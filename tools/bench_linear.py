"""Time the OFDM linear equalisers (LMMSEEqualizer whitened and unwhitened, ZFEqualizer, MFEqualizer, all fused
kernels of sb_ofdm_lmmse / sb_ofdm_equalize) and SymbolDemapper (sb_symbol_demap). CUDA events over many calls after
warm-up.

    python tools/bench_linear.py [--reps R] [--out FILE.json]

Equaliser shapes (14 x 76 grids, Kronecker pilots on symbols 2 and 11), one per kernel family:
  1. SISO 64-QAM, batch 2048: register kernel, K = 1, M = 1 (the link benchmark's single-antenna shape)
  2. 4 streams to 16 antennas, batch 1024: register kernel, K = 4, antennas in chunks
  3. two transmitters with 2 streams each to two 8-antenna receivers, each treating the other's streams as
     interference, batch 256: shared-memory kernel (S assembled from H_u H_u^H)
Algorithmic traffic: y and the channel columns read once (complex64), err_var and no read once (float32, full shape),
x_hat and no_eff written for the data symbols. All shapes are bound by those bytes (3.35 TB/s HBM, H100 SXM data sheet,
700 W); shape 3 also reports its FP32 operations. SymbolDemapper: 16 / 64 / 256-QAM, 10^7 symbols, 8 bytes read and
4 P bytes written per symbol. The card's name and power limit are read in the same run. Needs a GPU.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from bench_ml import card, time_ms     # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP32_FLOPS_PER_S = 67e12


def eq_shapes():
    # (name, num_tx, streams per tx, num_rx, rx antennas, association, batch)
    return [("1: SISO 64-QAM 14 x 76", 1, 1, 1, 1, np.ones((1, 1), int), 2048),
            ("2: 4 streams -> 16 antennas 14 x 76", 1, 4, 1, 16, np.ones((1, 1), int), 1024),
            ("3: 2 x 2 streams -> 2 x 8 antennas, interferers 14 x 76", 2, 2, 2, 8, np.eye(2, dtype=int), 256)]


def run_eq(name, tx, spt, rx, ra, assoc, b, reps):
    from sionna_b200.phy.ofdm import ResourceGrid, LMMSEEqualizer, ZFEqualizer, MFEqualizer
    from sionna_b200.phy.mimo import StreamManagement
    rg = ResourceGrid(14, 76, 15e3, num_tx=tx, num_streams_per_tx=spt, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[2, 11])
    sm = StreamManagement(assoc, spt)
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(1)

    def cn(*shape):
        return torch.complex(torch.randn(*shape, device=dev, generator=g), torch.randn(*shape, device=dev, generator=g))
    s_, f_ = 14, 76
    y = cn(b, rx, ra, s_, f_)
    h = cn(b, rx, ra, tx, spt, s_, f_)
    ev = 0.01 * torch.rand(h.shape, device=dev, generator=g)
    no = 0.05 + 0.01 * torch.rand(b, rx, ra, device=dev, generator=g)
    k, ku, txs = sm.num_streams_per_rx, sm.num_interfering_streams_per_rx, tx * spt
    re = b * rx * s_ * f_
    nd = rg.num_data_symbols
    nbytes = 8 * y.numel() + 8 * re * ra * (k + ku) + 4 * ev.numel() + 4 * no.numel() + 12 * b * txs * nd
    macs = re * (ra * (ra + 1) // 2 * ku + ra * ra * k) if ku else 0     # S assembly and its solve (shape 3)
    t_mem, t_flop = nbytes / HBM_BYTES_PER_S * 1e3, 8 * macs / FP32_FLOPS_PER_S * 1e3
    r = {"shape": name, "batch": b, "K": k, "M": ra, "interferers": ku, "resource_elements": re,
         "bytes": nbytes, "flops": 8 * macs, "bound_ms_bytes": round(t_mem, 4), "bound_ms_flops": round(t_flop, 4),
         "binds": "bytes" if t_mem >= t_flop else "flops"}
    for label, blk in (("lmmse", LMMSEEqualizer(rg, sm)),
                       ("lmmse_no_whitening", LMMSEEqualizer(rg, sm, whiten_interference=False)),
                       ("zf", ZFEqualizer(rg, sm)), ("mf", MFEqualizer(rg, sm))):
        ms = time_ms(lambda: blk(y, h, ev, no), reps)
        r[f"{label}_ms"] = round(ms, 4)
        r[f"{label}_REs_per_s"] = float(f"{re / (ms * 1e-3):.4g}")
        r[f"{label}_share_of_binding_roofline"] = round(max(t_mem, t_flop) / ms, 3)
    print(json.dumps(r), flush=True)
    return r


def run_sym(m, n, reps):
    from sionna_b200.phy.mapping import SymbolDemapper
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(2)
    y = torch.complex(torch.randn(n, device=dev, generator=g), torch.randn(n, device=dev, generator=g))
    dem = SymbolDemapper("qam", m)
    npts = 2 ** m
    nbytes = 8 * n + 4 * n * npts
    ms = time_ms(lambda: dem(y, 0.1), reps)
    r = {"shape": f"SymbolDemapper {npts}-QAM", "symbols": n, "bytes": nbytes, "ms": round(ms, 4),
         "symbols_per_s": float(f"{n / (ms * 1e-3):.4g}"),
         "share_of_hbm_roofline": round(nbytes / HBM_BYTES_PER_S * 1e3 / ms, 3)}
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_linear.py needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = [run_eq(*s, args.reps) for s in eq_shapes()]
    rows += [run_sym(m, 10_000_000, args.reps) for m in (4, 6, 8)]
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
