"""Time RZF precoding (sb_ofdm_precode through `RZFPrecoder` with the effective channel) and, on the same grid, the
receiver's `LMMSEEqualizer`, so the downlink's added cost reads against the receiver. CUDA events over many calls after
warm-up.

    python tools/bench_precoding.py [--reps R] [--out FILE.json]

Shapes (why these two: they bracket the per-element problem sizes the kernel serves, from the CDL tutorial's downlink
to massive MU-MIMO, where the cost moves from memory traffic to arithmetic):
  1. tutorial downlink: one 8-antenna BS to one 4-antenna UT (K = 4), 14 x 76 grid, guard carriers 5 / 6, DC null,
     batch 256.
  2. massive MU-MIMO: a 64-antenna BS to 8 UTs with 2 antennas each (K = 16), 14 x 1024 grid, batch 8.
Algorithmic traffic, from the shapes: h read once, x read, x_precoded and h_eff written (complex64). FLOPs: 8 per
complex multiply-add of the Gram matrix (K (K + 1) / 2 M), the solves (K^2 M), x_precoded (K M) and h_eff
(num_rx num_rx_ant K M on the effective subcarriers). Rooflines: 3.35 TB/s HBM and 67 TFLOP/s FP32 (H100 SXM data
sheet, 700 W); the larger bound binds. The card's name and power limit are read in the same run. Needs a GPU.
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


def shapes():
    from sionna_b200.phy.ofdm import ResourceGrid
    tut = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6,
                       num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                       pilot_ofdm_symbol_indices=[2, 11])
    mu = ResourceGrid(14, 1024, 30e3, num_tx=1, num_streams_per_tx=16)
    # (name, rg, association [num_rx, num_tx], num_rx_ant, num_tx_ant, batch)
    return [("1: tutorial downlink 8 -> 4", tut, np.ones((1, 1), np.int32), 4, 8, 256),
            ("2: massive MU-MIMO 64 -> 8 x 2", mu, np.ones((8, 1), np.int32), 2, 64, 8)]


def roofline(rg, rx, ra, tx, m, k, b):
    s_, f_, ne = rg.num_ofdm_symbols, rg.fft_size, rg.num_effective_subcarriers
    re = b * tx * s_ * f_
    elems = b * rx * ra * tx * m * s_ * f_ + re * k + re * m + b * rx * ra * tx * k * s_ * ne
    macs = re * (k * (k + 1) // 2 * m + k * k * m + k * m) + b * tx * s_ * ne * rx * ra * k * m
    nbytes, flops = 8 * elems, 8 * macs
    t_mem, t_flop = nbytes / HBM_BYTES_PER_S * 1e3, flops / FP32_FLOPS_PER_S * 1e3
    return {"bytes": nbytes, "flops": flops, "bound_ms_bytes": round(t_mem, 4), "bound_ms_flops": round(t_flop, 4),
            "binds": "bytes" if t_mem >= t_flop else "flops"}


def run(name, rg, assoc, ra, m, b, reps):
    from sionna_b200.phy.ofdm import RZFPrecoder, LMMSEEqualizer
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.channel import ApplyOFDMChannel
    from sionna_b200.phy.utils import complex_normal
    from sionna_b200.phy import config
    config.seed = 1
    rx, tx = assoc.shape
    sm = StreamManagement(assoc, rg.num_streams_per_tx)
    k, s_, f_ = sm.num_streams_per_tx, rg.num_ofdm_symbols, rg.fft_size
    h = complex_normal([b, rx, ra, tx, m, s_, f_])
    x = complex_normal([b, tx, k, s_, f_])
    prec = RZFPrecoder(rg, sm, return_effective_channel=True)
    xp, h_eff = prec(x, h)
    y = ApplyOFDMChannel()(xp, h, 0.01)
    eff = torch.as_tensor(np.asarray(rg.effective_subcarrier_ind), device=y.device)
    eq = LMMSEEqualizer(rg, sm)
    r = {"shape": name, "batch": b, "num_tx_ant": m, "num_streams_per_tx": k, "num_rx": rx, "num_rx_ant": ra,
         "grid": [s_, f_]}
    r.update(roofline(rg, rx, ra, tx, m, k, b))
    ms = time_ms(lambda: prec(x, h), reps)
    r["rzf_precoder_ms"] = round(ms, 4)
    r["achieved_GB_per_s"] = round(r["bytes"] / (ms * 1e-3) / 1e9, 1)
    r["achieved_GFLOP_per_s"] = round(r["flops"] / (ms * 1e-3) / 1e9, 1)
    r["share_of_binding_roofline"] = round(max(r["bound_ms_bytes"], r["bound_ms_flops"]) / ms, 3)
    x_only = RZFPrecoder(rg, sm)
    r["x_only_ms"] = round(time_ms(lambda: x_only(x, h), reps), 4)
    r["lmmse_equalizer_ms"] = round(time_ms(lambda: eq(y, h_eff, 0.0, 0.01), reps), 4)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_precoding.py needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = [run(*s, args.reps) for s in shapes()]
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
