"""Time the flat-fading channel (sb_flat_fading through FlatFadingChannel) against the unfused composition of the same
steps, and the Cholesky factor step (sb_chol_lower). CUDA events over many calls after warm-up.

    python tools/bench_flat_fading.py [--reps R] [--out FILE.json]

Shapes (why these: the tutorial / integration shape is what users run most, without h it is the pure generator
throughput, the per-column massive-MIMO shape moves the cost from memory traffic to the correlation products, and the
factor step is the set-up cost a fixed correlation pays once and a per-example one pays on every call):
  1. 4 -> 16, Kronecker 0.4 / 0.7, 2^20 channel uses, h returned, with noise;
  2. 4 -> 16, no correlation, 2^20 uses, h not returned, with noise;
  3. per-column one-ring, M = 64, K = 8, r_rx [8, 64, 64], 2^16 uses, h returned, with noise;
  4. the factor step: one n = 128 matrix, and 2^16 per-example n = 16 matrices.
Unfused composition beside each fused shape: complex_normal, then the model on the given h, then apply without noise,
then AWGN. Algorithmic traffic, from the shapes: x read, y written, h written when returned (complex64); the factors
(read once per CTA from L2) and the random draws (computed on chip) are not counted. FLOPs: 8 per complex multiply-add
of the correlation products (tx: M K (K + 1) / 2, rx or per column: K M (M + 1) / 2) and of y = h x (M K); the
Philox / Box-Muller work is not counted. Rooflines: 3.35 TB/s HBM and 67 TFLOP/s FP32 (H100 SXM data sheet, 700 W);
the larger bound binds. The card's name and power limit are read in the same run. Needs a GPU.
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from bench_ml import card, time_ms     # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FP32_FLOPS_PER_S = 67e12


def roofline(b, m, k, corr, want_h):
    elems = b * (k + m + (m * k if want_h else 0))
    macs = b * m * k
    if corr == "kronecker":
        macs += b * (m * k * (k + 1) // 2 + k * m * (m + 1) // 2)
    elif corr == "per_column":
        macs += b * k * m * (m + 1) // 2
    nbytes, flops = 8 * elems, 8 * macs
    t_mem, t_flop = nbytes / HBM_BYTES_PER_S * 1e3, flops / FP32_FLOPS_PER_S * 1e3
    return {"bytes": nbytes, "flops": flops, "bound_ms_bytes": round(t_mem, 4), "bound_ms_flops": round(t_flop, 4),
            "binds": "bytes" if t_mem >= t_flop else "flops"}


def run_channel(name, b, m, k, corr, want_h, reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.channel import (AWGN, ApplyFlatFadingChannel, FlatFadingChannel, KroneckerModel,
                                         PerColumnModel, exp_corr_mat, one_ring_corr_mat)
    from sionna_b200.phy.utils import complex_normal
    config.seed = 1
    model = {"none": None,
             "kronecker": KroneckerModel(exp_corr_mat(0.4, k), exp_corr_mat(0.7, m)),
             "per_column": PerColumnModel(one_ring_corr_mat(torch.linspace(-60, 60, k).numpy(), m, 0.5, 15))}[corr]
    chn = FlatFadingChannel(k, m, spatial_corr=model, return_channel=want_h)
    apply, awgn = ApplyFlatFadingChannel(), AWGN()
    x = complex_normal([b, k])
    no = 0.1

    def unfused():
        h = complex_normal([b, m, k])
        if model is not None:
            h = model(h)
        return awgn(apply(x, h), no)

    r = {"shape": name, "channel_uses": b, "num_rx_ant": m, "num_tx_ant": k, "correlation": corr, "h_returned": want_h}
    r.update(roofline(b, m, k, corr, want_h))
    ms = time_ms(lambda: chn(x, no), reps)
    r["fused_ms"] = round(ms, 4)
    r["achieved_GB_per_s"] = round(r["bytes"] / (ms * 1e-3) / 1e9, 1)
    r["achieved_GFLOP_per_s"] = round(r["flops"] / (ms * 1e-3) / 1e9, 1)
    r["share_of_binding_roofline"] = round(max(r["bound_ms_bytes"], r["bound_ms_flops"]) / ms, 3)
    r["unfused_ms"] = round(time_ms(unfused, reps), 4)
    print(json.dumps(r), flush=True)
    return r


def run_factor(name, count, n, reps):
    from sionna_b200.phy.channel import exp_corr_mat
    from sionna_b200.phy.channel.spatial_correlation import cholesky
    a = torch.rand(count).numpy() * 0.9 if count > 1 else 0.9
    r_ = exp_corr_mat(a, n)
    ms = time_ms(lambda: cholesky(r_), reps)
    flops = count * (8 * n ** 3 // 6)                   # n^3 / 6 complex multiply-adds per factorisation
    res = {"shape": name, "matrices": count, "n": n, "factor_ms": round(ms, 4), "flops": flops,
           "achieved_GFLOP_per_s": round(flops / (ms * 1e-3) / 1e9, 2)}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flat_fading.py needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = [run_channel("1: 4 -> 16 Kronecker 0.4 / 0.7, h returned", 1 << 20, 16, 4, "kronecker", True, args.reps),
            run_channel("2: 4 -> 16 uncorrelated, h not returned", 1 << 20, 16, 4, "none", False, args.reps),
            run_channel("3: per-column one-ring 64 x 8, h returned", 1 << 16, 64, 8, "per_column", True, args.reps),
            run_factor("4a: one n = 128 factor", 1, 128, args.reps),
            run_factor("4b: 2^16 per-example n = 16 factors", 1 << 16, 16, args.reps)]
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
