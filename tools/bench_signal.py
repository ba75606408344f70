"""Time the signal kernels (sb_convolve, the empirical PSD) with CUDA events after warm-up, beside cuDNN.

    python tools/bench_signal.py [--reps R] [--out FILE.json]

Shapes:
  1. the Pulse_Shaping_Basics chain: Upsampling(4) -> RRC (span 32, 129 taps) "full" on [128, 4000] -> matched RRC ->
     Downsampling(4, 128, 1000), and empirical_psd on [128, 4128];
  2. [4096, 16384] complex64 with 129 real taps, "same" (compute-bound);
  3. the same with 9 real taps (memory-bound);
  4. the same with 129 complex taps;
  5. shape 2 in complex128, computed natively in float64.
Beside each: torch.nn.functional.conv1d (cuDNN, TF32 off) in the shape's precision with the reference's real /
imaginary split (2 or 4 convolutions), and each arm's max error against the float64 oracle on the first rows.
Algorithmic FLOPs count 2 per real FMA (1, 2 or 4 real FMAs per tap and output for real x real, one complex operand,
complex x complex); bytes count x read once and y written once. The binding roofline is the larger of FLOPs over the
H100 SXM data-sheet rate (67 TFLOP/s FP32, 34 TFLOP/s FP64) and bytes over 3.35 TB/s. Needs a GPU.
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

PEAK = {"single": 67e12, "double": 34e12}
HBM = 3.35e12
ERR_ROWS = 8


def cudnn_conv(x, h, pad):
    """The reference's real / imaginary split on conv1d (cross-correlation, so the kernel is flipped)."""
    def c(a, k):
        return torch.nn.functional.conv1d(a[:, None, :], k.flip(0)[None, None, :], padding=pad)[:, 0, :]
    xr, xi = (x.real, x.imag) if x.is_complex() else (x, None)
    hr, hi = (h.real, h.imag) if h.is_complex() else (h, None)
    re, im = c(xr, hr), None
    if xi is not None:
        im = c(xi, hr)
    if hi is not None:
        im = c(xr, hi) if im is None else im + c(xr, hi)
        if xi is not None:
            re = re - c(xi, hi)
    return re if im is None else torch.complex(re, im)


def entry(name, precision, ms, outputs, flops, nbytes, err, cudnn_ms, cudnn_err):
    bound_flops, bound_bytes = flops / PEAK[precision], nbytes / HBM
    bound = "compute" if bound_flops >= bound_bytes else "memory"
    r = {"shape": name, "precision": precision, "ms": round(ms, 4), "outputs_per_s": outputs / (ms * 1e-3),
         "gflop": flops / 1e9, "gbytes": nbytes / 1e9, "roofline": bound,
         "share_of_roofline": max(bound_flops, bound_bytes) / (ms * 1e-3), "max_err": err,
         "cudnn_ms": round(cudnn_ms, 4), "cudnn_max_err": cudnn_err, "speedup_vs_cudnn": cudnn_ms / ms}
    print(json.dumps(r), flush=True)
    return r


def max_err(y, x, h, padding):
    from oracle import signal as O
    ref = O.convolve(x[:ERR_ROWS].cpu().numpy(), h.cpu().numpy(), padding)
    return float(np.abs(y[:ERR_ROWS].cpu().numpy() - ref).max() / np.abs(ref).max())


def fma_per_tap(x, h):
    return (2 if x.is_complex() else 1) * (2 if h.is_complex() else 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_signal needs a GPU"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from sionna_b200.phy import config
    from sionna_b200.phy.signal import (convolve, empirical_psd, Upsampling, Downsampling, RootRaisedCosineFilter)
    from sionna_b200.phy.signal import utils as U
    dev = torch.device("cuda", 0)
    config.device = dev
    head = card()
    print(json.dumps(head), flush=True)
    results = []
    g = torch.Generator(device=dev).manual_seed(0)

    # 1. the tutorial chain and its PSD
    rrcf = RootRaisedCosineFilter(32, 4, 0.22)
    up, down = Upsampling(4), Downsampling(4, 128, 1000)
    sym = torch.randn(128, 1000, dtype=torch.complex64, device=dev, generator=g)
    taps = rrcf(torch.ones(1, device=dev))                   # the prepared taps, for the cuDNN arm

    def chain():
        return down(rrcf(rrcf(up(sym))))

    def chain_cudnn():
        xu = torch.zeros(128, 4000, dtype=torch.complex64, device=dev)
        xu[:, ::4] = sym
        return cudnn_conv(cudnn_conv(xu, taps, 128), taps, 128)[:, 128::4][:, :1000]
    ms, cms = time_ms(chain, args.reps), time_ms(chain_cudnn, args.reps)
    d = float((chain() - chain_cudnn()).abs().max())
    outs = 128 * (4128 + 4256)
    results.append(entry("tutorial chain: up 4, RRC full [128, 4000], matched RRC, down 4", "single", ms, outs,
                         2 * 2 * 129 * outs, 8 * 128 * (4000 + 4128 + 4128 + 4256), None, cms, d))
    xp = torch.randn(128, 4128, dtype=torch.complex64, device=dev, generator=g)
    ms = time_ms(lambda: empirical_psd(xp, show=False, oversampling=4), args.reps)
    cms = time_ms(lambda: (torch.fft.fftshift(torch.fft.fft(xp) / 4128 ** 0.5, dim=-1).abs() ** 2).mean(0), args.reps)
    r = {"shape": "empirical_psd [128, 4128]", "ms": round(ms, 4), "torch_fft_ms": round(cms, 4),
         "gbytes": 8 * 128 * 4128 * 2 / 1e9}
    print(json.dumps(r), flush=True)
    results.append(r)
    xm = torch.randn(10 ** 6, 64, dtype=torch.complex64, device=dev, generator=g)
    ms = time_ms(lambda: U._power_mean(xm), args.reps)
    r = {"shape": "sb_power_mean [1e6, 64]", "ms": round(ms, 4), "share_of_hbm": 8 * 64e6 / HBM / (ms * 1e-3)}
    print(json.dumps(r), flush=True)
    results.append(r)

    # 2-5. [4096, 16384], "same"
    for name, k, hc, precision in (("129 real taps", 129, False, "single"), ("9 real taps", 9, False, "single"),
                                   ("129 complex taps", 129, True, "single"),
                                   ("129 real taps, complex128", 129, False, "double")):
        cdt = torch.complex64 if precision == "single" else torch.complex128
        rdt = torch.float32 if precision == "single" else torch.float64
        x = torch.randn(4096, 16384, dtype=cdt, device=dev, generator=g)
        h = torch.randn(k, dtype=cdt if hc else rdt, device=dev, generator=g)
        ms = time_ms(lambda: convolve(x, h, "same", precision=precision), args.reps)
        cms = time_ms(lambda: cudnn_conv(x, h, (k - 1) // 2), args.reps)
        err = max_err(convolve(x, h, "same", precision=precision), x, h, "same")
        cerr = max_err(cudnn_conv(x, h, (k - 1) // 2), x, h, "same")
        outs = x.numel()
        results.append(entry(f"[4096, 16384] {cdt}, {name}, same", precision, ms, outs,
                             2 * fma_per_tap(x, h) * k * outs, 2 * x.numel() * x.element_size(), err, cms, cerr))
        del x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": head, "reps": args.reps, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
