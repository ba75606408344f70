"""Time the maximum-likelihood MIMO detector (sb_ofdm_ml / sb_mimo_ml) alone, CUDA events after warm-up, on inputs
from the package's own chain (seeded), with LinearDetector on the same inputs for context.

    python tools/bench_ml.py [--reps R] [--out FILE.json]

Shapes:
  (a) configs[3]: 4 streams x 16 rx antennas, 16-QAM, 14 x 76 grid, batch 1024, TDL-A + LS(nn) estimate; app and maxlog
      (warp-per-element variant: 16^3 outer indices per element)
  (b) configs[4]'s PUSCH shape: 2 layers x 8 rx antennas, 16-QAM, 16 PRB, TDL-B + PUSCH LS estimate, batch 2048
      (thread-per-element variant: 256 candidates)
  (c) dense 2 x 2 QPSK sb_mimo_ml, 2^22 problems (thread-per-problem variant: 16 candidates)
Per shape: ms per call, data-carrying resource elements (problems) per second, candidate metrics per second and a share of the FP32
peak from the FP32 operations the kernel spends per candidate (FLOPS_PER_CANDIDATE below, FMA = 2). The card's name and
power limit are read in the same run. Needs a GPU; there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# FP32 operations per candidate vector in the enumeration's inner loop (mimo_ml.cu, ml_pass):
#   metric  t = b0 - R00 x0 (2 FMA), d = P1 + |t|^2 (2 FMA)                                         = 8 flops
#   maxlog  pass 1: metric + accumulator min + inner-loop min                                        = 10
#   app     pass 1 (10) + pass 2: inner-loop min (metric + min = 9) and sums (metric 8, 2 subtractions,
#           2 exp counted as 1 op each, 2 additions = 14)                                            = 33
FLOPS_PER_CANDIDATE = {"maxlog": 10, "app": 33}
FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32, at the 700 W power limit


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [v.strip() for v in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                                  # the timing does not depend on it; report what happened
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})"}


def time_ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps


def row(name, ms, problems, candidates, method, lin_ms):
    flops = FLOPS_PER_CANDIDATE[method] * candidates
    r = {"shape": name, "method": method, "ms_per_call": round(ms, 4), "problems_per_s": problems / (ms * 1e-3),
         "candidate_metrics_per_s": candidates / (ms * 1e-3), "flops_per_candidate": FLOPS_PER_CANDIDATE[method],
         "fp32_share_of_peak": flops / (ms * 1e-3) / FP32_PEAK, "linear_detector_ms": round(lin_ms, 4)}
    print(json.dumps(r), flush=True)
    return r


def data_res(rg):
    """Resource elements per frame (one receiver) that carry data for at least one stream: the ones the detector
    processes; pilot-only elements are skipped."""
    mask = np.asarray(rg.pilot_pattern.mask).astype(bool)
    return int((~mask).reshape(-1, mask.shape[-2] * mask.shape[-1]).any(0).sum())


def configs3(dev, reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.ofdm import (ResourceGrid, ResourceGridMapper, LSChannelEstimator, LinearDetector,
                                      MaximumLikelihoodDetector)
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.mapping import Mapper, BinarySource
    from sionna_b200.phy.channel import TDL, ApplyOFDMChannel, subcarrier_frequencies, cir_to_ofdm_channel
    config.seed = 1
    streams, rx_ant, m, batch, no = 4, 16, 4, 1024, 0.05
    rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=streams, cyclic_prefix_length=6,
                      num_guard_carriers=(5, 6), dc_null=True, pilot_pattern="kronecker",
                      pilot_ofdm_symbol_indices=[2, 11])                  # tools/bench_links.py, configs[3]
    sm = StreamManagement(np.array([[1]]), streams)
    b = BinarySource()([batch, 1, streams, rg.num_data_symbols * m])
    tdl = TDL("A", 300e-9, 3.5e9, num_rx_ant=rx_ant, num_tx_ant=streams)
    a, tau = tdl(batch, 14, 1.0 / rg.ofdm_symbol_duration)
    h = cir_to_ofdm_channel(subcarrier_frequencies(76, 15e3), a, tau, normalize=True)
    y = ApplyOFDMChannel()(ResourceGridMapper(rg)(Mapper("qam", m)(b)), h, no)
    h_hat, ev = LSChannelEstimator(rg, "nn")(y, no)
    lin = LinearDetector("lmmse", "bit", "app", rg, sm, "qam", m)
    lin_ms = time_ms(lambda: lin(y, h_hat, ev, no), reps)
    n_re = batch * data_res(rg)
    rows = []
    for method in ("maxlog", "app"):
        det = MaximumLikelihoodDetector("bit", method, rg, sm, "qam", m)
        ms = time_ms(lambda: det(y, h_hat, ev, no), reps, warm=1)
        rows.append(row("(a) configs[3] 4x16 16-QAM 14x76 batch 1024", ms, n_re, n_re * 16 ** 4, method, lin_ms))
    return rows


def configs4(dev, reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.nr import PUSCHConfig, PUSCHTransmitter, PUSCHReceiver
    from sionna_b200.phy.ofdm import MaximumLikelihoodDetector, LinearDetector
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.channel import TDL, ApplyOFDMChannel, subcarrier_frequencies, cir_to_ofdm_channel
    config.seed = 2
    batch, no = 2048, 0.05
    pc = PUSCHConfig(num_layers=2, num_antenna_ports=2)
    pc.carrier.n_size_grid = 16
    pc.dmrs.additional_position = 1
    pc.tb.mcs_index = 14
    tx = PUSCHTransmitter(pc)
    rg = tx.resource_grid
    rx = PUSCHReceiver(tx)
    x, _ = tx(batch)
    tdl = TDL("B", 100e-9, 3.5e9, num_rx_ant=8, num_tx_ant=2)
    a, tau = tdl(batch, rg.num_ofdm_symbols, 1.0 / rg.ofdm_symbol_duration)
    h = cir_to_ofdm_channel(subcarrier_frequencies(rg.fft_size, rg.subcarrier_spacing), a, tau, normalize=True)
    y = ApplyOFDMChannel()(x, h, no)
    h_hat, ev = rx._channel_estimator(y, no)
    sm = StreamManagement(np.ones((1, 1), bool), 2)
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", 4)
    lin_ms = time_ms(lambda: lin(y, h_hat, ev, no), reps)
    n_re = batch * data_res(rg)
    rows = []
    for method in ("maxlog", "app"):
        det = MaximumLikelihoodDetector("bit", method, rg, sm, "qam", 4)
        ms = time_ms(lambda: det(y, h_hat, ev, no), reps)
        rows.append(row(f"(b) configs[4] PUSCH 2 layers x 8 rx 16-QAM batch {batch}", ms, n_re, n_re * 16 ** 2, method,
                        lin_ms))
    return rows


def dense2x2(dev, reps):
    from sionna_b200.phy.mimo import MaximumLikelihoodDetector, LinearDetector
    from sionna_b200.phy.mapping import Mapper, BinarySource
    num, no = 1 << 22, 0.1
    g = torch.Generator(device="cpu").manual_seed(3)

    def crandn(*shape):
        return (torch.complex(torch.randn(*shape, generator=g), torch.randn(*shape, generator=g)) / np.sqrt(2)).to(dev)

    x = Mapper("qam", 2)(BinarySource(seed=4)([num, 2 * 2]))
    h = crandn(num, 2, 2)
    y = (h @ x[..., None])[..., 0] + crandn(num, 2) * np.sqrt(no)
    s = (no * torch.eye(2, dtype=torch.complex64, device=dev)).expand(num, 2, 2).contiguous()
    lin = LinearDetector("lmmse", "bit", "maxlog", "qam", 2)
    lin_ms = time_ms(lambda: lin(y, h, s), reps)
    rows = []
    for method in ("maxlog", "app"):
        det = MaximumLikelihoodDetector("bit", method, 2, "qam", 2)
        ms = time_ms(lambda: det(y, h, s), reps)
        rows.append(row(f"(c) dense 2x2 QPSK sb_mimo_ml, {num} problems", ms, num, num * 16, method, lin_ms))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ml.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = configs3(dev, args.reps) + configs4(dev, args.reps) + dense2x2(dev, args.reps)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
