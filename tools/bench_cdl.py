"""Time the CDL channel model: sb_cdl_coefficients (`CDL.synthesize`) alone, the random draws alone, the whole `CDL`
call, and the channel generation block around it. CUDA events over many launches after warm-up.

    python tools/bench_cdl.py [--reps R] [--out FILE.json]

Configurations (the reference's MIMO OFDM CDL tutorial): CDL-B, 300 ns, uplink, UT AntennaArray(1, 2, dual, cross,
38.901) (4 antennas), BS AntennaArray(1, 4, dual, cross, 38.901) (8 antennas), 2.6 GHz, 10 m/s.
  1. frequency domain: batch 4096, 14 steps at 1 / ofdm_symbol_duration of a 76 x 15 kHz grid (cyclic prefix 6);
     GenerateOFDMChannel timed as well.
  2. time domain: batch 64, 14 (76 + 6) + l_tot - 1 steps at the bandwidth 76 x 15 kHz; GenerateTimeChannel timed.
Rooflines from shapes: bytes written (the output, once) over 3.35 TB/s and FLOPs (8 per ray per output for the complex
multiply-add, 12 per ray per (antenna pair, cluster, time tile) for the ray coefficients) over 67 TFLOP/s FP32 (H100
SXM data sheet, 700 W); the larger bound binds. The card's name and power limit are read in the same run. Needs a GPU.
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
TIME_TILE = 16                         # kCdlTile in csrc/channel.cu


def model():
    from sionna_b200.phy.channel import CDL, AntennaArray
    fc = 2.6e9
    ut = AntennaArray(1, 2, "dual", "cross", "38.901", fc)
    bs = AntennaArray(1, 4, "dual", "cross", "38.901", fc)
    return CDL("B", 300e-9, fc, ut, bs, "uplink", min_speed=10.0)


def roofline(cdl, batch, steps):
    nr, nt, c = cdl.rx_array.num_ant, cdl.tx_array.num_ant, cdl.num_clusters
    outputs = batch * nr * nt * c * steps
    tiles = -(-steps // TIME_TILE)
    flops = outputs * 20 * 8 + batch * tiles * nr * nt * c * 20 * 12
    nbytes = outputs * 8
    t_mem, t_flop = nbytes / HBM_BYTES_PER_S * 1e3, flops / FP32_FLOPS_PER_S * 1e3
    return {"bytes_written": nbytes, "flops": flops, "phasors": batch * steps * c * 20,
            "bound_ms_bytes": round(t_mem, 4), "bound_ms_flops": round(t_flop, 4),
            "binds": "bytes" if t_mem >= t_flop else "flops"}


def run(name, batch, steps, fs, generate, reps):
    from sionna_b200.phy import config
    config.seed = 1
    cdl = model()
    draws = cdl.draws(batch)
    r = {"config": name, "batch": batch, "num_time_steps": steps, "sampling_frequency": fs}
    r.update(roofline(cdl, batch, steps))
    r["synthesize_ms"] = round(time_ms(lambda: cdl.synthesize(draws, steps, fs), reps), 4)
    r["draws_ms"] = round(time_ms(lambda: cdl.draws(batch), reps), 4)
    r["cdl_call_ms"] = round(time_ms(lambda: cdl(batch, steps, fs), reps), 4)
    gen = generate(cdl)
    r[gen[0] + "_ms"] = round(time_ms(lambda: gen[1](batch), max(reps // 4, 5)), 4)
    bound = max(r["bound_ms_bytes"], r["bound_ms_flops"])
    r["synthesize_share_of_bound"] = round(bound / r["synthesize_ms"], 3)
    r["synthesize_bytes_per_s"] = r["bytes_written"] / (r["synthesize_ms"] * 1e-3)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cdl.py needs a CUDA device")
    from sionna_b200.phy.ofdm import ResourceGrid
    from sionna_b200.phy.channel import GenerateOFDMChannel, GenerateTimeChannel, time_lag_discrete_time_channel
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rg = ResourceGrid(14, 76, 15e3, num_tx=1, num_streams_per_tx=4, cyclic_prefix_length=6)
    bw = 76 * 15e3
    l_min, l_max = time_lag_discrete_time_channel(bw)
    l_tot = l_max - l_min + 1
    rows = [
        run("1: frequency domain", 4096, 14, 1.0 / rg.ofdm_symbol_duration,
            lambda c: ("generate_ofdm_channel", GenerateOFDMChannel(c, rg)), args.reps),
        run("2: time domain", 64, 14 * (76 + 6) + l_tot - 1, bw,
            lambda c: ("generate_time_channel", GenerateTimeChannel(c, bw, 14 * (76 + 6), l_min, l_max)), args.reps),
    ]
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
