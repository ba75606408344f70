"""Time the EP and MMSE-PIC MIMO detectors (sb_ofdm_ep, sb_ofdm_mmse_pic) alone, CUDA events after warm-up, next to
LinearDetector and KBestDetector(k = 64) on the same inputs in the same process.

    python tools/bench_ep_pic.py [--reps R] [--out FILE.json]

Shapes:
  (a) configs[3]: 4 streams x 16 rx antennas, 16-QAM, 14 x 76 grid, batch 1024, TDL-A + LS(nn) estimate; EPDetector
      l = 10, MMSEPICDetector num_iter 1 and 3 with a non-zero prior (random LLRs), LinearDetector, KBestDetector k = 64.
  (b) the IDD tutorial's perfect-CSI link (tests/test_iterative_idd_gpu.py's Link: 4 UEs x 16 rx, 14 x 48 grid, LDPC5G
      k = 1152, n = 2304, min-sum 12 iterations), batch 64: one receive step per frame of the non-IDD LMMSE model and of
      IDD with 3 iterations.
Per row: ms per call and data-carrying resource elements (problems) per second. The card's name and power limit are
read in the same run. Needs a GPU; there is no CPU fallback.
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
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
from bench_ml import card, time_ms, data_res     # noqa: E402


def row(name, det_name, ms, problems, extra=None):
    r = {"shape": name, "detector": det_name, "ms_per_call": round(ms, 4), "problems_per_s": problems / (ms * 1e-3)}
    r.update(extra or {})
    print(json.dumps(r), flush=True)
    return r


def configs3(reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.ofdm import (ResourceGrid, ResourceGridMapper, LSChannelEstimator, LinearDetector,
                                      KBestDetector, EPDetector, MMSEPICDetector)
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
    prior = torch.randn(b.shape, device=b.device) * 2.0
    n_re = batch * data_res(rg)
    name = "(a) configs[3] 4x16 16-QAM 14x76 batch 1024"
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", m)
    lin_ms = time_ms(lambda: lin(y, h_hat, ev, no), reps)
    rows = [row(name, "LinearDetector", lin_ms, n_re)]
    kb = KBestDetector("bit", streams, 64, rg, sm, "qam", m)
    rows.append(row(name, "KBestDetector k=64", time_ms(lambda: kb(y, h_hat, ev, no), reps), n_re))
    ep = EPDetector("bit", rg, sm, m, l=10)
    rows.append(row(name, "EPDetector l=10", time_ms(lambda: ep(y, h_hat, ev, no), reps), n_re,
                    {"linear_detector_ms": round(lin_ms, 4)}))
    for it in (1, 3):
        pic = MMSEPICDetector("bit", "maxlog", rg, sm, it, "qam", m)
        rows.append(row(name, f"MMSEPICDetector num_iter={it} (random prior)",
                        time_ms(lambda: pic(y, h_hat, prior, ev, no), reps), n_re,
                        {"linear_detector_ms": round(lin_ms, 4)}))
    return rows


def idd_step(reps):
    from sionna_b200.phy import config
    from test_iterative_idd_gpu import Link
    config.seed = 3
    link, batch = Link(), 64
    _, y, h, no = link.frames(batch, -6.0)
    n_re = batch * data_res(link.rg)
    name = f"(b) IDD tutorial perfect CSI 4x16 16-QAM 14x48, LDPC5G (2304, 1152) min-sum 12, batch {batch}"
    rows = []
    for det_name, fn in (("non-IDD LMMSE receiver", lambda: link.lmmse_rx(y, h, no)),
                         ("IDD I=3 receiver", lambda: link.idd_rx(y, h, no, 3))):
        ms = time_ms(fn, reps)
        rows.append(row(name, det_name, ms, n_re, {"ms_per_frame": round(ms / batch, 5)}))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ep_pic.py needs a GPU")
    torch.cuda.set_device(0)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = configs3(args.reps) + idd_step(args.reps)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
