"""Time the K-Best MIMO detector (sb_ofdm_kbest) alone, CUDA events after warm-up, on inputs from the package's own
chain (seeded), next to LinearDetector and MaximumLikelihoodDetector on the same inputs.

    python tools/bench_kbest.py [--reps R] [--out FILE.json]

Shapes:
  (a) the 5G NR PUSCH tutorial's MU-MIMO uplink: 4 UEs x 2 codebook-precoded layers (8 streams), 16 rx antennas,
      16 PRB at 30 kHz, 16-QAM (MCS 14), DMRS type 2 / length 2 / one additional position, Rayleigh block fading,
      PUSCH LS estimate, batch 128; K-Best k = 64 in the complex and the real-valued representation. Plus one
      end-to-end PUSCHReceiver call (estimation, detection, layer demapping, LDPC decoding) with each detector.
  (b) configs[3]: 4 streams x 16 rx antennas, 16-QAM, 14 x 76 grid, batch 1024, TDL-A + LS(nn) estimate; K-Best
      k = 16 and 64 next to MaximumLikelihoodDetector (maxlog) and LinearDetector.
Per K-Best row: ms per call, data-carrying resource elements (problems) per second and child metrics per second (the
children the tree search scores: sum over layers of min(k, |C|^l) |C| per problem). The card's name and power limit
are read in the same run. Needs a GPU; there is no CPU fallback.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_ml import card, time_ms, data_res     # noqa: E402


def children(layers, points, k):
    """Child metrics the search scores per problem: layer l (0-based) has min(k, points^l) parents."""
    return sum(min(k, points ** l) * points for l in range(layers))


def row(name, det_name, ms, problems, child_metrics, ref):
    r = {"shape": name, "detector": det_name, "ms_per_call": round(ms, 4), "problems_per_s": problems / (ms * 1e-3)}
    if child_metrics:
        r["child_metrics_per_s"] = child_metrics / (ms * 1e-3)
    r.update(ref)
    print(json.dumps(r), flush=True)
    return r


def pusch_tutorial(dev, reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.nr import PUSCHConfig, PUSCHTransmitter, PUSCHReceiver
    from sionna_b200.phy.ofdm import KBestDetector, LinearDetector
    from sionna_b200.phy.mimo import StreamManagement
    from sionna_b200.phy.channel import RayleighBlockFading, OFDMChannel
    config.seed = 1
    num_tx, layers, batch, no = 4, 2, 128, 0.05
    pc = PUSCHConfig()
    pc.carrier.subcarrier_spacing = 30
    pc.carrier.n_size_grid = 16
    pc.num_antenna_ports = 4
    pc.num_layers = layers
    pc.precoding = "codebook"
    pc.tpmi = 1
    pc.dmrs.dmrs_port_set = list(range(layers))
    pc.dmrs.config_type = 2
    pc.dmrs.length = 2
    pc.dmrs.additional_position = 1
    pc.dmrs.num_cdm_groups_without_data = 3
    pc.tb.mcs_index = 14
    pc.tb.mcs_table = 1
    pcs = [pc]
    for i in range(1, num_tx):
        p = pc.clone()
        p.dmrs.dmrs_port_set = list(range(i * layers, (i + 1) * layers))
        pcs.append(p)
    tx = PUSCHTransmitter(pcs)
    rg = tx.resource_grid
    sm = StreamManagement(np.ones([1, num_tx], bool), layers)
    channel = OFDMChannel(RayleighBlockFading(1, 16, num_tx, 4), rg, normalize_channel=True)
    x, _ = tx(batch)
    y = channel(x, no)
    lin_rx = PUSCHReceiver(tx, stream_management=sm)
    h_hat, ev = lin_rx._channel_estimator(y, no)
    n_re = batch * data_res(rg)
    streams = num_tx * layers
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", 4)
    lin_ms = time_ms(lambda: lin(y, h_hat, ev, no), reps)
    name = f"(a) PUSCH tutorial {num_tx} UE x {layers} layers, 16 rx, 16 PRB, 16-QAM, batch {batch}"
    rows = [row(name, "LinearDetector", lin_ms, n_re, 0, {})]
    dets = {}
    for real_rep in (False, True):
        det = KBestDetector("bit", streams, 64, rg, sm, "qam", 4, use_real_rep=real_rep)
        dets[real_rep] = det
        ms = time_ms(lambda: det(y, h_hat, ev, no), reps)
        layers_, pts = (2 * streams, 4) if real_rep else (streams, 16)
        rows.append(row(name, f"KBestDetector k=64 real_rep={real_rep}", ms, n_re, n_re * children(layers_, pts, 64),
                        {"linear_detector_ms": round(lin_ms, 4)}))
    for det_name, rx in (("PUSCHReceiver LinearDetector", lin_rx),
                         ("PUSCHReceiver KBestDetector k=64", PUSCHReceiver(tx, mimo_detector=dets[False],
                                                                            stream_management=sm))):
        ms = time_ms(lambda: rx(y, no), max(1, reps // 2), warm=1)
        rows.append(row(name + " end to end", det_name, ms, n_re, 0, {}))
    return rows


def configs3(dev, reps):
    from sionna_b200.phy import config
    from sionna_b200.phy.ofdm import (ResourceGrid, ResourceGridMapper, LSChannelEstimator, LinearDetector,
                                      MaximumLikelihoodDetector, KBestDetector)
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
    n_re = batch * data_res(rg)
    name = "(b) configs[3] 4x16 16-QAM 14x76 batch 1024"
    lin = LinearDetector("lmmse", "bit", "maxlog", rg, sm, "qam", m)
    lin_ms = time_ms(lambda: lin(y, h_hat, ev, no), reps)
    ml = MaximumLikelihoodDetector("bit", "maxlog", rg, sm, "qam", m)
    ml_ms = time_ms(lambda: ml(y, h_hat, ev, no), reps, warm=1)
    rows = [row(name, "LinearDetector", lin_ms, n_re, 0, {}),
            row(name, "MaximumLikelihoodDetector maxlog", ml_ms, n_re, 0, {})]
    for k in (16, 64):
        det = KBestDetector("bit", streams, k, rg, sm, "qam", m)
        ms = time_ms(lambda: det(y, h_hat, ev, no), reps)
        rows.append(row(name, f"KBestDetector k={k}", ms, n_re, n_re * children(streams, 16, k),
                        {"linear_detector_ms": round(lin_ms, 4), "ml_maxlog_ms": round(ml_ms, 4)}))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_kbest.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = pusch_tutorial(dev, args.reps) + configs3(dev, args.reps)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
