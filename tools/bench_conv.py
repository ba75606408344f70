"""Time the convolutional decoders (sb_viterbi_decode / sb_bcjr_decode through ViterbiDecoder / BCJRDecoder) and the
float32 CPU oracle on the same inputs. CUDA events over many calls after warm-up.

    python tools/bench_conv.py [--reps R] [--cpu-batch B] [--out FILE.json]

Shapes (why these: the Polar-vs-LDPC tutorial's Viterbi decoder is what users run most, the GSM code is the packed-warp
path, k = 4096 sends the decisions through global memory, and BCJR at K = 5 / 8 keeps alpha on chip / in global memory):
  1. Viterbi K = 8, rate 1/2, k = 64, batch 10 000 (tutorial);
  2. Viterbi K = 5 (GSM), rate 1/2, k = 64, batch 10 000;
  3. Viterbi K = 8, rate 1/2, k = 4096, batch 256;
  4. BCJR map / log / maxlog at K = 5 and K = 8, rate 1/2, k = 64, batch 10 000, terminated.
Counted work: Viterbi ns ACS (two adds, one compare) per step and codeword; BCJR 2 ns state updates (forward and
backward) per step and codeword. Traffic: n floats in, k floats out per codeword. The CPU oracle (oracle/conv.py, NumPy)
decodes min(batch, --cpu-batch) codewords and is scaled to the batch; the host core count is reported beside it. The
card's name and power limit are read in the same run. Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from bench_ml import card, time_ms     # noqa: E402


def llrs(g, k, batch, terminate, snr_db=2.0, seed=0):
    from oracle import conv as O
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2, (batch, k))
    x = O.encode(u, g, False, terminate)
    no = 10 ** (-snr_db / 10)
    return (2 / no * ((2 * x - 1) + rng.normal(size=x.shape) * np.sqrt(no))).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cpu-batch", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_conv needs a GPU"
    from oracle import conv as O
    from sionna_b200.phy.fec.conv import ViterbiDecoder, BCJRDecoder, polynomial_selector
    rows = []
    cases = [("viterbi K=8 k=64 (tutorial)", "viterbi", 8, 64, 10000, False, None),
             ("viterbi K=5 k=64 (GSM)", "viterbi", 5, 64, 10000, False, None),
             ("viterbi K=8 k=4096 (global decisions)", "viterbi", 8, 4096, 256, False, None)]
    cases += [(f"bcjr {alg} K={K} k=64", "bcjr", K, 64, 10000, True, alg) for K in (5, 8)
              for alg in ("map", "log", "maxlog")]
    for name, kind, K, k, batch, terminate, alg in cases:
        g = polynomial_selector(1 / 2, K)
        y = llrs(g, k, batch, terminate)
        yd = torch.from_numpy(y).cuda()
        dec = ViterbiDecoder(gen_poly=g) if kind == "viterbi" else \
            BCJRDecoder(gen_poly=g, terminate=terminate, algorithm=alg, hard_out=False)
        ms = time_ms(lambda: dec(yd), a.reps, warm=3)
        ns, T = 2 ** (K - 1), y.shape[1] // 2
        cb = min(batch, a.cpu_batch)
        t0 = time.perf_counter()
        if kind == "viterbi":
            ref = O.viterbi(y[:cb], g, dtype=np.float32)
        else:
            ref = O.bcjr(y[:cb], g, terminate=terminate, algorithm=alg, dtype=np.float32)[:, :k]
        cpu_ms = (time.perf_counter() - t0) * 1e3 * batch / cb
        out = dec(yd)[:cb].cpu().numpy()
        agree = float(np.mean(out == ref)) if kind == "viterbi" else float(np.mean((out > 0) == (ref > 0)))
        updates = batch * T * ns * (1 if kind == "viterbi" else 2)
        r = {"shape": name, "batch": batch, "k": k, "states": ns, "ms_per_call": round(ms, 4),
             "info_bits_per_s": batch * k / (ms * 1e-3),
             ("acs_per_s" if kind == "viterbi" else "state_updates_per_s"): updates / (ms * 1e-3),
             "bytes_per_s": batch * (y.shape[1] + k) * 4 / (ms * 1e-3),
             "cpu_oracle_ms": round(cpu_ms, 1), "cpu_cores": os.cpu_count(), "agreement_with_oracle": agree}
        print(json.dumps(r), flush=True)
        rows.append(r)
    result = {"card": card(), "rows": rows}
    print(json.dumps(result["card"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
