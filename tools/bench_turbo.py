"""Time the turbo decoder (sb_turbo_decode through TurboDecoder) against the reference's algorithm composed from this
library's BCJRDecoder in a Python loop with torch glue, on the same inputs, and the encoder. CUDA events over many calls
after warm-up.

    python tools/bench_turbo.py [--reps R] [--out FILE.json]

Shapes (why these: k = 512 at batch 10 000 is the reference's BER test; k = 6144 is the 3GPP maximum, with alpha and the
extrinsic LLRs in the workspace; k = 40 is the smallest 3GPP size, all state on chip): LTE code (constraint length 4),
rate 1/3, terminated, 6 iterations, "map" and "maxlog". Counted work: 2 num_iter BCJR passes of T = k + 3 steps per
codeword ("codeword-steps"). The fused and composed outputs are compared bit for bit. The card's name and power limit
are read in the same run. Needs a GPU.
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
from bench_ml import card, time_ms     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_turbo needs a GPU"
    from sionna_b200.phy.fec.turbo import TurboEncoder, TurboDecoder
    from test_turbo_gpu import composed
    rows = []
    for k, batch in ((512, 10000), (6144, 1000), (40, 10000)):
        enc = TurboEncoder(constraint_length=4, rate=1 / 3, terminate=True)
        rng = np.random.default_rng(k)
        u = torch.from_numpy(rng.integers(0, 2, (batch, k)).astype(np.float32)).cuda()
        c = enc(u)
        no = 10 ** (-0.5 / 10)
        y = (2 / no * ((2 * c - 1) + torch.randn(c.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(k))
                       * np.sqrt(no))).contiguous()
        enc_ms = time_ms(lambda: enc(u), a.reps, warm=2)
        print(json.dumps({"shape": f"encoder k={k}", "batch": batch, "ms_per_call": round(enc_ms, 4),
                          "info_bits_per_s": batch * k / (enc_ms * 1e-3)}), flush=True)
        rows.append({"shape": f"encoder k={k}", "batch": batch, "ms_per_call": round(enc_ms, 4)})
        for alg in ("map", "maxlog"):
            dec = TurboDecoder(enc, num_iter=6, hard_out=False, algorithm=alg)
            fused_ms = time_ms(lambda: dec(y), a.reps, warm=2)
            comp_ms = time_ms(lambda: composed(dec, y), max(2, a.reps // 2), warm=1)
            same = bool(torch.equal(dec(y), composed(dec, y)))
            steps = batch * (k + 3) * 2 * 6
            r = {"shape": f"decoder {alg} k={k}", "batch": batch, "ms_per_call": round(fused_ms, 4),
                 "composed_ms_per_call": round(comp_ms, 4), "speedup": round(comp_ms / fused_ms, 2),
                 "info_bits_per_s": batch * k / (fused_ms * 1e-3), "codeword_steps_per_s": steps / (fused_ms * 1e-3),
                 "bit_identical_to_composed": same}
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
