"""Time OSDecoder (sb_osd_decode) and LinearEncoder (sb_gf2_encode) with CUDA events over many calls after warm-up.

    python tools/bench_osd.py [--reps R] [--out FILE.json]

Shapes: the Polar-vs-LDPC tutorial's 5G LDPC (64, 128) at t = 4, BCH(63, 45) t = 4 and BCH(127, 106) t = 2 (example
codes whose torch composition fits at a useful batch); the encoder on 802.11n (n = 648) and on the largest 5G generator's
shape (k = 8448, n = 25344, random G). Beside each OSD row: the reference's formulation (every candidate materialised as a [batch,
C(k, t), n] tensor, float32 softplus metric) composed from torch ops on the GPU at a batch that fits, and the NumPy
oracle's float64 discrepancy decoder on the host (single process; the host's core count is printed). LLRs of BPSK over
AWGN at Eb/N0 = 2 dB. Candidates/s counts sum_{t' <= t} C(k, t') per codeword (before pruning). Needs a GPU.
"""
import argparse
import itertools
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


def reference_osd(llr, gm, t):
    """fec/linear/decoding.py:253-478 composed from torch ops: [bs, C(k, t'), n] candidates per order."""
    bs, n = llr.shape
    k = gm.shape[0]
    llr = llr.clamp(-100., 100.)
    idx = torch.argsort(llr.abs(), dim=1, descending=True, stable=True)
    g = gm[None].expand(bs, k, n).gather(2, idx[:, None, :].expand(bs, k, n)).clone()
    piv = []
    for c in range(k):
        p = torch.argmax(g[:, c, :], dim=-1)
        piv.append(p)
        r = g.gather(2, p[:, None, None].expand(bs, k, 1)).squeeze(-1)
        r[:, c] = 0
        g = torch.remainder(g + r[:, :, None] * g[:, c:c + 1, :], 2)
    piv = torch.stack(piv, 1)
    key = torch.arange(n, device=llr.device)[None].expand(bs, n).clone()
    key.scatter_add_(1, piv, torch.full_like(piv, n))
    idx_mrb = torch.cat([piv, torch.argsort(key, dim=1)[:, :n - k]], 1)
    g = g.gather(2, idx_mrb[:, None, :].expand(bs, k, n))
    idx = idx.gather(1, idx_mrb)
    ls = llr.gather(1, idx)
    c0 = torch.remainder((ls[:, None, :k] > 0).float() @ g, 2).squeeze(1)

    def dist(cand):
        return torch.log(1. + torch.exp(ls[:, None, :] * (1 - 2 * cand))).mean(-1)
    best_c, best_d = c0, dist(c0[:, None])[:, 0]
    for ti in range(1, t + 1):
        ep = torch.tensor(list(itertools.combinations(range(k), ti)), device=llr.device)
        cand = torch.remainder(g[:, ep, :].sum(2) + c0[:, None], 2)
        d = dist(cand)
        i = torch.argmin(d, 1)
        dm = d.gather(1, i[:, None])[:, 0]
        cm = cand.gather(1, i[:, None, None].expand(bs, 1, n))[:, 0]
        upd = dm < best_d
        best_c = torch.where(upd[:, None], cm, best_c)
        best_d = torch.where(upd, dm, best_d)
    return torch.empty_like(best_c).scatter_(1, idx, best_c)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_osd needs a GPU"
    from sionna_b200.phy.fec.linear import LinearEncoder, OSDecoder
    from sionna_b200.phy.fec.utils import load_parity_check_examples, pcm2gm
    from oracle import linear_codes as O
    from math import comb
    sp = np.load(os.path.join(os.path.dirname(HERE), "tests", "golden", "ldpc_k64_n128_G.npy")).astype(int)
    g5 = np.zeros((64, 128), np.int64)
    g5[sp[0] - 1, sp[1] - 1] = 1
    rows = []
    shapes = (("5G LDPC (64,128) t=4", g5, 4, 2000, 2),
              ("BCH(63,45) t=4", pcm2gm(load_parity_check_examples(1)[0]), 4, 10000, 8),
              ("BCH(127,106) t=2", pcm2gm(load_parity_check_examples(2)[0]), 2, 10000, 64))
    for name, gm, t, batch, ref_batch in shapes:
        k, n = gm.shape
        rng = np.random.default_rng(k)
        u = rng.integers(0, 2, (batch, k))
        c = O.encode(u, gm)
        no = 1 / (10 ** 0.2 * k / n)
        llr_np = (4 * ((2. * c - 1) + rng.normal(size=c.shape) * np.sqrt(no / 2)) / no).astype(np.float32)
        llr = torch.from_numpy(llr_np).cuda()
        dec = OSDecoder(gm, t=t)
        ms = time_ms(lambda: dec(llr), a.reps, warm=1)
        cands = 1 + sum(comb(k, i) for i in range(1, t + 1))
        out = dec(llr)
        gm_t = torch.tensor(gm, dtype=torch.float32, device="cuda")
        ref_ms = time_ms(lambda: reference_osd(llr[:ref_batch], gm_t, t), 2, warm=1)
        ref_out = reference_osd(llr[:ref_batch], gm_t, t)
        agree = float((ref_out == out[:ref_batch]).all(1).float().mean())
        n_or = min(batch, 20 if t >= 4 else 200)
        t0 = time.perf_counter()
        for l in llr_np[:n_or]:
            O.osd_discrepancy(l, gm, t)
        or_s = (time.perf_counter() - t0) / n_or
        r = {"shape": name, "batch": batch, "ms_per_call": round(ms, 3),
             "codewords_per_s": round(batch / (ms * 1e-3)), "candidates_per_s": batch * cands / (ms * 1e-3),
             "reference_torch_batch": ref_batch, "reference_torch_ms": round(ref_ms, 3),
             "reference_torch_codewords_per_s": round(ref_batch / (ref_ms * 1e-3), 1),
             "speedup_per_codeword": round((ref_ms / ref_batch) / (ms / batch), 1),
             "decisions_equal_to_reference_torch": agree,
             "numpy_oracle_s_per_codeword": round(or_s, 4), "host_cores": os.cpu_count()}
        print(json.dumps(r), flush=True)
        rows.append(r)
    pcm4 = load_parity_check_examples(4)[0]
    rng = np.random.default_rng(0)
    for name, enc, batch in (("encoder 802.11n n=648", LinearEncoder(pcm4, is_pcm=True), 100000),
                             ("encoder random k=8448 n=25344", LinearEncoder(rng.integers(0, 2, (8448, 25344), dtype=np.uint8)), 1000)):
        u = torch.randint(0, 2, (batch, enc.k), device="cuda").float()
        ms = time_ms(lambda: enc(u), a.reps, warm=1)
        gm_t = enc.gm
        ref_ms = time_ms(lambda: torch.remainder(u @ gm_t, 2), a.reps, warm=1)
        same = bool(torch.equal(enc(u), torch.remainder(u @ gm_t, 2)))
        r = {"shape": name, "batch": batch, "ms_per_call": round(ms, 3),
             "codewords_per_s": round(batch / (ms * 1e-3)), "info_bits_per_s": batch * enc.k / (ms * 1e-3),
             "torch_fp32_matmul_mod2_ms": round(ref_ms, 3), "equal_to_matmul": same}
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
