"""Work model of the boxplus-phi QC decoder (csrc/ldpc_bp_qc.cu): warp-level phi evaluations per iteration.

    python tools/phi_work_model.py [--batch 512] [--ebno 2 0] [--seed 1]

The CPU oracle reproduces every message of the QC kernel bit for bit (math_mode=1, order="kernel"), so the v2c
messages entering each of the 20 iterations are taken from it (num_iter = t, return_state=True). The inputs are the
bench's (bench.make_inputs: k = 4224, n = 8448, the BPSK-equivalent logits of QPSK over AWGN with app demapping).
Edges are mapped to the kernel's layout: check (r, i) of block row r is lane i mod 32 of warp slice i // 32, and the
row's edges are its positions l = 0 .. deg-1 in ascending VN order. Per codeword the switch from the plain variant to
the voting ("SC") variant is emulated: the plain variant's probe raises the flag when every lane of a slice has
positions 0 and 1 saturated (|x| >= 16.635532), and the voting variant runs from the next iteration on.

Warp-level phi evaluations of one row slice (a pair evaluation counts 2), under three rules:
  (a) the code before the union mask: plain rows 2*deg; voting rows: a row vote (2 phi if every edge but the last is
      saturated in every lane), else per-pair votes (1) saturated pair, (2) p == 0 pair -> one shared phi(P), (3)
      P - p <= 8.5e-8 pair -> phi_max;
  (b) the union mask U (positions with |x| below the phi-zero bound t in some lane), as the kernel now runs it: plain rows 2*deg; voting
      rows 2 if U holds no edge but the last, else 2|U| + 1 (+1 only if some position is outside U);
  (b0) rule (b) with the voting variant from iteration 0 (no probe): the alternative switch;
  (c) a lower bound for any exact scheme without pooling work across lanes: every lane pays only for its own
      unsaturated edges (rule (b) per lane), summed over the lanes and divided by 32. Applied in every iteration.
The phi-zero bound t is the least float32 above which phi is +0 in the kernel's arithmetic (found with the oracle;
the kernel's SB_PHI_ZERO). Rule (a) needs p == 0 and P - p per lane: phi is evaluated in float64 there (a model, not
the kernel's arithmetic), with p == 0 for |x| >= t.
Nothing is written; the run takes about a minute per Eb/N0 on a few host cores and uses no GPU.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle import ldpc as O                                          # noqa: E402
import bench                                                         # noqa: E402

HI = np.float32(16.635532)
LO = np.float32(8.5e-8)
CLASS_NAMES = ["deg>20", "13-20", "9-12", "5-8", "3-4"]


def row_class(d):
    return 0 if d > 20 else 1 if d > 12 else 2 if d > 8 else 3 if d > 4 else 4


def phi_zero_threshold():
    """Least float32 t with phi(x) == +0 for every x in [t, 16.635532] in the kernel's arithmetic (phi is not monotone
    just below t, so every value from 14 up is evaluated)."""
    lo, hi = int(np.float32(14.0).view(np.uint32)), int(HI.view(np.uint32))
    xs = np.arange(lo, hi + 1, dtype=np.uint32).view(np.float32)
    nz = np.nonzero([O.phi(v, 1) != 0.0 for v in xs])[0]
    return xs[nz.max() + 1]


def phi64(a, t0):
    x = np.clip(a.astype(np.float64), float(LO), float(HI))
    p = np.log1p(2.0 / np.expm1(x))
    return np.where(a >= t0, 0.0, p)


class Layout:
    """Slot of every reference edge in a [rows, Dmax, slices * 32] array of one codeword."""

    def __init__(self, dec, z):
        cn, vn = dec.edges
        r, i, cb = cn // z, cn % z, vn // z
        self.R = int(r.max()) + 1
        self.S = (z + 31) // 32
        self.deg = np.bincount(r, minlength=self.R) // z
        self.D = int(self.deg.max())
        # position of the edge inside its check: rank of its block column among the block row's columns
        l = np.zeros(len(cn), np.int64)
        for rr in range(self.R):
            cols = np.unique(cb[r == rr])
            sel = r == rr
            l[sel] = np.searchsorted(cols, cb[sel])
        self.flat = (r * self.D + l) * (self.S * 32) + i
        self.cls = np.array([row_class(d) for d in self.deg])

    def magnitudes(self, st):
        """|v2c| [B, R, D, S, 32]; absent edges and lanes are +inf (saturated: neutral for every vote)."""
        B = st.shape[1]
        x = np.full((B, self.R * self.D * self.S * 32), np.inf, np.float32)
        x[:, self.flat] = np.abs(st.T)
        return x.reshape(B, self.R, self.D, self.S, 32)


def count_iteration(X, lay, sc, t0):
    """Warp-level phi per codeword and row class under rules a, b, c; probe result; |U| histogram of voting rows."""
    B = X.shape[0]
    out = {k: np.zeros((B, len(CLASS_NAMES))) for k in ("a", "b", "b0", "c")}
    hist = np.zeros(4)                                               # voting row slices with |U| = 0, 1, 2..deg-1, deg
    probe = np.zeros(B, bool)
    for r in range(lay.R):
        d, c = int(lay.deg[r]), int(lay.cls[r])
        x = X[:, r, :d]                                              # [B, d, S, 32]
        sat_all = ~(x < HI).any(-1)                                  # [B, d, S] saturated in every lane (old votes)
        probe |= (sat_all[:, 0] & sat_all[:, 1]).any(-1)
        unsat = x < t0                                               # phi(|x|) may be nonzero
        anyU = unsat.any(-1)                                         # [B, d, S]
        k = anyU.sum(1)                                              # [B, S]
        plain = np.full(k.shape, 2.0 * d)
        # (b)
        b_sc = np.where(anyU[:, :d - 1].any(1), 2 * k + (k < d), 2)
        # (c), per lane
        kl = unsat.sum(1)                                            # [B, S, 32]
        lane = np.where(kl == 0, 0, np.where(kl == 1, 2, 2 * kl + (kl < d)))
        active = np.isfinite(x).any(1)                               # lanes that exist
        c_all = (lane * active).sum(-1) / 32.0
        # (a) voting: row vote, else per-pair votes
        rowvote = sat_all[:, :d - 1].all(1)                          # [B, S]
        p = phi64(x, t0)                                             # [B, d, S, 32]
        P = p.sum(1, keepdims=True)
        pz = (p == 0).all(-1)                                        # [B, d, S]
        small = ((P - p) <= float(LO)).all(-1)
        old_any = ~sat_all
        a1 = np.zeros(k.shape)
        a2 = np.zeros(k.shape)
        shared = np.zeros(k.shape, bool)
        for l in range(0, d - 1, 2):
            a1 += 2 * (old_any[:, l] | old_any[:, l + 1])
            r2 = pz[:, l] & pz[:, l + 1]
            shared |= r2
            a2 += np.where(r2 | (small[:, l] & small[:, l + 1]), 0, 2)
        if d & 1:
            a1 += old_any[:, d - 1]
            r2 = pz[:, d - 1]
            shared |= r2
            a2 += np.where(r2 | small[:, d - 1], 0, 1)
        a_sc = np.where(rowvote, 2, a1 + a2 + shared)
        m = sc[:, None]
        out["a"][:, c] += np.where(m, a_sc, plain).sum(-1)
        out["b"][:, c] += np.where(m, b_sc, plain).sum(-1)
        out["b0"][:, c] += b_sc.sum(-1)
        out["c"][:, c] += c_all.sum(-1)
        ks = k[sc]
        hist += [(ks == 0).sum(), (ks == 1).sum(), ((ks > 1) & (ks < d)).sum(), (ks == d).sum()]
    return out, probe, hist


def run(ebno, batch, seed, iters, threads, t0):
    enc = O.LDPC5GEncoderRef(bench.K_INFO, bench.N_CODE)
    dec = O.LDPC5GDecoderRef(enc, hard_out=False, return_infobits=False, num_iter=iters, return_state=True)
    lay = Layout(dec, enc.z)
    llr = bench.make_inputs(seed, batch, ebno)
    sc = np.zeros(batch, bool)
    rows = []
    hist = np.zeros(4)
    per_cls = {k: np.zeros(len(CLASS_NAMES)) for k in "abc"}
    for t in range(iters):
        _, st = dec(llr, num_iter=t, math_mode=1, order="kernel", num_threads=threads)
        out, probe, h = count_iteration(lay.magnitudes(st), lay, sc, t0)
        hist += h
        for k in "abc":
            per_cls[k] += out[k].sum(0) / batch
        rows.append((t, sc.mean(), *(out[k].sum() / batch for k in ("a", "b", "c", "b0"))))
        sc = sc | probe
    return rows, per_cls, hist, lay


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--ebno", type=float, nargs="+", default=[2.0, 0.0])
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--threads", type=int, default=None)
    a = ap.parse_args()
    iters = bench.NUM_ITER
    t0 = phi_zero_threshold()
    print(f"phi(x) == +0 for x >= {t0:.9g} (kernel arithmetic); saturation bound {HI:.9g}")
    for ebno in a.ebno:
        rows, per_cls, hist, lay = run(ebno, a.batch, a.seed, iters, a.threads, t0)
        print(f"\nEb/N0 {ebno:g} dB, {a.batch} codewords, {iters} iterations; warp-level phi per codeword "
              f"({lay.R} block rows x {lay.S} slices)")
        print("| iter | SC share | (a) before | (b) union mask | (c) lower bound | b/a | (b0) voting from iteration 0 |")
        print("|---|---|---|---|---|---|---|")
        for t, s, ra, rb, rc, rb0 in rows:
            print(f"| {t} | {s:.3f} | {ra:.0f} | {rb:.0f} | {rc:.0f} | {rb / ra:.3f} | {rb0:.0f} |")
        tot = [sum(r[i] for r in rows) for i in (2, 3, 4, 5)]
        print(f"| all | {np.mean([r[1] for r in rows]):.3f} | {tot[0]:.0f} | {tot[1]:.0f} | {tot[2]:.0f} | "
              f"{tot[1] / tot[0]:.3f} | {tot[3]:.0f} |")
        sc_iters = [r[0] for r in rows if r[1] == 0]
        same = all(r[2] == r[3] for r in rows if r[1] == 0)
        print(f"iterations without SC codewords: {len(sc_iters)}; (a) == (b) in all of them: {same}")
        print("per row class, summed over iterations: " + "; ".join(
            f"{n}: a {per_cls['a'][i]:.0f} b {per_cls['b'][i]:.0f} c {per_cls['c'][i]:.0f}"
            for i, n in enumerate(CLASS_NAMES) if per_cls["a"][i] > 0))
        if hist.sum():
            h = hist / hist.sum()
            print(f"voting row slices: |U| = 0 {h[0]:.3f}, |U| = 1 {h[1]:.3f}, 1 < |U| < deg {h[2]:.3f}, "
                  f"|U| = deg {h[3]:.3f}")


if __name__ == "__main__":
    main()
