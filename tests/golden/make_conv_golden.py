"""Generate tests/golden/conv_golden.npz from the reference's convolutional-code goldens.

Needs /root/reference (build container only). Stores, for each of the four generator sets of
/root/reference/test/codes/conv/ (5/7, 64/74 as ('1101', '1111'), 5/7/7, 5/7/7/7; 10 x 500 information bits), the
information bits u, codewords x (packed), channel outputs y and Viterbi / BCJR decisions uhat of
test/unit/fec/test_conv_{encoding,decoding}.py, and the polynomial_selector table of fec/conv/utils.py:41-57 as
'rate:K' -> polynomials joined by ','.
"""
import os
import numpy as np

src = "/root/reference/test/codes/conv"
names = {"57": ("101", "111"), "6474": ("1101", "1111"), "577": ("101", "111", "111"),
         "5777": ("101", "111", "111", "111")}
files = {"57": "conv_rate_half_57_", "6474": "conv_rate_half_6474_", "577": "conv_rate_onethird_577_",
         "5777": "conv_rate_onefourth_5777_"}
out = {}
for key, stem in files.items():
    u = np.load(os.path.join(src, stem + "ref_u.npy"))
    x = np.load(os.path.join(src, stem + "ref_x.npy"))
    y = np.load(os.path.join(src, stem + "ref_y.npy"))
    uhat = np.load(os.path.join(src, stem + "ref_uhat.npy"))
    assert set(np.unique(u)) <= {0, 1} and set(np.unique(x)) <= {0, 1} and set(np.unique(uhat)) <= {0, 1}
    out[f"u_{key}"] = np.packbits(u.astype(np.uint8), axis=1)
    out[f"x_{key}"] = np.packbits(x.astype(np.uint8), axis=1)
    out[f"uhat_{key}"] = np.packbits(uhat.astype(np.uint8), axis=1)
    out[f"y_{key}"] = y.astype(np.float32) if y.dtype == np.float32 else y
    out[f"poly_{key}"] = np.array(names[key])
    out[f"shape_{key}"] = np.array([u.shape[1], x.shape[1]])
    print(key, u.shape, x.shape, y.dtype, y.shape, uhat.shape)

import sys, types
sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))     # the table module imports tf at load time
import importlib.util
spec = importlib.util.spec_from_file_location("ref_conv_utils", "/root/reference/src/sionna/phy/fec/conv/utils.py")
src_text = open(spec.origin).read()
start = src_text.index("def polynomial_selector")
ns = {}
exec(src_text[start:src_text.index("class Trellis")], ns)
table = []
for rate, tag in ((1 / 2, "1/2"), (1 / 3, "1/3")):
    for K in range(3, 9):
        table.append(f"{tag}:{K}:" + ",".join(ns["polynomial_selector"](rate, K)))
out["selector"] = np.array(table)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "conv_golden.npz"), **out)
