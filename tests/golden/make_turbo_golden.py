"""Pack the reference's turbo-code test vectors (test/codes/turbo/ref_k{40,112,168,432}_{u,x,y,uhat}.npy: LTE code,
constraint length 4, rate 1/3, terminated, 3GPP interleaver) into turbo_golden.npz: u, x and uhat bit-packed along the
last axis, y as float32, and each k. Data only.

    python tests/golden/make_turbo_golden.py [REFERENCE_ROOT]
"""
import os
import sys

import numpy as np

ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
src = os.path.join(ref, "test", "codes", "turbo")
out = {}
for k in (40, 112, 168, 432):
    for name in ("u", "x", "uhat"):
        a = np.load(os.path.join(src, f"ref_k{k}_{name}.npy"))
        out[f"{name}_{k}"] = np.packbits(a.astype(np.uint8), axis=-1)
        out[f"len_{name}_{k}"] = np.int32(a.shape[-1])
    out[f"y_{k}"] = np.load(os.path.join(src, f"ref_k{k}_y.npy")).astype(np.float32)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "turbo_golden.npz"), **out)
print({key: v.shape for key, v in out.items() if key.startswith(("u_", "y_"))})
