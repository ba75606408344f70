"""Run the reference's own make_systematic / pcm2gm (fec/utils.py, executed from the reference's source with NumPy, the
rest of that module not imported) on example code 3, the (3,6)-regular LDPC code that needs column swaps, and store
the generator (bit-packed along the last axis) and the column swaps in linear_golden.npz. Data only.

    python tests/golden/make_linear_golden.py [REFERENCE_ROOT]
"""
import ast
import os
import sys
import warnings

import numpy as np

ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
here = os.path.dirname(os.path.abspath(__file__))
src = open(os.path.join(ref, "src", "sionna", "phy", "fec", "utils.py")).read()
tree = ast.parse(src)
funcs = [f for f in tree.body if isinstance(f, ast.FunctionDef) and f.name in ("make_systematic", "pcm2gm",
                                                                                "verify_gm_pcm")]
ns = {"np": np, "warnings": warnings}
exec(compile(ast.Module(body=funcs, type_ignores=[]), "utils.py", "exec"), ns)
with np.load(os.path.join(here, "..", "..", "sionna_b200", "phy", "fec", "ldpc", "codes", "example_pcms.npz")) as d:
    pcm = np.array(d["pcm3"], dtype=np.int64)
_, swaps = ns["make_systematic"](pcm, is_pcm=True)
gm = ns["pcm2gm"](pcm).astype(np.uint8)
np.savez_compressed(os.path.join(here, "linear_golden.npz"), gm3=np.packbits(gm, axis=-1), n3=np.int32(gm.shape[1]),
                    swaps3=np.array(swaps, np.int32))
print(gm.shape, len(swaps))
