"""Run the reference's own pulse formulas (RaisedCosineFilter._raised_cosine, RootRaisedCosineFilter._root_raised_cosine,
SincFilter._sinc) and window builds (HannWindow / HammingWindow / BlackmanWindow.build), executed from the reference's
source with NumPy only (the rest of those modules not imported), over a grid that hits every singular point, and store
the coefficients in signal_golden.npz. Data only.

    python tests/golden/make_signal_golden.py [REFERENCE_ROOT]

Keys: "{rc,rrc}_b{beta}_s{sps}_n{span}" and "sinc_s{sps}_n{span}" (float32, sample times of a filter of span * sps
taps forced odd), "{hann,hamming,blackman}_{length}" (the window's coefficients as built, float64).
"""
import ast
import os
import sys

import numpy as np

ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
here = os.path.dirname(os.path.abspath(__file__))
sig = os.path.join(ref, "src", "sionna", "phy", "signal")


def methods(fname, wanted):
    """{(class, method): function} of the named methods of the module's classes, compiled without the module."""
    tree = ast.parse(open(os.path.join(sig, fname)).read())
    out = {}
    for cls in tree.body:
        if isinstance(cls, ast.ClassDef):
            for f in cls.body:
                if isinstance(f, ast.FunctionDef) and (cls.name, f.name) in wanted:
                    ns = {"np": np}
                    exec(compile(ast.Module(body=[f], type_ignores=[]), fname, "exec"), ns)
                    out[(cls.name, f.name)] = ns[f.name]
    return out


pulses = methods("filter.py", {("RaisedCosineFilter", "_raised_cosine"), ("RootRaisedCosineFilter", "_root_raised_cosine"),
                               ("SincFilter", "_sinc")})
windows = methods("window.py", {("HannWindow", "build"), ("HammingWindow", "build"), ("BlackmanWindow", "build")})


class _Holder:
    coefficients = None


out = {}
lengths = set()
for sps in (1, 2, 3, 4, 8):
    for span in (1, 7, 8, 32):
        length = 2 * (span * sps // 2) + 1
        lengths.add(length)
        t = (np.arange(-(length // 2), length - length // 2, dtype=np.float32) / np.float32(sps)).astype(np.float32)
        out[f"sinc_s{sps}_n{span}"] = np.asarray(pulses[("SincFilter", "_sinc")](None, t, 1.0), np.float32)
        for beta in (0, 0.25, 0.5, 1):
            out[f"rc_b{beta}_s{sps}_n{span}"] = pulses[("RaisedCosineFilter", "_raised_cosine")](None, t, 1.0, beta)
            out[f"rrc_b{beta}_s{sps}_n{span}"] = pulses[("RootRaisedCosineFilter", "_root_raised_cosine")](None, t, 1.0,
                                                                                                        beta)
for length in sorted(lengths | {2, 16}):
    for name in ("Hann", "Hamming", "Blackman"):
        h = _Holder()
        windows[(f"{name}Window", "build")](h, (length,))
        out[f"{name.lower()}_{length}"] = np.asarray(h.coefficients, np.float64)
np.savez_compressed(os.path.join(here, "signal_golden.npz"), **out)
print(len(out), "arrays")
