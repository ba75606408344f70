"""Build libsionna_b200.so in-tree with nvcc for sm_90a (no torch extension machinery needed:
the boundary is a plain C-ABI loaded with ctypes).

    python -m sionna_b200.csrc.build [--force]

Every source is compiled on its own (in parallel) and linked into one shared library. The LDPC / mapping sources are
built with -fmad=false: their arithmetic is specified operation by operation (explicit __f*_rn / fmaf calls) so that the
CPU oracle reproduces it bit for bit, and the compiler must not contract a*b+c on its own. The flat-fading source is
built the same way so that its random draws and noise equal sb_awgn's (phy_kernels.cu) bit for bit, and the convolutional
decoders so that their Viterbi path metrics equal the float32 oracle's bit for bit. The OFDM / MIMO / channel
sources are tolerance-checked floating-point kernels (FFT butterflies, complex MACs, Cholesky): they are built with the
default -fmad=true, which halves their instruction count.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "..", "libsionna_b200.so")
OBJ_DIR = os.path.join(HERE, "..", "..", "build", "obj")
EXACT = ["common.cu", "ldpc_bp.cu", "ldpc_bp_qc.cu", "ldpc_bp_flat.cu", "ldpc_enc.cu", "phy_kernels.cu",
         "flat_fading.cu", "conv.cu"]                                                                        # -fmad=false
FAST = ["ofdm_mimo.cu", "channel.cu", "frontend.cu", "mimo_ml.cu", "mimo_kbest.cu",
        "mimo_iterative.cu", "precoding.cu"]                                                     # -fmad=true
SOURCES = EXACT + FAST
HEADERS = ["sb_common.h", "sb_math.h", "sb_math2.cuh", "sb_logtab.h", "rng.cuh", "ldpc_graph.h", "ldpc_rules.cuh",
           "lmmse_diag.cuh", "dense_mimo.cuh", "demap_qam.cuh", "demap_prior.cuh", os.path.join("..", "..", "include", "sionna_b200.h")]
COMMON_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-Xcompiler", "-ffp-contract=off", "-Xptxas", "-v",
]


def _stale(lib, deps):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source into ``sionna_b200/libsionna_b200.so``; returns the library path."""
    srcs = [os.path.join(HERE, s) for s in SOURCES]
    hdrs = [os.path.join(HERE, h) for h in HEADERS]
    deps = srcs + hdrs + [os.path.abspath(__file__)]
    lib = os.path.abspath(LIB)
    if not force and not _stale(lib, deps):
        return lib
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(OBJ_DIR, exist_ok=True)
    newest_hdr = max(os.path.getmtime(h) for h in hdrs + [os.path.abspath(__file__)])

    def compile_one(name):
        src = os.path.join(HERE, name)
        obj = os.path.join(OBJ_DIR, name.replace(".cu", ".o"))
        log = obj + ".log"
        if not force and os.path.exists(obj) and os.path.exists(log) and \
                os.path.getmtime(obj) >= max(os.path.getmtime(src), newest_hdr):
            return name, 0, open(log).read()
        tmp = f"{obj}.tmp.{os.getpid()}"
        cmd = [nvcc] + COMMON_FLAGS + ["-fmad=false" if name in EXACT else "-fmad=true", "-c", "-o", tmp, src]
        res = subprocess.run(cmd, capture_output=True, text=True)
        text = res.stdout + res.stderr
        if res.returncode == 0:
            os.replace(tmp, obj)
            with open(log, "w") as f:
                f.write(text)
        elif os.path.exists(tmp):
            os.remove(tmp)
        return name, res.returncode, text

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    logs = "".join(f"==== {n} ====\n{t}" for n, _, t in results)
    failed = [n for n, rc, _ in results if rc != 0]
    if verbose or failed:
        sys.stderr.write(logs)
    if failed:
        raise RuntimeError("nvcc failed on " + ", ".join(failed))
    tmp = f"{lib}.tmp.{os.getpid()}"                        # atomic publish: concurrent builders (one per rank) cannot
    objs = [os.path.join(OBJ_DIR, s.replace(".cu", ".o")) for s in SOURCES]   # expose a half-written library
    res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-o", tmp] + objs,
                         capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed linking libsionna_b200.so")
    os.replace(tmp, lib)
    with open(os.path.join(HERE, "..", "build_ptxas.log"), "w") as f:
        f.write(logs)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
