"""Build the in-tree CUDA extension (C-ABI shared library) for sm_90a (H100) with nvcc.

    python -m lookoncetohear_b200.build [--force]

The .so lands in lookoncetohear_b200/lib/ (git-ignored build product).  nvcc cross-compiles without a GPU.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "liblookonce_b200.so")
SOURCES = ["sep_engine.cu", "embed_engine.cu", "umma_gemm.cu", "eval_metrics.cu", "render.cu", "resample.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--compiler-options", "-fPIC", "-shared", "-Xptxas", "-v"]


# test-only library: direct C entry points into the tensor-core GEMM and the LSTM recurrences (tests/kernels/).
# Hidden visibility + -Bsymbolic: its copy of the engine's symbols never binds to the product library's copy.
HARNESS_SRC = os.path.join(os.path.dirname(HERE), "tests", "kernels", "kernel_harness.cu")
HARNESS_LIB = os.path.join(LIBDIR, "libl2h_kernel_harness.so")
HARNESS_FLAGS = ["--compiler-options", "-fvisibility=hidden", "-Xlinker", "-Bsymbolic", "-I", CSRC]


def _fingerprint(extra_files=(), extra_flags=()):
    h = hashlib.sha256()
    inc = os.path.join(os.path.dirname(HERE), "include")
    for d in (CSRC, inc):
        for fn in sorted(os.listdir(d)):
            if fn.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(d, fn), "rb") as f:
                    h.update(fn.encode())
                    h.update(f.read())
    for p in extra_files:
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode())
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS + list(extra_flags)).encode())
    return h.hexdigest()


def nvcc_path():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isfile(c) or c == "nvcc"):
            return c
    return "nvcc"


def _compile(out, sources, fp, extra_flags, log_name, force, verbose):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = out + ".sha256"
    if not force and os.path.isfile(out) and os.path.isfile(stamp) and open(stamp).read().strip() == fp:
        return out
    cmd = [nvcc_path()] + NVCC_FLAGS + list(extra_flags) + ["-o", out] + list(sources)
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(LIBDIR, log_name), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-4000:])
    if verbose:
        print(log)
    with open(stamp, "w") as f:
        f.write(fp)
    return out


def build(force=False, verbose=False):
    """Compile if sources changed since the last build.  Returns the library path."""
    return _compile(LIB, [os.path.join(CSRC, s) for s in SOURCES], _fingerprint(), [], "build.log", force, verbose)


def build_harness(force=False, verbose=False):
    """The test-only kernel harness library (same flags as the product library), if its sources changed."""
    fp = _fingerprint([HARNESS_SRC], HARNESS_FLAGS)
    return _compile(HARNESS_LIB, [HARNESS_SRC], fp, HARNESS_FLAGS, "build_harness.log", force, verbose)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_harness(force="--force" in sys.argv, verbose="-v" in sys.argv))
