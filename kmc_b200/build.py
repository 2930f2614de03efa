"""Builds kmc_b200/libkmc_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache: the .so is built once, next to the package)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "kmc_b200.cu")
DEPS = sorted(os.path.join(HERE, "csrc", f) for f in os.listdir(os.path.join(HERE, "csrc")) if f.endswith((".cu", ".cuh", ".inl"))) + [
    os.path.join(os.path.dirname(HERE), "include", "kmc_b200.h")]
OUT = os.path.join(HERE, "libkmc_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# -ffp-contract=off: the host code rounds every product and sum on its own, as the reference's CPU code does (the estimator's recursion)
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
         "-Xcompiler", "-fvisibility=default", "-Xcompiler", "-ffp-contract=off"]


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s and %s is missing or stale" % (NVCC, OUT))
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT, SRC]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))


def build_variant(name, extra_flags):
    """Experiment builds (compile-time knobs) next to the product library: build/libkmc_b200_<name>.so, selected by scripts/ via KMCB200_LIB."""
    d = os.path.join(os.path.dirname(HERE), "build")
    os.makedirs(d, exist_ok=True)
    out = os.path.join(d, "libkmc_b200_%s.so" % name)
    subprocess.check_call([NVCC] + FLAGS + list(extra_flags) + ["-o", out, SRC])
    return out
