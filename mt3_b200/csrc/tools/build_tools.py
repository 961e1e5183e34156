"""Builds the test-only kernel harness library (libmt3kernels.so, loaded by tests/test_kernel_parity.py and
tests/test_decode_loop_kernels.py) next to this file (sm_90a).  A re-run is a no-op when the library is newer than the
kernel sources."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
HARNESS = os.path.join(HERE, "libmt3kernels.so")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr"]


def _stale(out, src):
    csrc = os.path.join(HERE, "..")
    deps = [src, os.path.abspath(__file__)] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".cu"))]
    return not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps)


def harness_stale():
    return _stale(HARNESS, os.path.join(HERE, "kernel_harness.cu"))


def main():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if harness_stale():
        subprocess.run([nvcc, *FLAGS, "-shared", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-o", HARNESS, os.path.join(HERE, "kernel_harness.cu")],
                       check=True)
        print("built", HARNESS)


if __name__ == "__main__":
    sys.exit(main())
