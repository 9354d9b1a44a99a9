"""Build tests/_build/idx_passes/libhostcheck_idx_passes.so: the pass planner of the device index build (plan_bucket_passes in
miniprot_b200/csrc/slices.hpp, exported by tests/hostcheck/hostcheck_idx_passes.cpp; CPU tests only).  It is compiled by nvcc for
sm_90a, as the library's sources that include slices.hpp are, so the header is checked under the compiler that builds the index."""
import os
import shutil
import subprocess

from build_hostcheck import CSRC, ROOT

OUT = os.path.join(ROOT, "tests", "_build", "idx_passes", "libhostcheck_idx_passes.so")


def nvcc():
    return shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")


def build(force=False):
    src = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_idx_passes.cpp")
    deps = [src, os.path.join(CSRC, "slices.hpp")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in deps):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    tmp = OUT + ".tmp"
    subprocess.run([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-x", "cu", "-shared", "-Xcompiler", "-fPIC,-Wall",
                    "-I" + CSRC, "-o", tmp, src], check=True)
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(force=True))
