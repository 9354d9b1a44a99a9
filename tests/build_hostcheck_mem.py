"""Build tests/_build/mem/libhostcheck_mem.so: the slice planner and MPB_DEVICE_MEM parser of the device-memory budget
(miniprot_b200/csrc/slices.hpp, exported by tests/hostcheck/hostcheck_mem.cpp; CPU tests only)."""
import os
import subprocess

from build_hostcheck import CSRC, ROOT

OUT = os.path.join(ROOT, "tests", "_build", "mem", "libhostcheck_mem.so")


def build(force=False):
    src = os.path.join(ROOT, "tests", "hostcheck", "hostcheck_mem.cpp")
    deps = [src, os.path.join(CSRC, "slices.hpp")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in deps):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    tmp = OUT + ".tmp"
    subprocess.run(["g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-I" + CSRC, "-o", tmp, src], check=True)
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(force=True))
