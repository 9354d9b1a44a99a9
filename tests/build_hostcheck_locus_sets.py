"""Build tests/_build/locus_sets/libhostcheck_locus_sets.so: the product's HOST sources + the C oracle backend with the set seeding
oracle, exporting mpb_map_locus_sets and the set file driver (tests/hostcheck/hostcheck_locus_sets.cpp; CPU tests of locus sets only)."""
import glob
import os
import subprocess

from build_hostcheck import CSRC, HOST_SRCS, ROOT

OUT = os.path.join(ROOT, "tests", "_build", "locus_sets", "libhostcheck_locus_sets.so")


def build(force=False):
    if os.environ.get("MPB_HOSTCHECK_LOCUS_SETS_SO"):  # a build made elsewhere
        return os.environ["MPB_HOSTCHECK_LOCUS_SETS_SO"]
    hc = os.path.join(ROOT, "tests", "hostcheck")
    srcs = [os.path.join(CSRC, s) for s in HOST_SRCS] + [os.path.join(hc, "hostcheck_locus_sets.cpp")]
    ora = sorted(glob.glob(os.path.join(ROOT, "oracle", "*.c")))
    deps = srcs + ora + [os.path.join(hc, f) for f in ("hostcheck.cpp", "hostcheck_loci.cpp", "hostcheck_loci_file.cpp")] + glob.glob(os.path.join(CSRC, "*.hpp")) + \
        glob.glob(os.path.join(ROOT, "include", "*.h")) + glob.glob(os.path.join(ROOT, "oracle", "*.h"))
    if not force and os.path.exists(OUT) and all(os.path.getmtime(OUT) >= os.path.getmtime(d) for d in deps):
        return OUT
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    objs = []
    for c in ora:
        o = os.path.join(os.path.dirname(OUT), "ora_" + os.path.basename(c) + ".o")
        subprocess.run(["gcc", "-std=c11", "-O2", "-g", "-fPIC", "-c", c, "-o", o], check=True)
        objs.append(o)
    tmp = OUT + ".tmp"
    cmd = ["g++", "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wno-unused-function", "-I" + os.path.join(ROOT, "include"),
           "-I" + CSRC, "-I" + os.path.join(ROOT, "oracle"), "-I" + hc, "-o", tmp] + srcs + objs + ["-lz", "-lpthread", "-lm"]
    subprocess.run(cmd, check=True)
    os.replace(tmp, OUT)
    return OUT


if __name__ == "__main__":
    print(build(force=True))
