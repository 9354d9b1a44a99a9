"""GPU: the debugging switches of the CLI (mp_dbg_flag) on the CUDA stages.  mp_map_file (hence mpb_map_file, and
mpb_map_file_multi under MPB_DEVICES) must print what the reference CLI prints with -t1 -- stdout and the QR / X / Y1 dump lines on
stderr, byte for byte; mpb_map_batch and mp_map the same dump lines, mp_map without QR lines.  --dbg-aflt on a slice of the
long-intron configuration gives the DP kernels whole-region global alignments of several hundred kb of rows."""
import os
import subprocess
import sys

import pytest

import dbg_lib
import miniprot_b200 as mp
import oracle_lib as ol

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    return dbg_lib.input_sets(str(tmp_path_factory.mktemp("dbg")))


def check(args, g, p, env=None):
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, args, g, p, env)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    assert dbg_lib.digest(out, err) == dbg_lib.ref_cli_dbg(args, g, p)
    return out, err


@pytest.mark.parametrize("switches", [" ".join(s) for s in dbg_lib.SWITCH_SETS])
@pytest.mark.parametrize("name", ["DPP3", "tiny", "tiny5", "short_ctg"])
def test_switches_golden(sets, name, switches):
    g, p = sets[name]
    check(switches.split(), g, p)


def test_aflt_splice_scores(tmp_path):
    check(["--dbg-aflt", "--spsc", dbg_lib.spsc_file(str(tmp_path))], ol.DPP3_GENOME, ol.DPP3_PROTEIN)


def test_no_refine_without_no_align_refused(sets):
    g, p = sets["tiny"]
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, ["--dbg-no-refine"], g, p)
    assert rc == -3 and out == b"" and b"--dbg-no-refine" in err


_BATCH_CHILD = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
import miniprot_b200 as mp
L = mp.lib()
mode, g, p = sys.argv[2:5]
names, seqs = [], []
for line in open(p):
    if line.startswith(">"): names.append(line[1:].split()[0]); seqs.append("")
    else: seqs[-1] += line.strip()
mi = mp.idx_load(g, 4)
mo = mp.mapopt()
mp.set_dbg_flag(mp.DBG_QNAME | mp.DBG_ANCHOR | mp.DBG_CHAIN)
L.mpb_map_batch.argtypes = [C.c_void_p, C.POINTER(mp.Idx), C.POINTER(mp.MapOpt), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
L.mpb_regs_free.argtypes = [C.c_int32, C.c_void_p, C.c_void_p]
L.mp_map.restype = C.c_void_p
L.mp_map.argtypes = [C.POINTER(mp.Idx), C.c_int, C.c_char_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(mp.MapOpt), C.c_char_p]
n = len(seqs)
if mode == "batch":
    c_seqs = (C.c_char_p * n)(*[s.encode() for s in seqs])
    c_names = (C.c_char_p * n)(*[s.encode() for s in names])
    c_lens = (C.c_int32 * n)(*[len(s) for s in seqs])
    n_reg, regs = (C.c_int32 * n)(), (C.c_void_p * n)()
    ctx = mp.Context(0)
    assert L.mpb_map_batch(ctx.h, mi, C.byref(mo), n, c_seqs, c_lens, c_names, n_reg, regs) == 0
    L.mpb_regs_free(n, n_reg, regs)
else:
    for s, nm in zip(seqs, names):
        nr = C.c_int(0)
        r = L.mp_map(mi, len(s), s.encode(), C.byref(nr), None, C.byref(mo), nm.encode())
        L.mpb_regs_free(1, C.byref(C.c_int32(nr.value)), C.byref(C.c_void_p(r)))
sys.stderr.flush()
"""


def test_map_batch_and_mp_map(sets):
    """mpb_map_batch prints the dump of mp_map_file (one mini-batch, QR tid 0); mp_map the same X / Y1 lines and no QR line, as
    the reference's mp_map does."""
    g, p = sets["tiny"]
    args = ["--dbg-qname", "--dbg-anchor", "--dbg-chain"]
    _, err = check(args, g, p)
    want = dbg_lib.dump_lines(err)
    got = {}
    for mode in ("batch", "single"):
        r = subprocess.run([sys.executable, "-c", _BATCH_CHILD, dbg_lib.ROOT, mode, g, p], capture_output=True, timeout=1800)
        assert r.returncode == 0, r.stderr.decode(errors="replace")[-2000:]
        got[mode] = dbg_lib.dump_lines(r.stderr)
    assert got["batch"] == want
    assert got["single"] == [l for l in want if not l.startswith(b"QR\t")]


def per_protein(lines):
    """Dump lines cut into one chunk per protein (a QR line and what follows it), QR tid blanked; and the tid of each chunk."""
    chunks, tids = [], []
    for l in lines:
        if l.startswith(b"QR\t"):
            f = l.rstrip(b"\n").split(b"\t")
            tids.append(int(f[3]))
            chunks.append([b"\t".join(f[:3]) + b"\n"])
        else:
            chunks[-1].append(l)
    return [b"".join(c) for c in chunks], tids


def test_two_contexts_one_device(sets):
    """MPB_DEVICES=0,0: stdout as with one context; the dump lines the same multiset, every protein's lines in one piece, QR tid the
    index of the context that mapped the protein, and both contexts at work (units of about 1000 residues)."""
    g, p = sets["tiny"]
    args = ["--dbg-qname", "--dbg-anchor", "--dbg-chain", "-K2000"]
    rc, out1, err1 = dbg_lib.run_cli(mp.LIB_PATH, args, g, p)
    assert rc == 0
    env = dict(os.environ, MPB_DEVICES="0,0")
    rc, out2, err2 = dbg_lib.run_cli(mp.LIB_PATH, args, g, p, env)
    assert rc == 0 and out2 == out1
    c1, t1 = per_protein(dbg_lib.dump_lines(err1))
    c2, t2 = per_protein(dbg_lib.dump_lines(err2))
    assert sorted(dbg_lib.dump_lines(err2)) != [] and len(c2) == len(c1) == 40
    assert sorted(c2) == sorted(c1) and set(t1) == {0} and set(t2) == {0, 1}
    # the proteins of one unit follow each other in input order: a chunk is preceded by its predecessor in the input unless the
    # context changes there or a new unit of the same context starts
    order = {c: i for i, c in enumerate(c1)}
    breaks = sum(1 for k in range(1, len(c2)) if order[c2[k]] != order[c2[k - 1]] + 1)
    assert breaks < len(c2) // 2


def test_aflt_long_introns(tmp_path):
    """--dbg-aflt on the first proteins of the scaled long-intron configuration (50-150 kb introns): one global alignment per region
    over several hundred kb of rows, on the column-pass traceback path, byte-identical to the reference."""
    g, p = dbg_lib.c4_slice(str(tmp_path))
    env = dict(os.environ, MPB_TRACE="1")
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, ["--dbg-aflt"], g, p, env)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    assert dbg_lib.digest(out, err) == dbg_lib.ref_cli_dbg(["--dbg-aflt"], g, p)
    longest = max(int(l.split(b"longest nl=")[1].split()[0]) for l in err.splitlines() if b"nasw tb " in l)
    assert longest > 100_000, longest
