"""GPU: the k-mer index build within a device-memory budget.  mp_idx_load builds on the default context; under a budget its scratch
(24 B per (bucket, block) pair) runs in passes over bucket ranges, and the .mpi must not change at all: byte for byte the automatic
build's and the reference CLI's (stored digests), for DPP3 and the small set at the default options, and for the awkward-contig
FASTA and the tiny set at every index option set the device build takes.  Budgets: the automatic mode (one pass on these genomes),
one half-way between the build's fixed arenas and what the automatic build held (several passes, every one within the budget), and
1 byte (the pass cap).  The budgets stay at a few hundred MB at most; no test fills the device or expects an allocation to fail."""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile

import pytest

import dbg_lib
import miniprot_b200 as mp
import oracle_lib as ol
from miniprot_b200 import synth
from test_gpu_dropin import write_odd_fasta
from test_gpu_index_options import INDEX_SETS, built_on_device, idxopt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
MB = 1 << 20
MAX_PASSES = 64  # kIdxMaxPasses (csrc/slices.hpp)


def default_ctx():
    L = mp.lib()
    L.mpb_ctx_default.restype = C.c_void_p
    return L.mpb_ctx_default()


def mem_stats(h) -> mp.MemStats:
    s = mp.MemStats()
    mp.lib().mpb_get_mem_stats(h, C.byref(s))
    return s


@pytest.fixture
def dctx():
    """The default context, its budget set back to automatic afterwards."""
    h = default_ctx()
    yield h
    assert mp.lib().mpb_ctx_set_mem_budget(h, 0) == 0


@pytest.fixture(scope="module")
def genomes(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("idx_budget"))
    return {"DPP3": ol.DPP3_GENOME, "small": synth.generate(synth.CONFIGS["small"], os.path.join(d, "small"))[0],
            "odd": write_odd_fasta(os.path.join(d, "odd.fa")), "tiny": synth.generate(synth.CONFIGS["tiny"], os.path.join(d, "tiny"))[0]}


def build(h, g, io, budget, path):
    """(.mpi bytes, mem stats) of mp_idx_load on the default context under `budget` (0: automatic).  The context's idle arenas are
    released first (a budget of 1 byte does that), so the peak is the build's own."""
    L = mp.lib()
    assert L.mpb_ctx_set_mem_budget(h, 1) == 0 and L.mpb_ctx_set_mem_budget(h, budget) == 0
    L.mpb_reset_stats(h)
    mi = mp.idx_load(g, 8, io)
    st = mem_stats(h)
    assert L.mp_idx_dump(path.encode(), mi) == 0
    L.mp_idx_destroy(mi)
    return open(path, "rb").read(), st


def middle_budget(st_auto, n_bucket):
    """Half-way between the build's fixed arenas, the bucket counters and starts (12 B per bucket), and what the automatic build
    held.  Automatic mode gives every arena a quarter of slack, so the scratch of its one pass is what it held beyond 15 B per
    bucket.  The small arenas left out (work units, the scan's block sums) only leave the passes a little less room: more of them."""
    return 12 * n_bucket + (st_auto.peak_held - 15 * n_bucket) // 2


CASES = [("DPP3", []), ("small", [])] + [(g, o) for g in ("odd", "tiny") for o in INDEX_SETS if built_on_device(idxopt(o))]


@pytest.mark.parametrize("name,opts", CASES, ids=[f"{g}-{' '.join(o) or 'defaults'}" for g, o in CASES])
def test_build_in_passes(genomes, dctx, tmp_path, name, opts):
    g, io = genomes[name], idxopt(opts)
    path = str(tmp_path / "i.mpi")
    want, st = build(dctx, g, io, 0, path)
    assert ol.file_digest(path) == ol.ref_index_file(g, opts)
    assert (st.n_index_passes, st.n_over_budget, st.budget) == (1, 0, 0)
    mid = middle_budget(st, mp.n_bucket(io))
    assert mid < 400 * MB, mid
    got, st = build(dctx, g, io, mid, path)
    assert got == want, f"{name} {opts}: the .mpi differs under a budget of {mid} bytes"
    assert st.n_index_passes >= 2 and st.n_over_budget == 0, (mid, st.n_index_passes, st.n_over_budget)
    assert st.peak_held <= mid, (st.peak_held, mid)
    got, st = build(dctx, g, io, 1, path)
    assert got == want, f"{name} {opts}: the .mpi differs under a budget of 1 byte"
    assert 1 < st.n_index_passes <= MAX_PASSES and st.n_over_budget > 0, (st.n_index_passes, st.n_over_budget)


def test_counters_reset(dctx, genomes, tmp_path):
    """mpb_reset_stats clears n_index_passes; every build adds its passes."""
    L = mp.lib()
    io = mp.idxopt()
    build(dctx, genomes["tiny"], io, 0, str(tmp_path / "a.mpi"))
    for _ in range(2):
        mi = mp.idx_load(genomes["tiny"], 8, io)
        L.mp_idx_destroy(mi)
    assert mem_stats(dctx).n_index_passes == 3
    L.mpb_reset_stats(dctx)
    assert mem_stats(dctx).n_index_passes == 0


def test_cli_maps_on_an_index_built_in_passes():
    """The CLI's path under MPB_DEVICE_MEM: mp_idx_load builds the tiny5 index from FASTA in several passes on the default context,
    and mp_map_file on it prints the reference's PAF."""
    with tempfile.TemporaryDirectory() as d:
        g, p = synth.generate(synth.CONFIGS["tiny5"], d)
        child = dbg_lib._CHILD.replace('C.c_int32.in_dll(L, "mp_verbose").value = 1', 'C.c_int32.in_dll(L, "mp_verbose").value = 3')
        assert child != dbg_lib._CHILD
        r = subprocess.run([sys.executable, "-c", child, ROOT, mp.LIB_PATH, g, p], capture_output=True, env=dict(os.environ, MPB_DEVICE_MEM="1k"),
                           timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout == open(os.path.join(GOLD, "tiny5.paf"), "rb").read()
    m = re.search(rb"built the k-mer tables on the device in [0-9.]+ s: \d+ kmer-block pairs in (\d+) passes", r.stderr)
    assert m and 1 < int(m.group(1)) <= MAX_PASSES, r.stderr[-2000:]
