"""GPU: mapping within a device-memory budget (mpb_ctx_set_mem_budget, MPB_DEVICE_MEM).  The seeding, refinement and DP stages run in
slices whose arenas fit the budget; the output must not change at all: byte for byte the unbudgeted context's and the stored goldens,
for every output format, the --dbg-* dumps, locus mode and the stage entry points.  The budgets are small (a few MB), so the tests
are light on a shared device; none of them fills the device or expects an allocation to fail."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import dbg_lib
import loci_file_lib
import loci_lib
import miniprot_b200 as mp
import oracle_lib as ol
from miniprot_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLD = os.path.join(ROOT, "tests", "golden")
MB = 1 << 20
# PAF, --gff, --aln, --trans, -u (MP_F_GFF, MP_F_SHOW_RESIDUE, MP_F_SHOW_TRANS, MP_F_SHOW_UNMAP)
FORMATS = {"paf": 0, "gff": 0x8, "aln": 0x80, "trans": 0x100, "unmap": 0x4}
GOLDENS = {("tiny5", "paf"): "tiny5.paf", ("tiny5", "gff"): "tiny5_gff.txt", ("DPP3", "paf"): "DPP3_default.paf", ("DPP3", "gff"): "DPP3_gff.txt"}


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("mem"))
    out = {"DPP3": (ol.DPP3_GENOME, ol.DPP3_PROTEIN)}
    for cfg in ("tiny5", "small"):
        out[cfg] = synth.generate(synth.CONFIGS[cfg], os.path.join(d, cfg))
    idx = {k: mp.idx_load(g, 8) for k, (g, _) in out.items()}
    yield out, idx, d
    for mi in idx.values():
        mp.lib().mp_idx_destroy(mi)


def budget_ctx(budget):
    c = mp.Context(0)
    assert c.set_mem_budget(budget) == 0
    return c


def map_with(budget, mi, p, out, flag=0):
    """(output bytes, mem stats) of mpb_map_file on a fresh context with this budget (0: automatic)"""
    c = budget_ctx(budget)
    mo = mp.mapopt()
    mo.flag |= flag
    mp.map_file(c, mi, p, out, mo)
    st = c.mem_stats()
    c.close()
    return open(out, "rb").read(), st


def check_within(st, budget):
    """a budget that every item fits on its own is kept: the arenas never held more than it at once"""
    if budget and st.n_over_budget == 0:
        assert st.peak_held <= budget, (st.peak_held, budget)


@pytest.mark.parametrize("name,budgets", [("tiny5", [8 * MB, 4 * MB, 2 * MB, 1]), ("DPP3", [4 * MB, 2 * MB, 1])])
@pytest.mark.parametrize("fmt", sorted(FORMATS))
def test_formats_identical(sets, name, budgets, fmt):
    (files, idx, d) = sets
    g, p = files[name]
    out = os.path.join(d, f"{name}_{fmt}.out")
    want, _ = map_with(0, idx[name], p, out, FORMATS[fmt])
    if (name, fmt) in GOLDENS:
        assert want == open(os.path.join(GOLD, GOLDENS[name, fmt]), "rb").read()
    for b in budgets:
        got, st = map_with(b, idx[name], p, out, FORMATS[fmt])
        assert got == want, f"{name} {fmt}: output differs under a budget of {b} bytes"
        check_within(st, b)


def test_slices_in_every_stage(sets):
    """The small set at budgets of a few MB: more than one slice in S1, S2 and S3 with every item within the budget, and the peak
    within it; then one protein per S1 slice."""
    (files, idx, d) = sets
    g, p = files["small"]
    out = os.path.join(d, "small.paf")
    want, st0 = map_with(0, idx["small"], p, out)
    assert st0.n_slices_seed == 1 and st0.n_slices_refine == 1 and st0.n_released == 0  # one batch, room to spare
    seen = []
    for b in (32 * MB, 24 * MB, 16 * MB, 12 * MB):
        got, st = map_with(b, idx["small"], p, out)
        assert got == want, b
        check_within(st, b)
        seen.append((st.n_over_budget, st.n_slices_seed, st.n_slices_refine, st.n_subwaves))
    assert any(o == 0 and s1 > 1 and s2 > 1 and s3 > st0.n_subwaves for o, s1, s2, s3 in seen), seen
    got, st = map_with(1, idx["small"], p, out)
    n_prot = sum(1 for line in open(p) if line.startswith(">"))
    assert got == want and st.n_slices_seed == n_prot and st.n_over_budget > 0


def test_automatic_c2_one_slice_no_release(tmp_path_factory):
    """Automatic mode on C2 (100 Mbp, 1000 proteins, one mini-batch at the default -K): one slice in every stage, nothing released,
    nothing over -- the path bench.py measures -- in the first run, which grows the arenas, and in the second, which fits them."""
    base = os.environ.get("MPB_BENCH_DIR") or str(tmp_path_factory.mktemp("c2"))
    g, p = synth.generate(synth.CONFIGS["C2"], os.path.join(base, "C2"))
    mi = mp.idx_load(g, 8)
    c = mp.Context(0)
    for _ in range(2):
        c.reset_stats()
        mp.map_file(c, mi, p, os.path.join(str(tmp_path_factory.mktemp("c2o")), "o.paf"))
        st = c.mem_stats()
        assert (st.n_slices_seed, st.n_slices_refine, st.n_released, st.n_over_budget, st.budget) == (1, 1, 0, 0, 0)
        assert st.n_subwaves == 3  # the three DP waves, none cut
    c.close()
    mp.lib().mp_idx_destroy(mi)


def test_c3s_sliced_matches_reference(tmp_path_factory):
    """The 3 Gbp / -I shape cut to 1 Gbp (~48 k anchors per protein, the large chaining class) at a 2 GiB budget: the 2000
    proteins' seeding and chaining run in at least four slices, and the PAF is still the reference CLI's (stored digest)."""
    import parity

    base = os.environ.get("MPB_BENCH_DIR") or str(tmp_path_factory.mktemp("cfg"))
    c = budget_ctx(2 << 30)
    rows = parity.run_config("C3s", ["-I"], os.path.join(base, "C3s"), min(os.cpu_count() or 8, 128), ctx=c)
    st = c.mem_stats()
    c.close()
    assert rows[0]["identical"], "C3s -I: PAF differs from the reference under a 2 GiB budget"
    assert rows[0]["anchors_per_protein"] > 16384 and st.n_slices_seed >= 4, (rows[0]["anchors_per_protein"], st.n_slices_seed)
    check_within(st, 2 << 30)


def test_automatic_one_slice_no_release(sets):
    """Automatic mode with room to spare: one slice per stage and batch, nothing released, nothing over."""
    (files, idx, d) = sets
    g, p = files["tiny5"]
    c = mp.Context(0)
    mo = mp.mapopt(mini_batch_size=5000)
    for _ in range(2):
        c.reset_stats()
        mp.map_file(c, idx["tiny5"], p, os.path.join(d, "auto.paf"), mo)
        st = c.mem_stats()
        n_batch = st.n_slices_seed  # one slice per batch
        assert n_batch > 1 and 0 < st.n_slices_refine <= n_batch and st.n_released == 0 and st.n_over_budget == 0 and st.budget == 0
        assert st.held == st.peak_held and st.allowance > st.held
    c.close()


def test_two_budgeted_contexts(sets):
    """Two contexts on device 0, each with a budget that slices its seeding, through mpb_map_file_multi: the same bytes."""
    (files, idx, d) = sets
    g, p = files["small"]
    want, _ = map_with(0, idx["small"], p, os.path.join(d, "m0.paf"))
    cs = [budget_ctx(3 * MB), budget_ctx(2 * MB)]
    out = os.path.join(d, "m2.paf")
    unit = 30000
    mp.map_file_multi(cs, idx["small"], p, out, mp.mapopt(mini_batch_size=2 * unit))
    assert open(out, "rb").read() == want
    st = [c.mem_stats() for c in cs]
    for c, s, b in zip(cs, st, (3 * MB, 2 * MB)):
        check_within(s, b)
        c.close()
    # units hold at most `unit` residues of whole proteins, so there are fewer than 2 * (residues / unit + 1) of them; a slice of
    # S1 holds a few dozen proteins at these budgets, i.e. several per unit
    residues = sum(len(s) for _, s in loci_lib.read_fasta(p))
    assert all(s.n_slices_seed > 0 for s in st)
    assert sum(s.n_slices_seed for s in st) > 2 * (residues // unit + 1), [s.n_slices_seed for s in st]


@pytest.fixture(scope="module")
def loci_cases(tmp_path_factory):
    return loci_lib.build_cases(str(tmp_path_factory.mktemp("mem_loci")))


@pytest.mark.parametrize("case", ["tiny", "DPP3"])
def test_map_loci(loci_cases, case):
    cs = loci_cases[case]
    mi = mp.idx_load(cs["genome"], 8)
    names, seqs, qid = loci_lib.index_of(cs)
    loci = loci_lib.loci_tuples(mi, cs, qid)
    mo = mp.mapopt()
    pafs, stats = [], []
    for b in (0, 2 * MB, 1):
        c = budget_ctx(b)
        rc, n_reg, reg = mp.map_loci(c, mi, mo, seqs, names, loci)
        assert rc == 0
        pafs.append(mp.loci_paf(mi, mo, seqs, names, loci, n_reg, reg))
        mp.free_loci_regs(n_reg, reg)
        stats.append(c.mem_stats())
        check_within(stats[-1], b)
        c.close()
    assert pafs[1] == pafs[0] and pafs[2] == pafs[0]
    assert loci_lib.digest(pafs[0]) == loci_lib.ref_answer(cs)
    assert stats[2].n_slices_loci == len(loci) and stats[0].n_slices_loci == 1
    mp.lib().mp_idx_destroy(mi)


def test_map_loci_file(loci_cases, tmp_path):
    cs = loci_cases["tiny"]
    mi = mp.idx_load_genome(cs["genome"])
    tsv = loci_file_lib.write_tsv(str(tmp_path / "l.tsv"), cs["loci"])
    outs = []
    for b in (0, 1):
        c = budget_ctx(b)
        mo = mp.mapopt()
        mo.flag |= 0x8
        out = str(tmp_path / f"o{b}.gff")
        mp.map_loci_file(c, mi, cs["proteins"], tsv, out, mo)
        outs.append(open(out, "rb").read())
        c.close()
    assert outs[0] == outs[1] and outs[0].count(b"\n") > 1
    mp.lib().mp_idx_destroy(mi)


def test_stage_entries(sets, loci_cases):
    """mpb_seed_batch, mpb_seed_loci_batch, mpb_refine_batch and mpb_nasw_batch under a budget of one item per slice give the
    unbudgeted arrays, array for array."""
    (files, idx, d) = sets
    g, p = files["tiny5"]
    mi = idx["tiny5"]
    recs = loci_lib.read_fasta(p)
    seqs = [s for _, s in recs]
    qid_of = {n: k for k, (n, _) in enumerate(recs)}
    nt = mi.contents.nt.contents
    ctg = {nt.ctg[i].name: (i, nt.ctg[i].len) for i in range(nt.n_ctg)}
    wins = []
    for line in open(os.path.join(GOLD, "tiny5.paf"), "rb"):
        f = line.split(b"\t")
        q = qid_of[f[0]]
        cid, clen = ctg[f[5]]
        ts, te = max(0, int(f[7]) - 2000), min(clen, int(f[8]) + 2000)
        rev = f[4] == b"-"
        wins.append((q, cid << 1 | rev, clen - te if rev else ts, clen - ts if rev else te))
    cs = loci_cases["tiny"]
    lmi = mp.idx_load(cs["genome"], 8)
    names, lseqs, qid = loci_lib.index_of(cs)
    loci = loci_lib.loci_tuples(lmi, cs, qid)
    rng = np.random.default_rng(3)
    opt = mp.nsopt()
    probs = []
    for it in range(40):
        a, b = ol.random_dp_problem(rng, al_max=(40, 150)[it % 2], flank=60)
        if len(a) >= 3:
            probs.append((a, b, (1, 4, 2)[it % 3], opt.io))
    res = []
    for b in (0, 1):
        c = budget_ctx(b)
        r = [mp.seed_batch(c, mi, 20000, seqs), mp.seed_loci_batch(c, lmi, 20000, lseqs, loci), mp.refine_batch(c, mi, mp.mapopt(), seqs, wins),
             mp.nasw_batch(c, opt, probs)]
        st = c.mem_stats()
        res.append((r, st))
        c.close()
    (want, st0), (got, st1) = res
    for a, b in zip(want[0] + want[1], got[0] + got[1]):
        assert np.array_equal(a, b)
    assert len(want[2]) == len(got[2]) and all(np.array_equal(a[0], b[0]) and a[1] == b[1] for a, b in zip(want[2], got[2]))
    assert want[3] == got[3]
    assert st1.n_slices_seed == len(seqs) and st1.n_slices_loci == len(loci) and st1.n_slices_refine == len(wins)
    assert st1.n_subwaves >= len(probs) and st1.n_over_budget > 0
    mp.lib().mp_idx_destroy(lmi)


_CHILD = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
import miniprot_b200 as mp
L = mp.lib()
s = mp.MemStats()
L.mpb_ctx_default.restype = C.c_void_p
L.mpb_get_mem_stats(L.mpb_ctx_default(), C.byref(s))
print(s.budget, s.n_slices_seed, s.n_slices_refine)
"""


def test_env_budget_reaches_the_default_context(sets):
    """MPB_DEVICE_MEM in the environment of a process that maps with mp_map_file (the CLI's call): the default context gets the
    budget, the stages slice, and the PAF and the --dbg-anchor / --dbg-chain dumps are still the reference's."""
    (files, idx, d) = sets
    g, p = files["tiny5"]
    args = ["--dbg-qname", "--dbg-anchor", "--dbg-chain"]
    env = dict(os.environ, MPB_DEVICE_MEM="1k")
    child = dbg_lib._CHILD.replace("sys.exit(0 if rc == 0 else 100 - rc)",
                                   "s = mp.MemStats(); L.mpb_ctx_default.restype = C.c_void_p; mp.lib().mpb_get_mem_stats(L.mpb_ctx_default(), C.byref(s))\n"
                                   "sys.stderr.write('MEM %d %d %d\\n' % (s.budget, s.n_slices_seed, s.n_slices_refine))\n"
                                   "sys.exit(0 if rc == 0 else 100 - rc)")
    r = subprocess.run([sys.executable, "-c", child, ROOT, mp.LIB_PATH, *args, g, p], capture_output=True, env=env, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    assert dbg_lib.digest(r.stdout, r.stderr) == dbg_lib.ref_cli_dbg(args, g, p)
    mem = [line.split() for line in r.stderr.splitlines() if line.startswith(b"MEM ")]
    assert mem and int(mem[0][1]) == 1024 and int(mem[0][2]) == 40 and int(mem[0][3]) > 1
    for bad in ("12gb", "-5", "x"):
        r = subprocess.run([sys.executable, "-c", _CHILD, ROOT], capture_output=True, env=dict(os.environ, MPB_DEVICE_MEM=bad), timeout=600)
        assert r.returncode == 0 and r.stdout.split()[0] == b"0" and b"MPB_DEVICE_MEM" in r.stderr


def test_api_checks():
    L = mp.lib()
    c = mp.Context(0)
    assert c.set_mem_budget(-1) == -1 and c.mem_stats().budget == 0
    assert L.mpb_ctx_set_mem_budget(None, 0) == -1
    assert c.set_mem_budget(5 * MB) == 0 and c.mem_stats().budget == 5 * MB
    assert c.set_mem_budget(0) == 0 and c.mem_stats().budget == 0
    c.close()
