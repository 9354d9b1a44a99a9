"""Locus sets (mpb_map_locus_sets, mpb_seed_locus_sets_batch, mpb_map_locus_sets_file*, tools/map_loci.py --sets) on the GPU.

* against the reference: every case of locus_sets_lib under every option set prints the reference's output for its sets (stored
  answers) through mpb_map_locus_sets_file, and the same bytes on two contexts with small units and in the serial form; default
  options through mpb_map_locus_sets + mpb_format_paf too;
* the DPP3 set that merges into the whole contig prints the whole-genome goldens;
* a memory budget small enough to run one set per slice gives the same bytes;
* sets of one locus give what mpb_map_loci gives for the pairs of every loci_lib case;
* stage parity: the set seeding gives the anchors of the C oracle over an index of each set's canonical genome, bit for bit;
* refusals, and tools/map_loci.py --sets end to end."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import loci_file_lib
import loci_lib
import locus_sets_lib
import miniprot_b200 as mp
import oracle_lib as ol
from test_gpu_stages import product_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    c = mp.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_pair():
    cs = [mp.Context(0), mp.Context(0)]
    yield cs
    for c in cs:
        c.close()


@pytest.fixture(scope="module")
def tool():
    return loci_file_lib.map_loci_tool()


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    d = tmp_path_factory.mktemp("locus_sets")
    cs = locus_sets_lib.build_cases(str(d))
    for name, case in cs.items():
        case["tsv"] = locus_sets_lib.write_tsv(str(d / f"{name}.tsv"), case["lines"])
    return cs


class tables:
    """the library's codon tables switched to genetic code `code` for the duration (what the CLI does for -T)"""

    def __init__(self, code):
        self.code = code

    def __enter__(self):
        assert mp.lib().ns_make_tables(self.code) == 0

    def __exit__(self, *exc):
        mp.lib().ns_make_tables(1)


def file_run(ctxs, mi, case, mo, path, tsv=None):
    """mpb_map_locus_sets_file_multi_path: (return code, output bytes or None when no file was created)"""
    if os.path.exists(path):
        os.unlink(path)
    ctxs = ctxs if isinstance(ctxs, list) else [ctxs]
    arr = (C.c_void_p * len(ctxs))(*[c.h if c else None for c in ctxs])
    rc = mp.lib().mpb_map_locus_sets_file_multi_path(arr, len(ctxs), mi, case["proteins"].encode(), (tsv or case["tsv"]).encode(), C.byref(mo),
                                                     str(path).encode())
    return rc, open(path, "rb").read() if os.path.exists(path) else None


def api_paf(ctx, mi, case, mo):
    """mpb_map_locus_sets + mpb_format_paf over the case's sets: (PAF bytes, regions per set)"""
    names, seqs, qid = loci_lib.index_of(case)
    off, loci = locus_sets_lib.set_arrays(mi, case, qid)
    sets = [loci[off[k]:off[k + 1]] for k in range(len(off) - 1)]
    rc, n_reg, reg = ctx.map_locus_sets(mi, mo, seqs, names, sets)
    assert rc == 0
    paf = mp.loci_paf(mi, mo, seqs, names, [s[0] for s in sets], n_reg, reg)
    regs = [mp.regions(reg[k], int(n_reg[k])) for k in range(len(sets))]
    mp.free_loci_regs(n_reg, reg)
    return paf, regs


@pytest.mark.parametrize("opts", list(locus_sets_lib.OPTION_SETS))
@pytest.mark.parametrize("name", locus_sets_lib.CASES)
def test_locus_sets_file_reference(ctx, ctx_pair, tool, cases, tmp_path, monkeypatch, name, opts):
    case, args = cases[name], locus_sets_lib.OPTION_SETS[opts]
    _, io, mo = tool.options([*case["args"], *args, "g", "p", "l"])
    mi = mp.idx_load_genome(case["genome"], io)
    with tables(io.trans_code):
        rc, out = file_run(ctx, mi, case, mo, tmp_path / "one")
        assert rc == 0
        assert loci_lib.digest(out) == locus_sets_lib.ref_answer(case, args)
        # two contexts, units of a few sets
        _, _, mo_small = tool.options([*case["args"], *args, "-K", "1500", "g", "p", "l"])
        assert file_run(ctx_pair, mi, case, mo_small, tmp_path / "two") == (0, out)
        # one context, one set per unit, one step after another on the calling thread
        monkeypatch.setenv("MPB_FILE_PIPELINE", "0")
        _, _, mo_one = tool.options([*case["args"], *args, "-K1", "g", "p", "l"])
        mp.map_locus_sets_file(ctx, mi, case["proteins"], case["tsv"], str(tmp_path / "serial"), mo_one)
        assert (tmp_path / "serial").read_bytes() == out
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", locus_sets_lib.CASES)
def test_locus_sets_api(ctx, cases, tool, name):
    """mpb_map_locus_sets + mpb_format_paf print the file driver's default PAF; the paralogs set has a primary and a secondary hit."""
    case = cases[name]
    _, io, mo = tool.options([*case["args"], "g", "p", "l"])
    mi = mp.idx_load(case["genome"], 4, io)
    with tables(io.trans_code):
        paf, regs = api_paf(ctx, mi, case, mo)
    assert loci_lib.digest(paf) == locus_sets_lib.ref_answer(case, [])
    if name == "paralogs":
        both = regs[0]
        assert len(both) >= 2 and {r[0][9] >> 1 for r in both} == {0}
        assert both[0][0][0] == both[0][0][1] and both[1][0][1] != both[1][0][0]  # id == parent: primary; the other copy secondary
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("args,golden", [([], "DPP3_default.paf"), (["-j2"], "DPP3_j2.paf"), (["--gff"], "DPP3_gff.txt"), (["--aln"], "DPP3_aln.txt"),
                                         (["--trans", "-u"], "DPP3_trans.txt")])
def test_whole_contig_set(ctx, tool, cases, tmp_path, args, golden):
    """[0, 1500) + [1500, L) of DPP3 merge into the whole contig: the reference's whole-genome output, byte for byte."""
    case = cases["DPP3"]
    tsv = locus_sets_lib.write_tsv(str(tmp_path / "whole.tsv"), [x for x in case["lines"] if x[4] == "whole"])
    _, io, mo = tool.options([*args, "g", "p", "l"])
    mi = mp.idx_load_genome(case["genome"], io)
    assert file_run(ctx, mi, case, mo, tmp_path / "out", tsv=tsv) == (0, open(os.path.join(ol.GOLDEN, golden), "rb").read())
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", ["paralogs", "tiny"])
def test_locus_sets_mem_budget(cases, tool, tmp_path, name):
    """A budget of one byte runs every set in slices of its own (and over the budget); the output is the same."""
    case = cases[name]
    _, io, mo = tool.options(["--gff", "g", "p", "l"])
    mi = mp.idx_load_genome(case["genome"], io)
    outs, stats = [], []
    for budget in (0, 1):
        c = mp.Context(0)
        try:
            assert c.set_mem_budget(budget) == 0
            rc, out = file_run(c, mi, case, mo, tmp_path / f"b{budget}")
            assert rc == 0
            outs.append(out)
            stats.append(c.mem_stats())
        finally:
            c.close()
    n_sets = len(locus_sets_lib.sets_of(case["lines"]))
    assert outs[0] == outs[1] and loci_lib.digest(outs[0]) == locus_sets_lib.ref_answer(case, ["--gff"])
    assert stats[0].n_slices_loci == 1 and stats[1].n_slices_loci == n_sets > 1 and stats[1].n_over_budget > 0
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", ["DPP3", "DPP3_N", "paralogs", "tiny", "tiny5", "tiny5_T2"])
def test_single_locus_sets(ctx, tmp_path, name):
    """Every pair of a loci_lib case as a set of its own gives mpb_map_loci's regions, and the stored PAF."""
    case = loci_lib.build_cases(str(tmp_path))[name]
    io = mp.idxopt()
    if case["args"]:
        io.trans_code = int(case["args"][0][2:])
    mi = mp.idx_load(case["genome"], 4, io)
    names, seqs, qid = loci_lib.index_of(case)
    loci = loci_lib.loci_tuples(mi, case, qid)
    mo = mp.mapopt()
    with tables(io.trans_code):  # the PAF's cs tags translate codons too
        rc, n1, r1 = mp.map_locus_sets(ctx, mi, mo, seqs, names, [[x] for x in loci])
        rc2, n2, r2 = mp.map_loci(ctx, mi, mo, seqs, names, loci)
        paf = mp.loci_paf(mi, mo, seqs, names, loci, n1, r1)
    assert rc == rc2 == 0 and list(n1) == list(n2)
    assert [mp.regions(r1[k], int(n1[k])) for k in range(len(loci))] == [mp.regions(r2[k], int(n2[k])) for k in range(len(loci))]
    assert loci_lib.digest(paf) == loci_lib.ref_answer(case)
    mp.free_loci_regs(n1, r1), mp.free_loci_regs(n2, r2)
    mp.lib().mp_idx_destroy(mi)


# ---- stage parity --------------------------------------------------------------------------------------------------------------

_NT4 = np.full(256, 4, np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    _NT4[_ch] = _NT4[_ch + 32] = _i


def oracle_set_anchors(io, recs, prot: bytes, max_occ: int):
    """The anchors of `prot` from an index of the records `recs` (a genome of those sequences alone: ora_sketch_nt4 over both
    strands of each, blocks numbered record by record, + strand then - strand), looked up and cut as map.c:126-177 does."""
    o, tab = ol.ora(), product_tables()
    pairs, boff = [], 0
    for seq in recs:
        fw = _NT4[np.frombuffer(seq, np.uint8)]
        rv = np.where(fw[::-1] < 4, 3 - fw[::-1], fw[::-1]).astype(np.uint8)
        nb = (len(seq) + (1 << io.bbit) - 1) >> io.bbit
        for s, b0 in ((fw, boff), (rv, boff + nb)):
            s = np.ascontiguousarray(s)
            out = np.zeros(len(s) + 1, np.uint64)
            n = o.ora_sketch_nt4(C.byref(tab), s.ctypes.data_as(C.c_void_p), C.c_int64(len(s)), io.min_aa_len, io.kmer, io.mod_bit, io.bbit, C.c_int64(b0),
                                 out.ctypes.data_as(C.c_void_p))
            pairs.append(out[:n])
        boff += 2 * nb
    pairs = np.unique(np.concatenate(pairs))
    sd = np.zeros(len(prot) + 1, np.uint64)
    n_sd = o.ora_sketch_prot(C.byref(tab), C.c_char_p(prot), len(prot), io.kmer, io.mod_bit, sd.ctypes.data_as(C.c_void_p))
    sd = np.sort(sd[:n_sd])
    b = sd >> np.uint64(32)
    lo = np.searchsorted(pairs, b << np.uint64(32))
    hi = np.searchsorted(pairs, (b + np.uint64(1)) << np.uint64(32))
    cnt = (hi - lo).astype(np.uint64)
    cap = max_occ
    if n_sd >= 8:
        c = np.sort(cnt)
        q25, q75 = int(c[int(n_sd * .25 + .499)]), int(c[int(n_sd * .75 + .499)])
        cap = min(cap, int(q75 + (q75 - q25) * 1.5 + 10.))
    a = [(int(pairs[j]) & 0xffffffff) << 32 | (int(sd[i]) & 0xffffffff) for i in range(n_sd) if int(cnt[i]) <= cap for j in range(lo[i], hi[i])]
    return np.array(sorted(a), np.uint64)


@pytest.mark.parametrize("name", ["paralogs", "DPP3", "tiny5"])
def test_seed_locus_sets_parity(ctx, cases, name):
    case = cases[name]
    mi = mp.idx_load(case["genome"], 4)
    io = mi.contents.opt
    genome = loci_lib.read_fasta(case["genome"])
    order = {n.decode(): i for i, (n, _) in enumerate(genome)}
    seq_of = dict(genome)
    names, seqs, qid = loci_lib.index_of(case)
    off, loci = locus_sets_lib.set_arrays(mi, case, qid)
    sets = [loci[off[k]:off[k + 1]] for k in range(len(off) - 1)]
    canon = [locus_sets_lib.canonical(r, order) for _, r in locus_sets_lib.sets_of(case["lines"])]
    n = 0
    for max_occ in (20000, 50, 1):
        got = mp.seed_locus_sets_batch(ctx, mi, max_occ, seqs, sets)
        for s, a, rs in zip(sets, got, canon):
            want = oracle_set_anchors(io, [seq_of[c.encode()][st:en] for c, st, en in rs], seqs[s[0][0]], max_occ)
            assert np.array_equal(a, want), (name, max_occ, rs, len(a), len(want))
            n += len(want)
    assert n > 0
    mp.lib().mp_idx_destroy(mi)


# ---- refusals, the tool --------------------------------------------------------------------------------------------------------

def test_locus_sets_refusals(ctx, cases, tool, tmp_path, capfd):
    mi = mp.idx_load(ol.DPP3_GENOME, 4)
    seqs, names = [b"MKVLAAGIVALLLAAGWWHHKKPLE", b"MKKLLPPAAGGHHWW"], [b"q", b"r"]
    mo = mp.mapopt()
    c0 = ctx.stats().n_anchors
    for bad in ([[(0, 0, 0, 100)], []], [[(0, 0, 0, 100), (1, 0, 200, 300)]], [[(0, 0, 0, 100), (0, 0, 60, 50)]], [[(0, 1, 0, 100)]], [[(2, 0, 0, 100)]]):
        rc, n_reg, _ = ctx.map_locus_sets(mi, mo, seqs, names, bad)
        assert rc == -1 and not n_reg.any(), bad
    for over in (dict(go=0), dict(ie_coef=100.0)):
        assert ctx.map_locus_sets(mi, mp.mapopt(**over), seqs, names, [[(0, 0, 0, 100), (0, 0, 500, 900)]])[0] == -3, over
    for bit in (mp.DBG_ANCHOR, mp.DBG_CHAIN, mp.DBG_NO_REFINE):
        old = mp.set_dbg_flag(bit)
        try:
            assert ctx.map_locus_sets(mi, mo, seqs, names, [[(0, 0, 0, 100), (0, 0, 500, 900)]])[0] == -3, bit
        finally:
            mp.set_dbg_flag(old)
    mp.lib().mp_idx_destroy(mi)
    io = mp.idxopt()
    io.min_aa_len = 41
    mi = mp.idx_load(ol.DPP3_GENOME, 4, io)
    assert ctx.map_locus_sets(mi, mo, seqs, names, [[(0, 0, 0, 100), (0, 0, 500, 900)]])[0] == -3
    mp.lib().mp_idx_destroy(mi)
    assert ctx.stats().n_anchors == c0  # nothing was seeded by any refused call
    # the file driver: file:line messages, nothing written
    case = cases["DPP3"]
    p, c = case["lines"][0][:2]
    tsv = tmp_path / "bad.tsv"
    tsv.write_text(f"{p}\t{c}\t0\t100\tA\n{p}\t{c}\t50\t50\tA\n")
    mi = mp.idx_load_genome(case["genome"])
    capfd.readouterr()
    assert file_run(ctx, mi, case, mo, tmp_path / "out", tsv=str(tsv)) == (-1, None)
    assert f"{tsv}:2:" in capfd.readouterr().err
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", ["paralogs", "tiny"])
def test_map_loci_tool_sets(cases, name):
    """tools/map_loci.py --sets on one context and on two; -I and --spsc stay refused."""
    case = cases[name]
    for extra in ([], ["--devices", "0,0", "-K2000"]):
        for args in ([], ["--gff"]):
            r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "map_loci.py"), "--sets", *args, *extra, case["genome"], case["proteins"], case["tsv"]],
                               capture_output=True)
            assert r.returncode == 0, r.stderr.decode()[-2000:]
            assert loci_lib.digest(r.stdout) == locus_sets_lib.ref_answer(case, args), (extra, r.stderr.decode()[-2000:])
    for refused in (["-I"], ["--spsc", "x.tsv"]):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "map_loci.py"), "--sets", *refused, case["genome"], case["proteins"], case["tsv"]],
                           capture_output=True)
        assert r.returncode != 0 and not r.stdout and refused[0].encode() in r.stderr
