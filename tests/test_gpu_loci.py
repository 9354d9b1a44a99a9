"""Locus mode (mpb_map_loci, mpb_seed_loci_batch) on the GPU.

* whole-contig locus: DPP3 against its single contig gives the whole-genome goldens (default and -j2);
* against the reference: every case of loci_lib gives the reference's PAF for its loci (stored answers), through the library and
  through tools/map_loci.py;
* stage parity: the locus seeding kernels give the anchors of the C oracle over an index of the locus alone, bit for bit, under the
  index options mapping serves and max_occ 20000 / 50 / 1;
* batch independence, a genome-only index (mpb_idx_load_meta) on a context that holds no index, what is uploaded, and refusals."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import dbg_lib
import loci_lib
import miniprot_b200 as mp
import oracle_lib as ol
from test_gpu_dropin import write_odd_fasta
from test_gpu_index_options import INDEX_SETS, _ids, idxopt, read_fasta
from test_gpu_stages import product_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx():
    c = mp.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    return loci_lib.build_cases(str(tmp_path_factory.mktemp("loci")))


def map_case(ctx, mi, case, mo=None):
    mo = mo or mp.mapopt()
    names, seqs, qid = loci_lib.index_of(case)
    loci = loci_lib.loci_tuples(mi, case, qid)
    rc, n_reg, reg = mp.map_loci(ctx, mi, mo, seqs, names, loci)
    assert rc == 0
    paf = mp.loci_paf(mi, mo, seqs, names, loci, n_reg, reg)
    regs = [mp.regions(reg[k], int(n_reg[k])) for k in range(len(loci))]
    mp.free_loci_regs(n_reg, reg)
    return paf, regs


def whole_contig_case():
    (cn, cs), = loci_lib.read_fasta(ol.DPP3_GENOME)
    p = loci_lib.read_fasta(ol.DPP3_PROTEIN)[0][0].decode()
    return {"genome": ol.DPP3_GENOME, "proteins": ol.DPP3_PROTEIN, "args": [], "loci": [(p, cn.decode(), 0, len(cs))]}


@pytest.mark.parametrize("sp_model,golden", [(1, "DPP3_default.paf"), (2, "DPP3_j2.paf")])
def test_whole_contig_locus(ctx, sp_model, golden):
    mi = mp.idx_load(ol.DPP3_GENOME, 4)
    paf, _ = map_case(ctx, mi, whole_contig_case(), mp.mapopt(sp_model=sp_model))
    assert paf == open(os.path.join(ol.GOLDEN, golden), "rb").read()
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", ["DPP3", "DPP3_N", "paralogs", "tiny", "tiny5"])
def test_loci_reference(ctx, cases, name):
    mi = mp.idx_load(cases[name]["genome"], 4)
    paf, regs = map_case(ctx, mi, cases[name])
    assert loci_lib.digest(paf) == loci_lib.ref_answer(cases[name])
    if name == "paralogs":
        assert len(regs[0]) >= 2 and regs[2] == []  # two copies in the first locus, nothing in random sequence
    mp.lib().mp_idx_destroy(mi)


def test_map_loci_tool(cases, tmp_path):
    """tools/map_loci.py (FASTA genome and .mpi) prints the same PAF."""
    for name in ("DPP3", "tiny5"):
        case = cases[name]
        tsv = tmp_path / f"{name}.tsv"
        tsv.write_text("".join(f"{p}\t{c}\t{st}\t{en}\n" for p, c, st, en in case["loci"]))
        genome = case["genome"]
        if name == "tiny5":
            mi = mp.idx_load(genome, 4)
            genome = str(tmp_path / "tiny5.mpi")
            assert mp.lib().mp_idx_dump(genome.encode(), mi) == 0
            mp.lib().mp_idx_destroy(mi)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "map_loci.py"), genome, case["proteins"], str(tsv)], capture_output=True, check=True)
        assert loci_lib.digest(r.stdout) == loci_lib.ref_answer(case), r.stderr.decode()[-2000:]


# ---- stage parity ----------------------------------------------------------------------------------------------------------

_NT4 = np.full(256, 4, np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    _NT4[_ch] = _NT4[_ch + 32] = _i


def oracle_locus_anchors(io, seq: bytes, prot: bytes, max_occ: int):
    """The anchors of `prot` from an index of `seq` alone (ora_sketch_nt4 over both strands, blocks of the - strand from
    ceil(len / 2^bbit)), looked up and cut as map.c:126-177 does."""
    o, tab = ol.ora(), product_tables()
    fw = _NT4[np.frombuffer(seq, np.uint8)]
    rv = np.where(fw[::-1] < 4, 3 - fw[::-1], fw[::-1]).astype(np.uint8)
    nb = (len(seq) + (1 << io.bbit) - 1) >> io.bbit
    pairs = []
    for s, boff in ((fw, 0), (rv, nb)):
        s = np.ascontiguousarray(s)
        out = np.zeros(len(s) + 1, np.uint64)
        n = o.ora_sketch_nt4(C.byref(tab), s.ctypes.data_as(C.c_void_p), C.c_int64(len(s)), io.min_aa_len, io.kmer, io.mod_bit, io.bbit, C.c_int64(boff),
                             out.ctypes.data_as(C.c_void_p))
        pairs.append(out[:n])
    pairs = np.sort(np.concatenate(pairs))
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


@pytest.fixture(scope="module")
def parity_inputs(tmp_path_factory, cases):
    """The tiny genome and the awkward contigs (stop-free ORF contig, poly-A, N runs) in one FASTA; loci of tile-boundary lengths,
    at contig starts and ends, shorter than a block, and the tiny genes with flanks."""
    d = tmp_path_factory.mktemp("loci_parity")
    tiny = cases["tiny"]
    ctgs = read_fasta(tiny["genome"]) + read_fasta(write_odd_fasta(str(d / "odd.fa")))
    path = str(d / "tiny_odd.fa")
    with open(path, "wb") as f:
        for n, s in ctgs:
            f.write(b">" + n.encode() + b"\n" + s + b"\n")
    cid = {n: i for i, (n, _) in enumerate(ctgs)}
    names, seqs, qid = loci_lib.index_of(tiny)
    loci = [(qid[p], cid[c], st, en) for p, c, st, en in tiny["loci"]]
    for n, s in ctgs[3:]:
        L = len(s)
        for lo, hi in ((0, min(L, 2047)), (0, min(L, 2049)), (0, min(L, 65536 + 100)), (max(0, L - 4297), L), (L // 3, min(L, L // 3 + 200)), (0, L)):
            if lo < hi:
                loci.append((len(loci) % len(seqs), cid[n], lo, hi))
    return path, ctgs, seqs, loci


@pytest.mark.parametrize("opts", [o for o in INDEX_SETS if dbg_lib.index_options(o)[0].get("min_aa_len", 30) <= 40], ids=_ids([o for o in INDEX_SETS if dbg_lib.index_options(o)[0].get("min_aa_len", 30) <= 40]))
def test_seed_loci_parity(ctx, parity_inputs, opts):
    path, ctgs, seqs, loci = parity_inputs
    io = idxopt(opts)
    mi = mp.idx_load(path, 8, io)
    n = 0
    for max_occ in (20000, 50, 1):
        got = mp.seed_loci_batch(ctx, mi, max_occ, seqs, loci)
        for (q, c, st, en), a in zip(loci, got):
            want = oracle_locus_anchors(io, ctgs[c][1][st:en], seqs[q], max_occ)
            assert np.array_equal(a, want), (opts, max_occ, q, c, st, en, len(a), len(want))
            n += len(want)
    assert n > 0
    mp.lib().mp_idx_destroy(mi)


# ---- batch independence, genome-only index, refusals -----------------------------------------------------------------------

def test_batch_independence(ctx, cases):
    case = cases["tiny5"]
    mi = mp.idx_load(case["genome"], 4)
    _, together = map_case(ctx, mi, case)
    _, small = map_case(ctx, mi, case, mp.mapopt(mini_batch_size=900))
    assert small == together
    alone = []
    for locus in case["loci"]:
        alone += map_case(ctx, mi, dict(case, loci=[locus]))[1]
    assert alone == together
    assert sum(len(r) for r in together) > 0
    mp.lib().mp_idx_destroy(mi)


def test_genome_only_index(cases, tmp_path):
    case = cases["tiny"]
    mi = mp.idx_load(case["genome"], 4)
    mpi = str(tmp_path / "tiny.mpi")
    assert mp.lib().mp_idx_dump(mpi.encode(), mi) == 0
    c = mp.Context(0)
    try:
        meta = mp.lib().mpb_idx_load_meta(mpi.encode())
        assert meta and not meta.contents.ki and not meta.contents.kb
        c.reset_stats()
        paf, _ = map_case(c, meta, case)
        assert loci_lib.digest(paf) == loci_lib.ref_answer(case)
        seq_bytes = (meta.contents.nt.contents.l_seq + 1) // 2
        first = c.stats().h2d_bytes
        assert seq_bytes <= first < seq_bytes + (1 << 20)  # the genome, never the k-mer tables (64 MiB at the defaults)
        # resident now: the next call uploads the proteins, the locus tables and the stages' work lists, nothing of the genome
        names, seqs, qid = loci_lib.index_of(case)
        residues = sum(len(seqs[qid[p]]) for p, _, _, _ in case["loci"])
        c.reset_stats()
        map_case(c, meta, case)
        again = c.stats().h2d_bytes
        assert residues <= again < seq_bytes // 10
        # an index uploaded in full: nothing of it is uploaded again
        assert mp.lib().mpb_idx_upload(c.h, mi) == 0
        c.reset_stats()
        paf2, _ = map_case(c, mi, case)
        assert paf2 == paf and c.stats().h2d_bytes == again
        mp.lib().mp_idx_destroy(meta)
    finally:
        c.close()
    mp.lib().mp_idx_destroy(mi)


def test_refusals(ctx, cases, tmp_path):
    mi = mp.idx_load(ol.DPP3_GENOME, 4)
    L = mi.contents.nt.contents.ctg[0].len
    seqs, names = [b"MKVLAAGIVALLLAAGWWHHKKPLE"], [b"q"]
    mo = mp.mapopt()
    c0 = ctx.stats().n_anchors
    for bad in [(1, 0, 0, 100), (-1, 0, 0, 100), (0, 1, 0, 100), (0, -1, 0, 100), (0, 0, -1, 100), (0, 0, 0, L + 1), (0, 0, 50, 50), (0, 0, 60, 50)]:
        rc, n_reg, _ = mp.map_loci(ctx, mi, mo, seqs, names, [(0, 0, 0, 100), bad])
        assert rc == -1 and not n_reg.any(), bad
    lib = mp.lib()
    lib.mpb_map_loci.restype = C.c_int
    assert lib.mpb_map_loci(None, C.cast(mi, C.c_void_p), C.byref(mo), 0, None, None, None, 0, None, None, None) == -1
    for over in (dict(go=0), dict(ie_coef=100.0)):
        rc, _, _ = mp.map_loci(ctx, mi, mp.mapopt(**over), seqs, names, [(0, 0, 0, 100)])
        assert rc == -3, over
    for bit in (mp.DBG_ANCHOR, mp.DBG_CHAIN, mp.DBG_QNAME, mp.DBG_MORE_DP, mp.DBG_NO_REFINE):
        old = mp.set_dbg_flag(bit)
        try:
            rc, _, _ = mp.map_loci(ctx, mi, mo, seqs, names, [(0, 0, 0, 100)])
        finally:
            mp.set_dbg_flag(old)
        assert rc == -3, bit
    mp.lib().mp_idx_destroy(mi)
    # --spsc scores on the index
    fa = str(tmp_path / "dpp3.fa")
    open(fa, "wb").write(b"".join(b">" + n + b"\n" + s + b"\n" for n, s in loci_lib.read_fasta(ol.DPP3_GENOME)))
    mi = mp.idx_load(fa, 4)
    lib.mp_set_spsc.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32]
    lib.mp_set_spsc(dbg_lib.spsc_file(str(tmp_path)).encode(), C.cast(mi, C.c_void_p), C.byref(mo), 0)
    rc, _, _ = mp.map_loci(ctx, mi, mo, seqs, names, [(0, 0, 0, 100)])
    assert rc == -3
    mp.lib().mp_idx_destroy(mi)
    # an index with -L above 40
    io = mp.idxopt()
    io.min_aa_len = 41
    mi = mp.idx_load(ol.DPP3_GENOME, 4, io)
    rc, _, _ = mp.map_loci(ctx, mi, mp.mapopt(), seqs, names, [(0, 0, 0, 100)])
    assert rc == -3
    mp.lib().mp_idx_destroy(mi)
    assert ctx.stats().n_anchors == c0  # nothing was seeded by any refused call
    # --no-kalloc is the one debugging bit locus mode takes
    mi = mp.idx_load(ol.DPP3_GENOME, 4)
    old = mp.set_dbg_flag(mp.DBG_NO_KALLOC)
    try:
        rc, n_reg, reg = mp.map_loci(ctx, mi, mo, seqs, names, [(0, 0, 0, 100)])
        assert rc == 0
        mp.free_loci_regs(n_reg, reg)
    finally:
        mp.set_dbg_flag(old)
    mp.lib().mp_idx_destroy(mi)
