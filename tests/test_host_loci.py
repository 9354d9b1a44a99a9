"""Locus mode (map_loci) on the CPU: the host orchestration -- locus views, batches, coordinate translation -- with the C oracle
as the stage backend (its locus seeding: ora_sketch_nt4 over each locus strand, sort + unique, lookup, max_occ, ora_chain).  Every
case must print the reference's PAF for its loci byte for byte (stored answers, loci_lib)."""
import ctypes as C
import os

import pytest

import build_hostcheck_loci
import loci_lib
import miniprot_b200 as mp


@pytest.fixture(scope="module")
def hc():
    L = C.CDLL(build_hostcheck_loci.build())
    L.mp_start()
    C.c_int32.in_dll(L, "mp_verbose").value = 1
    L.mp_idx_load.restype = C.POINTER(mp.Idx)
    L.mp_idx_load.argtypes = [C.c_char_p, C.POINTER(mp.IdxOpt), C.c_int32]
    L.mp_idx_destroy.argtypes = [C.POINTER(mp.Idx)]
    return L


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    return loci_lib.build_cases(str(tmp_path_factory.mktemp("loci")))


def run_case(L, case, **mo_over):
    io, mo = mp.IdxOpt(), mp.MapOpt()
    L.mp_idxopt_init(C.byref(io))
    L.mp_mapopt_init(C.byref(mo))
    for k, v in mo_over.items():
        setattr(mo, k, v)
    mi = L.mp_idx_load(case["genome"].encode(), C.byref(io), 4)
    assert mi
    names, seqs, qid = loci_lib.index_of(case)
    loci = loci_lib.loci_tuples(mi, case, qid)
    rc, n_reg, reg = mp.map_loci(None, mi, mo, seqs, names, loci, L=L, fn="hc_map_loci")
    assert rc == 0
    paf = mp.loci_paf(mi, mo, seqs, names, loci, n_reg, reg, L=L, fn="hc_format_paf")
    mp.free_loci_regs(n_reg, reg)
    L.mp_idx_destroy(mi)
    return paf


@pytest.mark.parametrize("name", ["DPP3", "DPP3_N", "paralogs", "tiny", "tiny5"])
def test_host_loci_reference(hc, cases, name):
    assert loci_lib.digest(run_case(hc, cases[name])) == loci_lib.ref_answer(cases[name])


def test_host_loci_small_batches(hc, cases):
    """Batches cut by mini_batch_size give the same answer."""
    assert loci_lib.digest(run_case(hc, cases["tiny"], mini_batch_size=700)) == loci_lib.ref_answer(cases["tiny"])


def test_host_loci_whole_contig(hc):
    """DPP3 against its whole contig as one locus prints the whole-genome golden."""
    case = {"genome": loci_lib.ol.DPP3_GENOME, "proteins": loci_lib.ol.DPP3_PROTEIN, "args": [], "loci": []}
    (cn, cs), = loci_lib.read_fasta(case["genome"])
    p = loci_lib.read_fasta(case["proteins"])[0][0].decode()
    case["loci"] = [(p, cn.decode(), 0, len(cs))]
    want = open(os.path.join(loci_lib.ol.GOLDEN, "DPP3_default.paf"), "rb").read()
    assert run_case(hc, case) == want


def test_host_loci_refusals(hc, cases):
    io, mo = mp.IdxOpt(), mp.MapOpt()
    hc.mp_idxopt_init(C.byref(io))
    hc.mp_mapopt_init(C.byref(mo))
    mi = hc.mp_idx_load(cases["DPP3"]["genome"].encode(), C.byref(io), 4)
    L = mi.contents.nt.contents.ctg[0].len
    seqs, names = [b"MKVLAAGIVALLLAAG"], [b"q"]
    for bad in [(1, 0, 0, 100), (-1, 0, 0, 100), (0, 1, 0, 100), (0, -1, 0, 100), (0, 0, -1, 100), (0, 0, 0, L + 1), (0, 0, 50, 50), (0, 0, 60, 50)]:
        rc, n_reg, _ = mp.map_loci(None, mi, mo, seqs, names, [(0, 0, 0, 100), bad], L=hc, fn="hc_map_loci")
        assert rc == -1 and not n_reg.any(), bad
    old = mp.set_dbg_flag(mp.DBG_ANCHOR, hc)
    try:
        rc, n_reg, _ = mp.map_loci(None, mi, mo, seqs, names, [(0, 0, 0, 100)], L=hc, fn="hc_map_loci")
        assert rc == -3 and not n_reg.any()
    finally:
        mp.set_dbg_flag(old, hc)
    hc.mp_idx_destroy(mi)
