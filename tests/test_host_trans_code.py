"""CPU twin of test_gpu_trans_code.py: NCBI genetic codes other than the standard one (-T).

* the product's host pipeline with the C oracle as stage backend (tests/hostcheck/hostcheck_dbg.cpp) prints what the reference CLI
  prints with -T<n> (stored digests, dbg_lib.ref_cli_dbg): PAF with the X / Y1 dump lines under every code of the GPU test's
  end-to-end runs, and GFF, --trans and --aln under two of them;
* the lock-step emulation of the DP kernels (pair-lane, block-wide and column-pass forms) equals the oracle under every code, and
  the oracle equals the reference's ns_global_gs16b (stored answers);
* the host index builder under every code writes the reference's -T<n> -d file, and locus mode under -T2 prints the reference's PAF.
"""
import ctypes as C

import numpy as np
import pytest

import build_hostcheck
import build_hostcheck_dbg
import build_hostcheck_loci
import dbg_lib
import loci_lib
import miniprot_b200 as mp
import oracle_lib as ol
from test_emu_nasw import emu
from test_gpu_dropin import write_odd_fasta
from test_host_loci import run_case


@pytest.fixture(scope="module")
def hc():
    return build_hostcheck_dbg.build()


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    return dbg_lib.input_sets(str(tmp_path_factory.mktemp("trans")))


# every code with the seed and chain dumps; the other formats (about ten seconds a run on the oracle backend) with the two codes of
# the most stop-codon records
CASES = [(c, f) for c in dbg_lib.TRANS_E2E_CODES for f in dbg_lib.TRANS_FORMATS if f == dbg_lib.INDEX_SWITCHES or c in (2, 23)]


@pytest.mark.parametrize("code,fmt", [(c, " ".join(f)) for c, f in CASES])
@pytest.mark.parametrize("name", ["tiny", "tiny5", "DPP3"])
def test_trans_code_golden(hc, sets, code, name, fmt):
    args = [f"-T{code}"] + fmt.split()
    g, p = sets[name]
    rc, out, err = dbg_lib.run_cli(hc, args, g, p)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    got, want = dbg_lib.digest(out, err), dbg_lib.ref_cli_dbg(args, g, p)
    assert (got["lines"], got["dump_lines"]) == (want["lines"], want["dump_lines"])
    assert got == want


@pytest.fixture(scope="module")
def emu_lib():
    lib = C.CDLL(build_hostcheck.build())
    lib.emu_nasw.restype = C.c_int
    lib.emu_nasw.argtypes = [C.c_void_p] * 5 + [C.c_int] * 6 + [C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_char_p, C.c_int] + \
        [C.c_void_p] * 4 + [C.c_int]
    return lib


@pytest.mark.parametrize("code", dbg_lib.TRANS_CODES)
def test_emu_trans_code(emu_lib, code):
    """Problems encoded with the standard code and with the code's own codons (one residue in twenty a stop codon of the code): the
    emulated pair-lane (-1), block-wide (0) and column-pass (1, 8) kernels against the oracle with the reference's tables of the code,
    and the oracle against the reference's ns_global_gs16b under -T<code>."""
    tab = ol.ref_tables_for(code)
    codon = ol.codon_array(tab)
    own = ol.codons_of(codon)
    mat, par = ol.default_mat(), dict(ol.DEFAULT_NASW)
    rng = np.random.default_rng(9100 + code)
    n_stop = n_differ = 0
    for it in range(24):
        mine = it % 2 == 1
        nt, aa = ol.random_dp_problem(rng, al_max=(30, 70, 140, 300)[it % 4], flank=40, intron_max=(0, 150, 400)[it % 3],
                                      codons=own if mine else None, p_stop=(0.05 if "*" in own else 0) if mine else 0.01)
        if len(nt) < 3:
            continue
        n_stop += ol.stop_rows(nt, codon)
        flag = (1, 4, 2)[it % 3]
        want = ol.ora_nasw(tab, nt, aa, flag, mat, par)
        assert list(ol.ref_nasw(nt, aa, flag, mat, par, code=code)) == list(want), (it, flag, len(nt), len(aa))
        n_differ += ol.ora_nasw(ol.ref_tables(), nt, aa, flag, mat, par) != want
        for Ccols in (-1, 0, 1, 8):
            got = emu(emu_lib, nt, aa, flag, Ccols, mat, par, tab)
            assert ((want[0] == got[0] and want[3] == got[3]) if flag == 1 else want[:3] == got[:3]), (it, flag, Ccols, want[:3], got[:3])
    assert n_stop >= 20 if (codon == 20).any() else n_stop == 0
    if not np.array_equal(codon, ol.codon_array(ol.ref_tables())):
        assert n_differ > 0


@pytest.fixture(scope="module")
def genomes(tmp_path_factory):
    from miniprot_b200 import synth

    d = tmp_path_factory.mktemp("trans_idx")
    return write_odd_fasta(str(d / "odd.fa")), synth.generate(synth.CONFIGS["tiny"], str(d / "tiny"))[0]


@pytest.mark.parametrize("code", dbg_lib.TRANS_CODES)
def test_host_index_trans_code(genomes, tmp_path, code):
    """The host index builder under -T<code> writes the reference's -T<code> -d file (awkward contigs and the tiny genome)."""
    L = mp.lib()
    io = mp.idxopt()
    io.trans_code = code
    for g in genomes:
        assert L.ns_make_tables(code) == 0
        try:
            mi = mp.idx_load(g, 4, io)
        finally:
            L.ns_make_tables(1)
        out = str(tmp_path / "o.mpi")
        assert L.mp_idx_dump(out.encode(), mi) == 0
        L.mp_idx_destroy(mi)
        assert ol.file_digest(out) == ol.ref_index_file(g, [f"-T{code}"])


def test_host_loci_trans_code(tmp_path):
    """Locus mode under -T2 with the oracle backend: the reference's PAF of each locus of tiny5 mapped on its own with -T2."""
    L = C.CDLL(build_hostcheck_loci.build())
    L.mp_start()
    C.c_int32.in_dll(L, "mp_verbose").value = 1
    L.mp_idx_load.restype = C.POINTER(mp.Idx)
    L.mp_idx_load.argtypes = [C.c_char_p, C.POINTER(mp.IdxOpt), C.c_int32]
    L.mp_idx_destroy.argtypes = [C.POINTER(mp.Idx)]
    case = loci_lib.build_cases(str(tmp_path))["tiny5_T2"]
    assert L.ns_make_tables(2) == 0
    try:
        paf = run_case(L, case)
    finally:
        L.ns_make_tables(1)
    assert loci_lib.digest(paf) == loci_lib.ref_answer(case)
