"""GPU stages under NCBI genetic codes other than the standard one (-T, ns_make_tables).  The kernels that read the codon tables:
the index build's ORF rule (a codon of code >= 20 closes an ORF) and k-mer letters (codon13; idx_build.cu, win_scan.cuh), the
refinement's window scan (seed_kernels.cu) and the DP prep kernels, which give each row its amino acid and, on stop-codon rows, the
frameshift penalty as gap extension (nasw_core.cuh make_row_rec, nasw_pair.cuh).  Each kernel takes the tables from a host copy
made at every call; these tests fail if any copy is cached or fixed to the standard code.

Each stage is compared bit for bit with its reference under the same code: the DP kernels and the seeding and refinement stages
with the C oracle given the live tables, the device-built index with the host builder's and the reference CLI's -T<n> -d output
(stored digests), and the whole pipeline with the reference CLI's -T<n> output (stored digests, dbg_lib)."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import dbg_lib
import loci_lib
import miniprot_b200 as mp
import oracle_lib as ol
from test_gpu_index_options import inputs, read_proteins, refine_inputs  # noqa: F401 (module fixtures)
from test_gpu_loci import map_case
from test_gpu_stages import _par, product_tables

pytestmark = pytest.mark.gpu

CODES, E2E_CODES, E2E_FORMATS = dbg_lib.TRANS_CODES, dbg_lib.TRANS_E2E_CODES, dbg_lib.TRANS_FORMATS
STOP = 20  # amino-acid code of '*' in ns_tab_aa20 / ns_tab_codon


@pytest.fixture(scope="module")
def ctx():
    c = mp.Context(0)
    yield c
    c.close()


@pytest.fixture
def use_code():
    """use_code(T): the library's tables switched to genetic code T (ns_make_tables must return 0); returns them as an oracle table
    bundle.  Code 1 is restored after the test, failed or not: the tables are process globals the rest of the session maps with."""
    L = mp.lib()

    def use(code):
        assert L.ns_make_tables(code) == 0, code
        return product_tables()
    yield use
    assert L.ns_make_tables(1) == 0


def tables_copy(code):
    """(oracle table bundle, arrays keeping it alive) of code `code`, copied out of the library, which is left at code 1."""
    L = mp.lib()
    assert L.ns_make_tables(code) == 0
    arrs = [np.ctypeslib.as_array((C.c_uint8 * n).in_dll(L, s)).copy()
            for s, n in (("ns_tab_nt4", 256), ("ns_tab_aa20", 256), ("ns_tab_aa13", 256), ("ns_tab_codon", 64), ("ns_tab_codon13", 64))]
    assert L.ns_make_tables(1) == 0
    return ol.tables_from_arrays(*arrs), arrs


@pytest.fixture(scope="module")
def std_tab():
    return tables_copy(1)


def stop_set(codon):
    return frozenset(int(c) for c in np.nonzero(codon == STOP)[0])


# ---- A. DP -------------------------------------------------------------------------------------------------------------------

FAMILIES = ["auto", "pair", "v3", "cols"]


def dp_problems(rng, own_codons):
    """(nt, aa, flag) triples of every width class (pair lanes <= 64 columns, block-wide CTAs of 1..8 warps, column passes beyond
    256): half encoded with the standard code (under another code some of its codons are stops, some standard stops are not),
    half with the code's own codons and one residue in twenty a stop codon of the code (codes 27, 28 and 31 have none)."""
    out = []
    for it in range(100):
        al_max = (24, 60, 120, 250, 400)[it % 5]
        own = it % 2 == 1
        nt, aa = ol.random_dp_problem(rng, al_max=al_max, flank=60, intron_max=(0, 150, 600)[it % 3], codons=own_codons if own else None,
                                      p_stop=(0.05 if "*" in own_codons else 0) if own else 0.01)
        if len(nt) >= 3:
            out.append((nt, aa, (1, 4, 2)[it % 3]))
    return out


STOP_SCORES = (None, 9)  # the matrix's stop-codon row as mp_mapopt_init leaves it, and as ns_set_stop_sc (-F) sets it


def nsopt_for(stop_sc):
    opt = mp.nsopt()
    if stop_sc is not None:
        mp.lib().ns_set_stop_sc(22, opt._mat_keepalive.ctypes.data_as(C.c_void_p), stop_sc)
    return opt


_dp_cases = {}


def dp_cases(code, tab, std_tab):
    """(problems, {stop score: ora_nasw answers under the live tables `tab`}, number of problems whose answer under code 1 is another
    one) of code `code`, computed once for the four kernel families."""
    if code not in _dp_cases:
        probs = dp_problems(np.random.default_rng(9000 + code), ol.codons_of(ol.codon_array(tab)))
        want, n_differ = {}, 0
        for stop_sc in STOP_SCORES:
            opt = nsopt_for(stop_sc)
            mat, par = opt._mat_keepalive, _par(opt)
            want[stop_sc] = [ol.ora_nasw(tab, nt, aa, flag, mat, par) for nt, aa, flag in probs]
            if stop_sc is None:
                n_differ = sum(ol.ora_nasw(std_tab, nt, aa, flag, mat, par) != w for (nt, aa, flag), w in zip(probs, want[stop_sc]))
        _dp_cases[code] = (probs, want, n_differ)
    return _dp_cases[code]


def classes_ran(st) -> set:
    return {(b, c) for b in range(2) for c in range(16) if st.n_class[b][c]}


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("code", CODES)
def test_nasw_trans_code(ctx, use_code, std_tab, code, family, monkeypatch):
    """mpb_nasw_batch against ora_nasw under code T, flags 1 / 4 / 2, with the default stop-codon score and with ns_set_stop_sc
    (-F): the production dispatch (auto), the pair-lane kernels for everything up to 64 columns (pair), the block-wide kernels
    (v3, in column passes beyond 256 columns) and the warp-per-problem column-pass kernels (cols)."""
    if family != "auto":
        monkeypatch.setenv("MPB_NASW_KERNEL", family)
    tab = use_code(code)
    codon = ol.codon_array(tab)
    probs, want, n_differ = dp_cases(code, tab, std_tab[0])
    assert max(len(aa) for _, aa, _ in probs) > 256
    n_stop = sum(ol.stop_rows(nt, codon) for nt, _, _ in probs)
    assert n_stop >= 100 if stop_set(codon) else n_stop == 0, n_stop  # the stop-row gap extension is exercised
    if not np.array_equal(codon, ol.codon_array(std_tab[0])):
        assert n_differ >= 10, n_differ  # kernels reading the standard code's tables would fail
    ctx.reset_stats()
    for stop_sc in STOP_SCORES:
        opt = nsopt_for(stop_sc)
        got = mp.nasw_batch(ctx, opt, [(nt, aa, flag, opt.io) for nt, aa, flag in probs])
        bad = [(flag, len(nt), len(aa), w[:3], g[:3]) for (nt, aa, flag), w, g in zip(probs, want[stop_sc], got)
               if not ((w[0] == g[0] and w[3] == g[3]) if flag == 1 else (w[:3] == g[:3]))]
        assert not bad, (stop_sc, len(bad), bad[:4])
    ran = classes_ran(ctx.stats())
    wide = {(b, c) for b in range(2) for c in range(4)}  # block-wide CTAs of 1, 2, 4, 8 warps
    cols = {(b, c) for b in range(2) for c in range(4, 9)}  # column-pass kernels; class 8: several passes
    pair = {(0, 9), (1, 9)}
    if family == "auto":
        assert (1, 9) in ran and ran & wide and not ran & cols, ran
    elif family == "pair":
        assert pair <= ran and not ran & cols, ran
    elif family == "v3":
        assert ran & wide and not ran & (cols | pair), ran
    else:
        assert ran & cols and ran & {(0, 8), (1, 8)} and not ran & (wide | pair), ran


# ---- B. index build ----------------------------------------------------------------------------------------------------------

def kmer_tables_digest(mi) -> str:
    idx = mi.contents
    ki = np.ctypeslib.as_array(C.cast(idx.ki, C.POINTER(C.c_int64)), shape=(mp.n_bucket(idx.opt),))
    kb = np.ctypeslib.as_array(C.cast(idx.kb, C.POINTER(C.c_uint32)), shape=(max(idx.n_kb, 1),))[:idx.n_kb]
    return ol._digest(ki, kb)


@pytest.fixture(scope="module")
def std_kmer_tables(inputs):  # noqa: F811
    """Digest of the k-mer tables (ki, kb) of the code-1 index of each input."""
    out = {}
    for tag in ("odd", "tiny"):
        mi = mp.idx_load(inputs[tag], 8)
        out[tag] = kmer_tables_digest(mi)
        mp.lib().mp_idx_destroy(mi)
    return out


@pytest.mark.parametrize("code", CODES)
def test_index_build_trans_code(inputs, std_kmer_tables, std_tab, use_code, code, monkeypatch, capfd):  # noqa: F811
    """The .mpi of the device build under -T<code> equals the host builder's and the reference CLI's (-T<code> -d).  Its k-mer tables
    differ from the code-1 index's wherever the stop codons differ, and equal them where the tables are code 1's."""
    L = mp.lib()
    verbose = C.c_int32.in_dll(L, "mp_verbose")
    io = mp.idxopt()
    io.trans_code = code
    codon = ol.codon_array(use_code(code))
    std = ol.codon_array(std_tab[0])
    for tag in ("odd", "tiny"):
        g = inputs[tag]
        files = {}
        for where in ("dev", "host"):
            if where == "host":
                monkeypatch.setenv("MPB_IDX_BUILD", "host")
            verbose.value = 3
            capfd.readouterr()
            mi = mp.idx_load(g, 8, io)
            verbose.value = 1
            err = capfd.readouterr().err
            monkeypatch.delenv("MPB_IDX_BUILD", raising=False)
            assert ("built the k-mer tables on the device" in err) == (where == "dev"), (tag, where, err[-500:])
            assert mi.contents.opt.trans_code == code
            if where == "dev":
                kt = kmer_tables_digest(mi)
            files[where] = str(inputs["dir"] / f"{tag}.T{code}.{where}.mpi")
            assert L.mp_idx_dump(files[where].encode(), mi) == 0
            L.mp_idx_destroy(mi)
        a, b = (open(files[x], "rb").read() for x in ("dev", "host"))
        assert a == b, tag
        assert ol.file_digest(files["dev"]) == ol.ref_index_file(g, [f"-T{code}"]), tag
        if stop_set(codon) != stop_set(std):
            assert kt != std_kmer_tables[tag], tag
        if np.array_equal(codon, std):
            assert kt == std_kmer_tables[tag], tag


# ---- C. seeding and refinement -----------------------------------------------------------------------------------------------

DEGENERATE_PROTEINS = [b"", b"MKV", b"M" * 40, b"ACDEFGHIKLMNPQRSTVWY" * 3 + b"XX*" + b"WWHHKK" * 5]


@pytest.mark.parametrize("code", E2E_CODES)
def test_seed_trans_code(ctx, inputs, use_code, code):  # noqa: F811
    """mpb_seed_batch against ora_seed_anchors on an index built under -T<code>, protein by protein, max_occ 20000 and 50."""
    tab = use_code(code)
    io = mp.idxopt()
    io.trans_code = code
    mi = mp.idx_load(inputs["tiny"], 8, io)
    idx = mi.contents
    seqs = read_proteins(inputs["tiny_prot"]) + DEGENERATE_PROTEINS
    ora = ol.ora()
    n_anchor = 0
    for max_occ in (20000, 50):
        got = mp.seed_batch(ctx, mi, max_occ, seqs)
        for s, a in zip(seqs, got):
            n_a = C.c_int64(0)
            ptr = ora.ora_seed_anchors(C.byref(tab), C.c_void_p(idx.ki), C.c_int64(idx.n_kb), C.c_void_p(idx.kb), C.c_int32(idx.opt.kmer),
                                       C.c_int32(idx.opt.mod_bit), C.c_int32(max_occ), C.c_char_p(s), C.c_int32(len(s)), C.byref(n_a))
            want = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint64)), shape=(max(n_a.value, 1),)).copy()[:n_a.value] if ptr else np.zeros(0, np.uint64)
            if ptr:
                ol._libc.free(C.c_void_p(ptr))
            assert np.array_equal(a, want), (max_occ, len(s), len(a), n_a.value)
            n_anchor += len(want)
    assert n_anchor > 0
    mp.lib().mp_idx_destroy(mi)


def oracle_refine(tab, par, min_aa_len, max_ava, nt, prot):
    ora = ol.ora()
    nb, sb = C.c_int32(0), C.c_int32(0)
    ptr = ora.ora_refine(C.byref(tab), C.byref(par), C.c_int32(min_aa_len), C.c_int32(max_ava), C.c_void_p(nt.ctypes.data), C.c_int64(len(nt)),
                         C.c_char_p(prot), C.c_int32(len(prot)), C.byref(nb), C.byref(sb))
    want = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint64)), shape=(max(nb.value, 1),)).copy()[:nb.value] if ptr else np.zeros(0, np.uint64)
    if ptr:
        ol._libc.free(C.c_void_p(ptr))
    return want, sb.value


@pytest.mark.parametrize("code", E2E_CODES)
def test_refine_trans_code(ctx, refine_inputs, std_tab, use_code, code):  # noqa: F811
    """mpb_refine_batch against ora_refine under -T<code>, window by window (both strands, contig ends, tile-boundary lengths, the
    stop-free and poly-A contigs, N runs), at the default refinement options."""
    path, seqs, windows, slices = refine_inputs
    tab = use_code(code)
    io = mp.idxopt()
    io.trans_code = code
    mi = mp.idx_load(path, 8, io)
    mo = mp.mapopt()
    got = mp.refine_batch(ctx, mi, mo, seqs, windows)
    par = mp.ChainPar(mo.max_intron, mo.max_gap, mo.bw, mo.max_chn_max_skip, mo.max_chn_iter, mo.min_chn_cnt, mo.min_chn_sc,
                      mo.chn_coef_log, 0 if (mo.flag & 0x1) else 1, mo.kmer2, 0)
    L_ = mi.contents.opt.min_aa_len
    n_hit, n_differ, bad = 0, 0, []
    for (q, vid, as_, ae), nt, (a, sc) in zip(windows, slices, got):
        want, sb = oracle_refine(tab, par, L_, mo.max_ava, nt, seqs[q])
        if not np.array_equal(a, want) or (len(want) and sc != sb):
            bad.append((q, vid, as_, ae, len(a), len(want), sc, sb))
        n_hit += len(want) > 0
        std, _ = oracle_refine(std_tab[0], par, L_, mo.max_ava, nt, seqs[q])
        n_differ += not np.array_equal(std, want)
    assert not bad, (len(bad), bad[:5])
    assert n_hit >= 10 and n_differ >= 5, (n_hit, n_differ)
    mp.lib().mp_idx_destroy(mi)


# ---- D. end to end -----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sets(inputs):  # noqa: F811
    return dbg_lib.input_sets(str(inputs["dir"] / "dbg"))


@pytest.mark.parametrize("fmt", E2E_FORMATS, ids=[" ".join(f) for f in E2E_FORMATS])
@pytest.mark.parametrize("name", ["tiny", "tiny5", "DPP3"])
@pytest.mark.parametrize("code", E2E_CODES)
def test_trans_code_end_to_end(sets, code, name, fmt):
    """The library under the reference's CLI with -T<code>: the PAF and X / Y1 dump lines, the GFF, the --trans and the --aln output
    equal the reference CLI's."""
    args = [f"-T{code}"] + fmt
    g, p = sets[name]
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, args, g, p)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    got, want = dbg_lib.digest(out, err), dbg_lib.ref_cli_dbg(args, g, p)
    assert (got["lines"], got["dump_lines"]) == (want["lines"], want["dump_lines"])
    assert got == want


def test_mpi_round_trip_trans_code(ctx, sets, use_code, tmp_path):
    """A -T2 index file byte-identical to the reference's -T2 -d output, loaded straight into device memory: loading it switches the
    tables to code 2 (the code is part of the file), and mapping with it prints the reference's -T2 PAF."""
    g, p = sets["tiny"]
    L = mp.lib()
    io = mp.idxopt()
    io.trans_code = 2
    use_code(2)
    mi0 = mp.idx_load(g, 4, io)
    mpi = str(tmp_path / "tiny.T2.mpi")
    assert L.mp_idx_dump(mpi.encode(), mi0) == 0
    L.mp_idx_destroy(mi0)
    assert ol.file_digest(mpi) == ol.ref_index_file(g, ["-T2"])
    code2 = ol.codon_array(product_tables())
    use_code(1)
    mi = mp.idx_load_device(ctx, mpi)
    assert mi.contents.opt.trans_code == 2 and np.array_equal(ol.codon_array(product_tables()), code2)
    out = str(tmp_path / "o.paf")
    mp.map_file(ctx, mi, p, out)
    L.mp_idx_destroy(mi)
    paf = open(out, "rb").read()
    want = dbg_lib.ref_cli_dbg(["-T2"] + E2E_FORMATS[0], g, p)  # the dump switches print to stderr only: stdout is the PAF
    assert (hashlib.sha256(paf).hexdigest(), paf.count(b"\n")) == (want["sha256"], want["lines"])


def test_loci_trans_code(ctx, use_code, tmp_path):
    """Locus mode under -T2: the loci of tiny5 give the reference's PAF of each locus mapped on its own with -T2."""
    case = loci_lib.build_cases(str(tmp_path))["tiny5_T2"]
    assert case["args"] == ["-T2"]
    use_code(2)
    io = mp.idxopt()
    io.trans_code = 2
    mi = mp.idx_load(case["genome"], 4, io)
    paf, _ = map_case(ctx, mi, case)
    mp.lib().mp_idx_destroy(mi)
    assert loci_lib.digest(paf) == loci_lib.ref_answer(case)
