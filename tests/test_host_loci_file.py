"""The locus file driver (loci_file_read + map_loci_file) on the CPU, with the C oracle as the stage backend and the locus seeding
oracle of hostcheck_loci.cpp: every case of loci_lib under every option set of loci_file_lib must print the reference's output for
its loci byte for byte (stored answers); bad input is refused before anything is written; the output does not depend on -K, on the
number of backends or on MPB_FILE_PIPELINE."""
import ctypes as C
import os

import pytest

import build_hostcheck_loci_file
import loci_file_lib
import loci_lib
import miniprot_b200 as mp


@pytest.fixture(scope="module")
def hc():
    L = C.CDLL(build_hostcheck_loci_file.build())
    L.mp_start()
    C.c_int32.in_dll(L, "mp_verbose").value = 1
    L.mpb_idx_load_genome.restype = C.POINTER(mp.Idx)
    L.mpb_idx_load_genome.argtypes = [C.c_char_p, C.POINTER(mp.IdxOpt)]
    L.mp_idx_destroy.argtypes = [C.POINTER(mp.Idx)]
    L.hc_map_loci_file.restype = C.c_int32
    L.hc_map_loci_file.argtypes = [C.POINTER(mp.Idx), C.c_char_p, C.c_char_p, C.POINTER(mp.MapOpt), C.c_int32, C.c_char_p]
    return L


@pytest.fixture(scope="module")
def tool():
    return loci_file_lib.map_loci_tool()


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    d = tmp_path_factory.mktemp("loci_file")
    cs = loci_lib.build_cases(str(d))
    for name, case in cs.items():
        case["tsv"] = loci_file_lib.write_tsv(str(d / f"{name}.tsv"), case["loci"])
    return cs


def run(hc, tool, case, args, tmp_path, n_backends=1, tsv=None, prot=None):
    """(return code, output bytes or None when no file was created) of the file driver on the case under CLI options `args`"""
    _, io, mo = tool.options([*args, "g", "p", "l"], L=hc)
    mi = hc.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
    assert mi and not mi.contents.ki and not mi.contents.kb and mi.contents.n_kb == 0
    out = tmp_path / "out"
    if out.exists():
        out.unlink()
    rc = hc.hc_map_loci_file(mi, (prot or case["proteins"]).encode(), (tsv or case["tsv"]).encode(), C.byref(mo), n_backends, str(out).encode())
    hc.mp_idx_destroy(mi)
    return rc, out.read_bytes() if out.exists() else None


@pytest.mark.parametrize("opts", list(loci_file_lib.OPTION_SETS))
@pytest.mark.parametrize("name", loci_file_lib.CASES)
def test_host_loci_file_reference(hc, tool, cases, tmp_path, name, opts):
    args = loci_file_lib.OPTION_SETS[opts]
    rc, out = run(hc, tool, cases[name], args, tmp_path)
    assert rc == 0
    assert loci_lib.digest(out) == loci_file_lib.ref_answer(cases[name], args)


def test_host_loci_file_default_is_loci_paf(hc, tool, cases, tmp_path):
    """With default options the file driver prints what mpb_map_loci + mpb_format_paf print (loci_lib's stored answer)."""
    for name in ("DPP3", "tiny5"):
        rc, out = run(hc, tool, cases[name], [], tmp_path)
        assert rc == 0 and loci_lib.digest(out) == loci_lib.ref_answer(cases[name])


@pytest.mark.parametrize("args,n_backends,serial", [(["-K1"], 1, False), (["-K1"], 3, False), (["-K700", "--gff"], 2, False), (["-K700", "--gff"], 1, True),
                                                    (["-K1", "--gtf", "-u"], 4, False)])
def test_host_loci_file_units(hc, tool, cases, tmp_path, monkeypatch, args, n_backends, serial):
    """One pair per unit, small units, several backends and the serial form give the bytes of one whole batch."""
    if serial:
        monkeypatch.setenv("MPB_FILE_PIPELINE", "0")
    case = cases["tiny"]
    rc, out = run(hc, tool, case, args, tmp_path, n_backends)
    assert rc == 0
    assert loci_lib.digest(out) == loci_file_lib.ref_answer(case, [a for a in args if not a.startswith("-K")])


def test_host_loci_file_duplicate_protein(hc, tool, cases, tmp_path):
    """A protein name that occurs twice stands for its last record."""
    case = cases["DPP3"]
    (pn, ps), = loci_lib.read_fasta(case["proteins"])
    prot = loci_lib.write_fasta(str(tmp_path / "dup.fa"), [(pn, ps[: len(ps) // 2]), (b"other", ps), (pn, ps)])
    rc, out = run(hc, tool, case, [], tmp_path, prot=prot)
    assert rc == 0 and loci_lib.digest(out) == loci_lib.ref_answer(case)


def test_host_loci_file_refusals(hc, tool, cases, tmp_path, capfd):
    case = cases["DPP3"]
    p, c, _, _ = case["loci"][0]
    L = len(loci_lib.read_fasta(case["genome"])[0][1])
    good = f"{p}\t{c}\t0\t100\n"
    bad_lines = {
        "too few fields": f"{p}\t{c}\t0\n",
        "non-integer start": f"{p}\t{c}\tx\t100\n",
        "non-integer end": f"{p}\t{c}\t0\t100bp\n",
        "unknown protein": f"nosuchprotein\t{c}\t0\t100\n",
        "unknown contig": f"{p}\tnosuchcontig\t0\t100\n",
        "negative start": f"{p}\t{c}\t-1\t100\n",
        "end past the contig": f"{p}\t{c}\t0\t{L + 1}\n",
        "empty range": f"{p}\t{c}\t50\t50\n",
        "reversed range": f"{p}\t{c}\t60\t50\n",
    }
    for why, line in bad_lines.items():
        tsv = tmp_path / "bad.tsv"
        tsv.write_text("# header\n\n" + good + line + good)
        capfd.readouterr()
        rc, out = run(hc, tool, case, ["--gff"], tmp_path, tsv=str(tsv))
        assert rc == -1 and out is None, why
        assert f"{tsv}:4:" in capfd.readouterr().err, why
    for prot, tsv in ((str(tmp_path / "missing.fa"), case["tsv"]), (case["proteins"], str(tmp_path / "missing.tsv"))):
        capfd.readouterr()
        rc, out = run(hc, tool, case, ["--gff"], tmp_path, tsv=tsv, prot=prot)
        assert rc == -1 and out is None
        assert "missing." in capfd.readouterr().err
    # what locus mode refuses: every debugging bit but --no-kalloc
    for bit in (mp.DBG_ANCHOR, mp.DBG_CHAIN, mp.DBG_QNAME, mp.DBG_MORE_DP, mp.DBG_NO_REFINE):
        old = mp.set_dbg_flag(bit, hc)
        try:
            rc, out = run(hc, tool, case, ["--gff"], tmp_path)
        finally:
            mp.set_dbg_flag(old, hc)
        assert rc == -3 and out is None, bit
    old = mp.set_dbg_flag(mp.DBG_NO_KALLOC, hc)
    try:
        rc, out = run(hc, tool, case, [], tmp_path)
    finally:
        mp.set_dbg_flag(old, hc)
    assert rc == 0 and loci_lib.digest(out) == loci_lib.ref_answer(case)


def test_host_loci_file_refuses_spsc(hc, tool, cases, tmp_path):
    import dbg_lib

    case = cases["DPP3"]
    _, io, mo = tool.options(["g", "p", "l"], L=hc)
    mi = hc.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
    hc.mp_set_spsc.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32]
    hc.mp_set_spsc(dbg_lib.spsc_file(str(tmp_path)).encode(), C.cast(mi, C.c_void_p), C.byref(mo), 0)
    out = tmp_path / "out"
    rc = hc.hc_map_loci_file(mi, case["proteins"].encode(), case["tsv"].encode(), C.byref(mo), 1, str(out).encode())
    hc.mp_idx_destroy(mi)
    assert rc == -3 and not out.exists()


def test_host_idx_load_genome_mpi(hc, tool, cases, tmp_path):
    """A .mpi file gives the same genome-only index as its FASTA (its stored options, io ignored) and the same output."""
    case = cases["tiny5"]
    L = hc
    L.mp_idx_load.restype = C.POINTER(mp.Idx)
    L.mp_idx_load.argtypes = [C.c_char_p, C.POINTER(mp.IdxOpt), C.c_int32]
    L.mp_idx_dump.argtypes = [C.c_char_p, C.POINTER(mp.Idx)]
    _, io, mo = tool.options(["g", "p", "l"], L=hc)
    full = L.mp_idx_load(case["genome"].encode(), C.byref(io), 4)
    mpi = str(tmp_path / "tiny5.mpi")
    assert L.mp_idx_dump(mpi.encode(), full) == 0
    L.mp_idx_destroy(full)
    other = mp.IdxOpt()
    L.mp_idxopt_init(C.byref(other))
    other.kmer = 4
    mi = L.mpb_idx_load_genome(mpi.encode(), C.byref(other))
    assert mi and not mi.contents.ki and not mi.contents.kb and mi.contents.n_kb == 0 and mi.contents.opt.kmer == io.kmer
    fa = L.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
    a, b = mi.contents, fa.contents
    assert (a.n_block, a.nt.contents.n_ctg, a.nt.contents.l_seq) == (b.n_block, b.nt.contents.n_ctg, b.nt.contents.l_seq)
    assert [C.cast(a.bo, C.POINTER(C.c_uint32))[i] for i in range(2 * a.nt.contents.n_ctg + 1)] == \
        [C.cast(b.bo, C.POINTER(C.c_uint32))[i] for i in range(2 * b.nt.contents.n_ctg + 1)]
    out = tmp_path / "out"
    assert hc.hc_map_loci_file(mi, case["proteins"].encode(), case["tsv"].encode(), C.byref(mo), 1, str(out).encode()) == 0
    assert loci_lib.digest(out.read_bytes()) == loci_file_lib.ref_answer(case, [])
    L.mp_idx_destroy(mi)
    L.mp_idx_destroy(fa)
    assert not L.mpb_idx_load_genome(str(tmp_path / "missing.fa").encode(), None)


def test_tool_options(hc, tool):
    """tools/map_loci.py reads the reference CLI's options in command-line order and refuses -I and --spsc."""
    _, io, mo = tool.options(["-S", "-G", "5k", "--gff-only", "-P", "XY", "--max-intron-out=51", "--gff-delim=:", "-K2M", "-k5", "-L35",
                              "--outs=0.9", "-j2", "g", "p", "l"], L=hc)
    assert (mo.max_intron, mo.bw, mo.max_ext, mo.io, mo.io_end) == (5000, 5000, 1000, 10000, 10000)
    assert mo.flag & (mp.MP_F_NO_SPLICE | 0x8 | 0x10) == mp.MP_F_NO_SPLICE | 0x18
    assert (mo.gff_prefix, mo.max_intron_flank, mo.gff_delim, mo.mini_batch_size, mo.sp_model) == (b"XY", 26, ord(":"), 2000000, 2)
    assert abs(mo.out_sim - 0.9) < 1e-6 and (io.kmer, io.min_aa_len) == (5, 35)
    for refused in (["-I"], ["--spsc", "x.tsv"]):
        with pytest.raises(SystemExit):
            tool.options([*refused, "g", "p", "l"], L=hc)
    assert os.path.basename(tool.__file__) == "map_loci.py"
