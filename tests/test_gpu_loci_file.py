"""The locus file driver (mpb_map_loci_file*, mpb_idx_load_genome, tools/map_loci.py) on the GPU.

* against the reference: every case of loci_lib under every option set of loci_file_lib prints the reference's output for its loci
  (stored answers) through mpb_map_loci_file, and the same bytes through mpb_map_loci_file_multi on two contexts of device 0 with
  small units and through the serial form (MPB_FILE_PIPELINE=0);
* tools/map_loci.py with a FASTA genome and with a .mpi file, on one context and on two;
* default options print what mpb_map_loci + mpb_format_paf print;
* a genome-only index uploads the packed genome and nothing of a k-mer table;
* refusals write nothing."""
import ctypes as C
import os
import subprocess
import sys

import pytest

import dbg_lib
import loci_file_lib
import loci_lib
import miniprot_b200 as mp

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
    d = tmp_path_factory.mktemp("loci_file")
    cs = loci_lib.build_cases(str(d))
    for name, case in cs.items():
        case["tsv"] = loci_file_lib.write_tsv(str(d / f"{name}.tsv"), case["loci"])
    return cs


_libc = C.CDLL(None)
_libc.fopen.restype, _libc.fopen.argtypes = C.c_void_p, [C.c_char_p, C.c_char_p]
_libc.fclose.argtypes = [C.c_void_p]


def map_to_stream(ctx, mi, case, mo, path):
    """mpb_map_loci_file into a C stream opened on path; (return code, bytes)"""
    L = mp.lib()
    L.mpb_map_loci_file.restype = C.c_int32
    L.mpb_map_loci_file.argtypes = [C.c_void_p, C.POINTER(mp.Idx), C.c_char_p, C.c_char_p, C.POINTER(mp.MapOpt), C.c_void_p]
    fp = _libc.fopen(str(path).encode(), b"wb")
    rc = L.mpb_map_loci_file(ctx.h, mi, case["proteins"].encode(), case["tsv"].encode(), C.byref(mo), fp)
    _libc.fclose(fp)
    return rc, open(path, "rb").read()


def multi_path(ctxs, mi, case, mo, path, tsv=None):
    """mpb_map_loci_file_multi_path's return code; the output file is removed first"""
    if os.path.exists(path):
        os.unlink(path)
    arr = (C.c_void_p * len(ctxs))(*[c.h if c else None for c in ctxs])
    return mp.lib().mpb_map_loci_file_multi_path(arr, len(ctxs), mi, case["proteins"].encode(), (tsv or case["tsv"]).encode(), C.byref(mo), str(path).encode())


@pytest.mark.parametrize("opts", list(loci_file_lib.OPTION_SETS))
@pytest.mark.parametrize("name", loci_file_lib.CASES)
def test_loci_file_reference(ctx, ctx_pair, tool, cases, tmp_path, monkeypatch, name, opts):
    case, args = cases[name], loci_file_lib.OPTION_SETS[opts]
    _, io, mo = tool.options([*args, "g", "p", "l"])
    mi = mp.idx_load_genome(case["genome"], io)
    rc, out = map_to_stream(ctx, mi, case, mo, tmp_path / "one")
    assert rc == 0
    assert loci_lib.digest(out) == loci_file_lib.ref_answer(case, args)
    # two contexts, units of a few pairs
    _, _, mo_small = tool.options([*args, "-K", "1500", "g", "p", "l"])
    assert multi_path(ctx_pair, mi, case, mo_small, tmp_path / "two") == 0
    assert (tmp_path / "two").read_bytes() == out
    # one context, one pair per unit, one step after another on the calling thread
    monkeypatch.setenv("MPB_FILE_PIPELINE", "0")
    _, _, mo_one = tool.options([*args, "-K1", "g", "p", "l"])
    mp.map_loci_file(ctx, mi, case["proteins"], case["tsv"], str(tmp_path / "serial"), mo_one)
    assert (tmp_path / "serial").read_bytes() == out
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("name", ["DPP3", "tiny5"])
def test_default_is_loci_paf(ctx, cases, tmp_path, name):
    """With default options the file driver prints what mpb_map_loci + mpb_format_paf print for the same pairs."""
    case = cases[name]
    mi = mp.idx_load(case["genome"], 4)
    names, seqs, qid = loci_lib.index_of(case)
    loci = loci_lib.loci_tuples(mi, case, qid)
    mo = mp.mapopt()
    rc, n_reg, reg = mp.map_loci(ctx, mi, mo, seqs, names, loci)
    assert rc == 0
    want = mp.loci_paf(mi, mo, seqs, names, loci, n_reg, reg)
    mp.free_loci_regs(n_reg, reg)
    mp.map_loci_file(ctx, mi, case["proteins"], case["tsv"], str(tmp_path / "out"), mo)
    assert (tmp_path / "out").read_bytes() == want and want
    mp.lib().mp_idx_destroy(mi)


@pytest.mark.parametrize("opts", ["default", "gff", "index_options"])
def test_map_loci_tool(cases, tmp_path, opts):
    """tools/map_loci.py with a FASTA genome and with a .mpi file, on one context and on two."""
    args = loci_file_lib.OPTION_SETS[opts]
    for name in ("DPP3", "tiny"):
        case = cases[name]
        genomes = [case["genome"]]
        if name == "tiny":
            io = mp.idxopt()
            for a in args:  # the .mpi file carries the index options
                if a[:2] in ("-k", "-M", "-L", "-b"):
                    setattr(io, {"-k": "kmer", "-M": "mod_bit", "-L": "min_aa_len", "-b": "bbit"}[a[:2]], int(a[2:]))
            mi = mp.idx_load(case["genome"], 4, io)
            genomes.append(str(tmp_path / "tiny.mpi"))
            assert mp.lib().mp_idx_dump(genomes[-1].encode(), mi) == 0
            mp.lib().mp_idx_destroy(mi)
        for genome in genomes:
            for devices in (["--devices", "0"], ["--devices", "0,0", "-K2000"]):
                cmd = [sys.executable, os.path.join(ROOT, "tools", "map_loci.py"), *args, *devices, genome, case["proteins"], case["tsv"]]
                r = subprocess.run(cmd, capture_output=True)
                assert r.returncode == 0, r.stderr.decode()[-2000:]
                assert loci_lib.digest(r.stdout) == loci_file_lib.ref_answer(case, args), (genome, devices, r.stderr.decode()[-2000:])


def test_map_loci_tool_refusals(cases):
    case = cases["DPP3"]
    for refused in (["-I"], ["--spsc", "x.tsv"]):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "map_loci.py"), *refused, case["genome"], case["proteins"], case["tsv"]],
                           capture_output=True)
        assert r.returncode != 0 and not r.stdout and refused[0].encode() in r.stderr


def test_genome_only_upload(cases, tmp_path):
    """idx_load_genome builds no k-mer table: a fresh context uploads the packed genome (plus the proteins and work lists)."""
    case = cases["tiny"]
    mi = mp.idx_load_genome(case["genome"])
    assert not mi.contents.ki and not mi.contents.kb and mi.contents.n_kb == 0
    c = mp.Context(0)
    try:
        c.reset_stats()
        mp.map_loci_file(c, mi, case["proteins"], case["tsv"], str(tmp_path / "out"), mp.mapopt())
        seq_bytes = (mi.contents.nt.contents.l_seq + 1) // 2
        assert seq_bytes <= c.stats().h2d_bytes <= seq_bytes + (1 << 20)
        assert loci_lib.digest((tmp_path / "out").read_bytes()) == loci_file_lib.ref_answer(case, [])
    finally:
        c.close()
    mp.lib().mp_idx_destroy(mi)


def test_refusals(ctx, ctx_pair, cases, tmp_path, capfd):
    case = cases["DPP3"]
    out = tmp_path / "out"
    mi = mp.idx_load_genome(case["genome"])
    c0 = ctx.stats().n_anchors
    p, c, _, _ = case["loci"][0]
    tsv = tmp_path / "bad.tsv"
    for line in (f"{p}\t{c}\t0\n", f"{p}\t{c}\t0\t1e3\n", f"other\t{c}\t0\t100\n", f"{p}\tother\t0\t100\n", f"{p}\t{c}\t100\t100\n"):
        tsv.write_text(f"{p}\t{c}\t0\t100\n" + line)
        capfd.readouterr()
        assert multi_path([ctx], mi, case, mp.mapopt(), out, str(tsv)) == -1 and not out.exists(), line
        assert f"{tsv}:2:" in capfd.readouterr().err
    assert multi_path([ctx], mi, dict(case, proteins=str(tmp_path / "none.fa")), mp.mapopt(), out) == -1 and not out.exists()
    assert multi_path([ctx_pair[0], ctx_pair[0]], mi, case, mp.mapopt(), out) == -1 and not out.exists()
    assert multi_path([ctx, None], mi, case, mp.mapopt(), out) == -1 and not out.exists()
    for over in (dict(go=0), dict(ie_coef=100.0)):
        assert multi_path([ctx], mi, case, mp.mapopt(**over), out) == -3 and not out.exists(), over
    for bit in (mp.DBG_ANCHOR, mp.DBG_CHAIN, mp.DBG_QNAME, mp.DBG_MORE_DP, mp.DBG_NO_REFINE):
        old = mp.set_dbg_flag(bit)
        try:
            rc = multi_path(ctx_pair, mi, case, mp.mapopt(), out)
        finally:
            mp.set_dbg_flag(old)
        assert rc == -3 and not out.exists(), bit
    mo = mp.mapopt()
    mp.lib().mp_set_spsc.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32]
    mp.lib().mp_set_spsc(dbg_lib.spsc_file(str(tmp_path)).encode(), C.cast(mi, C.c_void_p), C.byref(mo), 0)
    assert multi_path([ctx], mi, case, mo, out) == -3 and not out.exists()
    mp.lib().mp_idx_destroy(mi)
    io = mp.idxopt()
    io.min_aa_len = 41
    mi = mp.idx_load_genome(case["genome"], io)
    assert multi_path([ctx], mi, case, mp.mapopt(), out) == -3 and not out.exists()
    mp.lib().mp_idx_destroy(mi)
    assert ctx.stats().n_anchors == c0  # nothing was seeded by any refused call
