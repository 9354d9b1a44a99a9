"""Locus sets on the CPU (map_locus_sets, and loci_file_read + map_loci_file over sets), with the C oracle as the stage backend and
the set seeding oracle of hostcheck_locus_sets.cpp: every case of locus_sets_lib under every option set must print the reference's
output for its sets byte for byte (stored answers); a set merged into a whole contig prints the whole-contig goldens; a set of one
locus prints what the locus file driver prints; the output does not depend on -K, on the number of backends, on MPB_FILE_PIPELINE or
on the order of the lines within a set; bad input is refused before anything is written."""
import ctypes as C
import os

import numpy as np
import pytest

import build_hostcheck_locus_sets
import loci_file_lib
import loci_lib
import locus_sets_lib
import miniprot_b200 as mp
import oracle_lib as ol


@pytest.fixture(scope="module")
def hc():
    L = C.CDLL(build_hostcheck_locus_sets.build())
    L.mp_start()
    C.c_int32.in_dll(L, "mp_verbose").value = 1
    L.mpb_idx_load_genome.restype = C.POINTER(mp.Idx)
    L.mpb_idx_load_genome.argtypes = [C.c_char_p, C.POINTER(mp.IdxOpt)]
    L.mp_idx_destroy.argtypes = [C.POINTER(mp.Idx)]
    L.hc_map_locus_sets_file.restype = C.c_int32
    L.hc_map_locus_sets_file.argtypes = [C.POINTER(mp.Idx), C.c_char_p, C.c_char_p, C.POINTER(mp.MapOpt), C.c_int32, C.c_char_p, C.c_int32]
    return L


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


def run(hc, tool, case, args, tmp_path, n_backends=1, tsv=None, prot=None, sets=True):
    """(return code, output bytes or None when no file was created) of the set file driver on the case under CLI options `args`"""
    _, io, mo = tool.options([*case.get("args", []), *args, "g", "p", "l"], L=hc)
    mi = hc.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
    out = tmp_path / "out"
    if out.exists():
        out.unlink()
    assert hc.ns_make_tables(io.trans_code) == 0  # what the CLI does for -T
    try:
        rc = hc.hc_map_locus_sets_file(mi, (prot or case["proteins"]).encode(), (tsv or case["tsv"]).encode(), C.byref(mo), n_backends, str(out).encode(),
                                       int(sets))
    finally:
        hc.ns_make_tables(1)
    hc.mp_idx_destroy(mi)
    return rc, out.read_bytes() if out.exists() else None


@pytest.mark.parametrize("opts", list(locus_sets_lib.OPTION_SETS))
@pytest.mark.parametrize("name", locus_sets_lib.CASES)
def test_host_locus_sets_reference(hc, tool, cases, tmp_path, name, opts):
    args = locus_sets_lib.OPTION_SETS[opts]
    rc, out = run(hc, tool, cases[name], args, tmp_path)
    assert rc == 0
    assert loci_lib.digest(out) == locus_sets_lib.ref_answer(cases[name], args)


@pytest.mark.parametrize("args,golden", [([], "DPP3_default.paf"), (["-j2"], "DPP3_j2.paf"), (["-G2k"], "DPP3_G2k.paf"), (["--gff"], "DPP3_gff.txt"),
                                         (["--gtf"], "DPP3_gtf.txt"), (["--aln"], "DPP3_aln.txt"), (["--trans", "-u"], "DPP3_trans.txt"),
                                         (["--gff-only", "--gff-delim=#"], "DPP3_gff_only.txt")])
def test_host_locus_sets_whole_contig(hc, tool, cases, tmp_path, args, golden):
    """[0, 1500) + [1500, L) of DPP3 merge into the whole contig: the reference's whole-genome output, byte for byte."""
    case = cases["DPP3"]
    tsv = locus_sets_lib.write_tsv(str(tmp_path / "whole.tsv"), [x for x in case["lines"] if x[4] == "whole"])
    rc, out = run(hc, tool, case, args, tmp_path, tsv=tsv)
    assert rc == 0 and out == open(os.path.join(ol.GOLDEN, golden), "rb").read()


@pytest.mark.parametrize("name", ["DPP3", "paralogs", "tiny", "tiny5"])
def test_host_locus_sets_single_locus(hc, tool, cases, tmp_path, name):
    """Sets of one locus each print what the locus file driver prints for the pairs (its stored answers)."""
    base = loci_lib.build_cases(str(tmp_path))[name]
    tsv = locus_sets_lib.write_tsv(str(tmp_path / "single.tsv"), [(*x, f"s{k}") for k, x in enumerate(base["loci"])])
    for args in ([], ["--gff"], ["-u", "--outn=1"]):
        rc, out = run(hc, tool, base, args, tmp_path, tsv=tsv)
        assert rc == 0 and loci_lib.digest(out) == loci_file_lib.ref_answer(base, args)


@pytest.mark.parametrize("args,n_backends,serial", [(["-K1"], 1, False), (["-K1"], 3, False), (["-K700", "--gff"], 2, False), (["-K700", "--gff"], 1, True),
                                                    (["-K1", "--gtf", "-u"], 2, False)])
def test_host_locus_sets_units(hc, tool, cases, tmp_path, monkeypatch, args, n_backends, serial):
    """One set per unit, small units, several backends and the serial form give the bytes of one whole batch."""
    if serial:
        monkeypatch.setenv("MPB_FILE_PIPELINE", "0")
    case = cases["tiny"]
    rc, out = run(hc, tool, case, args, tmp_path, n_backends)
    assert rc == 0
    assert loci_lib.digest(out) == locus_sets_lib.ref_answer(case, [a for a in args if not a.startswith("-K")])


def test_host_locus_sets_line_order(hc, tool, cases, tmp_path):
    """The lines of a set in another order, interleaved with other sets' lines, give the same bytes (sets keep their first-line order)."""
    rng = np.random.default_rng(5)
    for name in ("tiny5", "paralogs", "DPP3"):
        case = cases[name]
        sets = locus_sets_lib.sets_of(case["lines"])
        key = lambda x: (x[0], x[4])  # noqa: E731
        first = {}
        for x in case["lines"]:
            first.setdefault(key(x), x)
        rest = [x for x in case["lines"] if first[key(x)] is not x]
        lines = list(first.values()) + [rest[k] for k in rng.permutation(len(rest))]
        assert len(first) == len(sets) and sorted(lines) == sorted(case["lines"])
        tsv = locus_sets_lib.write_tsv(str(tmp_path / "shuffled.tsv"), lines)
        for args in ([], ["--gff"]):
            rc, out = run(hc, tool, case, args, tmp_path, tsv=tsv)
            assert rc == 0 and loci_lib.digest(out) == locus_sets_lib.ref_answer(case, args), name


def test_host_locus_sets_api(hc, tool, cases, tmp_path):
    """map_locus_sets + mpb_format_paf print the file driver's PAF; every hit lies in a merged range of its set; a set of one locus gives
    map_loci's regions."""
    for name in ("paralogs", "tiny5"):
        case = cases[name]
        _, io, mo = tool.options([*case["args"], "g", "p", "l"], L=hc)
        mi = hc.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
        names, seqs, qid = loci_lib.index_of(case)
        off, loci = locus_sets_lib.set_arrays(mi, case, qid)
        sets = [loci[off[k]:off[k + 1]] for k in range(len(off) - 1)]
        rc, n_reg, reg = mp.map_locus_sets(None, mi, mo, seqs, names, sets, L=hc, fn="hc_map_locus_sets")
        assert rc == 0
        paf = mp.loci_paf(mi, mo, seqs, names, [s[0] for s in sets], n_reg, reg, L=hc, fn="hc_format_paf")
        assert loci_lib.digest(paf) == locus_sets_lib.ref_answer(case, [])
        nt = mi.contents.nt.contents
        for k, s in enumerate(sets):
            merged = locus_sets_lib.canonical([(c, a, b) for _, c, a, b in s], {i: i for i in range(nt.n_ctg)})
            for r in mp.regions(reg[k], int(n_reg[k])) if n_reg[k] else []:
                vid, vs, ve = r[0][9], r[0][12], r[0][13]
                cid, clen = vid >> 1, nt.ctg[vid >> 1].len
                st, en = (clen - ve, clen - vs) if vid & 1 else (vs, ve)
                assert any(c == cid and a <= st and en <= b for c, a, b in merged), (name, k)
        mp.free_loci_regs(n_reg, reg)
        # single-locus sets = map_loci
        pairs = loci[:6]
        rc, n1, r1 = mp.map_locus_sets(None, mi, mo, seqs, names, [[p] for p in pairs], L=hc, fn="hc_map_locus_sets")
        rc2, n2, r2 = mp.map_loci(None, mi, mo, seqs, names, pairs, L=hc, fn="hc_map_loci")
        assert rc == rc2 == 0 and list(n1) == list(n2)
        for k in range(len(pairs)):
            if n1[k]:
                assert mp.regions(r1[k], int(n1[k])) == mp.regions(r2[k], int(n2[k]))
        mp.free_loci_regs(n1, r1), mp.free_loci_regs(n2, r2)
        hc.mp_idx_destroy(mi)


def test_host_locus_sets_api_refusals(hc, tool, cases):
    case = cases["tiny"]
    _, io, mo = tool.options(["g", "p", "l"], L=hc)
    mi = hc.mpb_idx_load_genome(case["genome"].encode(), C.byref(io))
    names, seqs, qid = loci_lib.index_of(case)
    call = lambda sets: mp.map_locus_sets(None, mi, mo, seqs, names, sets, L=hc, fn="hc_map_locus_sets")[0]  # noqa: E731
    assert call([]) == 0
    assert call([[(0, 0, 100, 5000)], []]) == -1                    # an empty set
    assert call([[(0, 0, 100, 5000), (1, 0, 6000, 9000)]]) == -1    # loci of two proteins
    assert call([[(0, 0, 100, 5000), (0, 0, 5000, 4000)]]) == -1    # a malformed locus
    assert call([[(0, 7, 100, 5000)]]) == -1                        # no such contig
    assert call([[(0, 0, 100, 5000), (0, 0, 4000, 9000)]]) == 0     # overlapping loci are merged
    old = mp.set_dbg_flag(mp.DBG_CHAIN, hc)
    try:
        assert call([[(0, 0, 100, 5000)]]) == -3
    finally:
        mp.set_dbg_flag(old, hc)
    hc.mp_idx_destroy(mi)


def test_host_locus_sets_file_refusals(hc, tool, cases, tmp_path, capfd):
    case = cases["DPP3"]
    p, c = case["lines"][0][:2]
    L = len(loci_lib.read_fasta(case["genome"])[0][1])
    good = f"{p}\t{c}\t0\t100\tA\n"
    bad_lines = {
        "too few fields": f"{p}\t{c}\t0\n",
        "non-integer end": f"{p}\t{c}\t0\t100bp\tA\n",
        "unknown protein": f"nosuchprotein\t{c}\t0\t100\tA\n",
        "unknown contig": f"{p}\tnosuchcontig\t0\t100\n",
        "end past the contig": f"{p}\t{c}\t0\t{L + 1}\tA\n",
        "empty range": f"{p}\t{c}\t50\t50\tB\n",
    }
    for why, line in bad_lines.items():
        tsv = tmp_path / "bad.tsv"
        tsv.write_text("# header\n\n" + good + line + good)
        capfd.readouterr()
        rc, out = run(hc, tool, case, ["--gff"], tmp_path, tsv=str(tsv))
        assert rc == -1 and out is None, why
        assert f"{tsv}:4:" in capfd.readouterr().err, why
    for bit in (mp.DBG_ANCHOR, mp.DBG_QNAME, mp.DBG_NO_REFINE):
        old = mp.set_dbg_flag(bit, hc)
        try:
            rc, out = run(hc, tool, case, ["--gff"], tmp_path)
        finally:
            mp.set_dbg_flag(old, hc)
        assert rc == -3 and out is None, bit


def test_host_locus_sets_labels(hc, tool, cases, tmp_path):
    """Without --sets the 5th column is ignored (one set per line, the locus file driver's output); with it, lines of one protein and
    no label form one set, and further columns are ignored."""
    base = loci_lib.build_cases(str(tmp_path))["tiny"]
    tsv = locus_sets_lib.write_tsv(str(tmp_path / "labelled.tsv"), [(*x, "same") for x in base["loci"]])
    rc, out = run(hc, tool, base, [], tmp_path, tsv=tsv, sets=False)
    assert rc == 0 and loci_lib.digest(out) == loci_file_lib.ref_answer(base, [])
    case = cases["tiny5"]
    tsv = tmp_path / "extra.tsv"
    tsv.write_text("".join(f"{p}\t{c}\t{st}\t{en}" + (f"\t{lab}" if lab else "\t_none_") + "\textra\tcolumns\n" for p, c, st, en, lab in case["lines"]))
    rc, out = run(hc, tool, case, [], tmp_path, tsv=str(tsv))
    assert rc == 0 and loci_lib.digest(out) == locus_sets_lib.ref_answer(case, [])


def test_tool_sets_option(tool):
    """tools/map_loci.py --sets selects the set file driver; -I and --spsc stay refused with it."""
    assert tool.parser().parse_args(["--sets", "g", "p", "l"]).sets
    assert not tool.parser().parse_args(["g", "p", "l"]).sets
    for refused in (["-I"], ["--spsc", "x.tsv"]):
        with pytest.raises(SystemExit):
            tool.parser().parse_args(["--sets", *refused, "g", "p", "l"])
