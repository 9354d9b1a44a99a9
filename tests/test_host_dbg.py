"""CPU: the debugging switches of the CLI (mp_dbg_flag: --dbg-qname, --dbg-anchor, --dbg-chain, --dbg-no-refine, --dbg-aflt) served
by the product's host pipeline with the C oracle as stage backend (tests/hostcheck/hostcheck_dbg.cpp: the oracle that also returns
the seeds).  Stdout and the dump lines on stderr must equal what the reference CLI prints with -t1 (stored digests,
dbg_lib.ref_cli_dbg)."""
import os

import pytest

import build_hostcheck_dbg
import dbg_lib
import oracle_lib as ol

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def hc():
    return build_hostcheck_dbg.build()


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    return dbg_lib.input_sets(str(tmp_path_factory.mktemp("dbg")))


def check(hc, args, g, p):
    rc, out, err = dbg_lib.run_cli(hc, args, g, p)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    got, want = dbg_lib.digest(out, err), dbg_lib.ref_cli_dbg(args, g, p)
    assert (got["lines"], got["dump_lines"]) == (want["lines"], want["dump_lines"])
    assert got == want
    return out, err


@pytest.mark.parametrize("switches", [" ".join(s) for s in dbg_lib.SWITCH_SETS])
@pytest.mark.parametrize("name", ["DPP3", "tiny", "tiny5", "short_ctg"])
def test_switches_golden(hc, sets, name, switches):
    g, p = sets[name]
    out, err = check(hc, switches.split(), g, p)
    if "--dbg-qname" in switches:
        qr = [l for l in dbg_lib.dump_lines(err) if l.startswith(b"QR\t")]
        assert qr and all(l.rstrip(b"\n").split(b"\t")[3] == b"0" for l in qr)  # one context: tid 0


def test_aflt_splice_scores(hc, tmp_path):
    sp = dbg_lib.spsc_file(str(tmp_path))
    check(hc, ["--dbg-aflt", "--spsc", sp], ol.DPP3_GENOME, ol.DPP3_PROTEIN)


def test_chain_cut_at_contig_boundary(hc, sets):
    """Some Y1 line of the short-contig genome prints an anchor that lies on another contig than the region's (negative offset or
    past the contig's end): the case mp_dbg_chain prints with the kept contig's block offset."""
    g, p = sets["short_ctg"]
    _, err = check(hc, ["--dbg-chain"], g, p)
    offs = [int(l.split(b"\t")[5]) for l in dbg_lib.dump_lines(err)]
    assert offs and (min(offs) < 0 or max(offs) >= 25_000)


def test_no_refine_without_no_align_refused(hc, sets):
    g, p = sets["tiny"]
    for extra in ([], ["--gff"]):
        rc, out, err = dbg_lib.run_cli(hc, ["--dbg-no-refine", *extra], g, p)
        assert rc == -3 and out == b"" and b"--dbg-no-refine" in err


@pytest.mark.parametrize("name,golden", [("tiny", "tiny.paf"), ("tiny5", "tiny5.paf"), ("DPP3", "DPP3_default.paf")])
def test_all_bits_clear_unchanged(hc, sets, name, golden):
    g, p = sets[name]
    rc, out, err = dbg_lib.run_cli(hc, ["--no-kalloc"], g, p)
    assert rc == 0 and out == open(os.path.join(GOLD, golden), "rb").read() and dbg_lib.dump_lines(err) == []
