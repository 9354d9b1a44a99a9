"""CPU: the file driver (map_file: one reader, n mapper threads, the calling thread writing in input order) with n independent oracle
backends writes the reference's output, byte for byte, in every output format, for one backend as for several -- also when the work
units finish out of input order (HC_UNIT_DELAY) and when a unit holds a single protein."""
import ctypes as C
import gzip
import os
import subprocess
import sys

import pytest

import build_hostcheck_multi
import oracle_lib as ol
from miniprot_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(build_hostcheck_multi.build())
    lib.hc_map_file_multi.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32, C.c_int64, C.c_int32]
    return lib


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    d = tmp_path_factory.mktemp("sets")
    out = {"DPP3": (ol.DPP3_GENOME, ol.DPP3_PROTEIN)}
    for cfg in ("tiny", "tiny5"):
        out[cfg] = synth.generate(synth.CONFIGS[cfg], str(d / cfg))
    return out


def gold(name):
    path = os.path.join(GOLD, name)
    return gzip.open(path + ".gz", "rb").read() if os.path.exists(path + ".gz") else open(path, "rb").read()


def run(hc, g, p, out, n, flag=0, mini_batch=0):
    assert hc.hc_map_file_multi(g.encode(), p.encode(), out.encode(), flag, mini_batch, n) == 0
    return open(out, "rb").read()


@pytest.mark.parametrize("pipeline", ["1", "0"])
@pytest.mark.parametrize("mini_batch", [0, 1200, 1])
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_paf_golden(hc, sets, tmp_path, monkeypatch, n, mini_batch, pipeline):
    """MPB_FILE_PIPELINE=0 (the serial form, with one backend only) must not change the output."""
    monkeypatch.setenv("HC_UNIT_DELAY", str(7 * n + mini_batch))
    monkeypatch.setenv("MPB_FILE_PIPELINE", pipeline)
    for name, paf in (("tiny", "tiny.paf"), ("tiny5", "tiny5.paf")):
        g, p = sets[name]
        assert run(hc, g, p, str(tmp_path / "o.paf"), n, mini_batch=mini_batch) == gold(paf), name


@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_dpp3_paf_golden(hc, sets, tmp_path, monkeypatch, n):
    """The reference's DPP3 pair (the oracle DP is slow on it: one mini-batch size per mapper count)."""
    monkeypatch.setenv("HC_UNIT_DELAY", str(n))
    g, p = sets["DPP3"]
    assert run(hc, g, p, str(tmp_path / "o.paf"), n, mini_batch=(0, 1200, 1)[n % 3]) == gold("DPP3_default.paf")


FORMATS = {"gff": (0x8, None), "gtf": (0x20, None), "aln": (0x80, None), "trans": (0x100 | 0x4, None), "gff_only": (0x8 | 0x10, "#")}


@pytest.mark.parametrize("fmt", sorted(FORMATS))
@pytest.mark.parametrize("n", [1, 2, 3, 5])
def test_other_formats_golden(hc, sets, tmp_path, monkeypatch, n, fmt):
    """GFF3 / GTF number every printed hit with a counter that runs over the whole file: units mapped out of order must not
    disturb it."""
    flag, delim = FORMATS[fmt]
    if delim:
        monkeypatch.setenv("HC_GFF_DELIM", delim)
    monkeypatch.setenv("HC_UNIT_DELAY", str(11 * n))
    for mini_batch in (0, 1200, 1):
        g, p = sets["tiny5"]
        assert run(hc, g, p, str(tmp_path / "o.txt"), n, flag=flag, mini_batch=mini_batch) == gold(f"tiny5_{fmt}.txt"), mini_batch
    if n == 3:
        g, p = sets["DPP3"]
        assert run(hc, g, p, str(tmp_path / "d.txt"), n, flag=flag, mini_batch=1200) == gold(f"DPP3_{fmt}.txt")


def test_empty_and_missing_input(hc, sets, tmp_path):
    g, _ = sets["tiny"]
    empty = tmp_path / "empty.faa"
    empty.write_bytes(b"")
    assert run(hc, g, str(empty), str(tmp_path / "e.paf"), 3) == b""
    assert run(hc, g, str(empty), str(tmp_path / "e.gff"), 3, flag=0x8) == b"##gff-version 3\n"  # the header, as map_file writes it
    assert hc.hc_map_file_multi(g.encode(), str(tmp_path / "missing.faa").encode(), str(tmp_path / "m.paf").encode(), 0, 0, 3) == -1


_CHILD = r"""
import ctypes as C, sys, threading
lib = C.CDLL(sys.argv[1])
lib.hc_map_file_multi.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint32, C.c_int64, C.c_int32]
g, p, empty, out = (a.encode() for a in sys.argv[2:6])
assert lib.hc_map_file_multi(g, p, out, 0, 1, 4) == 0
assert lib.hc_map_file_multi(g, p, out, 0, 1, 1) == 0  # one mapper thread
assert lib.hc_map_file_multi(g, p, out, 0, 0, 1) == 0  # one unit: no thread
assert lib.hc_map_file_multi(g, empty, out, 0, 0, 4) == 0
assert lib.hc_map_file_multi(g, b"/nonexistent.faa", out, 0, 0, 4) == -1
assert threading.active_count() == 1
print("clean")
"""


def test_no_thread_left_behind(sets, tmp_path):
    """Every call -- a full file, an empty one, a missing one -- returns with its threads joined: the process exits normally, at
    once, with nothing left running."""
    g, p = sets["tiny"]
    empty = tmp_path / "empty.faa"
    empty.write_bytes(b"")
    env = dict(os.environ, HC_UNIT_DELAY="5")
    r = subprocess.run([sys.executable, "-c", _CHILD, build_hostcheck_multi.build(), g, p, str(empty), str(tmp_path / "o.paf")], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "clean", r.stderr
    assert open(tmp_path / "o.paf", "rb").read() == b""  # the last call that opened the output wrote nothing into it
