"""CPU: the product's host pipeline, with the C oracle as stage backend (tests/hostcheck/hostcheck_dbg.cpp), under index and
refinement options off the defaults (-k -M -L -b -l, dbg_lib.INDEX_OPTION_SETS).  Stdout and the X / Y1 dump lines must equal
what the reference CLI prints with -t1 (stored digests, dbg_lib.ref_cli_dbg).  The CPU twin of the end-to-end part of
test_gpu_index_options.py."""
import pytest

import build_hostcheck_dbg
import dbg_lib


@pytest.fixture(scope="module")
def hc():
    return build_hostcheck_dbg.build()


@pytest.fixture(scope="module")
def sets(tmp_path_factory):
    return dbg_lib.input_sets(str(tmp_path_factory.mktemp("idxopt")))


# -L 41 is past what the GPU window kernels take; the oracle backend has no such limit and maps like the reference
@pytest.mark.parametrize("opts", [" ".join(o) or "defaults" for o in dbg_lib.INDEX_OPTION_SETS + [["-L41"]]])
@pytest.mark.parametrize("name", ["tiny", "tiny5", "DPP3"])
def test_index_options_golden(hc, sets, name, opts):
    args = ([] if opts == "defaults" else opts.split()) + dbg_lib.INDEX_SWITCHES
    g, p = sets[name]
    rc, out, err = dbg_lib.run_cli(hc, args, g, p)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    got, want = dbg_lib.digest(out, err), dbg_lib.ref_cli_dbg(args, g, p)
    assert (got["lines"], got["dump_lines"]) == (want["lines"], want["dump_lines"])
    assert got == want
