"""GPU: several contexts in one process -- mpb_map_file_multi over two and three contexts, an index shared between contexts
(mpb_idx_share), mp_map / ns_global_gs16b called from several threads at once (with and without MPB_DEVICES), and, where
there are two GPUs, every stage with large shared-memory launches on device 1."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import miniprot_b200 as mp
import oracle_lib as ol
from miniprot_b200 import synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
SETS = {"tiny": ("tiny.paf", None), "tiny5": ("tiny5.paf", "tiny5_gff.txt"), "DPP3": ("DPP3_default.paf", "DPP3_gff.txt")}


def n_devices() -> int:
    import torch

    return torch.cuda.device_count()


two_gpus = pytest.mark.skipif(n_devices() < 2, reason="needs two GPUs: this machine has fewer")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("sets")
    out = {"DPP3": (ol.DPP3_GENOME, ol.DPP3_PROTEIN)}
    for cfg in ("tiny", "tiny5"):
        out[cfg] = synth.generate(synth.CONFIGS[cfg], str(d / cfg))
    return out


def gold(name):
    return open(os.path.join(GOLD, name), "rb").read()


def cells(ctxs):
    return sum(c.stats().dp_cells_ext + c.stats().dp_cells_tb for c in ctxs)


def check_sets(ctxs, inputs, tmp_path):
    """Every set through mpb_map_file_multi over ctxs with 1200-residue mini-batches: PAF and GFF3 equal the goldens; returns the
    DP cells the contexts computed."""
    for c in ctxs:
        c.reset_stats()
    for name, (paf, gff) in SETS.items():
        g, p = inputs[name]
        mi = mp.idx_load(g, 4)
        for flag, want in ((0, paf), (0x8, gff)):
            if want is None:
                continue
            out = str(tmp_path / f"{name}.{flag}.out")
            mp.map_file_multi(ctxs, mi, p, out, mp.mapopt(mini_batch_size=1200, flag=flag))
            assert open(out, "rb").read() == gold(want), (name, flag, len(ctxs))
        mp.lib().mp_idx_destroy(mi)
    return cells(ctxs)


@pytest.fixture(scope="module")
def one_ctx_cells(inputs, tmp_path_factory):
    c = mp.Context(0)
    n = check_sets([c], inputs, tmp_path_factory.mktemp("one"))
    c.close()
    return n


@pytest.mark.parametrize("n", [2, 3])
def test_map_file_multi_on_one_device(inputs, tmp_path, one_ctx_cells, n):
    ctxs = [mp.Context(0) for _ in range(n)]
    assert check_sets(ctxs, inputs, tmp_path) == one_ctx_cells  # the same DP work, spread over the contexts
    assert sum(c.stats().dp_cells_tb > 0 for c in ctxs) >= 2      # ... and really spread
    for c in ctxs:
        c.close()


def test_map_file_multi_refuses_a_repeated_context(inputs, tmp_path):
    c = mp.Context(0)
    g, p = inputs["tiny"]
    mi = mp.idx_load(g, 4)
    with pytest.raises(RuntimeError, match=r"\(-1\)"):
        mp.map_file_multi([c, c], mi, p, str(tmp_path / "o.paf"))
    mp.lib().mp_idx_destroy(mi)
    c.close()


def device_ptrs(ctx):
    p = [C.c_void_p() for _ in range(3)]
    rc = mp.lib().mpb_idx_device_ptrs(ctx.h, *[C.byref(x) for x in p])
    return None if rc else tuple(x.value for x in p)


def test_index_loaded_into_hbm_shared_on_one_device(inputs, tmp_path):
    """mpb_idx_load_device on A (no host copy of the k-mer tables), shared with B: B adopts A's buffers and maps the golden PAF;
    destroying the index clears both contexts."""
    g, p = inputs["tiny"]
    L = mp.lib()
    mi0 = mp.idx_load(g, 4)
    mpi = str(tmp_path / "t.mpi")
    assert L.mp_idx_dump(mpi.encode(), mi0) == 0
    L.mp_idx_destroy(mi0)
    a, b = mp.Context(0), mp.Context(0)
    mi = mp.idx_load_device(a, mpi)
    assert not mi.contents.ki
    mp.idx_share(b, a)
    assert device_ptrs(b) == device_ptrs(a) is not None  # adopted, not copied
    b.reset_stats()
    mp.map_file(b, mi, p, str(tmp_path / "o.paf"))
    assert open(tmp_path / "o.paf", "rb").read() == gold("tiny.paf")
    assert b.stats().dp_cells_tb > 0 and b.stats().h2d_bytes < os.path.getsize(mpi)  # the tables did not travel again
    L.mp_idx_destroy(mi)
    assert device_ptrs(a) is None and device_ptrs(b) is None
    a.close(), b.close()


def test_adopter_forgets_the_index_of_a_destroyed_owner(inputs, tmp_path):
    """A context that adopted another's index buffers forgets them when their owner goes, and takes the index again on its next call."""
    g, p = inputs["tiny"]
    mi = mp.idx_load(g, 4)
    a, b = mp.Context(0), mp.Context(0)
    assert mp.lib().mpb_idx_upload(a.h, mi) == 0
    mp.idx_share(b, a)
    assert device_ptrs(b) == device_ptrs(a)
    a.close()
    assert device_ptrs(b) is None
    mp.map_file(b, mi, p, str(tmp_path / "o.paf"))  # uploads from the host tables again
    assert open(tmp_path / "o.paf", "rb").read() == gold("tiny.paf")
    b.close()
    mp.lib().mp_idx_destroy(mi)


_THREADED = r"""
import ctypes as C, sys, threading
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import numpy as np
import miniprot_b200 as mp, oracle_lib as ol
from test_gpu_dropin import read_proteins, free_regions, NsRst

L = mp.lib()
L.mp_map.restype = C.c_void_p
L.mp_map.argtypes = [C.POINTER(mp.Idx), C.c_int, C.c_char_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(mp.MapOpt), C.c_char_p]
mo = mp.mapopt()

def map_all(mi, recs):
    out = []
    for name, seq in recs:
        n = C.c_int(0)
        reg = L.mp_map(mi, len(seq), seq, C.byref(n), None, C.byref(mo), name)
        out.append(mp.regions(reg, n.value))
        free_regions(reg, n.value)
    return out

def threaded(fn, parts):
    res, err = [None] * len(parts), []
    def run(k):
        try:
            res[k] = fn(parts[k])
        except BaseException as e:
            err.append(e)
    th = [threading.Thread(target=run, args=(k,)) for k in range(len(parts))]
    for t in th: t.start()
    for t in th: t.join()
    assert not err, err
    return res

n_reg = 0
for g, p in ((sys.argv[2], sys.argv[3]), (ol.DPP3_GENOME, ol.DPP3_PROTEIN)):
    mi = mp.idx_load(g, 4)
    recs = read_proteins(p)
    want = map_all(mi, recs)
    for rep in range(2):
        parts = [recs[k::4] for k in range(4)]
        got = threaded(lambda part: map_all(mi, part), parts)
        for k in range(4):
            assert got[k] == want[k::4], (g, k)
    n_reg += sum(len(r) for r in want)
    L.mp_idx_destroy(mi)
assert n_reg > 40

tab = ol.OraTab()
for f, sym in (("nt4", "ns_tab_nt4"), ("aa20", "ns_tab_aa20"), ("aa13", "ns_tab_aa13"), ("codon", "ns_tab_codon"), ("codon13", "ns_tab_codon13")):
    setattr(tab, f, C.addressof(C.c_uint8.in_dll(L, sym)))
f = L.ns_global_gs16b
f.restype = None

opt0 = mp.nsopt()
par = dict(go=opt0.go, ge=opt0.ge, io=opt0.io, fs=opt0.fs, xdrop=opt0.xdrop, end_bonus=opt0.end_bonus, sp=tuple(opt0.sp), sp_null_bonus=opt0.sp_null_bonus,
           ie_coef=opt0.ie_coef)

def dp_all(probs):
    opt = mp.nsopt()
    bad = 0
    for nt, aa, flag, w in probs:
        opt.flag = flag
        r = NsRst()
        f(None, nt.ctypes.data_as(C.c_char_p), C.c_int32(len(nt)), aa, C.c_int32(len(aa)), C.byref(opt), None, C.byref(r))
        if flag == 1:
            bad += not (w[0] == r.score and w[3] == [r.cigar[k] for k in range(r.n_cigar)])
            L.mpb_free(r.cigar)
        else:
            bad += w[:3] != (r.score, r.nt_len, r.aa_len)
    return bad

rng = np.random.default_rng(31)
probs = []
while len(probs) < 96:
    nt, aa = ol.random_dp_problem(rng, al_max=(60, 300)[len(probs) & 1], flank=50)
    if len(nt) >= 3:
        flag = (1, 2, 4)[len(probs) % 3]
        probs.append((nt, aa, flag, ol.ora_nasw(tab, nt, aa, flag, opt0._mat_keepalive, par)))  # the oracle, single-threaded
assert threaded(dp_all, [probs[k::4] for k in range(4)]) == [0] * 4
print("ok")
"""


@pytest.mark.parametrize("devices", [None, "0,0"])
def test_mp_map_from_four_threads(inputs, devices):
    """mp_map and ns_global_gs16b from four Python threads at once (ctypes releases the GIL), in a process of its own: every region
    equals the single-threaded result, every DP result the oracle's.  Without MPB_DEVICES the calls take turns on the default
    context; with MPB_DEVICES=0,0 they run on a pool of two contexts."""
    g, p = inputs["tiny"]
    env = dict(os.environ)
    env.pop("MPB_DEVICES", None)
    if devices:
        env["MPB_DEVICES"] = devices
    r = subprocess.run([sys.executable, "-c", _THREADED, ROOT, g, p], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "miniprot_b200_cli")), reason="the drop-in CLI is built by make -C oracle dropin")
def test_dropin_cli_with_two_contexts(tmp_path):
    """The reference's unmodified CLI linked against the library, with MPB_DEVICES=0,0: mp_map_file maps over two contexts and prints
    the reference's output."""
    env = dict(os.environ, MPB_DEVICES="0,0")
    for args, want in (([], "DPP3_default.paf"), (["--gff"], "DPP3_gff.txt")):
        out = subprocess.run([os.path.join(ROOT, "oracle", "_ref", "miniprot_b200_cli"), "-t4", *args, ol.DPP3_GENOME, ol.DPP3_PROTEIN], env=env,
                             check=True, capture_output=True).stdout
        assert out == gold(want), args


# ---------------------------------------------------------------- a second device

@two_gpus
def test_two_devices_share_by_peer_copy(inputs, tmp_path):
    a, b = mp.Context(0), mp.Context(1)
    g, p = inputs["tiny5"]
    mi = mp.idx_load(g, 4)
    assert mp.lib().mpb_idx_upload(a.h, mi) == 0
    mp.idx_share(b, a)
    assert device_ptrs(b) != device_ptrs(a)  # b's own copy, on its device
    b.reset_stats()
    mp.map_file(b, mi, p, str(tmp_path / "b.paf"), mp.mapopt(mini_batch_size=1200))
    assert open(tmp_path / "b.paf", "rb").read() == gold("tiny5.paf")
    assert b.stats().dp_cells_tb > 0
    mp.map_file_multi([a, b], mi, p, str(tmp_path / "ab.paf"), mp.mapopt(mini_batch_size=1200))
    assert open(tmp_path / "ab.paf", "rb").read() == gold("tiny5.paf")
    mp.lib().mp_idx_destroy(mi)
    a.close(), b.close()


@two_gpus
def test_two_devices_map_file_multi(inputs, tmp_path, one_ctx_cells):
    ctxs = [mp.Context(0), mp.Context(1)]
    assert check_sets(ctxs, inputs, tmp_path) == one_ctx_cells
    for c in ctxs:
        c.close()


def _product_tables():
    t = ol.OraTab()
    for f, sym in (("nt4", "ns_tab_nt4"), ("aa20", "ns_tab_aa20"), ("aa13", "ns_tab_aa13"), ("codon", "ns_tab_codon"), ("codon13", "ns_tab_codon13")):
        setattr(t, f, C.addressof(C.c_uint8.in_dll(mp.lib(), sym)))
    return t


@two_gpus
@pytest.mark.parametrize("family", ["auto", "cols"])
def test_nasw_batch_on_device_1(family, monkeypatch):
    """Problems of every width class on device 1 (a process whose first kernels ran on device 0): the 8-warp block-wide kernels,
    the column passes and the column-pass family need the shared-memory limit raised on device 1 as well."""
    c0, c1 = mp.Context(0), mp.Context(1)
    opt = mp.nsopt()
    rng = np.random.default_rng(5)
    mk = lambda al: ol.random_dp_problem(rng, al_max=al, flank=60)
    mp.nasw_batch(c0, opt, [(nt, aa, 1, opt.io) for nt, aa in (mk(250) for _ in range(8)) if len(nt) >= 3])
    if family != "auto":
        monkeypatch.setenv("MPB_NASW_KERNEL", family)
    probs = []
    for it in range(300):
        nt, aa = mk((30, 60, 120, 250, 600)[it % 5])
        if len(nt) >= 3:
            probs.append((nt, aa, (1, 4, 2)[it % 3], opt.io))
    got = mp.nasw_batch(c1, opt, probs)
    tab, par = _product_tables(), dict(go=opt.go, ge=opt.ge, io=opt.io, fs=opt.fs, xdrop=opt.xdrop, end_bonus=opt.end_bonus, sp=tuple(opt.sp),
                                      sp_null_bonus=opt.sp_null_bonus, ie_coef=opt.ie_coef)
    for (nt, aa, flag, io), g in zip(probs, got):
        w = ol.ora_nasw(tab, nt, aa, flag, opt._mat_keepalive, par)
        assert (w[0] == g[0] and w[3] == g[3]) if flag == 1 else (w[:3] == g[:3])
    c0.close(), c1.close()


@two_gpus
def test_sort_segments_on_device_1():
    c0, c1 = mp.Context(0), mp.Context(1)
    rng = np.random.default_rng(9)
    L = mp.lib()
    L.mpb_sort_segments.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    for c in (c0, c1):
        sizes = np.array([8192, 5000, 8192, 20000, 3], np.int64)
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        keys = rng.integers(0, 1 << 62, int(off[-1]), dtype=np.uint64)
        want = np.concatenate([np.sort(keys[off[s]:off[s + 1]]) for s in range(len(sizes))])
        assert L.mpb_sort_segments(c.h, len(sizes), off.ctypes.data, keys.ctypes.data) == 0
        assert np.array_equal(keys, want)
    c0.close(), c1.close()


@two_gpus
def test_chain_batch_on_device_1():
    """Problems large enough for the biggest shared-memory backtrack class (16384 anchors), on device 0 and then device 1: the
    results agree."""
    c0, c1 = mp.Context(0), mp.Context(1)
    rng = np.random.default_rng(3)
    par = mp.ChainPar(max_dist_x=20000, max_dist_y=20000, bw=20000, max_skip=25, max_iter=5000, min_cnt=3, min_sc=0, chn_coef_log=0.75,
                      is_spliced=1, kmer=6, bbit=8)
    lists = []
    for n in (16000, 12000, 300, 9000):
        blk = np.sort(rng.integers(0, 1 << 20, n)).astype(np.uint64)
        q = rng.integers(0, 4000, n).astype(np.uint64)
        lists.append(np.sort(blk << np.uint64(32) | q))
    r0, r1 = mp.chain_batch(c0, par, lists), mp.chain_batch(c1, par, lists)
    for (u0, b0), (u1, b1) in zip(r0, r1):
        assert np.array_equal(u0, u1) and np.array_equal(b0, b1)
    assert sum(len(u) for u, _ in r1) > 0
    c0.close(), c1.close()


@two_gpus
def test_event_bracket_on_device_1():
    c1 = mp.Context(1)
    L = mp.lib()
    L.mpb_event_begin(c1.h)
    mp.nasw_batch(c1, mp.nsopt(), [(np.array([0, 1, 2, 3] * 30, np.uint8), b"MKVL" * 10, 1, 29)])
    ms = L.mpb_event_end_ms(c1.h)
    assert 0 < ms < 10000
    c1.close()
