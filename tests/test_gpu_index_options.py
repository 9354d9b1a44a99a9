"""GPU stages under index and refinement options off the defaults (-k 6 -M 1 -L 30 -b 8, -l 5): the k-mer masks and bucket counts
(-k, -M), the ORF rule and the window kernels' tile halos (-L, and -l above -L), the block size (-b) and the refinement k-mer (-l).

Each stage against its reference, bit for bit: the device-built index against the host builder's and the reference CLI's -d
output (stored digests); seeding, refinement and chaining against the C oracle on the same inputs; the whole pipeline's PAF and
X / Y1 dump lines against the reference CLI's (stored digests, dbg_lib).  One table of option sets (dbg_lib.INDEX_OPTION_SETS)
serves every part."""
import ctypes as C

import numpy as np
import pytest

import dbg_lib
import miniprot_b200 as mp
import oracle_lib as ol
from miniprot_b200 import synth
from test_gpu_dropin import write_odd_fasta
from test_gpu_stages import product_tables

pytestmark = pytest.mark.gpu


def _index_args(opts):
    return [a for a in opts if not a.startswith("-l")]


# the option sets that change the index (-l is a mapping option)
INDEX_SETS = []
for _o in dbg_lib.INDEX_OPTION_SETS:
    if _index_args(_o) not in INDEX_SETS:
        INDEX_SETS.append(_index_args(_o))


def _ids(sets):
    return [" ".join(o) or "defaults" for o in sets]


def idxopt(opts) -> mp.IdxOpt:
    io = mp.idxopt()
    for f, v in dbg_lib.index_options(opts)[0].items():
        setattr(io, f, v)
    return io


def built_on_device(io) -> bool:
    """Where mp_idx_load builds the k-mer tables (idx_build.cu): on the device when the tile halos cover -L and the ORF rule
    needs no look-back beyond it (k <= L <= 40), and the bucket count fits (4k <= 28); on the host otherwise."""
    return io.kmer <= io.min_aa_len <= 40 and 4 * io.kmer <= 28


def read_fasta(path):
    """[(name, sequence bytes as written)] of a plain FASTA file."""
    out = []
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b">"):
                out.append([line[1:].split()[0].decode(), []])
            else:
                out[-1][1].append(line.strip())
    return [(n, b"".join(s)) for n, s in out]


def read_proteins(path):
    return [s for _, s in read_fasta(path)]


@pytest.fixture(scope="module")
def ctx():
    c = mp.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("idxopt")
    g, p = synth.generate(synth.CONFIGS["tiny"], str(d / "tiny"))
    return {"odd": write_odd_fasta(str(d / "odd.fa")), "tiny": g, "tiny_prot": p, "dir": d}


# ---- A. index build ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("opts", INDEX_SETS, ids=_ids(INDEX_SETS))
def test_index_build(inputs, opts, monkeypatch, capfd):
    """The .mpi of the device build equals the host builder's and the reference CLI's (-d) with the same options; the device
    path is taken exactly where built_on_device() says."""
    L = mp.lib()
    verbose = C.c_int32.in_dll(L, "mp_verbose")
    io = idxopt(opts)
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
            on_dev = "built the k-mer tables on the device" in err
            assert on_dev == (where == "dev" and built_on_device(io)), (tag, where, err[-500:])
            assert (mi.contents.opt.kmer, mi.contents.opt.mod_bit, mi.contents.opt.min_aa_len, mi.contents.opt.bbit) == \
                (io.kmer, io.mod_bit, io.min_aa_len, io.bbit)
            files[where] = str(inputs["dir"] / f"{tag}.{where}.mpi")
            assert L.mp_idx_dump(files[where].encode(), mi) == 0
            L.mp_idx_destroy(mi)
        a, b = (open(files[x], "rb").read() for x in ("dev", "host"))
        assert a == b, tag
        assert ol.file_digest(files["dev"]) == ol.ref_index_file(g, opts), tag


# ---- B. seeding ----------------------------------------------------------------------------------------------------------

DEGENERATE_PROTEINS = [b"", b"MKV", b"M" * 40, b"ACDEFGHIKLMNPQRSTVWY" * 3 + b"XX*" + b"WWHHKK" * 5]


@pytest.mark.parametrize("opts", INDEX_SETS, ids=_ids(INDEX_SETS))
def test_seed_options(ctx, inputs, opts):
    """mpb_seed_batch against ora_seed_anchors on an index built with the options, protein by protein, with the adaptive
    occupancy cut-off off (20000), biting (50) and at its floor (1)."""
    mi = mp.idx_load(inputs["tiny"], 8, idxopt(opts))
    idx = mi.contents
    seqs = read_proteins(inputs["tiny_prot"]) + DEGENERATE_PROTEINS
    tab = product_tables()
    ora = ol.ora()
    n_anchor = 0
    for max_occ in (20000, 50, 1):
        got = mp.seed_batch(ctx, mi, max_occ, seqs)
        assert len(got) == len(seqs)
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


# ---- C. refinement -------------------------------------------------------------------------------------------------------

# -L -> the -l values run on an index built with it: L < l (no k-mer of a short ORF is lost) and l > L + 1 (a k-mer reaches
# further back than the ORF rule, past the left tile halo of a narrow -L)
REFINE_GRID = {30: (5, 3, 7), 40: (7, 3), 12: (4,), 10: (4, 7), 6: (3, 7), 5: (5, 7), 4: (5, 4, 6), 1: (7, 3), 0: (5,)}
REFINE_CASES = [(L, l) for L, ls in REFINE_GRID.items() for l in ls]

_NT4 = np.full(256, 4, np.uint8)
for _i, _ch in enumerate(b"ACGT"):
    _NT4[_ch] = _NT4[_ch + 32] = _i
_COMP = bytes.maketrans(b"ACGTacgt", b"TGCAtgca")
_CODON = {}
for _i, _a in enumerate(ol._STD):
    _CODON["TCAG"[_i >> 4] + "TCAG"[(_i >> 2) & 3] + "TCAG"[_i & 3]] = _a


def translate(nt: bytes) -> bytes:
    s = nt.decode().upper()
    return "".join(_CODON.get(s[i:i + 3], "X") for i in range(0, len(s) - 2, 3)).encode()


@pytest.fixture(scope="module")
def refine_inputs(inputs):
    """(genome FASTA, proteins, windows, window slices): the tiny genome followed by the awkward contigs of write_odd_fasta in one
    FASTA.  Windows: both strands of every tiny protein's own 50 kb slot and of a foreign one; windows of 2047, 2048, 2049,
    4096 + 200 and tens of kb bases starting at contig offset 0 (the left halo lies before the contig) and ending at a contig's
    end, over the stop-free "orf" contig with a protein read off it in frame 0 (k-mers end near every tile start), over the poly-A
    contig with K / F runs (groups large enough for max_ava to drop) and over the contigs with N runs."""
    spec = synth.CONFIGS["tiny"]
    tiny_ctgs = read_fasta(inputs["tiny"])
    odd_ctgs = read_fasta(inputs["odd"])
    ctgs = tiny_ctgs + odd_ctgs
    path = str(inputs["dir"] / "tiny_odd.fa")
    with open(path, "wb") as f:
        for n, s in ctgs:
            f.write(b">" + n.encode() + b"\n" + s + b"\n")
    seqs = read_proteins(inputs["tiny_prot"])
    cid = {n: i for i, (n, _) in enumerate(ctgs)}
    orf, c13 = ctgs[cid["orf"]][1], ctgs[cid["c13"]][1]
    q_orf, q_c13, q_kf = len(seqs), len(seqs) + 1, len(seqs) + 2
    seqs += [translate(orf[3000:21000]), translate(c13[1500:4500]), b"K" * 30 + b"F" * 30 + b"MKV"]
    wins = []  # (qid, contig, lo, hi) on the forward strand; both strands are added below
    slot = spec.genome_len // spec.n_genes
    for q in range(spec.n_genes):
        for gslot in (q, (q + 17) % spec.n_genes):
            lo, hi = gslot * slot, (gslot + 1) * slot
            c = lo // spec.ctg_len
            wins.append((q, c, lo - c * spec.ctg_len, min(hi - c * spec.ctg_len, len(tiny_ctgs[c][1]))))
    c0 = len(tiny_ctgs[0][1])
    for lo, hi in ((0, 2047), (0, 2048), (0, 2049), (0, 4296), (c0 - 4296, c0), (c0 - 30000, c0)):
        wins.append((0, 0, lo, hi))
    o = cid["orf"]
    for lo, hi in ((0, 2047), (0, 2048), (0, 2049), (1000, 5296), (0, 30000), (1500, 61500), (250000, 300000)):
        wins += [(q_orf, o, lo, hi), (q_kf, o, lo, hi)]
    wins += [(q_kf, cid["polyA"], 0, 50000), (q_orf, cid["polyA"], 0, 50000), (0, cid["polyA"], 10000, 14296)]
    for n in ("c9", "c10", "c11", "c12", "c13"):  # 2047, 2048, 2049, 4187 and 70000 bases with a run of N
        c = cid[n]
        wins += [(q_c13, c, 0, len(ctgs[c][1])), (0, c, 0, len(ctgs[c][1]))]
    windows, slices = [], []
    for q, c, lo, hi in wins:
        c_len = len(ctgs[c][1])
        for rev in (0, 1):
            as_, ae = (lo, hi) if not rev else (c_len - hi, c_len - lo)
            sl = ctgs[c][1][lo:hi] if not rev else ctgs[c][1][lo:hi].translate(_COMP)[::-1]
            windows.append((q, c << 1 | rev, as_, ae))
            slices.append(_NT4[np.frombuffer(sl, np.uint8)])
    return path, seqs, windows, slices


@pytest.mark.parametrize("L,kmer2", REFINE_CASES, ids=[f"L{L}-l{l}" for L, l in REFINE_CASES])
def test_refine_options(ctx, refine_inputs, L, kmer2):
    """mpb_refine_batch against ora_refine, window by window, on an index built with -L (the index's min_aa_len is the ORF
    rule of the window scan) and with -l as the refinement k-mer, with max_ava at its default and at 4."""
    path, seqs, windows, slices = refine_inputs
    io = mp.idxopt()
    io.min_aa_len = L
    mi = mp.idx_load(path, 8, io)
    assert mi.contents.opt.min_aa_len == L
    tab = product_tables()
    ora = ol.ora()
    for max_ava in (1000, 4):
        mo = mp.mapopt(kmer2=kmer2, max_ava=max_ava)
        got = mp.refine_batch(ctx, mi, mo, seqs, windows)
        par = mp.ChainPar(mo.max_intron, mo.max_gap, mo.bw, mo.max_chn_max_skip, mo.max_chn_iter, mo.min_chn_cnt, mo.min_chn_sc,
                          mo.chn_coef_log, 0 if (mo.flag & 0x1) else 1, mo.kmer2, 0)
        n_hit, bad = 0, []
        for (q, vid, as_, ae), nt, (a, sc) in zip(windows, slices, got):
            nb, sb = C.c_int32(0), C.c_int32(0)
            ptr = ora.ora_refine(C.byref(tab), C.byref(par), C.c_int32(L), C.c_int32(max_ava), C.c_void_p(nt.ctypes.data), C.c_int64(len(nt)),
                                 C.c_char_p(seqs[q]), C.c_int32(len(seqs[q])), C.byref(nb), C.byref(sb))
            want = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint64)), shape=(max(nb.value, 1),)).copy()[:nb.value] if ptr else np.zeros(0, np.uint64)
            if ptr:
                ol._libc.free(C.c_void_p(ptr))
            if not np.array_equal(a, want) or (len(want) and sc != sb.value):
                bad.append((q, vid, as_, ae, len(a), len(want), sc, sb.value))
            n_hit += len(want) > 0
        assert not bad, (max_ava, len(bad), bad[:5])
        assert n_hit >= 20, max_ava  # the planted genes and the orf-contig protein are found
    mp.lib().mp_idx_destroy(mi)


def test_refine_refuses_min_orf_above_40(ctx, inputs):
    """-L 41 is beyond the window kernels' halos: mpb_refine_batch returns -3 with a message, like the mapping calls."""
    io = mp.idxopt()
    io.min_aa_len = 41
    mi = mp.idx_load(inputs["tiny"], 8, io)
    with pytest.raises(RuntimeError, match=r"\(-3\)"):
        mp.refine_batch(ctx, mi, mp.mapopt(), [b"MKVLAAGIVGLLLA"], [(0, 0, 0, 50000)])
    mp.lib().mp_idx_destroy(mi)


# ---- D. chaining ---------------------------------------------------------------------------------------------------------

CHAIN_CASES = [(m, k, b) for m in ("pre", "main") for b in (4, 6, 7, 9, 10) for k in (4, 5, 7)] + [("refine", k, 0) for k in (3, 4, 6, 7)]


@pytest.mark.parametrize("mode,kmer,bbit", CHAIN_CASES, ids=[f"{m}-k{k}-b{b}" for m, k, b in CHAIN_CASES])
def test_chain_options(ctx, mode, kmer, bbit):
    """mpb_chain_batch against ora_chain with the k-mer size (score floor) and block size (<< bbit distances) of the options, on
    problems of every size class: fused (<= 2048), shared memory (<= 16384) and global memory (above)."""
    rng = np.random.default_rng(7000 + 100 * kmer + bbit + {"pre": 0, "main": 20, "refine": 40}[mode])
    par = ol.chain_par(mode, kmer=kmer, bbit=bbit)
    sizes = [int(rng.integers(1, 80)) for _ in range(60)] + [1500, 2048, 2049, 5000, 9000, 16384, 16385, 21000]
    lists = [ol.random_chain_problem(rng, n, mode, bbit) for n in sizes]
    assert max(len(a) for a in lists) > 16384 and any(2048 < len(a) <= 16384 for a in lists)
    mpar = mp.ChainPar(**{f: getattr(par, f) for f, _ in mp.ChainPar._fields_})
    got = mp.chain_batch(ctx, mpar, lists)
    n_chain = 0
    for a, (u, b) in zip(lists, got):
        wu, wb = ol.ora_chain(par, a)
        assert len(wu) == len(u) and (wu == u).all() and len(wb) == len(b) and (wb == b).all(), (len(a), len(wu), len(u))
        n_chain += len(wu)
    assert n_chain > 0


# ---- E. end to end -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sets(inputs):
    return dbg_lib.input_sets(str(inputs["dir"] / "dbg"))


@pytest.mark.parametrize("opts", dbg_lib.INDEX_OPTION_SETS, ids=_ids(dbg_lib.INDEX_OPTION_SETS))
@pytest.mark.parametrize("name", ["tiny", "tiny5", "DPP3"])
def test_index_options_end_to_end(sets, name, opts):
    """The library under the reference's CLI with the options: PAF and the X (seeds) / Y1 (first-round chains) lines equal the
    reference CLI's."""
    args = opts + dbg_lib.INDEX_SWITCHES
    g, p = sets[name]
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, args, g, p)
    assert rc == 0, err.decode(errors="replace")[-2000:]
    got, want = dbg_lib.digest(out, err), dbg_lib.ref_cli_dbg(args, g, p)
    assert (got["lines"], got["dump_lines"]) == (want["lines"], want["dump_lines"])
    assert got["dump_sha256"] == want["dump_sha256"]  # seeds and chains first: they tell which stage diverged
    assert got == want


def test_min_orf_above_40_refused_end_to_end(sets):
    g, p = sets["tiny"]
    rc, out, err = dbg_lib.run_cli(mp.LIB_PATH, ["-L41"] + dbg_lib.INDEX_SWITCHES, g, p)
    assert rc == -3 and out == b"" and b"min ORF length 41" in err
