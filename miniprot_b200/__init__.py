"""miniprot_b200 -- Python mirror (ctypes) of the C ABI in include/miniprot_b200.h.

The product is ``libminiprot_b200.so`` (host orchestration in C++ + hand-written sm_90a CUDA kernels).  This
module only loads it and mirrors the reference-facing calls so that tests and bench.py read like a user of the
reference library: ``mp_idx_load`` -> ``mp_map_file`` / ``mpb_map_batch``.  There is no Python or CPU fallback: if
the library is missing, or no CUDA device is present, calls fail loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libminiprot_b200.so")
CSRC = os.path.join(_HERE, "csrc")

NS_F_CIGAR, NS_F_EXT_LEFT, NS_F_EXT_RIGHT = 1, 2, 4
MP_F_NO_SPLICE, MP_F_NO_ALIGN, MP_F_SHOW_UNMAP, MP_F_NO_PRE_CHAIN, MP_F_NO_CS = 0x1, 0x2, 0x4, 0x40, 0x200


BUILD_INFO = os.path.join(_HERE, "BUILD_INFO.json")
_SRC_GLOBS = ("csrc/Makefile", "csrc/*.cpp", "csrc/*.hpp", "csrc/cuda/*.cu", "csrc/cuda/*.cuh", "csrc/cuda/*.hpp", "../include/*.h")


def _sha256_file(path: str) -> str:
    import hashlib

    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 20), b""):
            h.update(blk)
    return h.hexdigest()


def source_fingerprint() -> str:
    """sha256 over the sources the library is compiled from (paths and contents, sorted)."""
    import glob
    import hashlib

    h = hashlib.sha256()
    for pat in _SRC_GLOBS:
        for path in sorted(glob.glob(os.path.join(_HERE, pat))):
            h.update(os.path.relpath(path, _HERE).encode() + b"\0" + _sha256_file(path).encode() + b"\n")
    return h.hexdigest()


def build(force: bool = False) -> str:
    """Compile the shared library in-tree with nvcc for sm_90a (no GPU needed to compile) and record what it was built from
    (BUILD_INFO.json next to the library: travels to the GPU box with it, stays out of the history like the library)."""
    import json
    import time

    if force:
        subprocess.run(["make", "-s", "-C", CSRC, "clean"], check=True)
    subprocess.run(["make", "-s", "-j8", "-C", CSRC], check=True)
    try:
        nvcc = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    except OSError:
        nvcc = "unknown"
    with open(BUILD_INFO, "w") as f:
        json.dump({"source_sha256": source_fingerprint(), "so_sha256": _sha256_file(LIB_PATH), "nvcc": nvcc,
                   "arch": "-gencode arch=compute_90a,code=sm_90a", "built_at": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime())}, f)
    return LIB_PATH


def build_info() -> dict:
    """What build() recorded, plus whether the library that is loaded now is that build and the sources are still the ones it was
    compiled from.  Never raises (bench.py and smoke() report it)."""
    import json

    try:
        with open(BUILD_INFO) as f:
            info = json.load(f)
        info["so_is_that_build"] = _sha256_file(LIB_PATH) == info.get("so_sha256")
        info["sources_unchanged_since"] = source_fingerprint() == info.get("source_sha256")
        return info
    except Exception as e:  # noqa: BLE001 -- a report, not a gate
        return {"error": f"{type(e).__name__}: {e}"}


class IdxOpt(C.Structure):  # mp_idxopt_t
    _fields_ = [("bbit", C.c_int32), ("min_aa_len", C.c_int32), ("kmer", C.c_int32), ("mod_bit", C.c_int32), ("trans_code", C.c_uint32)]


class MapOpt(C.Structure):  # mp_mapopt_t (include/miniprot_b200.h; reference miniprot.h:43-77)
    _fields_ = [("flag", C.c_uint32), ("mini_batch_size", C.c_int64), ("max_occ", C.c_int32), ("max_gap", C.c_int32),
                ("max_intron", C.c_int32), ("min_max_intron", C.c_int32), ("max_max_intron", C.c_int32), ("bw", C.c_int32),
                ("max_ext", C.c_int32), ("max_ava", C.c_int32), ("min_chn_cnt", C.c_int32), ("max_chn_max_skip", C.c_int32),
                ("max_chn_iter", C.c_int32), ("min_chn_sc", C.c_int32), ("chn_coef_log", C.c_float), ("mask_level", C.c_float),
                ("mask_len", C.c_int32), ("pri_ratio", C.c_float), ("out_sim", C.c_float), ("out_cov", C.c_float),
                ("best_n", C.c_int32), ("out_n", C.c_int32), ("kmer2", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32),
                ("io", C.c_int32), ("fs", C.c_int32), ("io_end", C.c_int32), ("ie_coef", C.c_float), ("sp_model", C.c_int32),
                ("sp_null_bonus", C.c_int32), ("sp_max_bonus", C.c_int32), ("sp_scale", C.c_float), ("xdrop", C.c_int32),
                ("end_bonus", C.c_int32), ("asize", C.c_int32), ("gff_delim", C.c_int32), ("max_intron_flank", C.c_int32),
                ("gff_prefix", C.c_char_p), ("mat", C.c_int8 * 484)]


class NsOpt(C.Structure):  # ns_opt_t
    _fields_ = [("flag", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32), ("io", C.c_int32), ("fs", C.c_int32),
                ("xdrop", C.c_int32), ("end_bonus", C.c_int32), ("asize", C.c_int32), ("sp", C.c_int32 * 6),
                ("sp_null_bonus", C.c_int32), ("ie_coef", C.c_float), ("sc", C.c_void_p), ("nt4", C.c_void_p),
                ("aa20", C.c_void_p), ("codon", C.c_void_p)]


class DpProblem(C.Structure):  # mpb_dp_problem_t
    _fields_ = [("nt", C.c_void_p), ("aa", C.c_char_p), ("ss", C.c_void_p), ("nl", C.c_int32), ("al", C.c_int32),
                ("flag", C.c_int32), ("io", C.c_int32)]


class DpResult(C.Structure):  # mpb_dp_result_t
    _fields_ = [("score", C.c_int32), ("nt_len", C.c_int32), ("aa_len", C.c_int32), ("n_cigar", C.c_int32),
                ("cigar", C.POINTER(C.c_uint32))]


class ChainPar(C.Structure):  # mpb_chain_par_t
    _fields_ = [("max_dist_x", C.c_int32), ("max_dist_y", C.c_int32), ("bw", C.c_int32), ("max_skip", C.c_int32),
                ("max_iter", C.c_int32), ("min_cnt", C.c_int32), ("min_sc", C.c_int32), ("chn_coef_log", C.c_float),
                ("is_spliced", C.c_int32), ("kmer", C.c_int32), ("bbit", C.c_int32)]


class Stats(C.Structure):  # mpb_stats_t
    _fields_ = [("dp_cells_ext", C.c_int64), ("dp_cells_tb", C.c_int64), ("n_dp_ext", C.c_int64), ("n_dp_tb", C.c_int64),
                ("n_anchors", C.c_int64), ("n_chain_problems", C.c_int64), ("n_refine_regions", C.c_int64),
                ("kernel_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("ms_seed", C.c_double),
                ("ms_chain", C.c_double), ("ms_refine", C.c_double), ("ms_dp_ext", C.c_double), ("ms_dp_tb", C.c_double), ("ms_wall", C.c_double * 6),
                ("ms_class", (C.c_double * 16) * 2), ("cells_class", (C.c_int64 * 16) * 2), ("n_class", (C.c_int64 * 16) * 2),
                ("ms_bt", C.c_double), ("ms_dp_wave", C.c_double), ("ms_prep", C.c_double)]


class MemStats(C.Structure):  # mpb_mem_stats_t
    _fields_ = [(f, C.c_int64) for f in ("budget", "allowance", "held", "peak_held", "n_slices_seed", "n_slices_loci", "n_slices_refine",
                                         "n_subwaves", "n_released", "bytes_released", "n_over_budget", "n_index_passes")]


class Extra(C.Structure):  # mp_extra_t without its trailing cigar[]
    _fields_ = [(f, C.c_int32) for f in ("dp_score", "dp_max", "dp_max2", "n_cigar", "m_cigar", "blen", "n_fs", "n_stop", "dist_stop",
                                         "dist_start", "n_iden", "n_plus")]


class Feat(C.Structure):  # mp_feat_t
    _fields_ = [("vs", C.c_int64), ("ve", C.c_int64), ("qs", C.c_int32), ("qe", C.c_int32), ("type", C.c_int16), ("phase", C.c_int16),
                ("n_fs", C.c_int32), ("n_stop", C.c_int32), ("score", C.c_int32), ("n_iden", C.c_int32), ("blen", C.c_int32),
                ("donor", C.c_uint8 * 2), ("acceptor", C.c_uint8 * 2)]


class Reg1(C.Structure):  # mp_reg1_t
    _fields_ = [(f, C.c_int32) for f in ("off", "cnt", "id", "parent", "n_sub", "subsc", "n_feat", "m_feat", "n_exon", "chn_sc", "chn_sc_ungap")] + \
        [("hash", C.c_uint32), ("vid", C.c_uint32), ("qs", C.c_int32), ("qe", C.c_int32), ("vs", C.c_int64), ("ve", C.c_int64),
         ("a", C.c_void_p), ("feat", C.POINTER(Feat)), ("p", C.POINTER(Extra))]


# what a caller of mp_map() / mpb_map_batch() gets per region (capacities and the anchor pointer, which is not valid after the
# call, left out)
REG_FIELDS = ("id", "parent", "n_sub", "subsc", "n_feat", "n_exon", "chn_sc", "chn_sc_ungap", "hash", "vid", "qs", "qe", "vs", "ve")
EXTRA_FIELDS = ("dp_score", "dp_max", "dp_max2", "n_cigar", "blen", "n_fs", "n_stop", "dist_stop", "dist_start", "n_iden", "n_plus")
FEAT_FIELDS = ("vs", "ve", "qs", "qe", "type", "phase", "n_fs", "n_stop", "score", "n_iden", "blen")


def regions(reg, n: int) -> list:
    """The n regions at `reg` (mp_reg1_t *) as plain values: [REG_FIELDS values, EXTRA_FIELDS values (None without r->p),
    CIGAR words, one list per feature (FEAT_FIELDS values + donor + acceptor)]."""
    rp = C.cast(reg, C.POINTER(Reg1))
    out = []
    for j in range(n):
        r = rp[j]
        extra, cigar = None, []
        if r.p:
            e = r.p.contents
            extra = [getattr(e, f) for f in EXTRA_FIELDS]
            words = C.cast(C.addressof(e) + C.sizeof(Extra), C.POINTER(C.c_uint32))
            cigar = [words[k] for k in range(e.n_cigar)]
        feats = [[getattr(r.feat[k], f) for f in FEAT_FIELDS] + list(r.feat[k].donor) + list(r.feat[k].acceptor)
                 for k in range(r.n_feat if r.feat else 0)]
        out.append([[getattr(r, f) for f in REG_FIELDS], extra, cigar, feats])
    return out


class Ctg(C.Structure):  # mp_ctg_t
    _fields_ = [("off", C.c_int64), ("len", C.c_int64), ("name", C.c_char_p)]


class NtDb(C.Structure):  # mp_ntdb_t
    _fields_ = [("n_ctg", C.c_int32), ("m_ctg", C.c_int32), ("l_name", C.c_int32), ("l_seq", C.c_int64), ("m_seq", C.c_int64),
                ("seq", C.c_void_p), ("ctg", C.POINTER(Ctg)), ("name", C.c_void_p), ("h", C.c_void_p), ("spsc", C.c_void_p)]


class Idx(C.Structure):  # mp_idx_t
    _fields_ = [("opt", IdxOpt), ("n_block", C.c_uint32), ("nt", C.POINTER(NtDb)), ("n_kb", C.c_int64), ("ki", C.c_void_p),
                ("bo", C.c_void_p), ("kb", C.c_void_p)]


_lib = None


def lib() -> C.CDLL:
    """The loaded shared library; raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with miniprot_b200.build() (needs nvcc); there is no fallback")
        L = C.CDLL(LIB_PATH)
        L.mpb_ctx_create.restype = C.c_void_p
        L.mpb_ctx_create.argtypes = [C.c_int]
        L.mpb_ctx_destroy.argtypes = [C.c_void_p]
        L.mp_idx_load.restype = C.POINTER(Idx)
        L.mp_idx_load.argtypes = [C.c_char_p, C.POINTER(IdxOpt), C.c_int32]
        L.mp_idx_restore.restype = C.POINTER(Idx)
        L.mp_idx_restore.argtypes = [C.c_char_p]
        L.mp_idx_dump.argtypes = [C.c_char_p, C.POINTER(Idx)]
        L.mp_idx_destroy.argtypes = [C.POINTER(Idx)]
        L.mpb_idx_upload.argtypes = [C.c_void_p, C.POINTER(Idx)]
        L.mpb_idx_load_device.restype = C.POINTER(Idx)
        L.mpb_idx_load_meta.restype = C.POINTER(Idx)
        L.mpb_idx_load_meta.argtypes = [C.c_char_p]
        L.mpb_idx_device_ptrs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.mpb_idx_load_device.argtypes = [C.c_void_p, C.c_char_p]
        L.mpb_idx_attach_device.argtypes = [C.c_void_p, C.POINTER(Idx), C.c_void_p, C.c_void_p, C.c_void_p]
        L.mpb_map_file_path.restype = C.c_int32
        L.mpb_map_file_path.argtypes = [C.c_void_p, C.POINTER(Idx), C.c_char_p, C.POINTER(MapOpt), C.c_char_p]
        L.mpb_map_file_multi_path.restype = C.c_int32
        L.mpb_map_file_multi_path.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Idx), C.c_char_p, C.POINTER(MapOpt), C.c_char_p]
        L.mpb_idx_load_genome.restype = C.POINTER(Idx)
        L.mpb_idx_load_genome.argtypes = [C.c_char_p, C.POINTER(IdxOpt)]
        L.mpb_map_loci_file_multi.restype = C.c_int32
        L.mpb_map_loci_file_multi.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Idx), C.c_char_p, C.c_char_p, C.POINTER(MapOpt), C.c_void_p]
        L.mpb_map_loci_file_multi_path.restype = C.c_int32
        L.mpb_map_loci_file_multi_path.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Idx), C.c_char_p, C.c_char_p, C.POINTER(MapOpt), C.c_char_p]
        L.mpb_map_locus_sets_file_multi.restype = C.c_int32
        L.mpb_map_locus_sets_file_multi.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Idx), C.c_char_p, C.c_char_p, C.POINTER(MapOpt), C.c_void_p]
        L.mpb_map_locus_sets_file_multi_path.restype = C.c_int32
        L.mpb_map_locus_sets_file_multi_path.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Idx), C.c_char_p, C.c_char_p, C.POINTER(MapOpt),
                                                         C.c_char_p]
        L.mpb_idx_share.argtypes = [C.c_void_p, C.c_void_p]
        L.mpb_event_begin.argtypes = [C.c_void_p]
        L.mpb_event_end_ms.restype = C.c_double
        L.mpb_event_end_ms.argtypes = [C.c_void_p]
        L.mpb_nasw_batch.argtypes = [C.c_void_p, C.POINTER(NsOpt), C.c_int32, C.POINTER(DpProblem), C.POINTER(DpResult)]
        L.mpb_chain_batch.argtypes = [C.c_void_p, C.POINTER(ChainPar), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(C.c_void_p), C.c_void_p, C.POINTER(C.c_void_p)]
        L.mpb_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        L.mpb_reset_stats.argtypes = [C.c_void_p]
        L.mpb_ctx_set_mem_budget.restype = C.c_int
        L.mpb_ctx_set_mem_budget.argtypes = [C.c_void_p, C.c_int64]
        L.mpb_get_mem_stats.argtypes = [C.c_void_p, C.POINTER(MemStats)]
        L.mpb_free.argtypes = [C.c_void_p]
        L.mp_mapopt_set_max_intron.argtypes = [C.POINTER(MapOpt), C.c_int64]
        L.mp_start()
        c_int32_p = C.POINTER(C.c_int32)
        C.c_int32.in_dll(L, "mp_verbose").value = 1
        _ = c_int32_p
        _lib = L
    return _lib


# mp_dbg_flag bits (include/miniprot_b200.h MP_DBG_*; the CLI's --dbg-* switches, reference mppriv.h:9-14)
DBG_NO_KALLOC, DBG_QNAME, DBG_NO_REFINE, DBG_MORE_DP, DBG_ANCHOR, DBG_CHAIN = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20
DBG_SWITCHES = {"--no-kalloc": DBG_NO_KALLOC, "--dbg-qname": DBG_QNAME, "--dbg-no-refine": DBG_NO_REFINE, "--dbg-aflt": DBG_MORE_DP,
                "--dbg-anchor": DBG_ANCHOR, "--dbg-chain": DBG_CHAIN}


def set_dbg_flag(bits: int, L: C.CDLL | None = None) -> int:
    """Set mp_dbg_flag (what main.c's --dbg-* switches set) in the library, or in `L` -- another library built from the same host
    sources; returns the previous value.  The mapping calls read it once per batch."""
    v = C.c_int32.in_dll(L or lib(), "mp_dbg_flag")
    old, v.value = v.value, bits
    return old


def n_bucket(io: IdxOpt) -> int:
    return 1 << (io.kmer * 4 - io.mod_bit)


class Context:
    """One GPU context (mpb_ctx_t).  Raises if there is no CUDA device -- the stages exist only as CUDA kernels."""

    def __init__(self, device: int = 0):
        self.h = lib().mpb_ctx_create(device)
        if not self.h:
            raise RuntimeError("mpb_ctx_create failed: no usable CUDA device (miniprot_b200 has no CPU fallback)")

    def close(self):
        if self.h:
            lib().mpb_ctx_destroy(self.h)
            self.h = None

    def stats(self) -> Stats:
        s = Stats()
        lib().mpb_get_stats(self.h, C.byref(s))
        return s

    def reset_stats(self):
        """Reset the counters of stats() and mem_stats() (the peak restarts at what the arenas hold)."""
        lib().mpb_reset_stats(self.h)

    def set_mem_budget(self, nbytes: int) -> int:
        """Cap the bytes the context's working arenas may hold at once (0: automatic, what the device has free less a sixteenth of it, at least 1 GiB).
        Stages then run in slices that fit; results do not change.  Returns 0, or -1 for a negative value."""
        return lib().mpb_ctx_set_mem_budget(self.h, nbytes)

    def mem_stats(self) -> MemStats:
        s = MemStats()
        lib().mpb_get_mem_stats(self.h, C.byref(s))
        return s

    def map_locus_sets(self, mi, mo: "MapOpt", seqs, names, sets):
        """map_locus_sets on this context: (rc, n_reg, reg) per set of `sets` (lists of (qid, cid, st, en))."""
        return map_locus_sets(self, mi, mo, seqs, names, sets)


def idxopt() -> IdxOpt:
    o = IdxOpt()
    lib().mp_idxopt_init(C.byref(o))
    return o


def mapopt(**over) -> MapOpt:
    o = MapOpt()
    lib().mp_mapopt_init(C.byref(o))
    for k, v in over.items():
        setattr(o, k, v)
    return o


def idx_load(path: str, n_threads: int = 8, io: IdxOpt | None = None):
    """mp_idx_load: build from FASTA or restore a .mpi file (index.c:231)."""
    io = io or idxopt()
    mi = lib().mp_idx_load(path.encode(), C.byref(io), n_threads)
    if not mi:
        raise RuntimeError(f"cannot load index from {path}")
    return mi


def idx_load_device(ctx: Context, path: str):
    """mpb_idx_load_device: restore a .mpi file straight into the context's HBM (no host copy of the k-mer tables)."""
    mi = lib().mpb_idx_load_device(ctx.h, path.encode())
    if not mi:
        raise RuntimeError(f"cannot load index {path} into device memory")
    return mi


def map_file(ctx: Context, mi, prot_path: str, out_path: str, mo: MapOpt | None = None) -> None:
    """mp_map_file with an explicit output path: FASTA proteins -> PAF, mini-batches mapped on the GPU."""
    mo = mo or mapopt()
    rc = lib().mpb_map_file_path(ctx.h, mi, prot_path.encode(), C.byref(mo), out_path.encode())
    if rc != 0:
        raise RuntimeError(f"mpb_map_file failed ({rc})")


def idx_share(dst: Context, src: Context) -> None:
    """mpb_idx_share: make the index resident in `src` resident in `dst` too (adopted on one device, copied device to device
    otherwise)."""
    if lib().mpb_idx_share(dst.h, src.h) != 0:
        raise RuntimeError("mpb_idx_share failed: the source context holds no index")


def map_file_multi(ctxs, mi, prot_path: str, out_path: str, mo: MapOpt | None = None) -> None:
    """mpb_map_file_multi: map_file over several distinct contexts at once (one mapper thread each); same output as map_file."""
    mo = mo or mapopt()
    arr = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    rc = lib().mpb_map_file_multi_path(arr, len(ctxs), mi, prot_path.encode(), C.byref(mo), out_path.encode())
    if rc != 0:
        raise RuntimeError(f"mpb_map_file_multi failed ({rc})")


def idx_load_genome(path: str, io: IdxOpt | None = None):
    """mpb_idx_load_genome: an index for locus mode only (genome and contig table of a FASTA, or the head of a .mpi file; no k-mer
    table)."""
    mi = lib().mpb_idx_load_genome(path.encode(), C.byref(io) if io is not None else None)
    if not mi:
        raise RuntimeError(f"cannot read a genome from {path}")
    return mi


def map_loci_file(ctxs, mi, prot_path: str, loci_path: str, out_path: str = "-", mo: MapOpt | None = None, sets: bool = False) -> None:
    """mpb_map_loci_file_multi: proteins (FASTA) against the loci of a TSV (`protein contig start end`) on one Context or a list of
    distinct ones, in the output format of `mo`; out_path "-" is this process's standard output.  sets: mpb_map_locus_sets_file_multi,
    the lines of one (protein, 5th-column label) forming one set (map_locus_sets_file)."""
    mo = mo or mapopt()
    ctxs = [ctxs] if isinstance(ctxs, Context) else list(ctxs)
    arr = (C.c_void_p * len(ctxs))(*[c.h for c in ctxs])
    L = lib()
    if out_path == "-":
        import sys

        sys.stdout.flush()
        libc = C.CDLL(None)
        libc.fdopen.restype, libc.fdopen.argtypes = C.c_void_p, [C.c_int, C.c_char_p]
        libc.fclose.argtypes = [C.c_void_p]
        fp = libc.fdopen(os.dup(sys.stdout.fileno()), b"wb")
        f = L.mpb_map_locus_sets_file_multi if sets else L.mpb_map_loci_file_multi
        rc = f(arr, len(ctxs), mi, prot_path.encode(), loci_path.encode(), C.byref(mo), fp)
        libc.fclose(fp)
    else:
        f = L.mpb_map_locus_sets_file_multi_path if sets else L.mpb_map_loci_file_multi_path
        rc = f(arr, len(ctxs), mi, prot_path.encode(), loci_path.encode(), C.byref(mo), out_path.encode())
    if rc != 0:
        raise RuntimeError(f"{'mpb_map_locus_sets_file' if sets else 'mpb_map_loci_file'} failed ({rc})")


def map_locus_sets_file(ctxs, mi, prot_path: str, loci_path: str, out_path: str = "-", mo: MapOpt | None = None) -> None:
    """mpb_map_locus_sets_file_multi: as map_loci_file, but the lines of the TSV of one protein and one set label (an optional 5th
    column; no label: all lines of the protein) form one set, aligned as the reference aligns the protein against a genome of the
    set's ranges alone."""
    map_loci_file(ctxs, mi, prot_path, loci_path, out_path, mo, sets=True)


def nsopt(mat=None, **over) -> NsOpt:
    """ns_opt_t with miniprot's mapping defaults (align.c:50-60 applied to options.c:42-90)."""
    import numpy as np

    o = NsOpt()
    L = lib()
    L.ns_opt_init(C.byref(o))
    mo = mapopt()
    o.go, o.ge, o.io, o.fs, o.xdrop, o.end_bonus, o.ie_coef, o.sp_null_bonus = mo.go, mo.ge, mo.io, mo.fs, mo.xdrop, mo.end_bonus, mo.ie_coef, mo.sp_null_bonus
    L.ns_opt_set_sp(C.byref(o), 1)
    if mat is None:
        mat = np.ctypeslib.as_array(mo.mat).astype(np.int8).copy()
    o._mat_keepalive = mat
    o.sc = mat.ctypes.data
    for k, v in over.items():
        if k == "sp":
            for i in range(6):
                o.sp[i] = v[i]
        else:
            setattr(o, k, v)
    return o


def nasw_batch(ctx: Context, opt: NsOpt, problems):
    """problems: list of (nt uint8 ndarray codes 0..4, aa bytes, flag, io).  Returns list of (score, nt_len, aa_len, cigar list)."""
    import numpy as np

    n = len(problems)
    P = (DpProblem * n)()
    R = (DpResult * n)()
    keep = []
    for i, (nt, aa, flag, io) in enumerate(problems):
        nt = np.ascontiguousarray(nt, dtype=np.uint8)
        keep.append(nt)
        P[i].nt, P[i].aa, P[i].ss, P[i].nl, P[i].al, P[i].flag, P[i].io = nt.ctypes.data, aa, None, len(nt), len(aa), flag, io
    rc = lib().mpb_nasw_batch(ctx.h, C.byref(opt), n, P, R)
    if rc != 0:
        raise RuntimeError(f"mpb_nasw_batch failed ({rc})")
    out = []
    for i in range(n):
        cig = [R[i].cigar[k] for k in range(R[i].n_cigar)]
        if R[i].n_cigar:
            lib().mpb_free(R[i].cigar)
        out.append((R[i].score, R[i].nt_len, R[i].aa_len, cig))
    return out


def seed_batch(ctx: Context, mi, max_occ: int, seqs):
    """mpb_seed_batch: sketch + index lookup + sort for a list of protein byte strings; returns one sorted uint64 anchor
    array (block<<32 | qpos) per protein."""
    import numpy as np

    n = len(seqs)
    arr = (C.c_char_p * n)(*seqs)
    lens = np.array([len(s) for s in seqs], np.int32)
    off = np.zeros(n + 1, np.int64)
    ap = C.c_void_p()
    L = lib()
    L.mpb_seed_batch.restype = C.c_int
    L.mpb_seed_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    rc = L.mpb_seed_batch(ctx.h, C.cast(mi, C.c_void_p), max_occ, n, C.cast(arr, C.c_void_p), lens.ctypes.data, off.ctypes.data, C.byref(ap))
    if rc != 0:
        raise RuntimeError("mpb_seed_batch failed")
    a = np.ctypeslib.as_array(C.cast(ap, C.POINTER(C.c_uint64)), shape=(max(int(off[n]), 1),)).copy()[:int(off[n])]
    L.mpb_free(ap)
    return [a[off[i]:off[i + 1]] for i in range(n)]


class Locus(C.Structure):  # mpb_locus_t
    _fields_ = [("qid", C.c_int32), ("cid", C.c_int32), ("st", C.c_int64), ("en", C.c_int64)]


def _loci_args(seqs, loci, names=None):
    import numpy as np

    n, nl = len(seqs), len(loci)
    arr = (C.c_char_p * max(n, 1))(*seqs)
    nam = (C.c_char_p * max(n, 1))(*(names or [b"*"] * n))
    lens = np.array([len(s) for s in seqs] or [0], np.int32)
    loc = (Locus * max(nl, 1))(*[Locus(*l) for l in loci])
    return n, nl, arr, nam, lens, loc


def map_loci(ctx: Context, mi, mo: MapOpt, seqs, names, loci, L: C.CDLL | None = None, fn: str = "mpb_map_loci"):
    """mpb_map_loci: loci = list of (qid, cid, st, en).  Returns (rc, n_reg int32 array, reg array of mp_reg1_t pointers); free the
    regions with free_loci_regs.  `L` / `fn`: another library exporting the same call without its context argument (the CPU tests'
    oracle-backed hc_map_loci), ctx is then None."""
    import numpy as np

    n, nl, arr, nam, lens, loc = _loci_args(seqs, loci, names)
    n_reg = np.zeros(max(nl, 1), np.int32)
    reg = (C.c_void_p * max(nl, 1))()
    f = getattr(L or lib(), fn)
    f.restype = C.c_int
    f.argtypes = ([C.c_void_p] if ctx is not None else []) + [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                                              C.c_void_p, C.c_void_p]
    args = [C.cast(mi, C.c_void_p), C.cast(C.pointer(mo), C.c_void_p), n, C.cast(arr, C.c_void_p), lens.ctypes.data, C.cast(nam, C.c_void_p), nl,
            C.cast(loc, C.c_void_p), n_reg.ctypes.data, C.cast(reg, C.c_void_p)]
    rc = f(*([ctx.h] if ctx is not None else []), *args)
    return rc, n_reg[:nl], reg


def _set_args(sets):
    import numpy as np

    off = np.array([0] + [len(x) for x in sets], np.int64).cumsum()
    flat = [l for x in sets for l in x]
    return off, len(flat), (Locus * max(len(flat), 1))(*[Locus(*l) for l in flat])


def map_locus_sets(ctx: Context, mi, mo: MapOpt, seqs, names, sets, L: C.CDLL | None = None, fn: str = "mpb_map_locus_sets"):
    """mpb_map_locus_sets: sets = list of lists of (qid, cid, st, en), the loci of one set naming one protein.  Returns (rc, n_reg
    int32 array, reg array of mp_reg1_t pointers), one entry per set; free the regions with free_loci_regs.  `L` / `fn`: another
    library exporting the same call without its context argument (the CPU tests' oracle-backed hc_map_locus_sets), ctx is then None."""
    import numpy as np

    n, _, arr, nam, lens, _ = _loci_args(seqs, [], names)
    off, _, loc = _set_args(sets)
    ns = len(sets)
    n_reg = np.zeros(max(ns, 1), np.int32)
    reg = (C.c_void_p * max(ns, 1))()
    f = getattr(L or lib(), fn)
    f.restype = C.c_int
    f.argtypes = ([C.c_void_p] if ctx is not None else []) + [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                                              C.c_void_p, C.c_void_p, C.c_void_p]
    args = [C.cast(mi, C.c_void_p), C.cast(C.pointer(mo), C.c_void_p), n, C.cast(arr, C.c_void_p), lens.ctypes.data, C.cast(nam, C.c_void_p), ns,
            off.ctypes.data, C.cast(loc, C.c_void_p), n_reg.ctypes.data, C.cast(reg, C.c_void_p)]
    rc = f(*([ctx.h] if ctx is not None else []), *args)
    return rc, n_reg[:ns], reg


def free_loci_regs(n_reg, reg) -> None:
    """What mpb_regs_free does, with the C library's free (the regions of either library are libc-allocated)."""
    import ctypes.util

    libc = C.CDLL(ctypes.util.find_library("c"))
    libc.free.argtypes = [C.c_void_p]
    for k in range(len(n_reg)):
        if not reg[k]:
            continue
        rp = C.cast(reg[k], C.POINTER(Reg1))
        for j in range(int(n_reg[k])):
            libc.free(C.cast(rp[j].feat, C.c_void_p)), libc.free(C.cast(rp[j].p, C.c_void_p))
        libc.free(reg[k])


def loci_paf(mi, mo: MapOpt, seqs, names, loci, n_reg, reg, L: C.CDLL | None = None, fn: str = "mpb_format_paf") -> bytes:
    """The PAF lines of map_loci's regions, pair by pair: the hits the reference's writer prints for a protein (map.c:293-326: the
    first out_n, with a positive score of at least out_sim times the best and a query coverage of at least out_cov), formatted by
    mpb_format_paf (or `fn` of `L`) with the real index."""
    f = getattr(L or lib(), fn)
    f.restype = C.c_int64
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int32, C.c_char_p, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    buf, ln, cap = C.c_void_p(), C.c_int64(0), C.c_int64(0)
    for k, (qid, _, _, _) in enumerate(loci):
        nr = int(n_reg[k])
        if nr == 0:
            continue
        rp = C.cast(reg[k], C.POINTER(Reg1))
        sc = lambda r: r.p.contents.dp_max if r.p else r.chn_sc  # noqa: E731
        best = sc(rp[0])
        for j in range(min(nr, mo.out_n)):
            r = rp[j]
            if sc(r) <= 0 or sc(r) < best * mo.out_sim or r.qe - r.qs < len(seqs[qid]) * mo.out_cov:
                continue
            f(C.cast(mi, C.c_void_p), C.cast(C.pointer(mo), C.c_void_p), names[qid], len(seqs[qid]), seqs[qid], C.addressof(r), C.byref(buf), C.byref(ln), C.byref(cap))
    out = C.string_at(buf, ln.value) if ln.value else b""
    if buf:
        free = (L or lib()).mpb_free if L is None else C.CDLL(None).free
        free.argtypes = [C.c_void_p]
        free(buf)
    return out


def seed_loci_batch(ctx: Context, mi, max_occ: int, seqs, loci):
    """mpb_seed_loci_batch: the sorted, max_occ-filtered anchors (block<<32 | qpos, blocks of an index of the locus alone) of every
    (qid, cid, st, en) pair."""
    import numpy as np

    n, nl, arr, _, lens, loc = _loci_args(seqs, loci)
    off = np.zeros(nl + 1, np.int64)
    ap = C.c_void_p()
    L = lib()
    L.mpb_seed_loci_batch.restype = C.c_int
    L.mpb_seed_loci_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.POINTER(C.c_void_p)]
    rc = L.mpb_seed_loci_batch(ctx.h, C.cast(mi, C.c_void_p), max_occ, n, C.cast(arr, C.c_void_p), lens.ctypes.data, nl, C.cast(loc, C.c_void_p),
                               off.ctypes.data, C.byref(ap))
    if rc != 0:
        raise RuntimeError(f"mpb_seed_loci_batch failed ({rc})")
    a = np.ctypeslib.as_array(C.cast(ap, C.POINTER(C.c_uint64)), shape=(max(int(off[nl]), 1),)).copy()[:int(off[nl])]
    L.mpb_free(ap)
    return [a[off[k]:off[k + 1]] for k in range(nl)]


def seed_locus_sets_batch(ctx: Context, mi, max_occ: int, seqs, sets):
    """mpb_seed_locus_sets_batch: the sorted, max_occ-filtered anchors (block<<32 | qpos, blocks of an index of the set's merged,
    sorted ranges alone) of every set (a list of (qid, cid, st, en))."""
    import numpy as np

    n, _, arr, _, lens, _ = _loci_args(seqs, [])
    so, _, loc = _set_args(sets)
    ns = len(sets)
    off = np.zeros(ns + 1, np.int64)
    ap = C.c_void_p()
    L = lib()
    L.mpb_seed_locus_sets_batch.restype = C.c_int
    L.mpb_seed_locus_sets_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.POINTER(C.c_void_p)]
    rc = L.mpb_seed_locus_sets_batch(ctx.h, C.cast(mi, C.c_void_p), max_occ, n, C.cast(arr, C.c_void_p), lens.ctypes.data, ns, so.ctypes.data,
                                     C.cast(loc, C.c_void_p), off.ctypes.data, C.byref(ap))
    if rc != 0:
        raise RuntimeError(f"mpb_seed_locus_sets_batch failed ({rc})")
    a = np.ctypeslib.as_array(C.cast(ap, C.POINTER(C.c_uint64)), shape=(max(int(off[ns]), 1),)).copy()[:int(off[ns])]
    L.mpb_free(ap)
    return [a[off[k]:off[k + 1]] for k in range(ns)]


class Window(C.Structure):  # mpb_window_t
    _fields_ = [("qid", C.c_int32), ("vid", C.c_uint32), ("as_", C.c_int64), ("ae", C.c_int64)]


def refine_batch(ctx: Context, mi, mo, seqs, windows):
    """mpb_refine_batch: windows = list of (qid, vid, as, ae).  Returns one (anchors uint64 array, score) per window."""
    import numpy as np

    n, nw = len(seqs), len(windows)
    arr = (C.c_char_p * n)(*seqs)
    lens = np.array([len(s) for s in seqs], np.int32)
    win = (Window * max(nw, 1))(*[Window(*w) for w in windows])
    off = np.zeros(nw + 1, np.int64)
    sc = np.zeros(max(nw, 1), np.int32)
    ap = C.c_void_p()
    L = lib()
    L.mpb_refine_batch.restype = C.c_int
    L.mpb_refine_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
                                   C.c_void_p]
    rc = L.mpb_refine_batch(ctx.h, C.cast(mi, C.c_void_p), C.cast(C.pointer(mo), C.c_void_p), n, C.cast(arr, C.c_void_p), lens.ctypes.data, nw,
                            C.cast(win, C.c_void_p), off.ctypes.data, C.byref(ap), sc.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"mpb_refine_batch failed ({rc})")
    a = np.ctypeslib.as_array(C.cast(ap, C.POINTER(C.c_uint64)), shape=(max(int(off[nw]), 1),)).copy()[:int(off[nw])]
    L.mpb_free(ap)
    return [(a[off[k]:off[k + 1]], int(sc[k])) for k in range(nw)]


def chain_batch(ctx: Context, par: ChainPar, anchor_lists):
    """anchor_lists: list of sorted uint64 arrays.  Returns list of (u array, b array) per problem."""
    import numpy as np

    n = len(anchor_lists)
    off = np.zeros(n + 1, np.int64)
    for i, a in enumerate(anchor_lists):
        off[i + 1] = off[i] + len(a)
    a = np.ascontiguousarray(np.concatenate(anchor_lists) if n else np.zeros(0, np.uint64), dtype=np.uint64)
    u_off = np.zeros(n + 1, np.int64)
    b_off = np.zeros(n + 1, np.int64)
    up, bp = C.c_void_p(), C.c_void_p()
    rc = lib().mpb_chain_batch(ctx.h, C.byref(par), n, off.ctypes.data, a.ctypes.data, u_off.ctypes.data, C.byref(up), b_off.ctypes.data, C.byref(bp))
    if rc != 0:
        raise RuntimeError("mpb_chain_batch failed")
    u = np.ctypeslib.as_array(C.cast(up, C.POINTER(C.c_uint64)), shape=(max(int(u_off[n]), 1),)).copy()[:int(u_off[n])]
    b = np.ctypeslib.as_array(C.cast(bp, C.POINTER(C.c_uint64)), shape=(max(int(b_off[n]), 1),)).copy()[:int(b_off[n])]
    lib().mpb_free(up)
    lib().mpb_free(bp)
    return [(u[u_off[i]:u_off[i + 1]], b[b_off[i]:b_off[i + 1]]) for i in range(n)]
