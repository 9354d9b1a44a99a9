"""ctypes bindings for the two CHECKERS (test infrastructure only):

* ``oracle/_ref/libref.so``  - the unmodified reference, every symbol renamed ``ref_*``
* ``oracle/liboracle.so``    - the plain-C restatement of the hot path

plus seeded random problem generators shared by the CPU and GPU parity tests.

The reference is only built where its sources are (oracle/Makefile).  Everything the tests ask it is therefore also stored:
``tests/golden/reference_calls.json.gz`` maps a digest of each question (function + inputs) to the reference's answer, and
``reference()`` answers from there.  ``MPB_RECORD_REFERENCE=1`` asks the compiled reference instead and writes the answers
back (tests/golden/make_golden.py does that for the whole suite).
"""
from __future__ import annotations

import atexit
import ctypes as C
import gzip
import hashlib
import json
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORA_DIR = os.path.join(ROOT, "oracle")
REF_SO = os.path.join(ORA_DIR, "_ref", "libref.so")
REF_BIN = os.path.join(ORA_DIR, "_ref", "miniprot")
ORA_SO = os.path.join(ORA_DIR, "liboracle.so")
GOLDEN = os.path.join(ROOT, "tests", "golden")
DPP3_GENOME, DPP3_PROTEIN = os.path.join(GOLDEN, "DPP3-hs.gen.fa.gz"), os.path.join(GOLDEN, "DPP3-mm.pep.fa.gz")  # the reference's bundled test pair
RECORD_PATH = os.path.join(GOLDEN, "reference_calls.json.gz")
RECORDING = os.environ.get("MPB_RECORD_REFERENCE") == "1"
_record = None


def _answers() -> dict:
    global _record
    if _record is None:
        _record = {}
        if os.path.exists(RECORD_PATH):
            with gzip.open(RECORD_PATH, "rt") as f:
                _record = json.load(f)
        if RECORDING:
            atexit.register(_save)
    return _record


def _save():
    with gzip.open(RECORD_PATH + ".tmp", "wt", compresslevel=9) as f:
        json.dump(_record, f, sort_keys=True, separators=(",", ":"))
    os.replace(RECORD_PATH + ".tmp", RECORD_PATH)


def _digest(*parts) -> str:
    h = hashlib.sha256()
    for p in parts:
        if isinstance(p, np.ndarray):
            p = np.ascontiguousarray(p).tobytes()
        elif isinstance(p, str):
            p = p.encode()
        elif not isinstance(p, (bytes, bytearray)):
            p = repr(p).encode()
        h.update(len(p).to_bytes(8, "little") + bytes(p))
    return h.hexdigest()


def file_digest(path: str) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def reference(compute, *question):
    """The compiled reference's answer to `question` (a function name and its inputs): the stored one, or -- when recording,
    or for a question never stored where oracle/_ref is built -- compute() run against the reference.  JSON types only."""
    k = _digest(*question)[:40]
    rec = _answers()
    if k in rec and not RECORDING:
        return rec[k]
    if not (have_ref() and os.path.exists(REF_BIN)):
        raise LookupError(f"no stored reference answer for {question[0]!r} on these inputs, and oracle/_ref is not built: "
                          "regenerate tests/golden/reference_calls.json.gz with tests/golden/make_golden.py")
    v = json.loads(json.dumps(compute()))
    if RECORDING:
        rec[k] = v
    return v


def ref_cli(args, genome: str, proteins: str | None = None, threads: int = 8) -> dict:
    """{"sha256", "lines"} of what the reference CLI prints for `args genome [proteins]` (input files keyed by content)."""
    files = [genome] + ([proteins] if proteins else [])

    def run():
        out = subprocess.run([REF_BIN, f"-t{threads}", *args, *files], check=True, capture_output=True).stdout
        return {"sha256": hashlib.sha256(out).hexdigest(), "lines": out.count(b"\n")}
    # a file named among the options (--spsc FILE) is keyed by its content too
    return reference(run, "cli", [file_digest(a) if os.path.isfile(a) else a for a in args], [file_digest(f) for f in files])


def ref_index_file(genome: str, args=()) -> str:
    """sha256 of the .mpi file the reference CLI writes for `args -d FILE genome` (args: index options such as -k5 -L12)."""
    def run():
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            out = os.path.join(d, "ref.mpi")
            subprocess.run([REF_BIN, "-t4", *args, "-d", out, genome], check=True, capture_output=True)
            return file_digest(out)
    return reference(run, "cli -d", file_digest(genome), *([list(args)] if args else []))


def build_oracle():
    subprocess.run(["make", "-s", "-C", ORA_DIR, "all"], check=True, stdout=subprocess.DEVNULL)


class NsOpt(C.Structure):  # reference nasw.h:61-71 (== include/nasw_b200.h ns_opt_t)
    _fields_ = [("flag", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32), ("io", C.c_int32), ("fs", C.c_int32),
                ("xdrop", C.c_int32), ("end_bonus", C.c_int32), ("asize", C.c_int32), ("sp", C.c_int32 * 6),
                ("sp_null_bonus", C.c_int32), ("ie_coef", C.c_float), ("sc", C.c_void_p), ("nt4", C.c_void_p),
                ("aa20", C.c_void_p), ("codon", C.c_void_p)]


class NsRst(C.Structure):  # reference nasw.h:73-78
    _fields_ = [("n_cigar", C.c_int32), ("m_cigar", C.c_int32), ("nt_len", C.c_int32), ("aa_len", C.c_int32),
                ("score", C.c_int32), ("cigar", C.POINTER(C.c_uint32))]


class OraTab(C.Structure):
    _fields_ = [("nt4", C.c_void_p), ("aa20", C.c_void_p), ("aa13", C.c_void_p), ("codon", C.c_void_p), ("codon13", C.c_void_p)]


class OraNaswPar(C.Structure):
    _fields_ = [("flag", C.c_int32), ("go", C.c_int32), ("ge", C.c_int32), ("io", C.c_int32), ("fs", C.c_int32),
                ("xdrop", C.c_int32), ("end_bonus", C.c_int32), ("sp", C.c_int32 * 6), ("sp_null_bonus", C.c_int32),
                ("ie_coef", C.c_float), ("mat", C.c_void_p)]


class OraNaswRst(C.Structure):
    _fields_ = [("score", C.c_int32), ("nt_len", C.c_int32), ("aa_len", C.c_int32), ("n_cigar", C.c_int32),
                ("m_cigar", C.c_int32), ("cigar", C.POINTER(C.c_uint32))]


class ChainPar(C.Structure):
    _fields_ = [("max_dist_x", C.c_int32), ("max_dist_y", C.c_int32), ("bw", C.c_int32), ("max_skip", C.c_int32),
                ("max_iter", C.c_int32), ("min_cnt", C.c_int32), ("min_sc", C.c_int32), ("chn_coef_log", C.c_float),
                ("is_spliced", C.c_int32), ("kmer", C.c_int32), ("bbit", C.c_int32)]


_ref = None
_ora = None
_libc = C.CDLL(None)
_libc.free.argtypes = [C.c_void_p]


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        _ref = C.CDLL(REF_SO)
        _ref.ref_mp_start()
        _ref.ref_mp_chain.restype = C.c_void_p
        _ref.ref_mp_chain.argtypes = [C.c_int32] * 7 + [C.c_float] + [C.c_int32] * 3 + [C.c_int64, C.c_void_p,
                                                                                       C.POINTER(C.c_int32),
                                                                                       C.POINTER(C.c_void_p), C.c_void_p]
        _ref.ref_kmalloc.restype = C.c_void_p
        _ref.ref_kmalloc.argtypes = [C.c_void_p, C.c_size_t]
        _ref.ref_ns_global_gs16b.argtypes = [C.c_void_p, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(NsOpt),
                                             C.c_void_p, C.POINTER(NsRst)]
    return _ref


def ora():
    global _ora
    if _ora is None:
        if not os.path.exists(ORA_SO):
            build_oracle()
        _ora = C.CDLL(ORA_SO)
        _ora.ora_chain.restype = C.c_void_p
        _ora.ora_chain.argtypes = [C.POINTER(ChainPar), C.c_int64, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]
        _ora.ora_seed_anchors.restype = C.c_void_p
        _ora.ora_refine.restype = C.c_void_p
        _ora.ora_hash32_mask.restype = C.c_uint32
        _ora.ora_hash32_mask.argtypes = [C.c_uint32, C.c_uint32]
        _ora.ora_sketch_nt4.restype = C.c_int64
    return _ora


_TABLES = (("nt4", "ns_tab_nt4", 256), ("aa20", "ns_tab_aa20", 256), ("aa13", "ns_tab_aa13", 256), ("codon", "ns_tab_codon", 64),
           ("codon13", "ns_tab_codon13", 64))
_tab_keepalive = {}


def ref_tables() -> OraTab:
    """Oracle table bundle holding the REFERENCE's tables (as set up by ref_mp_start())."""
    return ref_tables_for(1)


def ref_tables_for(code: int) -> OraTab:
    """Oracle table bundle holding the reference's tables of NCBI genetic code `code` (ref_ns_make_tables, -T); the reference is
    left at code 1."""
    if code not in _tab_keepalive:
        def run():
            r = ref()
            assert r.ref_ns_make_tables(code) == 0, code
            try:
                return {f: bytes((C.c_uint8 * n).in_dll(r, "ref_" + sym)).hex() for f, sym, n in _TABLES}
            finally:
                r.ref_ns_make_tables(1)
        r = reference(run, "tables", *([code] if code != 1 else []))
        arrs = {f: np.frombuffer(bytes.fromhex(r[f]), np.uint8).copy() for f, _, _ in _TABLES}
        t = OraTab()
        for f, _, _ in _TABLES:
            setattr(t, f, arrs[f].ctypes.data)
        _tab_keepalive[code] = (t, arrs)
    return _tab_keepalive[code][0]


def codon_array(tab: OraTab) -> np.ndarray:
    """The 64 amino-acid codes (0..20, 20 = stop) of a table bundle's codon table, indexed by b1 << 4 | b2 << 2 | b3 (A, C, G, T = 0..3)."""
    return np.ctypeslib.as_array((C.c_uint8 * 64).from_address(tab.codon)).copy()


def stop_rows(nt: np.ndarray, codon: np.ndarray) -> int:
    """Rows of a DP problem (nucleotide codes 0..4) whose codon, the three bases ending at the row, is a stop codon (20) of `codon`."""
    nt = np.asarray(nt, np.int64)
    a, b, d = nt[:-2], nt[1:-1], nt[2:]
    ok = (a < 4) & (b < 4) & (d < 4)
    return int((codon[(a << 4 | b << 2 | d)[ok]] == 20).sum())


def codons_of(codon: np.ndarray) -> dict:
    """{amino-acid letter: [codon as three base codes]} of a codon table (codon_array): what random_dp_problem(codons=) encodes with."""
    out = {}
    for c in range(64):
        out.setdefault("ARNDCQEGHILKMFPSTWYV*X"[int(codon[c])], []).append([c >> 4, (c >> 2) & 3, c & 3])
    return out


def tables_from_arrays(nt4, aa20, aa13, codon, codon13):
    """Oracle table bundle from numpy uint8 arrays (kept alive by the caller)."""
    t = OraTab()
    t.nt4, t.aa20, t.aa13, t.codon, t.codon13 = (a.ctypes.data for a in (nt4, aa20, aa13, codon, codon13))
    return t


DEFAULT_NASW = dict(go=11, ge=1, io=29, fs=23, xdrop=100, end_bonus=5, sp=(8, 15, 21, 30, 0, 0), sp_null_bonus=-7,
                    ie_coef=0.5)


def default_mat() -> np.ndarray:
    """BLOSUM62 22x22 with the miniprot stop-codon row (options.c:87-88), as the reference sets it up."""
    def run():
        r = ref()
        m = np.ctypeslib.as_array((C.c_int8 * 484).in_dll(r, "ref_ns_mat_blosum62")).copy()
        r.ref_ns_set_stop_sc(22, m.ctypes.data_as(C.c_void_p), 23)
        return m.tobytes().hex()
    return np.frombuffer(bytes.fromhex(reference(run, "default_mat")), np.int8).copy()


def ref_set_stop_sc(m: np.ndarray, sc: int) -> None:
    """The reference's ns_set_stop_sc(22, m, sc) (-C), applied to m in place."""
    def run():
        x = m.copy()
        ref().ref_ns_set_stop_sc(22, x.ctypes.data_as(C.c_void_p), sc)
        return x.tobytes().hex()
    m[:] = np.frombuffer(bytes.fromhex(reference(run, "ns_set_stop_sc", m, sc)), np.int8)


def ref_nasw(nt: np.ndarray, aa: bytes, flag: int, mat: np.ndarray, par: dict, ss=None, code: int = 1):
    """The reference's ns_global_gs16b under NCBI genetic code `code` (-T); the reference is left at code 1."""
    def run():
        r = ref()
        o = NsOpt()
        r.ref_ns_opt_init(C.byref(o))
        for k in ("go", "ge", "io", "fs", "xdrop", "end_bonus", "sp_null_bonus", "ie_coef"):
            setattr(o, k, par[k])
        for i in range(6):
            o.sp[i] = par["sp"][i]
        o.flag = flag
        o.sc = mat.ctypes.data
        rst = NsRst()
        ssp = ss.ctypes.data_as(C.c_void_p) if ss is not None else None
        assert r.ref_ns_make_tables(code) == 0, code  # o.codon points at the reference's live table
        try:
            r.ref_ns_global_gs16b(None, nt.tobytes(), len(nt), aa, len(aa), C.byref(o), ssp, C.byref(rst))
        finally:
            r.ref_ns_make_tables(1)
        cig = [rst.cigar[i] for i in range(rst.n_cigar)]
        if rst.n_cigar:
            _libc.free(rst.cigar)
        return rst.score, rst.nt_len, rst.aa_len, cig
    pars = tuple((k, par[k]) for k in ("go", "ge", "io", "fs", "xdrop", "end_bonus", "sp_null_bonus", "ie_coef")) + (tuple(par["sp"]),)
    v = reference(run, "ns_global_gs16b", np.ascontiguousarray(nt, np.uint8), aa, flag, np.ascontiguousarray(mat, np.int8), pars,
                  b"" if ss is None else np.ascontiguousarray(ss, np.uint8), ss is None, *([("code", code)] if code != 1 else []))
    return v[0], v[1], v[2], v[3]


def ora_nasw(tab: OraTab, nt: np.ndarray, aa: bytes, flag: int, mat: np.ndarray, par: dict, ss=None):
    o = ora()
    p = OraNaswPar()
    for k in ("go", "ge", "io", "fs", "xdrop", "end_bonus", "sp_null_bonus", "ie_coef"):
        setattr(p, k, par[k])
    for i in range(6):
        p.sp[i] = par["sp"][i]
    p.flag = flag
    p.mat = mat.ctypes.data
    rst = OraNaswRst()
    nt = np.ascontiguousarray(nt, dtype=np.uint8)
    ssp = ss.ctypes.data_as(C.c_void_p) if ss is not None else None
    o.ora_nasw(C.byref(tab), C.byref(p), nt.ctypes.data_as(C.c_void_p), len(nt), aa, len(aa), ssp, C.byref(rst))
    cig = [rst.cigar[i] for i in range(rst.n_cigar)]
    if rst.n_cigar:
        _libc.free(rst.cigar)
    return rst.score, rst.nt_len, rst.aa_len, cig


# ------------------------------------------------------------------ random problem generators

_AA = "ARNDCQEGHILKMFPSTWYV"
_STD = "FFLLSSSSYY**CC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG"
_T2A = {"T": 3, "C": 1, "A": 0, "G": 2}
_AA2COD = {}
for _i, _a in enumerate(_STD):
    _c = ("TCAG"[_i >> 4], "TCAG"[(_i >> 2) & 3], "TCAG"[_i & 3])
    _AA2COD.setdefault(_a, []).append([_T2A[x] for x in _c])


def random_dp_problem(rng: np.random.Generator, al_max=60, intron_max=400, p_sub=0.2, p_indel=0.03, p_fs=0.02, p_n=0.002,
                      flank=30, codons=None, p_stop=0.01):
    """A protein and a nucleotide string (codes 0..4) that encodes a mutated, intron-interrupted copy of it: with the standard
    code, or with `codons` (codons_of() of another genetic code); a residue is replaced by a stop codon with probability p_stop."""
    cod_of = codons or _AA2COD
    al = int(rng.integers(1, al_max + 1))
    prot = [int(x) for x in rng.integers(0, 20, size=al)]
    nt = []
    nt += [int(x) for x in rng.integers(0, 4, size=int(rng.integers(0, flank + 1)))]
    for a in prot:
        r = rng.random()
        if r < p_indel / 2:
            continue  # residue missing from the genome (insertion in the protein)
        if r < p_indel:
            extra = cod_of[_AA[int(rng.integers(0, 20))]]
            nt += extra[int(rng.integers(0, len(extra)))]  # extra codon (deletion)
        aa = _AA[a] if rng.random() >= p_sub else _AA[int(rng.integers(0, 20))]
        if rng.random() < p_stop:
            aa = "*"
        cods = cod_of[aa]
        cod = list(cods[int(rng.integers(0, len(cods)))])
        if rng.random() < p_fs:
            if rng.random() < 0.5:
                cod.pop(int(rng.integers(0, 3)))
            else:
                cod.insert(int(rng.integers(0, 3)), int(rng.integers(0, 4)))
        if rng.random() < 0.08 and intron_max > 0:  # intron at a random phase inside this codon
            ph = int(rng.integers(0, len(cod) + 1))
            il = int(rng.integers(20, intron_max + 1))
            body = [int(x) for x in rng.integers(0, 4, size=il)]
            if rng.random() < 0.9:
                body[0:2] = [2, 3]
                body[2] = int(rng.choice([0, 2]))
                body[-3] = int(rng.choice([1, 3]))
                body[-2:] = [0, 2]
            cod = cod[:ph] + body + cod[ph:]
        nt += cod
    nt += [int(x) for x in rng.integers(0, 4, size=int(rng.integers(0, flank + 1)))]
    nt = np.array(nt, dtype=np.uint8)
    if len(nt) and p_n > 0:
        nt[rng.random(len(nt)) < p_n] = 4
    aa = "".join(_AA[a] for a in prot)
    if rng.random() < 0.1 and al > 2:
        k = int(rng.integers(0, al))
        aa = aa[:k] + "X" + aa[k + 1:]
    return nt, aa.encode()


def random_chain_problem(rng: np.random.Generator, n: int, mode: str, bbit: int = 8):
    """Sorted anchors for the three mp_chain call regimes: 'pre', 'main' (block ids of 1 << bbit bases) and 'refine' (base
    resolution)."""
    if mode in ("pre", "main"):
        nb = max(4, n // 3)
        x = np.sort(rng.integers(1000, 1000 + nb, size=n)).astype(np.uint64)
        base = rng.integers(5, 400, size=n)
        # plant collinear runs: qpos follows block id * the residues of a block (85 = 256/3 at bbit 8) within clusters
        f = max(1, (1 << bbit) // 3)
        y = ((x.astype(np.int64) - 1000) * f % max(380, 4 * f + 40) + rng.integers(0, 40, size=n) + 5).astype(np.uint64)
        y = np.where(rng.random(n) < 0.3, base.astype(np.uint64), y)
    else:
        x = np.sort(rng.integers(14, 14 + 6 * n + 50, size=n)).astype(np.uint64)
        y = (x.astype(np.int64) // 3 + rng.integers(-3, 4, size=n)).clip(4, 2000).astype(np.uint64)
        y = np.where(rng.random(n) < 0.2, rng.integers(4, 500, size=n).astype(np.uint64), y)
    a = np.unique((x << np.uint64(32)) | y)
    return np.ascontiguousarray(a, dtype=np.uint64)


CHAIN_MODES = {
    "pre": dict(max_dist_x=256, max_dist_y=256, bw=256, max_skip=25, max_iter=1000000, min_cnt=2, min_sc=0,
                chn_coef_log=0.75, is_spliced=1, kmer=6, bbit=8),
    "main": dict(max_dist_x=200000, max_dist_y=1000, bw=200000, max_skip=25, max_iter=1000000, min_cnt=3, min_sc=0,
                 chn_coef_log=0.75, is_spliced=1, kmer=6, bbit=8),
    "refine": dict(max_dist_x=200000, max_dist_y=1000, bw=200000, max_skip=25, max_iter=1000000, min_cnt=3, min_sc=0,
                   chn_coef_log=0.75, is_spliced=1, kmer=5, bbit=0),
}


def chain_par(mode: str, **over) -> ChainPar:
    d = dict(CHAIN_MODES[mode])
    d.update(over)
    return ChainPar(**d)


def chain_answer(u: np.ndarray, b: np.ndarray) -> dict:
    """A chaining result (u, b arrays) as stored: number of chains and a digest of both arrays."""
    return {"n_u": len(u), "sha256": _digest(np.ascontiguousarray(u, np.uint64), np.ascontiguousarray(b, np.uint64))}


def ref_chain(par: ChainPar, a: np.ndarray) -> dict:
    """chain_answer() of the reference's mp_chain on sorted anchors `a`."""
    def run():
        r = ref()
        n = len(a)
        buf = r.ref_kmalloc(None, max(8 * n, 8))  # mp_chain frees its input
        C.memmove(buf, a.ctypes.data, 8 * n)
        n_u = C.c_int32(0)
        u = C.c_void_p(0)
        b = r.ref_mp_chain(par.max_dist_x, par.max_dist_y, par.bw, par.max_skip, par.max_iter, par.min_cnt, par.min_sc,
                           par.chn_coef_log, par.is_spliced, par.kmer, par.bbit, n, buf, C.byref(n_u), C.byref(u), None)
        return chain_answer(*_take_chain(n_u.value, u.value, b))
    return reference(run, "mp_chain", bytes(par), np.ascontiguousarray(a, np.uint64))


def _take_chain(n_u, u_ptr, b_ptr):
    if n_u == 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    u = np.ctypeslib.as_array(C.cast(u_ptr, C.POINTER(C.c_uint64)), shape=(n_u,)).copy()
    nb = int((u & np.uint64(0xffffffff)).sum())
    b = np.ctypeslib.as_array(C.cast(b_ptr, C.POINTER(C.c_uint64)), shape=(nb,)).copy()
    _libc.free(u_ptr)
    _libc.free(b_ptr)
    return u, b


def ora_chain(par: ChainPar, a: np.ndarray):
    o = ora()
    n_u = C.c_int32(0)
    u = C.c_void_p(0)
    b = o.ora_chain(C.byref(par), len(a), a.ctypes.data_as(C.c_void_p), C.byref(n_u), C.byref(u))
    return _take_chain(n_u.value, u.value, b)
