"""The --dbg-* switches of the CLI (mp_dbg_flag) run the way the reference's main.c runs them, against any library that exports the
reference's entry points: the oracle-backed host library of the CPU tests or libminiprot_b200.so.  Shared by test_host_dbg.py and
test_gpu_dbg.py, and by tools/fuzz_cli.py for the dump lines.

A child process parses the few options below as main.c does (main.c:114-201; -k -M -L -b -T -l only in the attached form -k5),
builds the tables of the genetic code (-T), loads the index, sets mp_dbg_flag and calls
mp_map_file: stdout is the PAF / GFF, stderr carries the dump lines, exactly where the reference CLI prints them."""
import hashlib
import json
import os
import subprocess
import sys

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle_lib as ol  # noqa: E402
from miniprot_b200 import synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DUMP_PREFIXES = (b"QR\t", b"X\t", b"Y1\t")
# what the reference CLI prints for the cases of test_host_dbg / test_gpu_dbg, keyed by a digest of the options and the input files'
# contents; `python tests/dbg_lib.py --record` rewrites it from oracle/_ref/miniprot
RECORD_PATH = os.path.join(ROOT, "tests", "golden", "dbg_reference_calls.json")
_record = None

# the switch sets of the tests (each one a list of CLI options)
SWITCH_SETS = [["--dbg-qname", "--dbg-anchor", "--dbg-chain"], ["--dbg-aflt"], ["--dbg-aflt", "--gff"], ["--dbg-aflt", "-j2"],
               ["--dbg-no-refine", "-A"], ["--dbg-qname", "--dbg-chain", "--dbg-no-refine", "-A"]]

# index and refinement options off the defaults (-k 6 -M 1 -L 30 -b 8, -l 5), one CLI option list each: the k-mer masks and bucket
# counts (-k, -M), the ORF rule and the window kernels' halos (-L; below -k the index is built on the host, below -l only the
# refinement sees it), the block size (-b) and the refinement k-mer (-l).  4k <= 28 and -l <= 7 (a 32-bit k-mer word).
INDEX_OPTION_SETS = [[], ["-k5"], ["-k4", "-M0"], ["-M0"], ["-M2"], ["-L6"], ["-L5"], ["-L1"], ["-L0"], ["-L4"], ["-L10"], ["-L40"],
                     ["-b6"], ["-b7"], ["-b9"], ["-b10"], ["-l3"], ["-l4"], ["-l6"], ["-l7"], ["-l7", "-L5"], ["-l6", "-L4"],
                     ["-l7", "-L1"], ["-k5", "-M0", "-L12", "-b9", "-l4"]]
INDEX_SWITCHES = ["--dbg-anchor", "--dbg-chain"]  # the X (seeds) and Y1 (first-round chains) lines show which stage diverged
# NCBI genetic codes (-T): every code ns_make_tables defines, and those the end-to-end runs take -- their output on tiny, tiny5 and
# DPP3 differs from code 1's and from each other's (code 11 has code 1's tables), with the output formats below.
TRANS_CODES = [1, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14, 15, 16, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33]
TRANS_E2E_CODES = [2, 3, 6, 9, 14, 22, 23, 27, 31, 33]
TRANS_FORMATS = [INDEX_SWITCHES, ["--gff"], ["--trans"], ["--aln"]]
_IDX_FIELD = {"-k": "kmer", "-M": "mod_bit", "-L": "min_aa_len", "-b": "bbit", "-T": "trans_code"}


def index_options(opts) -> tuple:
    """({IdxOpt field: value}, {MapOpt field: value}) of an option list of INDEX_OPTION_SETS (main.c:114-121)."""
    io, mo = {}, {}
    for a in opts:
        if a[:2] in _IDX_FIELD:
            io[_IDX_FIELD[a[:2]]] = int(a[2:])
        elif a[:2] == "-l":
            mo["kmer2"] = int(a[2:])
        else:
            raise ValueError(a)
    return io, mo

_CHILD = r"""
import ctypes as C, os, sys
sys.path.insert(0, sys.argv[1])
import miniprot_b200 as mp
L = C.CDLL(sys.argv[2])
args = sys.argv[3:]
files = [a for i, a in enumerate(args) if not a.startswith("-") and not (i > 0 and args[i - 1] == "--spsc")]
L.mp_start()
C.c_int32.in_dll(L, "mp_verbose").value = 1
io, mo = mp.IdxOpt(), mp.MapOpt()
L.mp_idxopt_init(C.byref(io))
L.mp_mapopt_init(C.byref(mo))
dbg, spsc = 0, None
for i, a in enumerate(args):
    if a in mp.DBG_SWITCHES: dbg |= mp.DBG_SWITCHES[a]
    elif a == "-A": mo.flag |= 0x2
    elif a == "--gff": mo.flag |= 0x8
    elif a.startswith("-j"): mo.sp_model = int(a[2:])
    elif a == "--spsc": spsc = args[i + 1]
    elif a.startswith("-K"): mo.mini_batch_size = int(a[2:])
    elif a == "--aln": mo.flag |= 0x80
    elif a == "--trans": mo.flag |= 0x100
    elif a[:2] in ("-k", "-M", "-L", "-b", "-T"): setattr(io, {"-k": "kmer", "-M": "mod_bit", "-L": "min_aa_len", "-b": "bbit", "-T": "trans_code"}[a[:2]], int(a[2:]))
    elif a[:2] == "-l": mo.kmer2 = int(a[2:])
if L.ns_make_tables(io.trans_code) < 0:
    sys.stderr.write(f"[ERROR] failed to find translation table {io.trans_code}\n")
    sys.exit(101)
L.mp_idx_load.restype = C.c_void_p
L.mp_idx_load.argtypes = [C.c_char_p, C.c_void_p, C.c_int32]
mi = L.mp_idx_load(files[0].encode(), C.byref(io), 4)
assert mi
if spsc:
    L.mp_set_spsc.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_int32]
    L.mp_set_spsc(spsc.encode(), mi, C.byref(mo), 0)
mp.set_dbg_flag(dbg, L)
L.mp_map_file.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int]
rc = L.mp_map_file(mi, files[1].encode(), C.byref(mo), 1)
sys.stdout.flush()
L.mp_idx_destroy.argtypes = [C.c_void_p]
L.mp_idx_destroy(mi)
sys.exit(0 if rc == 0 else 100 - rc)
"""


def dump_lines(stderr: bytes) -> list:
    """The lines of the --dbg-* dumps (QR / X / Y1) among everything else on stderr, in order."""
    return [l for l in stderr.splitlines(keepends=True) if l.startswith(DUMP_PREFIXES)]


def digest(out: bytes, err: bytes) -> dict:
    """What ol.ref_cli_dbg() stores for one run."""
    d = b"".join(dump_lines(err))
    return {"sha256": hashlib.sha256(out).hexdigest(), "lines": out.count(b"\n"), "dump_sha256": hashlib.sha256(d).hexdigest(),
            "dump_lines": d.count(b"\n")}


def ref_cli_dbg(args, genome: str, proteins: str) -> dict:
    """digest() of what the reference CLI prints for `-t1 args genome proteins` (one worker thread: the dump lines come protein after
    protein): the stored answer, or -- when recording -- the answer of oracle/_ref/miniprot."""
    global _record
    if _record is None:
        _record = json.load(open(RECORD_PATH)) if os.path.exists(RECORD_PATH) else {}
    key = ol._digest("cli -t1 dbg", [ol.file_digest(a) if os.path.isfile(a) else a for a in args], [ol.file_digest(f) for f in (genome, proteins)])[:40]
    if key in _record and not ol.RECORDING:
        return _record[key]
    if not os.path.exists(ol.REF_BIN):
        raise LookupError(f"no stored reference answer for {args!r} on these inputs, and oracle/_ref is not built: record it with "
                          "python tests/dbg_lib.py --record")
    r = subprocess.run([ol.REF_BIN, "-t1", *args, genome, proteins], check=True, capture_output=True)
    _record[key] = digest(r.stdout, r.stderr)
    return _record[key]


def save_record():
    with open(RECORD_PATH + ".tmp", "w") as f:
        json.dump(_record, f, sort_keys=True, indent=1)
        f.write("\n")
    os.replace(RECORD_PATH + ".tmp", RECORD_PATH)


def run_cli(lib_path: str, args, genome: str, proteins: str, env=None):
    """(return code of mp_map_file, stdout, stderr) of `args genome proteins` through `lib_path`."""
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, lib_path, *args, genome, proteins], capture_output=True,
                       env=env if env is not None else os.environ.copy(), timeout=3600)
    if r.returncode not in (0, 100 + 3, 100 + 1):
        raise RuntimeError(f"the child failed ({r.returncode}): {r.stderr.decode(errors='replace')[-2000:]}")
    return (0 if r.returncode == 0 else 100 - r.returncode), r.stdout, r.stderr


def short_contig_genome(d: str) -> str:
    """The tiny genome cut into 25 kb contigs: chains that cross a contig boundary are cut (hit.c:32-76), so some Y1 lines print
    anchors of the other contig with the kept one's block offset."""
    g, _ = synth.generate(synth.CONFIGS["tiny"], d)
    seq = []
    out = os.path.join(d, "short_ctg.fa")
    with open(g) as f:
        for line in f:
            if not line.startswith(">"):
                seq.append(line.strip())
    s = "".join(seq)
    with open(out, "w") as f:
        for i in range(0, len(s), 25_000):
            f.write(f">s{i // 25_000}\n{s[i:i + 25_000]}\n")
    return out


def input_sets(d: str) -> dict:
    """name -> (genome, proteins): DPP3, the synthetic golden sets (tiny5 is the divergent one) and the short-contig genome."""
    out = {"DPP3": (ol.DPP3_GENOME, ol.DPP3_PROTEIN)}
    for cfg in ("tiny", "tiny5"):
        out[cfg] = synth.generate(synth.CONFIGS[cfg], os.path.join(d, cfg))
    out["short_ctg"] = (short_contig_genome(os.path.join(d, "tiny")), out["tiny"][1])
    return out


def spsc_file(d: str) -> str:
    """A splice-score file over the DPP3 genome (the --dbg-aflt --spsc case)."""
    import gzip

    fa = os.path.join(d, "dpp3.fa")
    with gzip.open(ol.DPP3_GENOME, "rb") as f, open(fa, "wb") as o:
        o.write(f.read())
    return synth.make_spsc(fa, os.path.join(d, "dpp3.spsc"), seed=6)


def c4_slice(d: str, n: int = 12) -> tuple:
    """(genome, proteins): the scaled long-intron configuration C4s with its first n proteins only -- region of 50-150 kb introns,
    so --dbg-aflt aligns several hundred kb of rows per region in one problem."""
    g, p = synth.generate(synth.CONFIGS["C4s"], os.path.join(d, "C4s"))
    out = os.path.join(d, "C4s", f"first{n}.faa")
    k = 0
    with open(p) as f, open(out, "w") as o:
        for line in f:
            if line.startswith(">"):
                k += 1
                if k > n:
                    break
            o.write(line)
    return g, out


if __name__ == "__main__":  # --record: the reference's answers for every case of the two test files (needs oracle/_ref)
    import tempfile

    assert sys.argv[1:] == ["--record"], "usage: python tests/dbg_lib.py --record"
    ol.RECORDING = True
    _record = {}
    with tempfile.TemporaryDirectory() as d:
        sets = input_sets(d)
        for name in ("DPP3", "tiny", "tiny5", "short_ctg"):
            for sw in SWITCH_SETS:
                ref_cli_dbg(sw, *sets[name])
        ref_cli_dbg(["--dbg-chain"], *sets["short_ctg"])
        ref_cli_dbg(["--dbg-qname", "--dbg-anchor", "--dbg-chain"], *sets["tiny"])
        ref_cli_dbg(["--dbg-aflt", "--spsc", spsc_file(d)], ol.DPP3_GENOME, ol.DPP3_PROTEIN)
        ref_cli_dbg(["--dbg-aflt"], *c4_slice(d))
        for name in ("DPP3", "tiny", "tiny5"):  # test_host_index_options / test_gpu_index_options
            for opts in INDEX_OPTION_SETS + [["-L41"]]:
                ref_cli_dbg(opts + INDEX_SWITCHES, *sets[name])
            for code in TRANS_E2E_CODES:  # test_host_trans_code / test_gpu_trans_code
                for fmt in TRANS_FORMATS:
                    ref_cli_dbg([f"-T{code}"] + fmt, *sets[name])
    save_record()
    print(len(_record), "answers written to", RECORD_PATH)
