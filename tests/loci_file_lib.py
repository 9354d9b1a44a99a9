"""The locus file driver (mpb_map_loci_file*): the cases of test_gpu_loci_file.py / test_host_loci_file.py and the reference's
answers for them.

A case of loci_lib (its genome, proteins and loci) is run under each option set of OPTION_SETS.  The answer: for every locus, in
order, the reference CLI with those options maps the protein against a FASTA that holds only genome[contig][st:en]; its output is
moved to the real contig -- contig name and length in PAF columns 6-7 (also in the ##PAF lines), st added to PAF columns 8-9 and
GFF / GTF columns 4-5, the contig's name in GFF / GTF column 1 -- its ids renumbered by one counter over the whole output, and the
"##gff-version 3" line kept once at the top.  The answers are stored as digests in tests/golden/loci_file_reference_calls.json;
`python tests/loci_file_lib.py --record` rewrites them from oracle/_ref/miniprot (make -C oracle)."""
import json
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import importlib.util  # noqa: E402

import loci_lib  # noqa: E402
import oracle_lib as ol  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORD_PATH = os.path.join(ROOT, "tests", "golden", "loci_file_reference_calls.json")
CASES = ["DPP3", "DPP3_N", "paralogs", "tiny", "tiny5"]
OPTION_SETS = {
    "default": [],
    "gff": ["--gff"],
    "gff_only_P": ["--gff-only", "-P", "XY"],
    "gtf": ["--gtf"],
    "gtf_unmapped": ["--gtf", "-u"],
    "aln": ["--aln"],
    "trans_gff": ["--trans", "--gff"],
    "unmapped_outn1": ["-u", "--outn=1"],
    "outs_outc": ["--outs=0.99", "--outc=0.5"],
    "j2_no_cs": ["-j2", "--no-cs"],
    "no_splice": ["-S"],
    "aln_flank_delim": ["--aln", "--max-intron-out=50", "--gff-delim=:"],
    "index_options": ["-k5", "-M2", "-L35", "-b7"],
}
_record = None


def map_loci_tool():
    """tools/map_loci.py as a module (its option parser)."""
    spec = importlib.util.spec_from_file_location("map_loci_tool", os.path.join(ROOT, "tools", "map_loci.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def write_tsv(path, loci):
    with open(path, "w") as f:
        f.write("# protein\tcontig\tstart\tend\n\n")
        f.writelines(f"{p}\t{c}\t{st}\t{en}\n" for p, c, st, en in loci)
    return path


def _key(case, args) -> str:
    return ol._digest("loci_file", ol.file_digest(case["genome"]), ol.file_digest(case["proteins"]), list(args), [list(x) for x in case["loci"]])[:40]


def _id_pattern(prefix: bytes):
    """the numbered ids of GFF3 (ID= / Parent=) and GTF (gene_id / transcript_id) attributes: (head, prefix + infix, number)"""
    return re.compile(rb'((?:ID=|Parent=|gene_id "|transcript_id ")' + re.escape(prefix) + rb"[GT]?)(\d+)")


def translate(out: bytes, ctg: bytes, clen: int, st: int, id_pat, id_base: int):
    """One locus run's output in contig coordinates, ids moved up by id_base; returns (lines, the largest id it used)."""
    lines, top = [], 0

    def renumber(m):
        nonlocal top
        top = max(top, int(m.group(2)))
        return m.group(1) + b"%.6d" % (int(m.group(2)) + id_base)

    for line in out.splitlines(keepends=True):
        if line.startswith(b"##gff-version"):
            continue
        t = line.split(b"\t")
        if t[0] == b"##PAF" and len(t) > 9 and t[6] == b"locus":
            t[6], t[7], t[8], t[9] = ctg, str(clen).encode(), str(int(t[8]) + st).encode(), str(int(t[9]) + st).encode()
        elif not line.startswith(b"#") and len(t) > 8 and t[5] == b"locus":  # PAF
            t[5], t[6], t[7], t[8] = ctg, str(clen).encode(), str(int(t[7]) + st).encode(), str(int(t[8]) + st).encode()
        elif not line.startswith(b"#") and len(t) == 9 and t[0] == b"locus":  # GFF3 / GTF
            t[0], t[3], t[4] = ctg, str(int(t[3]) + st).encode(), str(int(t[4]) + st).encode()
            t[8] = id_pat.sub(renumber, t[8])
        lines.append(b"\t".join(t))
    return lines, top


def reference_output(case, args) -> bytes:
    """What the reference CLI prints for every locus of the case under `args`, translated and concatenated (needs oracle/_ref)."""
    genome = dict(loci_lib.read_fasta(case["genome"]))
    prots = dict(loci_lib.read_fasta(case["proteins"]))
    prefix = args[args.index("-P") + 1].encode() if "-P" in args else b"MP"
    id_pat = _id_pattern(prefix)
    with tempfile.TemporaryDirectory() as d:
        def run(k):
            p, c, st, en = case["loci"][k]
            gf = loci_lib.write_fasta(os.path.join(d, f"locus{k}.fa"), [(b"locus", genome[c.encode()][st:en])])
            pf = loci_lib.write_fasta(os.path.join(d, f"prot{k}.fa"), [(p.encode(), prots[p.encode()])])
            return subprocess.run([ol.REF_BIN, "-t1", *args, gf, pf], check=True, capture_output=True).stdout
        with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
            outs = list(ex.map(run, range(len(case["loci"]))))
    res = [b"##gff-version 3\n"] if any(a in ("--gff", "--gff-only") for a in args) else []
    base = 0
    for (p, c, st, en), out in zip(case["loci"], outs):
        lines, top = translate(out, c.encode(), len(genome[c.encode()]), st, id_pat, base)
        res += lines
        base += top
    return b"".join(res)


def ref_answer(case, args) -> dict:
    """loci_lib.digest() of reference_output(case, args): the stored answer, or -- when recording -- the compiled reference's."""
    global _record
    if _record is None:
        _record = json.load(open(RECORD_PATH)) if os.path.exists(RECORD_PATH) else {}
    k = _key(case, args)
    if k in _record and not ol.RECORDING:
        return _record[k]
    if not os.path.exists(ol.REF_BIN):
        raise LookupError("no stored reference answer for this case, and oracle/_ref is not built: record it with python tests/loci_file_lib.py --record")
    _record[k] = loci_lib.digest(reference_output(case, args))
    return _record[k]


if __name__ == "__main__":
    assert sys.argv[1:] == ["--record"], "usage: python tests/loci_file_lib.py --record"
    ol.RECORDING = True
    _record = {}
    with tempfile.TemporaryDirectory() as d:
        cases = loci_lib.build_cases(d)
        for name in CASES:
            for set_name, args in OPTION_SETS.items():
                print(name, set_name, ref_answer(cases[name], args), flush=True)
    with open(RECORD_PATH + ".tmp", "w") as f:
        json.dump(_record, f, sort_keys=True, indent=1)
        f.write("\n")
    os.replace(RECORD_PATH + ".tmp", RECORD_PATH)
    print(len(_record), "answers written to", RECORD_PATH)
