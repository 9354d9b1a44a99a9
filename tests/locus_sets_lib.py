"""Locus sets (mpb_map_locus_sets, mpb_map_locus_sets_file*): the cases of test_gpu_locus_sets.py / test_host_locus_sets.py and the
reference's answers for them.

A case is a genome of loci_lib.build_cases, its proteins and the lines of a set file: (protein, contig, start, end, label or None).
The lines of one (protein, label) form a set, sets in the order of their first line.  The answer, under each option set of
OPTION_SETS: for every set, the reference CLI with those options maps the protein against a FASTA of the set's canonical genome -- its
ranges, those of one contig that overlap or abut merged, sorted by (contig order in the genome, start), one record each with a name
of its own -- and its output is moved to the real contigs: the record's contig name and length in PAF columns 6-7 (also in the ##PAF
lines), the record's start added to PAF columns 8-9 and GFF / GTF columns 4-5, the contig's name in GFF / GTF column 1; ids are
renumbered by one counter over the whole output and "##gff-version 3" is kept once at the top.  The answers are stored as digests in
tests/golden/locus_sets_reference_calls.json; `python tests/locus_sets_lib.py --record` rewrites them from oracle/_ref/miniprot
(make -C oracle)."""
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

import loci_file_lib  # noqa: E402
import loci_lib  # noqa: E402
import oracle_lib as ol  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORD_PATH = os.path.join(ROOT, "tests", "golden", "locus_sets_reference_calls.json")
CASES = ["paralogs", "DPP3", "tiny", "tiny5", "tiny5_T2"]
OPTION_SETS = dict(loci_file_lib.OPTION_SETS, N1=["-N1"], N0_unmapped=["-N0", "-u"], p095=["-p0.95"], outn2_gff=["--outn=2", "--gff"])
_record = None


def _tsv_line(p, c, st, en, label):
    return f"{p}\t{c}\t{st}\t{en}" + (f"\t{label}" if label is not None else "") + "\n"


def write_tsv(path, lines):
    with open(path, "w") as f:
        f.write("# protein\tcontig\tstart\tend\tset\n\n")
        f.writelines(_tsv_line(*x) for x in lines)
    return path


def sets_of(lines):
    """[(protein, [(contig, st, en)])]: the sets of a set file's lines, in the order of their first line."""
    order, loci = [], {}
    for p, c, st, en, label in lines:
        k = (p, label)
        if k not in loci:
            order.append(k)
            loci[k] = []
        loci[k].append((c, st, en))
    return [(k[0], loci[k]) for k in order]


def canonical(ranges, ctg_order):
    """The merged ranges of a set, sorted by (contig index, start): ranges of one contig that overlap or abut become their union."""
    out = []
    for c, st, en in sorted(ranges, key=lambda r: (ctg_order[r[0]], r[1])):
        if out and out[-1][0] == c and st <= out[-1][2]:
            out[-1][2] = max(out[-1][2], en)
        else:
            out.append([c, st, en])
    return [tuple(r) for r in out]


def build_cases(d: str) -> dict:
    """name -> {"genome", "proteins", "args", "lines"}: the set-file cases on the genomes of loci_lib.build_cases."""
    base = loci_lib.build_cases(d)
    rng = np.random.default_rng(23)
    cases = {}
    # paralogs: both diverged copies (para [0, 12000) and [15000, 27000)) and the random contig in one set, so that which copy is
    # primary and which secondary is decided across ranges; and each copy alone
    b = base["paralogs"]
    p = b["loci"][0][0]
    cases["paralogs"] = dict(genome=b["genome"], proteins=b["proteins"], args=[], lines=[
        (p, "para", 0, 13000, "both"), (p, "para", 14500, 28000, "both"), (p, "rand", 0, 5000, "both"),
        (p, "para", 0, 13000, "copy1"), (p, "para", 14500, 28000, "copy2")])
    # DPP3: [0, 1500) + [1500, L) abut and merge into the whole contig; three exon-only ranges as another set
    b = base["DPP3"]
    p, c, _, L = b["loci"][0]
    cases["DPP3"] = dict(genome=b["genome"], proteins=b["proteins"], args=[], lines=[
        (p, c, 1500, L, "whole"), (p, c, 4325, 4572, "exons"), (p, c, 0, 1500, "whole"), (p, c, 5063, 5163, "exons"), (p, c, 2953, 3153, "exons")])
    # synthetic genes: each protein with its gene +- 100 bp (every other one as two overlapping lines), the genes of three other
    # proteins as decoys and a range of a second contig; the lines shuffled over the file; tiny adds labelled sets of one protein
    for cfg in ("tiny", "tiny5"):
        b = base[cfg]
        ctg_len = {x.decode(): len(y) for x, y in loci_lib.read_fasta(b["genome"])}
        ctgs = list(ctg_len)
        hits = loci_lib.paf_hits(os.path.join(ol.GOLDEN, f"{cfg}.paf"))
        first = {}
        for h in hits:
            first.setdefault(h[0], h)
        genes = list(first.values())[:8]
        lines = []
        for i, (q, c, s, e, _) in enumerate(genes):
            lo, hi = max(0, s - 100), min(ctg_len[c], e + 100)
            if i % 2 == 0:
                m = (lo + hi) // 2
                lines += [(q, c, lo, m + 50, None), (q, c, m - 50, hi, None)]
            else:
                lines.append((q, c, lo, hi, None))
            for j in (1, 2, 3):
                _, dc, ds, de, _ = genes[(i + j) % len(genes)]
                lines.append((q, dc, ds, de, None))
            c2 = ctgs[(ctgs.index(c) + 1) % len(ctgs)]
            lines.append((q, c2, 300000 + 1000 * i, 304000 + 1000 * i, None))
        lines = [lines[k] for k in rng.permutation(len(lines))]
        if cfg == "tiny":
            q, c, s, e, _ = genes[0]
            _, dc, ds, de, _ = genes[1]
            lines += [(q, c, s, e, "gene"), (q, dc, ds, de, "decoy"), (q, c, 0, 20000, "decoy"), (q, c, max(0, s - 5000), e + 5000, "gene")]
        cases[cfg] = dict(genome=b["genome"], proteins=b["proteins"], args=[], lines=lines)
    cases["tiny5_T2"] = dict(cases["tiny5"], args=["-T2"])
    return cases


def _key(case, args) -> str:
    return ol._digest("locus_sets", ol.file_digest(case["genome"]), ol.file_digest(case["proteins"]), list(case["args"]) + list(args),
                      [list(x) for x in case["lines"]])[:40]


def translate(out: bytes, recs: dict, id_pat, id_base: int):
    """One set run's output on the real contigs (recs: record name -> (contig, contig length, start)), ids moved up by id_base;
    returns (lines, the largest id it used)."""
    lines, top = [], 0

    def renumber(m):
        nonlocal top
        top = max(top, int(m.group(2)))
        return m.group(1) + b"%.6d" % (int(m.group(2)) + id_base)

    for line in out.splitlines(keepends=True):
        if line.startswith(b"##gff-version"):
            continue
        t = line.split(b"\t")
        if t[0] == b"##PAF" and len(t) > 9 and t[6] in recs:
            c, clen, st = recs[t[6]]
            t[6], t[7], t[8], t[9] = c, str(clen).encode(), str(int(t[8]) + st).encode(), str(int(t[9]) + st).encode()
        elif not line.startswith(b"#") and len(t) > 8 and t[5] in recs:  # PAF
            c, clen, st = recs[t[5]]
            t[5], t[6], t[7], t[8] = c, str(clen).encode(), str(int(t[7]) + st).encode(), str(int(t[8]) + st).encode()
        elif not line.startswith(b"#") and len(t) == 9 and t[0] in recs:  # GFF3 / GTF
            c, _, st = recs[t[0]]
            t[0], t[3], t[4] = c, str(int(t[3]) + st).encode(), str(int(t[4]) + st).encode()
            t[8] = id_pat.sub(renumber, t[8])
        lines.append(b"\t".join(t))
    return lines, top


def reference_output(case, args) -> bytes:
    """What the reference CLI prints for every set of the case under `args`, translated and concatenated (needs oracle/_ref)."""
    genome = loci_lib.read_fasta(case["genome"])
    order = {n.decode(): i for i, (n, _) in enumerate(genome)}
    genome = dict(genome)
    prots = dict(loci_lib.read_fasta(case["proteins"]))
    prefix = args[args.index("-P") + 1].encode() if "-P" in args else b"MP"
    id_pat = loci_file_lib._id_pattern(prefix)
    sets = [(p, canonical(r, order)) for p, r in sets_of(case["lines"])]
    with tempfile.TemporaryDirectory() as d:
        def run(k):
            p, rs = sets[k]
            recs = [(b"set%d_r%d" % (k, i), genome[c.encode()][st:en]) for i, (c, st, en) in enumerate(rs)]
            gf = loci_lib.write_fasta(os.path.join(d, f"set{k}.fa"), recs)
            pf = loci_lib.write_fasta(os.path.join(d, f"prot{k}.fa"), [(p.encode(), prots[p.encode()])])
            return subprocess.run([ol.REF_BIN, "-t1", *case["args"], *args, gf, pf], check=True, capture_output=True).stdout
        with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
            outs = list(ex.map(run, range(len(sets))))
    res = [b"##gff-version 3\n"] if any(a in ("--gff", "--gff-only") for a in args) else []
    base = 0
    for k, ((p, rs), out) in enumerate(zip(sets, outs)):
        recs = {b"set%d_r%d" % (k, i): (c.encode(), len(genome[c.encode()]), st) for i, (c, st, en) in enumerate(rs)}
        lines, top = translate(out, recs, id_pat, base)
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
        raise LookupError("no stored reference answer for this case, and oracle/_ref is not built: record it with python tests/locus_sets_lib.py --record")
    _record[k] = loci_lib.digest(reference_output(case, args))
    return _record[k]


def set_arrays(mi, case, qid):
    """(set_off, loci) of the case's sets for mpb_map_locus_sets, in the order of the file: loci as (qid, cid, st, en) tuples."""
    nt = mi.contents.nt.contents
    cid = {nt.ctg[i].name.decode(): i for i in range(nt.n_ctg)}
    off, loci = [0], []
    for p, rs in sets_of(case["lines"]):
        loci += [(qid[p], cid[c], st, en) for c, st, en in rs]
        off.append(len(loci))
    return off, loci


if __name__ == "__main__":
    assert sys.argv[1:] == ["--record"], "usage: python tests/locus_sets_lib.py --record"
    ol.RECORDING = True
    _record = {}
    with tempfile.TemporaryDirectory() as d:
        cases = build_cases(d)
        for name in CASES:
            for set_name, args in OPTION_SETS.items():
                print(name, set_name, ref_answer(cases[name], args), flush=True)
    with open(RECORD_PATH + ".tmp", "w") as f:
        json.dump(_record, f, sort_keys=True, indent=1)
        f.write("\n")
    os.replace(RECORD_PATH + ".tmp", RECORD_PATH)
    print(len(_record), "answers written to", RECORD_PATH)
