"""Locus mode (mpb_map_loci): the cases of test_gpu_loci.py / test_host_loci.py and the reference's answers for them.

For a case, the reference CLI maps each protein against a FASTA that holds only genome[cid][st:en]; its PAF lines, with columns 6-9
moved to the real contig (name, length, start + st, end + st), concatenated in the order of the loci, are the answer.  The answers are
stored as digests in tests/golden/loci_reference_calls.json; `python tests/loci_lib.py --record` rewrites them from oracle/_ref/miniprot.
Every input is generated at test time (DPP3 and seeded synthetic genomes)."""
import gzip
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle_lib as ol  # noqa: E402
from miniprot_b200 import synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORD_PATH = os.path.join(ROOT, "tests", "golden", "loci_reference_calls.json")
_record = None


def read_fasta(path):
    """[(name, sequence bytes)] of a FASTA file (gzip or plain)."""
    out = []
    with (gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")) as f:
        for line in f:
            if line.startswith(b">"):
                out.append([line[1:].split()[0], []])
            elif out:
                out[-1][1].append(line.strip())
    return [(n, b"".join(s)) for n, s in out]


def write_fasta(path, recs):
    with open(path, "wb") as f:
        for n, s in recs:
            f.write(b">" + n + b"\n" + s + b"\n")
    return path


def paf_hits(path):
    """(protein, contig, start, end, strand) of the lines of a PAF file."""
    out = []
    for line in open(path):
        t = line.split("\t")
        out.append((t[0], t[5], int(t[7]), int(t[8]), t[4]))
    return out


def _mutate(rng, s: bytes, p: float) -> bytes:
    a = np.frombuffer(s, np.uint8).copy()
    m = rng.random(len(a)) < p
    a[m] = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, int(m.sum()))]
    return a.tobytes()


def _rand(rng, n: int) -> bytes:
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)].tobytes()


def _around(hits, ctg_len, flank, n):
    """loci of the first n hits with `flank` bases on each side, clipped to the contig"""
    return [(p, c, max(0, s - flank), min(ctg_len[c], e + flank)) for p, c, s, e, _ in hits[:n]]


def build_cases(d: str) -> dict:
    """name -> {"genome", "proteins", "loci": [(protein, contig, st, en)], "args": [CLI options]}."""
    rng = np.random.default_rng(11)
    cases = {}
    # DPP3: one gene over the whole 27 kb contig; CDS 1 is [0, 270), intron 1 is [270, 2972), the last CDS ends at 27030 (DPP3_gff.txt)
    g = read_fasta(ol.DPP3_GENOME)
    (cn, cs), = g
    p = read_fasta(ol.DPP3_PROTEIN)[0][0].decode()
    c, L = cn.decode(), len(cs)
    cases["DPP3"] = dict(genome=ol.DPP3_GENOME, proteins=ol.DPP3_PROTEIN, args=[], loci=[
        (p, c, 0, L), (p, c, 0, 27030), (p, c, 150, L), (p, c, 0, 26950), (p, c, 0, 1500), (p, c, 1500, L),
        (p, c, 2953, 3153), (p, c, 4325, 4572), (p, c, 5063, 5163), (p, c, 0, 31), (p, c, L - 97, L)])
    # an N run inside intron 2 and one inside exon 3
    s = bytearray(cs)
    s[3500:3600] = b"N" * 100
    s[4400:4420] = b"N" * 20
    gN = write_fasta(os.path.join(d, "dpp3N.fa"), [(cn, bytes(s))])
    cases["DPP3_N"] = dict(genome=gN, proteins=ol.DPP3_PROTEIN, args=[], loci=[(p, c, 0, L), (p, c, 2000, 6000)])
    # two diverged copies of the first 12 kb of the gene in one contig (secondary hits), random sequence (no hit)
    para = cs[:12000] + _rand(rng, 3000) + _mutate(rng, cs[:12000], 0.005) + _rand(rng, 2000)
    gP = write_fasta(os.path.join(d, "para.fa"), [(b"para", para), (b"rand", _rand(rng, 5000))])
    cases["paralogs"] = dict(genome=gP, proteins=ol.DPP3_PROTEIN, args=[], loci=[
        (p, "para", 0, len(para)), (p, "para", 12000, 15000), (p, "rand", 0, 5000), (p, "para", 14000, len(para))])
    # synthetic genes on both strands, 0 / 100 / 5000 bp flanks; one protein against several loci in one call; the divergent set
    # with frameshifts (tiny5, the error model of C5)
    for cfg, n in (("tiny", 8), ("tiny5", 10)):
        gg, pp = synth.generate(synth.CONFIGS[cfg], os.path.join(d, cfg))
        ctg_len = {x.decode(): len(y) for x, y in read_fasta(gg)}
        hits = paf_hits(os.path.join(ol.GOLDEN, f"{cfg}.paf"))
        loci = _around(hits, ctg_len, 0, n) + _around(hits, ctg_len, 100, n) + _around(hits, ctg_len, 5000, n // 2)
        q0, c0 = hits[0][0], hits[0][1]
        loci += [(q0, hh[1], max(0, hh[2] - 100), hh[3] + 100) for hh in hits[1:4]] + [(q0, c0, 0, 20000), (q0, c0, ctg_len[c0] - 20000, ctg_len[c0])]
        cases[cfg] = dict(genome=gg, proteins=pp, args=[], loci=loci)
    # the divergent set under the vertebrate mitochondrial code (-T2: AGA / AGG are stops, TGA is W, ATA is M)
    cases["tiny5_T2"] = dict(cases["tiny5"], args=["-T2"])
    return cases


def _key(case) -> str:
    return ol._digest("loci", ol.file_digest(case["genome"]), ol.file_digest(case["proteins"]), case["args"], [list(x) for x in case["loci"]])[:40]


def digest(paf: bytes) -> dict:
    return {"sha256": hashlib.sha256(paf).hexdigest(), "lines": paf.count(b"\n")}


def translate(line: bytes, ctg: bytes, clen: int, st: int) -> bytes:
    """A PAF line of the locus FASTA in the coordinates of the real contig (columns 6-9)."""
    t = line.split(b"\t")
    t[5], t[6], t[7], t[8] = ctg, str(clen).encode(), str(int(t[7]) + st).encode(), str(int(t[8]) + st).encode()
    return b"\t".join(t)


def reference_paf(case) -> bytes:
    """What the reference CLI prints for every locus of the case, translated and concatenated (needs oracle/_ref)."""
    genome = dict(read_fasta(case["genome"]))
    prots = dict(read_fasta(case["proteins"]))
    out = []
    with tempfile.TemporaryDirectory() as d:
        for p, c, st, en in case["loci"]:
            gf = write_fasta(os.path.join(d, "locus.fa"), [(b"locus", genome[c.encode()][st:en])])
            pf = write_fasta(os.path.join(d, "prot.fa"), [(p.encode(), prots[p.encode()])])
            r = subprocess.run([ol.REF_BIN, *case["args"], gf, pf], check=True, capture_output=True).stdout
            out += [translate(line, c.encode(), len(genome[c.encode()]), st) for line in r.splitlines(keepends=True)]
    return b"".join(out)


def ref_answer(case) -> dict:
    """digest() of reference_paf(case): the stored answer, or -- when recording -- the compiled reference's."""
    global _record
    if _record is None:
        _record = json.load(open(RECORD_PATH)) if os.path.exists(RECORD_PATH) else {}
    k = _key(case)
    if k in _record and not ol.RECORDING:
        return _record[k]
    if not os.path.exists(ol.REF_BIN):
        raise LookupError("no stored reference answer for this locus case, and oracle/_ref is not built: record it with python tests/loci_lib.py --record")
    _record[k] = digest(reference_paf(case))
    return _record[k]


def index_of(case):
    """(names, sequences) of the case's proteins and the (qid, cid, st, en) tuples of its loci, for the index `mi` of its genome."""
    prots = read_fasta(case["proteins"])
    qid = {n.decode(): i for i, (n, _) in enumerate(prots)}
    return [n for n, _ in prots], [s for _, s in prots], qid


def loci_tuples(mi, case, qid):
    nt = mi.contents.nt.contents
    cid = {nt.ctg[i].name.decode(): i for i in range(nt.n_ctg)}
    return [(qid[p], cid[c], st, en) for p, c, st, en in case["loci"]]


if __name__ == "__main__":
    assert sys.argv[1:] == ["--record"], "usage: python tests/loci_lib.py --record"
    ol.RECORDING = True
    _record = {}
    with tempfile.TemporaryDirectory() as d:
        for name, case in build_cases(d).items():
            print(name, ref_answer(case))
    with open(RECORD_PATH + ".tmp", "w") as f:
        json.dump(_record, f, sort_keys=True, indent=1)
        f.write("\n")
    os.replace(RECORD_PATH + ".tmp", RECORD_PATH)
    print(len(_record), "answers written to", RECORD_PATH)
