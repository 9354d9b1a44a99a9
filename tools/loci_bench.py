"""Throughput of locus mode (mpb_map_loci) on the C2 synthetic workload: each planted protein against its gene locus +- 10 kb.

    python tools/loci_bench.py [--workload C2] [--flank 10000] [--repeats 3] [--ref-sample 20] [--sets K]

The loci come from a whole-genome mpb_map_batch of the same proteins (the primary hit of each protein, widened by the flank and
clipped to its contig).  Reported, with the device name and power limit beside the numbers:
  * pairs/s of mpb_map_loci over all pairs in one call (the genome resident; best of the repeats);
  * proteins/s of the whole-genome mpb_map_batch of the same proteins (the k-mer index resident), for context;
  * loci/s of the reference CLI (oracle/_ref/miniprot, where it is built) run the way one maps a known locus without this library --
    extract the locus to a FASTA, index it and map the protein, one run per locus -- on a sample of the loci, on the host;
  * with --sets K: each protein gets a locus set (mpb_map_locus_sets) of its gene locus plus the loci of the K - 1 proteins after it
    as decoys; sets/s over all sets in one call, beside pairs/s of mpb_map_loci over the same (protein, locus) pairs.
Inputs go to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import miniprot_b200 as mp  # noqa: E402
from miniprot_b200 import synth  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "miniprot")


def read_fasta(path):
    out = []
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b">"):
                out.append([line[1:].split()[0], []])
            elif out:
                out[-1][1].append(line.strip())
    return [(n, b"".join(s)) for n, s in out]


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().split(",")[:2]]
        return {"device": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 -- a report
        return {"device": f"unknown ({type(e).__name__})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C2", choices=sorted(synth.CONFIGS))
    ap.add_argument("--flank", type=int, default=10_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--ref-sample", type=int, default=20)
    ap.add_argument("--sets", type=int, default=0, metavar="K", help="also time sets of each gene locus and K - 1 decoy loci")
    a = ap.parse_args()
    L = mp.lib()
    res = {"workload": a.workload, "flank": a.flank, **device_info()}
    with tempfile.TemporaryDirectory() as d:
        g, p = synth.generate(synth.CONFIGS[a.workload], d)
        prots = read_fasta(p)
        names, seqs = [n for n, _ in prots], [s for _, s in prots]
        ctx = mp.Context(0)
        mi = mp.idx_load(g, os.cpu_count() or 8)
        assert L.mpb_idx_upload(ctx.h, mi) == 0
        n = len(seqs)
        arr = (mp.C.c_char_p * n)(*seqs)
        nam = (mp.C.c_char_p * n)(*names)
        lens = (mp.C.c_int32 * n)(*[len(s) for s in seqs])
        n_reg = (mp.C.c_int32 * n)()
        reg = (mp.C.c_void_p * n)()
        L.mpb_map_batch.argtypes = [mp.C.c_void_p, mp.C.c_void_p, mp.C.c_void_p, mp.C.c_int32, mp.C.c_void_p, mp.C.c_void_p, mp.C.c_void_p, mp.C.c_void_p, mp.C.c_void_p]
        L.mpb_regs_free.argtypes = [mp.C.c_int32, mp.C.c_void_p, mp.C.c_void_p]
        mo = mp.mapopt()
        whole = []
        for _ in range(a.repeats + 1):
            t0 = time.perf_counter()
            assert L.mpb_map_batch(ctx.h, mp.C.cast(mi, mp.C.c_void_p), mp.C.byref(mo), n, arr, lens, nam, n_reg, reg) == 0
            whole.append(time.perf_counter() - t0)
            loci = []
            nt = mi.contents.nt.contents
            for q in range(n):
                if n_reg[q] == 0:
                    continue
                r = mp.C.cast(reg[q], mp.C.POINTER(mp.Reg1))[0]
                c = r.vid >> 1
                clen = nt.ctg[c].len
                st, en = (r.vs, r.ve) if not (r.vid & 1) else (clen - r.ve, clen - r.vs)
                loci.append((q, c, max(0, st - a.flank), min(clen, en + a.flank)))
            L.mpb_regs_free(n, n_reg, reg)
        res["whole_genome_proteins_per_s"] = round(n / min(whole[1:]), 1)
        res["pairs"] = len(loci)
        times = []
        for _ in range(a.repeats + 1):
            t0 = time.perf_counter()
            rc, nr, rg = mp.map_loci(ctx, mi, mo, seqs, names, loci)
            times.append(time.perf_counter() - t0)
            assert rc == 0
            mp.free_loci_regs(nr, rg)
        res["loci_pairs_per_s"] = round(len(loci) / min(times[1:]), 1)
        res["loci_bp_mean"] = round(sum(en - st for _, _, st, en in loci) / max(1, len(loci)))
        if a.sets > 0:
            sets = [[(q, c, st, en)] + [(q,) + loci[(i + j) % len(loci)][1:] for j in range(1, a.sets)] for i, (q, c, st, en) in enumerate(loci)]
            pairs = [x for s in sets for x in s]
            ts, tp = [], []
            for _ in range(a.repeats + 1):
                t0 = time.perf_counter()
                rc, nr, rg = mp.map_locus_sets(ctx, mi, mo, seqs, names, sets)
                ts.append(time.perf_counter() - t0)
                assert rc == 0
                mp.free_loci_regs(nr, rg)
                t0 = time.perf_counter()
                rc, nr, rg = mp.map_loci(ctx, mi, mo, seqs, names, pairs)
                tp.append(time.perf_counter() - t0)
                assert rc == 0
                mp.free_loci_regs(nr, rg)
            res["set_size"], res["sets"] = a.sets, len(sets)
            res["locus_sets_per_s"] = round(len(sets) / min(ts[1:]), 1)
            res["same_loci_pairs_per_s"] = round(len(pairs) / min(tp[1:]), 1)
        if os.path.exists(REF_BIN) and a.ref_sample > 0:
            genome = dict(read_fasta(g))
            ctg_names = [nt.ctg[i].name for i in range(nt.n_ctg)]
            sample = loci[:a.ref_sample]
            t0 = time.perf_counter()
            for q, c, st, en in sample:
                gf, pf = os.path.join(d, "locus.fa"), os.path.join(d, "prot.fa")
                with open(gf, "wb") as f:
                    f.write(b">locus\n" + genome[ctg_names[c]][st:en] + b"\n")
                with open(pf, "wb") as f:
                    f.write(b">" + names[q] + b"\n" + seqs[q] + b"\n")
                subprocess.run([REF_BIN, gf, pf], check=True, capture_output=True)
            res["reference_extract_index_map_loci_per_s"] = round(len(sample) / (time.perf_counter() - t0), 2)
            res["reference_sample"] = len(sample)
        L.mp_idx_destroy(mi)
        ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
