"""Align proteins to genomic loci on the GPU: PAF on stdout, as the reference prints it for each locus, in genome coordinates.

    python tools/map_loci.py GENOME PROTEINS LOCI [-j2] [-K residues]

GENOME is a FASTA file or a .mpi index (only its genome section is read: the loci are seeded without a k-mer table), PROTEINS a
FASTA file, LOCI a TSV of `protein contig start end` (0-based, end exclusive, forward strand; both strands are searched).  Lines
come in the order of the loci."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import miniprot_b200 as mp  # noqa: E402


def read_fasta(path):
    import gzip

    out = []
    with (gzip.open(path, "rb") if path.endswith(".gz") else open(path, "rb")) as f:
        for line in f:
            if line.startswith(b">"):
                out.append([line[1:].split()[0], []])
            elif out:
                out[-1][1].append(line.strip())
    return [(n, b"".join(s)) for n, s in out]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("genome")
    ap.add_argument("proteins")
    ap.add_argument("loci")
    ap.add_argument("-j", type=int, default=None, help="splice model (as the reference's -j)")
    ap.add_argument("-K", type=int, default=None, help="residues per batch (as the reference's -K)")
    a = ap.parse_args()
    L = mp.lib()
    with open(a.genome, "rb") as f:
        is_mpi = f.read(3) == b"MPI"
    mi = L.mpb_idx_load_meta(a.genome.encode()) if is_mpi else mp.idx_load(a.genome, 4)
    if not mi:
        sys.exit(f"cannot read {a.genome}")
    prots = read_fasta(a.proteins)
    qid = {n: i for i, (n, _) in enumerate(prots)}
    nt = mi.contents.nt.contents
    cid = {nt.ctg[i].name: i for i in range(nt.n_ctg)}
    loci = []
    for ln, line in enumerate(open(a.loci, "rb"), 1):
        t = line.split()
        if not t or t[0].startswith(b"#"):
            continue
        if len(t) < 4 or t[0] not in qid or t[1] not in cid:
            sys.exit(f"{a.loci}:{ln}: expected `protein contig start end` with a known protein and contig")
        loci.append((qid[t[0]], cid[t[1]], int(t[2]), int(t[3])))
    mo = mp.mapopt()
    if a.j is not None:
        mo.sp_model = a.j
    if a.K is not None:
        mo.mini_batch_size = a.K
    ctx = mp.Context(0)
    names, seqs = [n for n, _ in prots], [s for _, s in prots]
    rc, n_reg, reg = mp.map_loci(ctx, mi, mo, seqs, names, loci)
    if rc != 0:
        sys.exit(f"mpb_map_loci failed ({rc})")
    sys.stdout.buffer.write(mp.loci_paf(mi, mo, seqs, names, loci, n_reg, reg))
    sys.stdout.flush()
    mp.free_loci_regs(n_reg, reg)
    L.mp_idx_destroy(mi)
    ctx.close()


if __name__ == "__main__":
    main()
