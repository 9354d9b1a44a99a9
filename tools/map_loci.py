"""Align proteins to genomic loci on the GPU: for every locus, what the reference CLI prints with the same options when that locus
alone is the genome, moved to the coordinates of the real contig.

    python tools/map_loci.py [options] GENOME PROTEINS LOCI > out.paf
    python tools/map_loci.py --gff [options] GENOME PROTEINS LOCI > out.gff

GENOME is a FASTA file (gzip allowed) or a .mpi index; either way only its genome is read: the loci are seeded without a k-mer
table, and the index options -k -M -L -b -T apply to a FASTA only (a .mpi file carries its own).  PROTEINS is a FASTA file, LOCI a
TSV of `protein contig start end` (0-based, end exclusive, forward strand; both strands are searched).  Output comes in the order
of the loci: PAF (columns 6-9 on the contig), or GFF3 / GTF (columns 1, 4 and 5 on the contig) with ids numbered over the whole
file.  The options are the reference CLI's that mean something for one locus; -I (a max intron per locus) and --spsc are refused.
--devices 0,1 aligns on one GPU context per entry (repeats allowed); the output is the same.

--sets aligns each protein against all of its loci at once, as the reference aligns it against a genome made of those loci alone:
hits across the loci are ranked together (one primary, the rest secondary; -N, -p, --outn, --outs and -u per set), and overlapping
or abutting loci of one contig are merged.  An optional 5th column of LOCI labels the line's set: the lines of one protein and one
label form one set, and without a label all lines of a protein do.  Sets come out in the order of their first line."""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import miniprot_b200 as mp  # noqa: E402


def parse_num(s: str) -> int:
    """A count with an optional K / M / G suffix (decimal), rounded, as the CLI reads -K, -G, -c and the like."""
    for suffix, mult in (("k", 1e3), ("m", 1e6), ("g", 1e9)):
        if s.lower().endswith(suffix):
            return int(float(s[:-1]) * mult + .499)
    return int(float(s) + .499)


def _set(field, conv=int):
    return lambda io, mo, L, v: setattr(mo, field, conv(v))


def _flag(bits):
    def f(io, mo, L, v):
        mo.flag |= bits
    return f


def _no_splice(io, mo, L, v):  # -S: no introns; max intron, band and extension 1000, intron open 10000
    mo.flag |= mp.MP_F_NO_SPLICE
    mo.bw = mo.max_intron = mo.max_ext = 1000
    mo.io = mo.io_end = 10000


def _max_intron(io, mo, L, v):
    mo.bw = mo.max_intron = parse_num(v)


def _idx(field):
    return lambda io, mo, L, v: setattr(io, field, int(v))


# option -> (takes a value, how it is applied, help); applied in command-line order, as the CLI does
F_GFF, F_NO_PAF, F_GTF, F_SHOW_RESIDUE, F_SHOW_TRANS = 0x8, 0x10, 0x20, 0x80, 0x100
OPTIONS = {
    # indexing (FASTA genomes)
    "-k": (True, _idx("kmer"), "k-mer size"),
    "-M": (True, _idx("mod_bit"), "modimisers bit (sample rate 1/2**M)"),
    "-L": (True, _idx("min_aa_len"), "min ORF length to index"),
    "-b": (True, _idx("bbit"), "bits per block"),
    "-T": (True, _idx("trans_code"), "NCBI translation table"),
    # mapping
    "-S": (False, _no_splice, "no splicing (max intron, band and extension 1000, intron open 10000)"),
    "-c": (True, _set("max_occ", parse_num), "max k-mer occurrence"),
    "-G": (True, _max_intron, "max intron size"),
    "-w": (True, _set("chn_coef_log", float), "weight of the log gap penalty"),
    "-n": (True, _set("min_chn_cnt", parse_num), "min number of syncmers in a chain"),
    "-m": (True, _set("min_chn_sc", parse_num), "min chaining score"),
    "-l": (True, _set("kmer2"), "k-mer size of the second round of chaining"),
    "-e": (True, _set("max_ext", parse_num), "max extension of the second round and the alignment"),
    "-p": (True, _set("pri_ratio", float), "min secondary-to-primary score ratio"),
    "-N": (True, _set("best_n", parse_num), "consider at most this many secondary alignments"),
    "-g": (True, _set("max_gap", parse_num), "max gap in a chain"),
    "--max-skip": (True, _set("max_chn_max_skip", parse_num), "max skipped anchors in chaining"),
    "--no-pre-chain": (False, _flag(mp.MP_F_NO_PRE_CHAIN), "no pre-chaining"),
    # alignment
    "-O": (True, _set("go"), "gap open penalty"),
    "-E": (True, _set("ge"), "gap extension penalty"),
    "-J": (True, _set("io"), "intron open penalty"),
    "--J2": (True, _set("io_end"), "intron open penalty near the ends"),
    "-F": (True, lambda io, mo, L, v: L.mp_mapopt_set_fs(C.byref(mo), int(v)), "frameshift / in-frame stop penalty"),
    "-C": (True, _set("sp_scale", float), "weight of the splice penalty"),
    "-B": (True, _set("end_bonus"), "bonus for reaching the query ends"),
    "-j": (True, _set("sp_model"), "splice model: 2 vertebrate/insect, 1 general, 0 none"),
    "--xdrop": (True, _set("xdrop"), "x-drop of the extension"),
    "--ie-coef": (True, _set("ie_coef", float), "coefficient of the extension length penalty"),
    # output
    "--gff": (False, _flag(F_GFF), "GFF3"),
    "--gff-only": (False, _flag(F_GFF | F_NO_PAF), "GFF3 without the ##PAF lines"),
    "--gtf": (False, _flag(F_GTF), "basic GTF"),
    "--aln": (False, _flag(F_SHOW_RESIDUE), "residue alignment"),
    "--trans": (False, _flag(F_SHOW_TRANS), "translated protein sequences"),
    "-P": (True, lambda io, mo, L, v: setattr(mo, "gff_prefix", v.encode()), "prefix of the GFF3 / GTF ids"),
    "-u": (False, _flag(mp.MP_F_SHOW_UNMAP), "print pairs without a hit"),
    "--outn": (True, _set("out_n", parse_num), "print up to this many hits per pair"),
    "--outs": (True, _set("out_sim", float), "print hits scoring at least this times the best"),
    "--outc": (True, _set("out_cov", float), "print hits covering at least this fraction of the protein"),
    "--gff-delim": (True, lambda io, mo, L, v: setattr(mo, "gff_delim", ord(v[0])), "ids as protein name, this character, rank"),
    "--max-intron-out": (True, lambda io, mo, L, v: setattr(mo, "max_intron_flank", (parse_num(v) + 1) // 2), "abbreviate longer introns in --aln"),
    "--no-cs": (False, _flag(mp.MP_F_NO_CS), "no cs tag"),
    "-K": (True, _set("mini_batch_size", parse_num), "residues per batch"),
}
REFUSED = {"-I": "-I would give every locus a max intron of its own; set one with -G",
           "--spsc": "locus mode does not take --spsc splice scores"}


class _Apply(argparse.Action):
    def __call__(self, parser, ns, value, option_string=None):
        if option_string in REFUSED:
            parser.error(f"{option_string}: {REFUSED[option_string]}")
        ns.apply.append((option_string, value))


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0], allow_abbrev=False)
    ap.add_argument("genome")
    ap.add_argument("proteins")
    ap.add_argument("loci")
    ap.set_defaults(apply=[])
    for opt, (has_value, _, hlp) in OPTIONS.items():
        ap.add_argument(opt, action=_Apply, nargs=None if has_value else 0, help=hlp, metavar="V" if has_value else None)
    ap.add_argument("-I", action=_Apply, nargs=0, help="refused: " + REFUSED["-I"])
    ap.add_argument("--spsc", action=_Apply, help="refused: " + REFUSED["--spsc"], metavar="FILE")
    ap.add_argument("--devices", default="0", help="GPU contexts to align on, one per entry (repeats allowed) [0]")
    ap.add_argument("--sets", action="store_true", help="align each (protein, 5th-column label) set of loci together, ranked as one genome")
    return ap


def options(argv, L=None):
    """(parsed arguments, index options, mapping options) of a command line; L: the library whose mp_*opt_init / mp_mapopt_set_fs
    to use (the product's by default)."""
    L = L or mp.lib()
    a = parser().parse_args(argv)
    io, mo = mp.IdxOpt(), mp.MapOpt()
    L.mp_idxopt_init(C.byref(io))
    L.mp_mapopt_init(C.byref(mo))
    for opt, v in a.apply:
        OPTIONS[opt][1](io, mo, L, v)
    return a, io, mo


def main(argv=None):
    a, io, mo = options(sys.argv[1:] if argv is None else argv)
    L = mp.lib()
    if L.mp_mapopt_check(C.byref(mo)) < 0:
        sys.exit(1)
    if L.ns_make_tables(io.trans_code) < 0:
        sys.exit(f"no translation table {io.trans_code}")
    try:
        devices = [int(d) for d in a.devices.split(",")]
    except ValueError:
        sys.exit(f"--devices {a.devices}: expected a comma-separated list of device numbers")
    mi = mp.idx_load_genome(a.genome, io)
    ctxs = [mp.Context(d) for d in devices]
    try:
        mp.map_loci_file(ctxs, mi, a.proteins, a.loci, "-", mo, sets=a.sets)
    except RuntimeError as e:
        sys.exit(str(e))
    finally:
        L.mp_idx_destroy(mi)
        for c in ctxs:
            c.close()


if __name__ == "__main__":
    main()
