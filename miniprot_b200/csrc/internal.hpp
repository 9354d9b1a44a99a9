// internal.hpp -- declarations shared by the host side of libminiprot_b200 (not installed).
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <unordered_map>
#include <vector>
#include "miniprot_b200.h"
#include "flagsort.hpp"

namespace mpb {

// ---------------------------------------------------------------- sorting (flagsort.hpp)
void sort_u64(uint64_t *beg, uint64_t *end);      // plain ascending sort of full 64-bit keys (radix_sort_mp64)
void sort_128x(mp128_t *beg, mp128_t *end);       // by .x, reference tie order (radix_sort_mp128x)

// ---------------------------------------------------------------- genome store (ntdb.cpp)
mp_ntdb_t *ntdb_read_fasta(const char *fn);                                  // ntseq.c:29
void ntdb_destroy(mp_ntdb_t *db);
int32_t ntdb_read_spsc(mp_ntdb_t *nt, const char *fn, int32_t max_sc); // ntseq.c:234
void ntdb_dump(FILE *fp, const mp_ntdb_t *db);                               // ntseq.c:163
mp_ntdb_t *ntdb_restore(FILE *fp);                                           // ntseq.c:176
// bases [st,en) of contig cid as codes 0..4, reverse-complemented if rev (ntseq.c:89)
int64_t nt_fetch(const mp_ntdb_t *db, int32_t cid, int64_t st, int64_t en, int32_t rev, uint8_t *out);
// same in the coordinates of strand vid = cid<<1|rev (ntseq.c:108)
int64_t nt_fetch_v(const mp_ntdb_t *db, uint32_t vid, int64_t st, int64_t en, uint8_t *out);
static inline uint8_t nt_at_v(const mp_ntdb_t *db, uint32_t vid, int64_t pos) // one base in strand coordinates
{
	const mp_ctg_t *c = &db->ctg[vid >> 1];
	int64_t g = c->off + ((vid & 1) ? c->len - 1 - pos : pos);
	uint8_t b = db->seq[g >> 1] >> ((g & 1) * 4) & 0xf;
	return (vid & 1) ? (b >= 4 ? b : (uint8_t)(3 - b)) : b;
}

// ---------------------------------------------------------------- index (index.cpp)
extern void (*g_idx_destroy_hook)(const mp_idx_t *);                           // set by the CUDA backend
extern int (*g_idx_build_hook)(mp_idx_t *);                                    // device index builder; non-zero return = build on the host
int32_t idx_block2vid(const mp_idx_t *mi, uint32_t block);                  // index.c:41
mp_idx_t *idx_restore_head(FILE *fp);                                        // .mpi up to (not including) ki / kb
static inline uint32_t idx_n_bucket(const mp_idxopt_t *io) { return 1U << (io->kmer * 4 - io->mod_bit); }
uint32_t hash32_mask(uint32_t key, uint32_t mask);                           // sketch.c:7
// genome-side sketch of one strand (sketch.c:62); host code, used by the index builder only
void sketch_strand(const uint8_t *seq, int64_t len, int32_t min_aa_len, int32_t kmer, int32_t mod_bit, int32_t bbit,
                   int64_t boff, std::vector<uint64_t> &out);

// ---------------------------------------------------------------- stage interface
// The mapping of one mini-batch is a fixed sequence of host bookkeeping steps and three kinds of
// device stages.  The product implements the stages with CUDA kernels (cuda/backend.cu); the CPU
// test-suite plugs the C oracle in (tests/hostcheck) to check the host logic without a GPU.
struct Batch {
	int32_t n = 0;
	const char *const *seq = 0;
	const int32_t *len = 0;
	const char *const *name = 0;
};

struct ChainSet {                // result of one chaining stage over many problems
	std::vector<int64_t> u_off;  // [n+1] into u
	std::vector<int64_t> a_off;  // [n+1] into a
	std::vector<uint64_t> u;     // score<<32 | n_anchors, per chain (chain.c:160 *_u)
	std::vector<uint64_t> a;     // compacted anchors
	// --dbg-anchor (map.c:179-184): set by the caller of seed_chain to have the seeds of each query returned as well -- sorted,
	// max_occ-filtered, before any chaining -- in seed[seed_off[q], seed_off[q+1]).  Left empty otherwise.
	bool want_seeds = false;
	std::vector<int64_t> seed_off;
	std::vector<uint64_t> seed;
};

struct RefineJob {               // one second-round window (map.c:32-47)
	int32_t qid;
	uint32_t vid;
	int64_t as, ae;              // window on strand vid
};

struct RefineSet {
	std::vector<int64_t> off;    // [n+1] into a
	std::vector<uint64_t> a;     // best chain per job: (nt end pos in window)<<32 | aa end pos
	std::vector<int32_t> sc;     // its chain score; off[i+1]==off[i] means "no chain"
};

struct DpJob {                   // one ns_global_gs16b call (align.c:288/296/73/323/330)
	int32_t qid;
	uint32_t vid;
	int64_t nt_st;               // slice start on strand vid
	int32_t nl;
	int32_t aa_st, al;
	int32_t flag;                // NS_F_*
	int32_t io;
	int64_t win_st = -1;         // start of the region's window on strand vid: the --spsc byte of that one position reads "unset" (ntseq.c:130-156)
};

struct DpSet {
	std::vector<int32_t> score, nt_len, aa_len;
	std::vector<int64_t> cig_off; // [n+1]
	std::vector<uint32_t> cig;
};

struct Stages {
	virtual ~Stages() {}
	// map.c:155-195: sketch, lookup, sort, pre-chain, main chain -- per query; the seeds too when out.want_seeds is set
	virtual void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) = 0;
	// map.c:41-97 per window
	virtual void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) = 0;
	// nasw DP over genome slices
	virtual void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) = 0;
	// brackets of one map_batch() call (a backend may keep per-batch state resident between the stages); optional
	virtual void batch_begin(const Batch & /*b*/) {}
	virtual void batch_end() {}
	// wall-clock accounting of the dispatcher's phases (0 S1, 1 H1, 2 S2, 3 H2, 4 S3 waves, 5 H3); optional
	virtual void note_wall(int /*phase*/, double /*ms*/) {}
	// called on a host thread before it first calls the stages (the mapper threads of the file drivers): a device backend makes its
	// device current there and keeps the thread on the device's NUMA node; optional
	virtual void thread_init() {}
	// Locus mode (map_loci).  loci_view(mi, view): until loci_view(0, 0), the stages called with `view` -- an index whose contigs are
	// slices of mi's genome and that has no k-mer tables (LocusView) -- read mi's genome.  False: the backend has no locus mode.
	virtual bool loci_view(const mp_idx_t * /*mi*/, const mp_idx_t * /*view*/) { return false; }
	// S1 of locus mode: query q is seeded against contig q of `view` alone, as the reference seeds from an index of that locus
	// (index.c:52-136 over a one-record FASTA), then chained as in seed_chain
	virtual void seed_chain_loci(const mp_idx_t * /*view*/, const mp_mapopt_t * /*opt*/, const Batch & /*b*/, ChainSet & /*out*/) {}
	// Locus sets (map_sets).  True: seed_chain_locus_sets seeds a query against several contigs of `view` together.
	virtual bool locus_sets() { return false; }
	// S1 of a batch of locus sets: query q is seeded against contigs [ctg_off[q], ctg_off[q+1]) of `view` together, as the reference
	// seeds from an index of a genome made of those contigs alone, then chained as in seed_chain.  Called for queries of several
	// contigs only when locus_sets() is true; the default serves queries of one contig each (ctg_off[q] == q) with seed_chain_loci.
	virtual void seed_chain_locus_sets(const mp_idx_t *view, const int32_t * /*ctg_off*/, const mp_mapopt_t *opt, const Batch &b, ChainSet &out)
	{
		seed_chain_loci(view, opt, b, out);
	}
};

// ---------------------------------------------------------------- locus mode (pipeline.cpp)
// The index of one batch of loci: contig k is the range [st, en) of contig cid of rng[k], a view into mi's packed genome (nothing is
// copied), with block ids numbered over these contigs as index.c:11-26 numbers a genome's; ki / kb stay null.  Contig names are the
// real contigs'.  rng[k].qid is not read.
struct LocusView {
	mp_idx_t idx;
	mp_ntdb_t nt;
	std::vector<mp_ctg_t> ctg;
	std::vector<uint32_t> bo;
	LocusView(const mp_idx_t *mi, int32_t n, const mpb_locus_t *rng);
	LocusView(const LocusView &) = delete;
	LocusView &operator=(const LocusView &) = delete;
};
// -1 for a malformed locus (qid or cid out of range, st < 0, en > contig length, st >= en); -3 with a message for what locus mode
// refuses (--spsc scores, any mp_dbg_flag bit but MP_DBG_NO_KALLOC); else 0
int check_loci(const mp_idx_t *mi, int32_t n_seq, int32_t n_loci, const mpb_locus_t *loci);
// Locus sets in canonical form: set s is protein rng[off[s]].qid against the genome made of the ranges rng[off[s], off[s+1]) --
// sorted by (cid, st), ranges of one contig that overlap or abut merged into their union.  A pair of locus mode is a set of one range.
struct LocusSets {
	std::vector<int64_t> off{0};
	std::vector<mpb_locus_t> rng;
	int32_t n() const { return (int32_t)off.size() - 1; }
	int64_t n_rng(int32_t s) const { return off[(size_t)s + 1] - off[(size_t)s]; }
	void add(const mpb_locus_t *loci, int64_t n); // one set of n loci of one protein, any order
};
// The canonical sets of set s = loci[set_off[s], set_off[s+1]): -1 for a malformed locus, a null or decreasing set_off, an empty set
// or a set whose loci name different proteins; check_loci()'s -3 refusals; else 0 with `out` filled.
int locus_sets_make(const mp_idx_t *mi, int32_t n_seq, int32_t n_sets, const int64_t *set_off, const mpb_locus_t *loci, LocusSets &out);
// Sets [s_lo, s_hi) of ls on a backend, the protein of a set being seqs/lens/names[qid]: batches of whole sets, up to
// opt->mini_batch_size residues and fewer than 2^31 blocks, each through map_batch over the LocusView of its sets' ranges with the
// set seeding stage; n_reg_out / reg_out[s - s_lo] receive set s's regions in the coordinates of mi's contigs.  -3 (nothing mapped)
// for a backend without locus mode, or one without set seeding when a set has several ranges; else 0.
int map_sets(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *const *seqs, const int32_t *lens, const char *const *names, const LocusSets &ls,
             int32_t s_lo, int32_t s_hi, int32_t *n_reg_out, mp_reg1_t **reg_out);
// mpb_map_locus_sets on a backend: locus_sets_make()'s code, or map_sets over all the sets.
int map_locus_sets(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names,
                   int32_t n_sets, const int64_t *set_off, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out);
// mpb_map_loci on a backend: check_loci()'s code, or every pair mapped as a set of one locus (map_sets).
int map_loci(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names,
             int32_t n_loci, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out);
// The inputs of the locus file drivers, read whole: proteins (a repeated name stands for its last record), the pairs of the loci file
// in its order, and the sets the driver maps -- one per pair, or with `by_set` one per (protein, label) in the order of their first line.
struct LociFile {
	std::vector<std::string> names, seqs;
	std::vector<const char*> sp, np;
	std::vector<int32_t> len;
	std::vector<mpb_locus_t> loci;
	LocusSets sets;
	bool by_set = false;
	std::unordered_map<std::string, int32_t> qid;
	void add_protein(const std::string &name, const std::string &seq);
};
// Reads prot_fn (FASTA, gzip or plain) and loci_fn (`protein contig start end` per line, 0-based, end exclusive; blank and '#' lines
// skipped; further fields ignored, except that with by_set a 5th field is the line's set label: the lines of one protein and one label,
// or of one protein and no label, form one set).  -1 with "file:line: why" on stderr for an unreadable file, a malformed line, an
// unknown protein or contig, or a bad range; then check_loci()'s -3 refusals; else 0.
int loci_file_read(const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, LociFile &in, bool by_set = false);
// mpb_map_loci_file_multi / mpb_map_locus_sets_file_multi on n backends (the file driver's pipeline, with map_sets as the mapper): for
// every set of `in`, in order, the output of the reference given the set's ranges alone as the genome, in contig coordinates; ids
// numbered over the whole output.  Returns 0, -1 for n < 1, or -3 (nothing written) for a backend without locus mode or set seeding.
int32_t map_loci_file(Stages *const *st, int n, const mp_idx_t *mi, const LociFile &in, const mp_mapopt_t *opt, FILE *out);

// ---------------------------------------------------------------- host pipeline (pipeline.cpp, hits.cpp, align.cpp)
// The --dbg-* switches (mp_dbg_flag, MP_DBG_*) are read once per call.  Their dumps go to stderr, one contiguous block per batch:
// per protein a QR line (only when qr_tid >= 0; the reference prints it in worker_for, map.c:268, so mp_map prints none), its X
// lines and its Y1 lines.  qr_tid is the tid field of the QR lines: the index of the context that maps the batch.
void map_batch(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, int32_t *n_reg_out, mp_reg1_t **reg_out, int32_t qr_tid = -1);
// --dbg-no-refine without -A: the reference aligns regions that have no refined anchors and crashes (mp_align, r->a == NULL).
// True, with a message on stderr, when mp_dbg_flag and opt ask for that: the callers then map nothing and return -3.
bool bad_dbg_flags(const mp_mapopt_t *opt);
// The file drivers (map.c:273-343): map_file_multi and map_loci_file run one ordered pipeline over n distinct backends.  One reader
// thread cuts the input into units of max(1, mini_batch_size / n) residues, one mapper thread per backend (after its thread_init)
// maps the next unit, and the calling thread writes the units in input order, with one hit-id counter over the whole output.  At
// most 2n + 1 units are read but not yet written.  With one backend, an input of one unit or MPB_FILE_PIPELINE=0 runs everything on
// the calling thread.  No thread outlives the call.
// map_file_multi: a protein FASTA; the QR lines of --dbg-qname carry the index of the backend as tid.  -1 for n < 1 or an input
// that cannot be opened, -3 for bad_dbg_flags, else 0.  map_file is the same with one backend.
int32_t map_file_multi(Stages *const *st, int n, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out);
inline int32_t map_file(Stages *st, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out) { return map_file_multi(&st, 1, mi, fn, opt, out); }

struct Str {                      // growable output buffer
	char *s = 0; int64_t l = 0, m = 0;
	void reserve(int64_t extra);
	void put(const char *p, int64_t n);
	void puts(const char *p) { put(p, (int64_t)strlen(p)); }
	void putc(char c) { reserve(1); s[l++] = c; s[l] = 0; }
	void puti(int64_t v);
};
void format_hit(Str &out, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq,
                const mp_reg1_t *r);
// everything the reference prints for one hit (PAF, --aln / --trans blocks, GFF3 or GTF, format.c:453); id = running number of
// the hit in the whole output, hit_idx = its rank for this protein (1-based); r == 0: the unmapped line of -u.  nt_lim >= 0: the
// genome on strand r->vid ends there for this hit (the end of its locus in locus mode); the only read past r->ve is --aln's codon.
void format_output(Str &out, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq,
                   const mp_reg1_t *r, int64_t id, int32_t hit_idx, int64_t nt_lim = -1);

// hits.cpp (hit.c)
mp_reg1_t *regs_from_chains(const mp_idx_t *mi, int32_t n_u, const uint64_t *u, const uint64_t *a, int32_t *n_reg); // hit.c:32
void regs_sort(int32_t *n_regs, mp_reg1_t *r);                                                                      // hit.c:97
void regs_set_parent(float mask_level, int32_t mask_len, int32_t n, mp_reg1_t *r, int32_t sub_diff, int32_t hard);  // hit.c:128
void regs_select_sub(float pri_ratio, int32_t min_diff, int32_t best_n, int32_t *n_, mp_reg1_t *r);                 // hit.c:212
void regs_select_multi_exon(int32_t n, mp_reg1_t *r, int32_t single_penalty);                                       // hit.c:238
void regs_max_ext(const mp_ntdb_t *nt, int32_t n_reg, mp_reg1_t *reg, const uint64_t *a, int32_t min_ext, int32_t max_ext,
                  std::vector<uint64_t> &ext);                                                                       // hit.c:252
int32_t chain_score_ungapped(int32_t n_a, const uint64_t *a, int32_t kmer);                                         // hit.c:18

} // namespace mpb
