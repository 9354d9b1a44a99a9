// internal.hpp -- declarations shared by the host side of libminiprot_b200 (not installed).
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
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
	// map.c:155-195: sketch, lookup, sort, pre-chain, main chain -- per query
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
	// called on a host thread before it first calls the stages (the mapper threads of map_file_multi): a device backend makes its
	// device current there and keeps the thread on the device's NUMA node; optional
	virtual void thread_init() {}
};

// ---------------------------------------------------------------- host pipeline (pipeline.cpp, hits.cpp, align.cpp)
void map_batch(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, int32_t *n_reg_out, mp_reg1_t **reg_out);
int32_t map_file(Stages *st, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out);
// map_file over n backends at once (one mapper thread each); n == 1 is map_file.  The stages must be distinct.
int32_t map_file_multi(Stages *const *st, int n, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out);

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
// the hit in the whole output, hit_idx = its rank for this protein (1-based); r == 0: the unmapped line of -u
void format_output(Str &out, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq,
                   const mp_reg1_t *r, int64_t id, int32_t hit_idx);

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
