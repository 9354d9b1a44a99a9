// seed_dev.hpp -- descriptors and launcher prototypes of the seeding / window-join kernels (seed_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct mpb_ctx_s;

namespace mpb {
namespace cuda {

constexpr int SEED_THREADS = 128;
constexpr int WIN_TILE = 2048;                 // window positions per shared-memory tile
constexpr int WIN_SMEM_SPAN = WIN_TILE + 256;  // + halos of 3*(max(min_aa_len,kmer)+1) on the left, 3*min_aa_len on the right
constexpr int WIN_MAX_MIN_AA = 40;             // largest min_aa_len the halos cover
constexpr int WIN_MAX_KMER = 7;                // largest k-mer (index -k, refinement -l): 4 bits a residue in a 32-bit word
static_assert(WIN_MAX_KMER <= WIN_MAX_MIN_AA && 3 * (WIN_MAX_MIN_AA + 1) + 3 * WIN_MAX_MIN_AA <= WIN_SMEM_SPAN - WIN_TILE,
              "the tile halos must fit in the shared-memory span for every min_aa_len <= WIN_MAX_MIN_AA and kmer <= WIN_MAX_KMER");

struct SeedConst {          // passed by value (constant bank)
	uint8_t aa13[256];      // residue char -> 4-bit reduced alphabet (>= 14: stop / unknown)
	uint8_t codon[64];      // codon -> amino acid (20 = stop)
	uint8_t codon13[64];    // codon -> reduced alphabet
	int32_t kmer, mod_bit, max_occ;
	int64_t n_kb;
};

struct WinJob {             // one refinement window
	int64_t g_start;        // nibble index of window position 0
	int32_t dir, comp;
	int64_t len;
	int32_t qid, pad_;
	int64_t grp_off;        // per-job group counters live at grp[grp_off .. grp_off + n_pk[qid])
};

struct LocusStrand {        // one strand of a locus (locus seeding)
	int64_t g_start;        // nibble index of strand position 0
	int32_t dir, comp;
	int64_t len;
	uint32_t boff;          // its first block id
	int32_t qid;            // the protein it is joined with
};
struct LocusUnit { int32_t strand, pad_; int64_t pos_lo, pos_hi; }; // the tiles of one locus strand that one CTA scans

void seed_launch_sketch(cudaStream_t st, const char *aa, const int32_t *aa_off, int n_q, const SeedConst &cst, const int64_t *ki, uint32_t *sd_hash, int32_t *sd_pos,
                        int64_t *sd_cnt, int64_t *sd_aoff, int32_t *n_sd, int64_t *tot);
void seed_launch_expand(cudaStream_t st, const int32_t *aa_off, int n_q, const int64_t *ki, const uint32_t *kb, const uint32_t *sd_hash, const int32_t *sd_pos,
                        const int64_t *sd_cnt, const int64_t *sd_aoff, const int32_t *n_sd, const int64_t *a_off, uint64_t *a);
void seed_launch_prot_kmer(cudaStream_t st, const char *aa, const int32_t *aa_off, int n_q, const SeedConst &cst, int kmer, int mod_bit, uint64_t *keys, int32_t *n_out);
void locus_launch_join(cudaStream_t st, bool emit, const LocusUnit *units, int n_units, const LocusStrand *strands, const uint8_t *packed, const SeedConst &cst,
                       int min_aa_len, int bbit, const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, const int64_t *unit_off, int64_t *unit_n, uint64_t *out);
void locus_launch_unique(cudaStream_t st, const uint64_t *keys, const int64_t *seg, int n_q, uint64_t *uniq, uint32_t *blk, int64_t *n_u);
void locus_launch_occ(cudaStream_t st, const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, int n_q, const uint64_t *uniq, const int64_t *seg, const int64_t *n_u,
                      int32_t max_occ, uint32_t *sd_idx, int32_t *sd_pos, int64_t *sd_lo, int64_t *sd_cnt, int64_t *sd_aoff, int64_t *tot);
void win_launch_count(cudaStream_t st, const WinJob *jobs, int n_jobs, const uint8_t *packed, const SeedConst &cst, int kmer, int min_aa_len, int max_ava,
                      const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, int32_t *grp, int64_t *n_a);
void win_launch_emit(cudaStream_t st, const WinJob *jobs, int n_jobs, const uint8_t *packed, const SeedConst &cst, int kmer, int min_aa_len, const uint64_t *pk,
                     const int32_t *aa_off, const int32_t *n_pk, const int32_t *grp, const int64_t *a_off, uint64_t *a);

// segmented ascending sort of 64-bit keys (device-wide primitive; see seg_sort.cu)
// segmented ascending sort of 64-bit keys, in place (seg_sort.cu); the segment bounds are host arrays
void seg_sort_u64(mpb_ctx_s *ctx, cudaStream_t st, uint64_t *keys, uint64_t *tmp, int n_seg, const int64_t *h_begin, const int64_t *h_end);

} // namespace cuda
} // namespace mpb
