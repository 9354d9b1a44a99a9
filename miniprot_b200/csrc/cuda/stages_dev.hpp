// stages_dev.hpp -- host entry points of the seeding/chaining and refinement stages (seed_chain.cu, refine.cu).
#pragma once
#include "ctx.hpp"
#include "chain_core.cuh"

namespace mpb {
namespace cuda {

// S1 (map.c:155-195): per protein sketch -> index lookup -> anchor sort -> pre-chain -> main chain
void seed_chain_run(mpb_ctx_s *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa,
                    ChainSet &out);
// S2 (map.c:41-97): per window 5-mer join with the protein + base-level chain, best chain kept
void refine_run(mpb_ctx_s *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa,
                const std::vector<RefineJob> &jobs, RefineSet &out);

// S1 of locus mode (map_sets): query q seeded against contigs [ctg_off[q], ctg_off[q+1]) of the locus view vi together -- its set's
// ranges; one contig per query for a pair -- without a k-mer table; then the same chains
void seed_chain_loci_run(mpb_ctx_s *ctx, const mp_idx_t *vi, const int32_t *ctg_off, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off,
                         const char *d_aa, ChainSet &out);
void seed_loci_batch_run(mpb_ctx_s *ctx, const mp_idx_t *vi, const int32_t *ctg_off, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off,
                         const char *d_aa, std::vector<int64_t> &a_off, std::vector<uint64_t> &a);

void seed_batch_run(mpb_ctx_s *ctx, const mp_idx_t *mi, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa,
                    std::vector<int64_t> &a_off, std::vector<uint64_t> &a);
void chain_batch_run(mpb_ctx_s *ctx, const chn::Par &par, int n_prob, const int64_t *a_off, const uint64_t *a, std::vector<int32_t> &n_u, std::vector<int32_t> &n_b,
                     std::vector<uint64_t> &u, std::vector<uint64_t> &bb);

} // namespace cuda
} // namespace mpb
