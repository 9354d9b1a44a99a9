// ctx.hpp -- the per-process, per-GPU context behind mpb_ctx_t (host side of the CUDA backend).
#pragma once
#include <mutex>
#include <vector>
#include "../internal.hpp"
#include "devbuf.hpp"
#include "nasw_dev.hpp"

struct mpb_ctx_s {
	int device = 0;
	// taken by every mpb_* entry point that uses the context: concurrent calls on one context take turns (the stream, the arenas
	// and the resident index are the context's alone).  Internal paths below an entry point never take it again.
	mutable std::mutex mu;
	cudaStream_t stream = 0;
	cudaEvent_t ev0 = 0, ev1 = 0;
	cudaEvent_t ev_bench[2] = {0, 0}; // mpb_event_begin / mpb_event_end_ms
	// side streams: size classes of one DP wave (and independent stage pieces) run concurrently; each class is bounded
	// by its longest problem, so serialising them on one stream would add the critical paths up
	static const int N_SIDE = 32; // 0..8 are high-priority streams (extension classes of a DP wave: their long problems must be dispatched first; 3, the widest class, highest), 9..17 normal
	cudaStream_t side[N_SIDE] = {0};
	cudaEvent_t ev_fork = 0, ev_fork2 = 0, ev_join[N_SIDE] = {0}, ev_k0[N_SIDE] = {0}, ev_k1[N_SIDE] = {0}, ev_km[N_SIDE] = {0};
	cudaEvent_t ev_w0 = 0, ev_w1 = 0, ev_p0 = 0; // timing of a DP wave on the main stream: before the prep kernel, at the fork, after the last join

	// resident read-only index (uploaded once, adopted from an NCCL broadcast, or shared by another context: mpb_idx_share)
	const mp_idx_t *mi = 0;
	mpb_ctx_s *idx_owner = 0; // the context whose ki / kb / seq buffers this one adopted (same device), else null
	uint8_t *d_seq = 0;       // 4-bit genome, (l_seq+1)/2 bytes
	int64_t *d_ki = 0;        // n_bucket + 1 entries (a sentinel n_kb is appended on upload)
	uint32_t *d_kb = 0;
	uint32_t *d_bo = 0;       // 2*n_ctg + 1
	int64_t *d_ctg = 0;       // per contig {off, len}
	bool own_index = false;
	mpb::cuda::DevBuf own_ki, own_kb, own_seq, own_bo, own_ctg;
	// --spsc splice scores as a dense table: one byte per base and strand, [strand * l_seq + offset of the base in the packed genome]
	// (0xff = no score), built from mi->nt->spsc when a DP wave first needs it
	uint8_t *d_ss = 0;
	const void *ss_src = 0;   // the mi->nt->spsc the table was built from
	int64_t ss_l_seq = 0;
	mpb::cuda::DevBuf own_ss;

	// nasw arenas
	mpb::cuda::DevBuf b_jobs, b_order, b_chunks, b_rw, b_aa, b_out, b_carry, b_tb, b_cigar, b_cigpack, b_cigoff, b_packed, b_units;
	mpb::cuda::PinBuf h_out, h_cigar;
	// chaining / seeding / refinement arenas
	mpb::cuda::DevBuf b_c[16];
	mpb::cuda::PinBuf h_c[4];
	// the working arenas above (every DevBuf except the resident index and the --spsc table) and their budget
	mpb::cuda::Ledger mem;

	mpb_stats_t stats;
	mpb::Stages *stages = 0;

	void time_begin() { cudaEventRecord(ev0, stream); }
	double time_end() { cudaEventRecord(ev1, stream); cudaEventSynchronize(ev1); float ms = 0; cudaEventElapsedTime(&ms, ev0, ev1); return ms; }
};

namespace mpb {
namespace cuda {

// One nasw wave over device-resident sequences.  `packed` is the nibble array the jobs' g_start refer to,
// `d_aa` the residue buffer their aa_off refer to.  jobs[].{g_start,dir,comp,nl,al,aa_off,flag,io} must be set.
int idx_build_device(mpb_ctx_s *c, mp_idx_t *mi); // idx_build.cu: ki / kb of mi from its packed genome, resident in c->own_ki / own_kb
void nasw_run(mpb_ctx_s *ctx, const uint8_t *packed, const uint8_t *d_ss, const char *d_aa, const ns_opt_t *base, std::vector<DpDev> &jobs, DpSet &out);

int nasw_check_ie_coef(float ie_coef); // 0 if the extension length penalty fits the kernels' step table

// chaining stage over many independent problems (chain_kernels.cu)
struct ChainPar { int32_t max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc; float chn_coef_log; int32_t is_spliced, kmer, bbit; };

} // namespace cuda
} // namespace mpb
