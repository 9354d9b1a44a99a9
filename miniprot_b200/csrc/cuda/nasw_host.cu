// nasw_host.cu -- host side of the nasw stage: lays a wave of DP problems out in HBM, launches the kernels
// of nasw_kernels.cu size class by size class, and brings (score, nt_len, aa_len, CIGAR) back.
//
// HBM layout of one wave (all grow-only arenas of the context):
//   jobs[]    DpDev descriptors                              order[]  job ids grouped by (kind, C), longest first
//   rw[]      32-byte row records (triple-major for the      carry[]  one int4 per row for problems wider than a pass
//             block-wide kernels, nasw_core.cuh v3_triples)
//   tb[]      16-bit traceback words, wavefront-major        cigar[]  per-problem CIGAR slots (filled from the end)
//   out[]     int4 {score, nt_len, aa_len, n_cigar}
// A wave whose traceback or row-word footprint exceeds the budget is cut into sub-waves.
#include <algorithm>
#include <numeric>
#include "ctx.hpp"
#include "nasw_core.cuh"
#include "nasw_pair.cuh"

namespace mpb {
namespace cuda {

// A sub-wave's two big arenas stay within a fifth of the H100's 80 GB, next to the resident index (about 8 GB at 3 Gbp) and the
// other stages' arenas; a C2 wave needs a tenth of that.
static const size_t kTbBudget = (size_t)12 << 30;   // bytes of traceback words per sub-wave
static const size_t kRwBudget = (size_t)4 << 30;    // bytes of row records per sub-wave

static inline int pick_C(int al)
{
	const int W8 = (al + 7) / 8 * 8;
	return W8 <= 32 ? 1 : W8 <= 64 ? 2 : W8 <= 128 ? 4 : 8;
}

// Kernel family: the block-wide wavefront (one thread per column, nasw_v3_kernel) serves every problem; those wider than 256
// padded columns run in column passes inside the same kernel.  MPB_NASW_KERNEL=cols forces the warp-per-problem column-pass
// family for everything (A/B measurements and tests only).
// Per nucleotide row the block-wide kernel is the faster one, and a mini-batch is latency bound -- its waves last as long as
// their longest problem (100 k-row extensions).
// The A/B switches of the dispatcher are read from the environment at every nasw_run into a value of its own (tests switch the
// family between calls), never into a global: DP waves of several contexts run concurrently on different host threads.
struct Switches {
	int forced_family = 0; // MPB_NASW_KERNEL=cols|v3|pair (A/B switch for tests and measurements): 1, 2, 3
	int pass_warps = 8;
	int wide_warps = 4;    // passes of a problem wider than 256 columns: 128 columns each (MPB_NASW_WIDE_WARPS=8: 256)
	bool split_long = false; // MPB_NASW_SPLIT=1: long extensions of 129..256 columns as two 4-warp column passes (measured slower, see below)
	static Switches from_env()
	{
		Switches s;
		const char *e = getenv("MPB_NASW_KERNEL"), *pw = getenv("MPB_NASW_PASS_WARPS"), *ww = getenv("MPB_NASW_WIDE_WARPS"), *sp = getenv("MPB_NASW_SPLIT");
		s.pass_warps = pw && atoi(pw) == 2 ? 2 : 8;
		s.wide_warps = ww && atoi(ww) == 8 ? 8 : 4;
		s.split_long = sp && atoi(sp) != 0;
		s.forced_family = !e ? 0 : strcmp(e, "cols") == 0 ? 1 : strcmp(e, "v3") == 0 ? 2 : strcmp(e, "pair") == 0 ? 3 : 0;
		return s;
	}
};
static inline bool use_v3(const Switches &sw)
{
	return sw.forced_family != 1; // default: latency first (a wave is bounded by its longest problems); wide problems run in passes
}
// Warps per CTA of the block-wide kernels.  A problem wider than one CTA (256 columns) runs as column PASSES, one CTA per pass,
// all passes of a problem concurrently (pass q a few dozen rows behind pass q - 1, linked by a per-row carry array and a progress
// counter), so a 350-column extension over a 100 k-row window costs the rows of one pass, not of two.  MPB_NASW_PASS_WARPS=2
// cuts every problem wider than 64 columns into 64-column passes instead: per row a two-warp CTA is the faster one, but the
// publishing fence, the carry traffic and above all the start-up lag of each further pass (short global alignments!) cost more
// than that gains over a whole C2 step, so CTAs of up to 8 warps stay the default.
constexpr int NCLS_ = 13;
static inline int v3_warps(const Switches &sw, int al)
{
	const int nw = ((al + 7) / 8 * 8 + 31) / 32;
	const int r = nw <= 1 ? 1 : nw <= 2 ? 2 : nw <= 4 ? 4 : 8;
	// wider than one CTA anyway: passes of 128 columns (four warps meet at the barrier of a macro-step instead of eight, which on
	// 350 columns x 100 k rows beats two 8-warp passes)
	if (nw > 8 && sw.wide_warps < 8) return sw.wide_warps;
	return r < sw.pass_warps ? r : sw.pass_warps;
}

// Pair-lane kernels (nasw_pair.cuh: two columns per thread as packed int16x2) serve every problem whose scores provably stay
// inside their value domain and whose padded width fits 8 warps; MPB_NASW_KERNEL=v3|cols keeps them out (A/B measurements).
static nsw::PairLimits pair_limits(const ns_opt_t *o) { return nsw::pair_limits(o->sc, o->sp); }
// Which problems they serve by default is a measured choice (tools/dp_bench.py and bench.py A/B): global alignments of up to 64
// padded columns, where one warp of the pair-lane kernel replaces one or two warps of the block-wide kernel and is faster.
// Score-only extensions stay on the block-wide kernels: there the pair-lane form needs more cycles per row -- its 64 columns per
// warp do not pay for the 32-bit row-maximum bookkeeping that an extension carries per cell.  MPB_NASW_KERNEL=pair sends every
// problem of up to 64 columns to them (tests, A/B).
static inline bool use_pair(const Switches &sw, const DpDev &j, const ns_opt_t *o, const nsw::PairLimits &l)
{
	if (sw.forced_family == 1 || sw.forced_family == 2) return false;
	const int W8 = (j.al + 7) / 8 * 8;
	if (W8 > nsw::PAIR_MAX_W8 || j.nl < 3) return false;
	if (j.ss_off >= 0) return false; // --spsc makes donor / acceptor entries negative: outside the value-domain argument of the pair-lane kernels
	if (sw.forced_family != 3) {
		const bool is_tb = !(j.flag & (NS_F_EXT_LEFT | NS_F_EXT_RIGHT));
		if (!is_tb) return false;
	}
	return nsw::pair_eligible(j.al, o->go, o->ge, j.io, o->fs, o->end_bonus, l.smin, l.smax, l.dmax, l.amax);
}

static void fill_const(const ns_opt_t *o, NaswConst &c)
{
	memcpy(c.mat, o->sc, 484);
	memcpy(c.aa20, ns_tab_aa20, 256);
	memcpy(c.codon, ns_tab_codon, 64);
	for (int i = 0; i < 6; ++i) c.sp[i] = o->sp[i];
	c.go = o->go, c.ge = o->ge, c.fs = o->fs, c.xdrop = o->xdrop, c.end_bonus = o->end_bonus, c.ie_coef = o->ie_coef;
	c.aa_x = ns_tab_aa20[(uint8_t)'X'];
	c.sp_null_bonus = o->sp_null_bonus;
	nsw::pen_table_build(o->ie_coef, c.pen);
}

// The extension length penalty reaches the kernels as a step table (nasw_core.cuh PenTable).  A coefficient so large that the
// table cannot hold all its steps below 2^31 is refused up front (0 = fine).
int nasw_check_ie_coef(float ie_coef)
{
	nsw::PenTable t;
	nsw::pen_table_build(ie_coef, t);
	if (t.n < nsw::PEN_STEPS) return 0;
	return nsw::ext_len_penalty(ie_coef, 2147483646) == t.val[t.n - 1] ? 0 : -1;
}

// run jobs[lo, hi) as one sub-wave
static void run_subwave(mpb_ctx_s *ctx, const Switches &sw, const uint8_t *packed, const uint8_t *d_ss, const char *d_aa, const NaswConst &cst, const ns_opt_t *nso,
                        std::vector<DpDev> &jobs, size_t lo, size_t hi, DpSet &out)
{
	const int n = (int)(hi - lo);
	if (n == 0) return;
	cudaStream_t st = ctx->stream;
	const double t_in = mp_realtime();
	int64_t rw_tot = 0, tb_tot = 0, cig_tot = 0, carry_tot = 0;
	std::vector<PrepChunk> chunks, pchunks; // row-record chunks of the 32-bit families, pair-record chunks of the pair-lane family
	bool wide3[2][NCLS_] = { { false } }; // does a block-wide class hold problems of more than one pass?
	std::vector<int> unsupported;
	const nsw::PairLimits plim = pair_limits(nso);
	constexpr int NCLS = NCLS_;
	std::vector<int> order[2][NCLS]; // [is_tb][class]: 0..3 block-wide wavefront with 1/2/4/8 warps; 4..7 column passes C = 1/2/4/8; 8 multi-pass; 9 pair-lane kernels (one warp per problem)
	for (int k = 0; k < n; ++k) {
		DpDev &j = jobs[lo + k];
		const bool is_tb = !(j.flag & (NS_F_EXT_LEFT | NS_F_EXT_RIGHT));
		if (!is_tb && j.al > nsw::CODE_MAX_AL) { // the row maximum carries its column in at most 15 bits (nasw_core.cuh code_bits): the problem is not
			// run and reports nt_len = -1, which the caller treats as "this alignment failed" (the region is dropped with a warning)
			unsupported.push_back(k);
			j.C = 0, j.pad_ = 32, j.rw_off = 0, j.tb_off = j.cig_off = 0, j.cig_cap = 0, j.carry_off = 0;
			continue;
		}
		if (use_pair(sw, j, nso, plim)) { // pair-lane kernels: pair records (96 B per triple of rows), wavefront-major traceback of 64 columns per warp
			const int W8 = (j.al + 7) / 8 * 8, K = nsw::pair_rec_slots(j.nl), n_macro = nsw::pair_n_macro(j.nl, W8);
			j.C = 0, j.pad_ = 64;
			j.rw_off = rw_tot, rw_tot += (int64_t)192 * nsw::pair_rec_blocks(j.nl); // two parities x blocks x 192 sixteen-byte fields, in units of 32 bytes
			j.tb_off = j.cig_off = 0, j.cig_cap = 0, j.carry_off = 0;
			if (is_tb) {
				j.tb_off = tb_tot, tb_tot += (int64_t)3 * (n_macro + 2) * j.pad_;
				j.cig_cap = j.nl + j.al + 4;
				j.cig_off = cig_tot, cig_tot += j.cig_cap;
			}
			const int n_tri = 2 * K; // record indices 0 .. 2K-1 (the tail past the last real triple is never read unmasked)
			for (int m = 0; m < n_tri; m += 1024) pchunks.push_back(PrepChunk{ k, m, std::min(1024, n_tri - m), 0 });
			order[is_tb][9].push_back(k);
			(is_tb ? ctx->stats.dp_cells_tb : ctx->stats.dp_cells_ext) += (int64_t)j.nl * j.al;
			(is_tb ? ctx->stats.n_dp_tb : ctx->stats.n_dp_ext) += 1;
			continue;
		}
		const bool v3 = use_v3(sw);
		int nw = v3_warps(sw, j.al);
		// A long extension of 129..256 columns is a pole of its wave on one 8-warp CTA (eight warps at one barrier).  Two concurrent
		// column passes of four warps (fewer cycles per row each, linked by the carry row; class 10) looked like the way out and are NOT:
		// on C2 the pass pipeline costs about twice the rows of a lone CTA, as it does for the 350-column problems that need it.  Opt-in only.
		const bool split = sw.split_long && v3 && !is_tb && nw == 8 && j.nl >= 32768 && (j.al + 7) / 8 * 8 <= 256 && (j.al + 7) / 8 * 8 > 128;
		if (split) nw = 4;
		j.C = v3 ? 0 : pick_C(j.al);
		j.pad_ = v3 ? 32 * nw : 0;
		const int Wp = v3 ? 32 * nw : 32 * j.C, W8 = (j.al + 7) / 8 * 8, n_pass = (W8 + Wp - 1) / Wp;
		const int T = v3 ? (j.nl > 2 ? 3 * ((j.nl - 2 + 2) / 3 + Wp + 2) : 0) : (j.nl > 2 ? j.nl - 2 + 32 + 6 : 0); // rows of the wavefront-major traceback buffer
		// row records: 32 B per row; block-wide problems store them per triple of rows, field-major (nasw_core.cuh v3_triples)
		const int rec_rows = v3 ? 2 + 3 * nsw::v3_triples(j.nl) : j.nl + 1;
		j.rw_off = rw_tot, rw_tot += (rec_rows + 3) / 4 * 4;
		j.tb_off = j.cig_off = 0, j.cig_cap = 0, j.carry_off = 0;
		(void)0;
		if (is_tb) {
			j.tb_off = tb_tot, tb_tot += (int64_t)n_pass * T * Wp;
			j.cig_cap = j.nl + j.al + 4;
			j.cig_off = cig_tot, cig_tot += j.cig_cap;
		}
		if (n_pass > 1) j.carry_off = carry_tot, carry_tot += ((int64_t)j.nl + 3 * Wp + 64) * 4; // four ints per row; slack: the feeder of a later pass reads ahead of the rows it needs, past the last row during the ramp-down
		for (int r = 0; r < rec_rows; r += PREP_ROWS) chunks.push_back(PrepChunk{ k, r, std::min(PREP_ROWS, rec_rows - r), 0 });
		const int cls = split ? 10 : v3 ? (nw == 1 ? 0 : nw == 2 ? 1 : nw == 4 ? 2 : 3) : n_pass > 1 ? 8 : j.C == 1 ? 4 : j.C == 2 ? 5 : j.C == 4 ? 6 : 7;
		if (v3 && n_pass > 1) wide3[is_tb][cls] = true;
		order[is_tb][cls].push_back(k);
		(is_tb ? ctx->stats.dp_cells_tb : ctx->stats.dp_cells_ext) += (int64_t)j.nl * j.al;
		(is_tb ? ctx->stats.n_dp_tb : ctx->stats.n_dp_ext) += 1;
	}
	std::vector<int> flat;
	size_t first[2][NCLS], count[2][NCLS];
	for (int b = 0; b < 2; ++b)
		for (int c = 0; c < NCLS; ++c) {
			std::vector<int> &v = order[b][c];
			std::stable_sort(v.begin(), v.end(), [&](int x, int y) { return jobs[lo + x].nl > jobs[lo + y].nl; });
			first[b][c] = flat.size(), count[b][c] = v.size();
			flat.insert(flat.end(), v.begin(), v.end());
		}
	// units of the multi-pass launches: (slot in the class's order list, pass), passes of a problem consecutive
	std::vector<int2> units;
	int unit_first[2][NCLS] = { { 0 } }, unit_count[2][NCLS] = { { 0 } }, n_units_tot = 0;
	for (int b = 0; b < 2; ++b)
		for (int c = 0; c < NCLS; ++c) {
			unit_first[b][c] = (int)units.size();
			if (wide3[b][c])
				for (size_t s = 0; s < count[b][c]; ++s) {
					const DpDev &jj = jobs[lo + flat[first[b][c] + s]];
					const int Wp = jj.pad_, np = ((jj.al + 7) / 8 * 8 + Wp - 1) / Wp;
					for (int q = 0; q < np; ++q) units.push_back(make_int2((int)s, q));
				}
			unit_count[b][c] = (int)units.size() - unit_first[b][c];
		}
	n_units_tot = (int)units.size();
	if (n_units_tot) {
		ctx->b_units.reserve((sizeof(int2) + sizeof(int)) * (size_t)n_units_tot + 64);
		MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_units.p, units.data(), sizeof(int2) * units.size(), cudaMemcpyHostToDevice, st));
		MPB_CUDA_OK(cudaMemsetAsync(ctx->b_units.as<int2>() + n_units_tot, 0, sizeof(int) * (size_t)n_units_tot, st));
	}
	ctx->b_jobs.reserve(sizeof(DpDev) * n);
	ctx->b_order.reserve(sizeof(int) * (flat.size() + 1));
	ctx->b_chunks.reserve(sizeof(PrepChunk) * (chunks.size() + pchunks.size() + 1));
	ctx->b_rw.reserve(32 * (size_t)(rw_tot + 4));
	ctx->b_out.reserve(sizeof(int4) * n);
	ctx->b_carry.reserve(sizeof(int) * (size_t)(carry_tot + 4));
	ctx->b_tb.reserve(sizeof(uint16_t) * (size_t)(tb_tot + 8));
	ctx->b_cigar.reserve(sizeof(uint32_t) * (size_t)(cig_tot + 4));
	ctx->h_out.reserve(sizeof(int4) * n);
	ctx->h_cigar.reserve(sizeof(uint32_t) * (size_t)(cig_tot + 4));
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_jobs.p, jobs.data() + lo, sizeof(DpDev) * n, cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_order.p, flat.data(), sizeof(int) * flat.size(), cudaMemcpyHostToDevice, st));
	if (!chunks.empty()) MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_chunks.p, chunks.data(), sizeof(PrepChunk) * chunks.size(), cudaMemcpyHostToDevice, st));
	if (!pchunks.empty())
		MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_chunks.as<PrepChunk>() + chunks.size(), pchunks.data(), sizeof(PrepChunk) * pchunks.size(), cudaMemcpyHostToDevice, st));
	ctx->stats.h2d_bytes += sizeof(DpDev) * n + sizeof(int) * flat.size() + sizeof(PrepChunk) * (chunks.size() + pchunks.size());
	const DpDev *dj = ctx->b_jobs.as<DpDev>();
	const int *dord = ctx->b_order.as<int>();
	MPB_CUDA_OK(cudaEventRecord(ctx->ev_p0, st));
	nasw_launch_prep(st, dj, ctx->b_chunks.as<PrepChunk>(), (int)chunks.size(), packed, d_ss, cst, ctx->b_rw.as<int4>());
	nasw_launch_prep_pair(st, dj, ctx->b_chunks.as<PrepChunk>() + chunks.size(), (int)pchunks.size(), packed, d_ss, cst, ctx->b_rw.as<int4>());
	ctx->stats.kernel_launches += (chunks.empty() ? 0 : 1) + (pchunks.empty() ? 0 : 1);
	static const int Cs[NCLS] = { 1, 2, 4, 8, 1, 2, 4, 8, 16, 1, 2, 4, 8 }; // warps per problem (classes 0..3, 9..12) or columns per lane (4..8)
	// Scheduling of a big wave.  It is bounded by its longest extensions (100 k rows next to thousands of short problems):
	//  * the extension classes run on high-priority streams and are ordered longest first, so those problems start at once.
	// MPB_NASW_WSM=<warps per SM> caps the residency of the block-wide launches (measurements only).
	static const int wsm_env = getenv("MPB_NASW_WSM") ? atoi(getenv("MPB_NASW_WSM")) : -1;
	// fork: every (kind, size class) runs on its own stream -- each is bounded by its longest problem
	struct Group { int sid, b, c; size_t first, count; };
	std::vector<Group> groups;
	for (int b = 0; b < 2; ++b)
		for (int c = NCLS - 1; c >= 0; --c)
			if (count[b][c]) groups.push_back(Group{ b * NCLS + c, b, c, first[b][c], count[b][c] });
	MPB_CUDA_OK(cudaEventRecord(ctx->ev_w0, st));
	MPB_CUDA_OK(cudaEventRecord(ctx->ev_fork, st));
	for (const Group &g : groups) {
		cudaStream_t ss = ctx->side[g.sid];
		const int b = g.b, c = g.c, cnt = (int)g.count;
		const int *ord = dord + g.first;
		MPB_CUDA_OK(cudaStreamWaitEvent(ss, ctx->ev_fork, 0));
		MPB_CUDA_OK(cudaEventRecord(ctx->ev_k0[g.sid], ss));
		if (c == 9) {
			nasw_launch_pair(ss, b == 1, dj, ord, cnt, ctx->b_rw.as<int4>(), d_aa, cst, ctx->b_out.as<int4>(), ctx->b_tb.as<uint16_t>());
			ctx->stats.kernel_launches += 1;
			MPB_CUDA_OK(cudaEventRecord(ctx->ev_km[g.sid], ss));
			if (b == 1) {
				nasw_launch_bt(ss, dj, ord, cnt, ctx->b_tb.as<uint16_t>(), ctx->b_cigar.as<uint32_t>(), ctx->b_out.as<int4>());
				ctx->stats.kernel_launches += 1;
			}
		} else if (c < 4 || c == 10) {
			const bool multi = wide3[b][c];
			const int2 *d_units = 0;
			int *d_prog = 0, n_launch = cnt;
			if (multi) { // one CTA per (problem, column pass): the passes of a problem run concurrently, linked by progress counters
				d_units = ctx->b_units.as<int2>() + unit_first[b][c], d_prog = (int*)(ctx->b_units.as<int2>() + n_units_tot) + unit_first[b][c];
				n_launch = unit_count[b][c];
			}
			nasw_launch_v3(ss, c == 10 ? 4 : Cs[c], b == 1, dj, ord, n_launch, ctx->b_rw.as<int4>(), d_aa, cst, ctx->b_out.as<int4>(), ctx->b_tb.as<uint16_t>(),
			               wsm_env > 0 ? wsm_env : 0, ctx->b_carry.as<int>(), multi, d_units, d_prog);
			ctx->stats.kernel_launches += 1;
			MPB_CUDA_OK(cudaEventRecord(ctx->ev_km[g.sid], ss));
			if (b == 1) {
				nasw_launch_bt(ss, dj, ord, cnt, ctx->b_tb.as<uint16_t>(), ctx->b_cigar.as<uint32_t>(), ctx->b_out.as<int4>());
				ctx->stats.kernel_launches += 1;
			}
		} else if (b == 0) {
			nasw_launch_ext(ss, Cs[c], dj, ord, cnt, ctx->b_rw.as<int4>(), d_aa, cst, ctx->b_out.as<int4>(), ctx->b_carry.as<int>());
			MPB_CUDA_OK(cudaEventRecord(ctx->ev_km[g.sid], ss));
			ctx->stats.kernel_launches += 1;
		} else {
			nasw_launch_tb(ss, Cs[c], dj, ord, cnt, ctx->b_rw.as<int4>(), d_aa, cst, ctx->b_out.as<int4>(), ctx->b_carry.as<int>(), ctx->b_tb.as<uint16_t>());
			MPB_CUDA_OK(cudaEventRecord(ctx->ev_km[g.sid], ss));
			nasw_launch_bt(ss, dj, ord, cnt, ctx->b_tb.as<uint16_t>(), ctx->b_cigar.as<uint32_t>(), ctx->b_out.as<int4>());
			ctx->stats.kernel_launches += 2;
		}
		MPB_CUDA_OK(cudaEventRecord(ctx->ev_k1[g.sid], ss));
		MPB_CUDA_OK(cudaEventRecord(ctx->ev_join[g.sid], ss));
		MPB_CUDA_OK(cudaStreamWaitEvent(st, ctx->ev_join[g.sid], 0));
	}
	MPB_CUDA_OK(cudaEventRecord(ctx->ev_w1, st));
	// results: scores first; the CIGARs are packed back to back on the device and only what was produced is copied
	if (cig_tot) {
		ctx->b_cigpack.reserve(sizeof(uint32_t) * (size_t)(cig_tot + 4));
		ctx->b_cigoff.reserve(sizeof(int64_t) * (size_t)(n + 1));
		nasw_launch_pack(st, dj, n, ctx->b_out.as<int4>(), ctx->b_cigar.as<uint32_t>(), ctx->b_cigoff.as<int64_t>(), ctx->b_cigpack.as<uint32_t>());
		ctx->stats.kernel_launches += 2;
	}
	const double t_launched = mp_realtime();
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->h_out.p, ctx->b_out.p, sizeof(int4) * n, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	const double t_synced = mp_realtime();
	MPB_CUDA_OK(cudaGetLastError());
	const int4 *ho = ctx->h_out.as<int4>();
	int64_t cig_used = 0;
	for (int k = 0; k < n; ++k)
		if (jobs[lo + k].cig_cap > 0) cig_used += ho[k].w;
	if (cig_used) {
		MPB_CUDA_OK(cudaMemcpyAsync(ctx->h_cigar.p, ctx->b_cigpack.p, sizeof(uint32_t) * (size_t)cig_used, cudaMemcpyDeviceToHost, st));
		MPB_CUDA_OK(cudaStreamSynchronize(st));
	}
	{
		float ms = 0;
		cudaEventElapsedTime(&ms, ctx->ev_w0, ctx->ev_w1);
		ctx->stats.ms_dp_wave += ms;
		cudaEventElapsedTime(&ms, ctx->ev_p0, ctx->ev_w0);
		ctx->stats.ms_prep += ms;
	}
	static const bool trace = getenv("MPB_TRACE") != 0; // per-class durations of every wave on stderr (diagnostics only)
	for (const Group &g : groups) { // sum of the classes' own durations (they overlap in time; the wave's wall time is what the step pays)
		float ms = 0, ms_dp = 0;
		cudaEventElapsedTime(&ms, ctx->ev_k0[g.sid], ctx->ev_k1[g.sid]);
		cudaEventElapsedTime(&ms_dp, ctx->ev_k0[g.sid], ctx->ev_km[g.sid]);
		(g.b == 0 ? ctx->stats.ms_dp_ext : ctx->stats.ms_dp_tb) += ms;
		ctx->stats.ms_class[g.b][g.c] += ms_dp, ctx->stats.n_class[g.b][g.c] += 1, ctx->stats.ms_bt += ms - ms_dp;
		for (size_t k = 0; k < g.count; ++k) {
			const DpDev &jj = jobs[lo + flat[g.first + k]];
			ctx->stats.cells_class[g.b][g.c] += (int64_t)jj.nl * jj.al;
		}
		if (trace) {
			int hist[5] = { 0 };
			double hc[5] = { 0 }, cells = 0;
			for (size_t k = 0; k < g.count; ++k) {
				const DpDev &jj = jobs[lo + flat[g.first + k]];
				const int q = jj.nl >= 65536 ? 0 : jj.nl >= 32768 ? 1 : jj.nl >= 16384 ? 2 : jj.nl >= 8192 ? 3 : 4;
				++hist[q], hc[q] += (double)jj.nl * jj.al * 1e-6, cells += (double)jj.nl * jj.al * 1e-6;
			}
			const DpDev &j0 = jobs[lo + flat[g.first]];
			fprintf(stderr, "[mpb-trace] nasw %s class %d%s: %zu jobs, longest nl=%d al=%d, %.1f Mcell, %.2f ms | nl>=64k %d (%.0f Mc), >=32k %d (%.0f), >=16k %d (%.0f), >=8k %d (%.0f), <8k %d (%.0f)\n",
			        g.b ? "tb " : "ext", g.c, "", g.count, j0.nl, j0.al, cells, ms, hist[0], hc[0], hist[1], hc[1], hist[2], hc[2], hist[3], hc[3], hist[4], hc[4]);
		}
	}
	ctx->stats.d2h_bytes += sizeof(int4) * n + sizeof(uint32_t) * (size_t)cig_used;
	const uint32_t *hc = ctx->h_cigar.as<uint32_t>();
	int64_t off = 0;
	for (int k = 0; k < n; ++k) {
		const DpDev &j = jobs[lo + k];
		out.score[lo + k] = ho[k].x, out.nt_len[lo + k] = ho[k].y, out.aa_len[lo + k] = ho[k].z;
		if (ho[k].y == -2 && ho[k].z == -2) { // the watchdog of the pair-lane kernels (nasw_pair_kernels.cu): never in a correct run
			fprintf(stderr, "[miniprot_b200] nasw: the warps of problem %d (nl=%d al=%d flag=%d) stopped waiting for each other\n", k, j.nl, j.al, j.flag);
			abort();
		}
		if (!unsupported.empty() && std::find(unsupported.begin(), unsupported.end(), k) != unsupported.end()) {
			out.score[lo + k] = INT32_MIN, out.nt_len[lo + k] = -1, out.aa_len[lo + k] = 0;
			out.cig_off[lo + k + 1] = (int64_t)out.cig.size();
			continue;
		}
		if (j.cig_cap > 0 && ho[k].w > 0) {
			out.cig.insert(out.cig.end(), hc + off, hc + off + ho[k].w);
			off += ho[k].w;
		}
		out.cig_off[lo + k + 1] = (int64_t)out.cig.size();
	}
	if (trace)
		fprintf(stderr, "[mpb-trace] nasw wave: %d problems, host prepare+launch %.2f ms, wait %.2f ms, results %.2f ms\n", n, (t_launched - t_in) * 1e3,
		        (t_synced - t_launched) * 1e3, (mp_realtime() - t_synced) * 1e3);
}

void nasw_run(mpb_ctx_s *ctx, const uint8_t *packed, const uint8_t *d_ss, const char *d_aa, const ns_opt_t *base, std::vector<DpDev> &jobs, DpSet &out)
{
	const size_t n = jobs.size();
	out.score.assign(n, 0), out.nt_len.assign(n, 0), out.aa_len.assign(n, 0);
	out.cig.clear(), out.cig_off.assign(n + 1, 0);
	if (n == 0) return;
	const Switches sw = Switches::from_env();
	NaswConst cst;
	fill_const(base, cst);
	size_t lo = 0;
	while (lo < n) {
		size_t hi = lo, tb_bytes = 0, rw_bytes = 0;
		while (hi < n) {
			const DpDev &j = jobs[hi];
			const bool is_tb = !(j.flag & (NS_F_EXT_LEFT | NS_F_EXT_RIGHT));
			const bool v3 = use_v3(sw);
			const int C = pick_C(j.al), Wp = v3 ? 32 * v3_warps(sw, j.al) : 32 * C, W8 = (j.al + 7) / 8 * 8, n_pass = (W8 + Wp - 1) / Wp;
			const size_t tbb = is_tb ? (size_t)n_pass * (size_t)(j.nl + 3 * Wp + 64) * Wp * 2 : 0, rwb = (size_t)(j.nl + 20) * 32;
			if (hi > lo && (tb_bytes + tbb > kTbBudget || rw_bytes + rwb > kRwBudget)) break;
			tb_bytes += tbb, rw_bytes += rwb, ++hi;
		}
		run_subwave(ctx, sw, packed, d_ss, d_aa, cst, base, jobs, lo, hi, out);
		lo = hi;
	}
}

} // namespace cuda
} // namespace mpb
