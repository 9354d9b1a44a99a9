// nasw_kernels.cu -- sm_90a kernels of the splice/frameshift-aware protein-to-DNA DP ("nasw").
//
// Replaces reference nasw-sse.c:340 ns_global_gs16b (striped SSE2, one problem per CPU thread) by:
//
//   nasw_prep_kernel   one thread per nucleotide row: unpack the 4-bit genome slice (strand / reversal aware), translate the
//                      codon ending at the row, evaluate the donor / acceptor rules (nasw-sse.c:91-210) and emit the 32-byte
//                      row record with every per-row constant of the recurrences precombined.  HBM-bound.
//   nasw_v3_kernel     the production DP kernel ("block-wide wavefront"): one CTA of 1/2/4/8 warps per problem, one thread
//                      per protein column, three rows per macro-step, skewed so that a column's left neighbour finished
//                      the same rows one macro-step earlier (warp shuffles inside a warp, 48 bytes of shared memory and a
//                      barrier between warps).  TB = false: score-only extension (80 % of all DP cells) with the
//                      warp-parallel x-drop bookkeeping; TB = true: global alignment that also streams one 16-bit
//                      traceback word per cell in wavefront-major order.  MP: problems wider than 256 columns in column
//                      passes with a per-row carry.  Latency bound (row-to-row dependency), see DESIGN.md section 4.
//   nasw_ext_kernel /  the first design, kept as the A/B family (MPB_NASW_KERNEL=cols): one warp per problem, lane l owns
//   nasw_tb_kernel     C protein columns, one row per step, column passes of 32*C with a carry array.
//   nasw_bt_kernel     one warp per problem walks the traceback words a run at a time and writes the CIGAR.
//   nasw_cigoff/cigpack_kernel   pack the CIGARs of a wave back to back before the device-to-host copy.
#include <algorithm>
#include <cuda_runtime.h>
#include <stdint.h>
#include "nasw_core.cuh"
#include "nasw_dev.hpp"
#include "nasw_warp.cuh"
#include "smem_attr.hpp"

namespace mpb {
namespace cuda {

using namespace nsw;

__device__ __forceinline__ unsigned long long globaltimer_ns()
{
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}

// nucleotide code of row k of a job: nibble (g_start + dir*k) of the packed genome, complemented on the - strand
__device__ __forceinline__ int job_code(const uint8_t *packed, const DpDev &j, int k)
{
	const int64_t g = j.g_start + (int64_t)j.dir * k;
	int b = packed[g >> 1] >> ((g & 1) * 4) & 0xf;
	if (j.comp) b = b < 4 ? 3 - b : b;
	return b;
}

// --spsc byte of the nucleotide of row k (-1: this problem has none); the table is laid out like the genome, one byte per base and strand
__device__ __forceinline__ int job_spsc(const uint8_t *ss, const DpDev &j, int k)
{
	if (j.ss_off < 0) return -1;
	const int64_t g = j.ss_off + j.g_start + (int64_t)j.dir * k;
	return g == j.ss_excl ? 0xff : (int)ss[g];
}

// ------------------------------------------------------------------ prep
// One CTA per chunk of <= PREP_ROWS rows of one problem: phase 1 evaluates the per-row splice / codon rules into shared
// memory (with a halo of 2 rows before and 1 after), phase 2 combines rows i-2..i+1 into the 32-byte record of row i.
__global__ void __launch_bounds__(256) nasw_prep_kernel(const DpDev *jobs, const PrepChunk *chunks, int n_chunks, const uint8_t *packed,
                                                        const uint8_t *ss, NaswConst cst, int4 *rec)
{
	__shared__ uint32_t w[PREP_ROWS + 4];
	const int ck = blockIdx.x;
	if (ck >= n_chunks) return;
	const PrepChunk c = chunks[ck];
	const DpDev job = jobs[c.job];
	auto code = [&](int k) { return job_code(packed, job, k); };
	auto sbyte = [&](int k) { return job_spsc(ss, job, k); };
	const SpscPar sq = { (job.io + 1) / 2 - 1, cst.sp_null_bonus };
	for (int x = threadIdx.x; x < c.n_rows + 3; x += blockDim.x) { // smem slot x <-> row c.row0 - 2 + x
		int r = c.row0 - 2 + x;
		r = r < 0 ? 0 : (r > job.nl ? job.nl : r);
		w[x] = (job.flag & NS_F_EXT_LEFT) ? prep_row_left(code, job.nl, r, cst.sp, cst.codon, cst.aa_x, sbyte, sq) : prep_row_forward(code, job.nl, r, cst.sp, cst.codon, cst.aa_x, sbyte, sq);
	}
	__syncthreads();
	Par par;
	par.go = cst.go, par.ge = cst.ge, par.io = job.io, par.fs = cst.fs, par.gei_stop = cst.fs;
	const int M = v3_triples(job.nl);
	for (int x = threadIdx.x; x < c.n_rows; x += blockDim.x) {
		const RowRec r = make_row_rec(par, w[x], w[x + 1], w[x + 2], w[x + 3]);
		const int i = c.row0 + x;
		int4 *dst, *dst2;
		if (job.C == 0) { // block-wide kernels: triple-major, field-major (nasw_core.cuh v3_triples); rows 0 and 1 are never read
			if (i < 2) continue;
			const int m = (i - 2) / 3, k = (i - 2) - 3 * m;
			dst = rec + job.rw_off * 2 + (int64_t)(2 * k) * M + m, dst2 = dst + M;
		} else dst = rec + (job.rw_off + i) * 2, dst2 = dst + 1;
		*dst = make_int4(r.cA, r.cB, r.cC, r.gei);
		*dst2 = make_int4(r.aA, r.aB, r.aC, r.nas);
	}
}

// residue code of logical column jg (reversed for left extension)
__device__ __forceinline__ int col_residue(const char *aa, const NaswConst &cst, const DpDev &j, int jg)
{
	const int p = (j.flag & NS_F_EXT_LEFT) ? j.al - 1 - jg : jg;
	return cst.aa20[(uint8_t)aa[j.aa_off + p]];
}

__device__ __forceinline__ void build_profile(int *prof, int Wp, int pass, const char *aa, const NaswConst &cst, const DpDev &job, int lane)
{
	for (int j = lane; j < Wp; j += 32) {
		const int jg = pass * Wp + j;
		if (jg < job.al) {
			const int r = col_residue(aa, cst, job, jg);
			for (int a = 0; a < 22; ++a) prof[a * Wp + j] = cst.mat[a * 22 + r];
		} else {
			for (int a = 0; a < 22; ++a) prof[a * Wp + j] = NEG;
		}
	}
	__syncwarp();
}

// environment of one column of the block-wide kernels: triple-major row records (nasw_core.cuh v3_triples) and the profile
struct DevEnv3 {
	const int4 *rec;     // field 0 of triple 0
	int M;               // triples per field array
	const int *prof;     // profile in shared memory, already offset to this column
	int Wp;
	const int4 *cur;     // steady-state cursor: field 0 of the next triple to fetch
	__device__ __forceinline__ void load3(const int4 *q, RowRec &r0, RowRec &r1, RowRec &r2) const
	{
		const int4 a0 = __ldg(q), b0 = __ldg(q + M), a1 = __ldg(q + 2 * M), b1 = __ldg(q + 3 * M), a2 = __ldg(q + 4 * M), b2 = __ldg(q + 5 * M);
		r0.cA = a0.x, r0.cB = a0.y, r0.cC = a0.z, r0.gei = a0.w, r0.aA = b0.x, r0.aB = b0.y, r0.aC = b0.z, r0.nas = b0.w;
		r1.cA = a1.x, r1.cB = a1.y, r1.cC = a1.z, r1.gei = a1.w, r1.aA = b1.x, r1.aB = b1.y, r1.aC = b1.z, r1.nas = b1.w;
		r2.cA = a2.x, r2.cB = a2.y, r2.cC = a2.z, r2.gei = a2.w, r2.aA = b2.x, r2.aB = b2.y, r2.aC = b2.z, r2.nas = b2.w;
	}
	// triple m (clamped: whatever a clamped index delivers belongs to rows that are never computed)
	__device__ __forceinline__ void rec3(int m, RowRec &r0, RowRec &r1, RowRec &r2) const { load3(rec + (m < 0 ? 0 : (m >= M ? M - 1 : m)), r0, r1, r2); }
	__device__ __forceinline__ void seek3(int m) { cur = rec + m; }
	__device__ __forceinline__ void next3(RowRec &r0, RowRec &r1, RowRec &r2) { load3(cur, r0, r1, r2), ++cur; }
	// columns 0..5 pull one field array each towards L1, 24 triples ahead of the front (column x's cursor + x = column 0's)
	__device__ __forceinline__ void prefetch_ahead(int x) const
	{
		const int4 *q = cur + x + 24;
		if (q < rec + M) asm volatile("prefetch.global.L1 [%0];" :: "l"(q + (int64_t)x * M));
	}
	__device__ __forceinline__ int profile_stride() const { return Wp; }
	__device__ __forceinline__ const int *profile(int nas) const { return prof + nas * Wp; }
};

// what a lane needs from its surroundings (see nasw_core.cuh ExtLane/TbLane)
struct DevEnv {
	const int4 *rec;     // row records of this problem (2 x int4 per row)
	int nl;
	const int *prof;     // profile of this warp for this pass, already offset to the lane's first column
	int Wp;
	int *cy;             // per-row carry between column passes
	__device__ __forceinline__ RowRec row_rec(int i) const
	{
		i = i < 0 ? 0 : (i > nl ? nl : i);
		const int4 a = __ldg(rec + 2 * i), b = __ldg(rec + 2 * i + 1);
		RowRec r;
		r.cA = a.x, r.cB = a.y, r.cC = a.z, r.gei = a.w, r.aA = b.x, r.aB = b.y, r.aC = b.z, r.nas = b.w;
		return r;
	}
	__device__ __forceinline__ int profile_stride() const { return Wp; }
	__device__ __forceinline__ void prefetch_row(int i) const
	{
		if (i <= nl) asm volatile("prefetch.global.L1 [%0];" :: "l"(rec + 2 * (i < 0 ? 0 : i)));
	}
	__device__ __forceinline__ const int *profile(int nas) const { return prof + nas * Wp; }
	__device__ __forceinline__ void carry_load3(int i, int &a, int &b, int &c) const { a = cy[(int64_t)i * 3], b = cy[(int64_t)i * 3 + 1], c = cy[(int64_t)i * 3 + 2]; }
	__device__ __forceinline__ void carry_store3(int i, int a, int b, int c) const { cy[(int64_t)i * 3] = a, cy[(int64_t)i * 3 + 1] = b, cy[(int64_t)i * 3 + 2] = c; }
	__device__ __forceinline__ void carry_load4(int i, int &a, int &b, int &c, int &d) const
	{
		const int4 v = *reinterpret_cast<const int4*>(cy + (int64_t)i * 4);
		a = v.x, b = v.y, c = v.z, d = v.w;
	}
	__device__ __forceinline__ void carry_store4(int i, int a, int b, int c, int d) const { *reinterpret_cast<int4*>(cy + (int64_t)i * 4) = make_int4(a, b, c, d); }
};

// ------------------------------------------------------------------ extension (score only)
template <int C, bool MULTI>
__global__ void __launch_bounds__(NASW_WARPS * 32) nasw_ext_kernel(const DpDev *jobs, const int *order, int n_jobs, const int4 *rec, const char *aa,
                                                                  NaswConst cst, int4 *out, int *carry)
{
	extern __shared__ int smem[];
	constexpr int Wp = 32 * C;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int slot = blockIdx.x * NASW_WARPS + warp;
	if (slot >= n_jobs) return;
	const int jid = order[slot];
	const DpDev job = jobs[jid];
	int *prof = smem + warp * 22 * Wp;
	LaneGeom g;
	g.lane = lane, g.nl = job.nl, g.al = job.al, g.W8 = (job.al + 7) / 8 * 8;
	g.n_pass = (g.W8 + Wp - 1) / Wp;
	const int T = g.nl > 2 ? g.nl - 2 + 32 : 0;
	Par par;
	par.go = cst.go, par.ge = cst.ge, par.io = job.io, par.fs = cst.fs, par.gei_stop = cst.fs;
	ExtTracker trk;
	trk.init(code_bits(g.al));
	DevEnv env;
	env.rec = rec + job.rw_off * 2, env.nl = g.nl, env.prof = prof + lane * C, env.Wp = Wp, env.cy = carry + job.carry_off;

	for (int pass = 0; pass < g.n_pass; ++pass) {
		build_profile(prof, Wp, pass, aa, cst, job, lane);
		g.pass = pass, g.col0 = pass * Wp + lane * C, g.live = g.col0 < g.W8;
		ExtLane<C, MULTI> L;
		L.init(g, cst.end_bonus, par.fs, env);
#define NSW_EXT_STEP(P) { \
			const int rH = __shfl_up_sync(0xffffffffu, L.outH, 1), rI = __shfl_up_sync(0xffffffffu, L.outI, 1), rB = __shfl_up_sync(0xffffffffu, L.outB, 1); \
			const int row_i = L.template step<P>(g, par, t + P, rH, rI, rB, env); \
			if (row_i >= 0 && pass == g.n_pass - 1) trk.row(row_i, L.outB, g.al * 3, cst.pen, cst.xdrop); /* only lane 31's tracker is read */ }
		for (int t = 0; t < T; t += 6) { // unrolled by the phase period so that row rotation is register renaming
			NSW_EXT_STEP(0)
			if (t == 0) L.after_first_step(g);
			NSW_EXT_STEP(1) NSW_EXT_STEP(2) NSW_EXT_STEP(3) NSW_EXT_STEP(4) NSW_EXT_STEP(5)
			if (pass == g.n_pass - 1 && (t % 12) == 6) {
				if (__shfl_sync(0xffffffffu, (int)trk.stopped, 31)) break;
			}
		}
#undef NSW_EXT_STEP
		__syncwarp();
	}
	if (lane == 31) {
		int4 r;
		r.x = trk.max_sc, r.y = trk.max_i + 1;
		r.z = trk.aa_len(g.al);
		r.w = 0;
		out[jid] = r;
	}
}

// ------------------------------------------------------------------ global alignment with traceback
// one traceback word per cell, wavefront-major [pass][step][32*C]: a warp step is one coalesced 64*C-byte store
template <int C>
__device__ __forceinline__ void store_words(uint16_t *dst, const uint32_t *wd)
{
	if (C == 1) dst[0] = (uint16_t)wd[0];
	else if (C == 2) *reinterpret_cast<uint32_t*>(dst) = wd[0] | wd[C > 1 ? 1 : 0] << 16;
	else {
#pragma unroll
		for (int k = 0; k < C; k += 4) {
			uint2 v;
			v.x = wd[k] | wd[k + 1 < C ? k + 1 : k] << 16, v.y = wd[k + 2 < C ? k + 2 : k] | wd[k + 3 < C ? k + 3 : k] << 16;
			*reinterpret_cast<uint2*>(dst + k) = v;
		}
	}
}

template <int C, bool MULTI>
__global__ void __launch_bounds__(NASW_WARPS * 32) nasw_tb_kernel(const DpDev *jobs, const int *order, int n_jobs, const int4 *rec, const char *aa,
                                                                 NaswConst cst, int4 *out, int *carry, uint16_t *tb)
{
	extern __shared__ int smem[];
	constexpr int Wp = 32 * C;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int slot = blockIdx.x * NASW_WARPS + warp;
	if (slot >= n_jobs) return;
	const int jid = order[slot];
	const DpDev job = jobs[jid];
	int *prof = smem + warp * 22 * Wp;
	LaneGeom g;
	g.lane = lane, g.nl = job.nl, g.al = job.al, g.W8 = (job.al + 7) / 8 * 8;
	g.n_pass = (g.W8 + Wp - 1) / Wp;
	const int T = g.nl > 2 ? g.nl - 2 + 32 : 0;
	Par par;
	par.go = cst.go, par.ge = cst.ge, par.io = job.io, par.fs = cst.fs, par.gei_stop = cst.fs;
	DevEnv env;
	env.rec = rec + job.rw_off * 2, env.nl = g.nl, env.prof = prof + lane * C, env.Wp = Wp, env.cy = carry + job.carry_off;
	int score = NEG;

	for (int pass = 0; pass < g.n_pass; ++pass) {
		build_profile(prof, Wp, pass, aa, cst, job, lane);
		g.pass = pass, g.col0 = pass * Wp + lane * C, g.live = g.col0 < g.W8;
		TbLane<C, MULTI> L;
		L.init(g, par.fs, env);
		uint16_t *tbp = tb + job.tb_off + (int64_t)pass * T * Wp + lane * C;
#define NSW_TB_STEP(P) { \
			const int rH = __shfl_up_sync(0xffffffffu, L.outH, 1), rF = __shfl_up_sync(0xffffffffu, L.outF, 1); \
			const int rS = __shfl_up_sync(0xffffffffu, L.outS, 1), rI = __shfl_up_sync(0xffffffffu, L.outI, 1); \
			uint32_t wd[C]; \
			if (L.template step<P>(g, par, t + P, rH, rF, rS, rI, env, wd)) store_words<C>(tbp + (int64_t)(t + P) * Wp, wd); }
		for (int t = 0; t < T; t += 6) {
			NSW_TB_STEP(0)
			if (t == 0) L.after_first_step(g);
			NSW_TB_STEP(1) NSW_TB_STEP(2) NSW_TB_STEP(3) NSW_TB_STEP(4) NSW_TB_STEP(5)
		}
#undef NSW_TB_STEP
		if (L.k_end >= 0) score = L.score;
		__syncwarp();
	}
	// the lane that owns column al-1 (in its pass) holds H(nl-1, al-1)
	const int owner = g.al > 0 ? ((g.al - 1) % Wp) / C : 0;
	score = __shfl_sync(0xffffffffu, score, owner);
	if (lane == 0) out[jid] = make_int4(score, g.nl, g.al, 0);
}

// ------------------------------------------------------------------ block-wide wavefront (one thread per column, 3 rows per step)
// CTA = NW warps = 32*NW columns of ONE problem; see nasw_core.cuh::Lane3.  TB = false: score-only extension (result by the
// last thread's tracker); TB = true: global alignment, one 16-bit word per cell to tb[(3T + r) * 32NW + x].
// MP (multi-pass, widest instantiation only): a problem wider than the block's Wp columns runs in passes of Wp columns; the last
// column of a pass leaves what the column to its right needs (H, insertion chain, running row maximum / first-pass H, segment
// chain: one int4 per row) in the carry array, the first column of the next pass reads it back two macro-steps ahead.
template <int NW, bool TB, bool MP>
__global__ void __launch_bounds__(NW * 32) nasw_v3_kernel(const DpDev *jobs, const int *order, int n_jobs, const int4 *rec, const char *aa, NaswConst cst,
                                                          int4 *out, uint16_t *tb, int4 *carry_all, const int2 *units, int *progress)
{
	extern __shared__ int smem[];
	constexpr int Wp = 32 * NW;
	__shared__ __align__(16) int xchg[2][NW + 1][12]; // [parity][warp + 1]: last column of each warp; slot 0 = the constant boundary left of column 0
	__shared__ int ring[TB ? 32 : 32 * 32];           // [slot][lane] row maxima waiting for the warp tracker (WarpTracker)
	__shared__ int stop_flag[2]; // written by the last column during macro-step Tm into slot Tm & 1, read by everyone after that step's barrier
	if ((int)blockIdx.x >= n_jobs) return;
	// MP: one CTA per (problem, column pass), listed in units[] pass after pass: the passes of a problem run CONCURRENTLY, pass q
	// a few dozen rows behind pass q - 1, whose last column publishes how many of its carry rows are complete (progress[])
	const int unit_pass = MP ? units[blockIdx.x].y : 0;
	const int jid = order[MP ? units[blockIdx.x].x : (int)blockIdx.x];
	const DpDev job = jobs[jid];
	const int x = threadIdx.x, lane = x & 31, warp = x >> 5;
	const int W8all = (job.al + 7) / 8 * 8, n_pass = MP ? (W8all + Wp - 1) / Wp : 1;
	volatile int *prog_out = MP ? progress + blockIdx.x : 0;
	volatile const int *prog_in = MP && unit_pass > 0 ? progress + blockIdx.x - 1 : 0;
	int4 *carry = MP ? carry_all + job.carry_off / 4 : 0; // one int4 per row
	Par par;
	par.go = cst.go, par.ge = cst.ge, par.io = job.io, par.fs = cst.fs, par.gei_stop = cst.fs;
	WarpTracker trk; // meaningful in the warp that owns the last column (of the last pass)
	trk.init(code_bits(job.al));
	int tb_score = NEG;
	for (int pass = unit_pass; pass <= unit_pass; ++pass) {
	// carry_out: the last column of a pass that has a successor writes its outputs to the carry row array; feeder: in a later pass, one
	// thread off the first column's warp (lane 1 of warp 1) brings the carry rows in
	const bool last_pass = pass == n_pass - 1, carry_out = MP && !last_pass && x == Wp - 1, feeder = MP && pass > 0 && x == 33;
	Geo3 g;
	g.x = x, g.col = pass * Wp + x, g.nl = job.nl, g.al = job.al, g.W8 = W8all, g.live = g.col < g.W8, g.first = g.col == 0;
	// profile: 22 x Wp, column x of row a at smem[a * Wp + x]
	{
		int rcode = -1;
		if (g.col < job.al) rcode = col_residue(aa, cst, job, g.col);
		for (int a = 0; a < 22; ++a) smem[a * Wp + x] = rcode >= 0 ? cst.mat[a * 22 + rcode] : NEG;
	}
	if (x == 0) stop_flag[0] = stop_flag[1] = 0;
	if (x < 24 && !(MP && pass > 0)) xchg[x / 12][0][x % 12] = (!TB && x % 12 >= 6 && x % 12 < 9) ? INT32_MIN : NEG; // (a later pass: slot 0 is fed from the carry rows)
	__syncthreads();
	const uint32_t xr[2] = { smem_addr(&xchg[0][warp][0]), smem_addr(&xchg[1][warp][0]) };         // what lane 0 receives from
	const uint32_t xw[2] = { smem_addr(&xchg[0][warp + (warp < NW - 1)][0]), smem_addr(&xchg[1][warp + (warp < NW - 1)][0]) }; // what lane 31 sends to
	const uint32_t sf = smem_addr(stop_flag), ring_w = smem_addr(ring) + lane * 4, ring_r = smem_addr(ring) + lane * 128 + 124;
	(void)xw, (void)ring_w, (void)ring_r;
	DevEnv3 env;
	env.rec = rec + job.rw_off * 2, env.M = v3_triples(g.nl), env.prof = smem + x, env.Wp = Wp, env.cur = env.rec;
	Lane3<TB> L;
	L.init(g, cst.end_bonus, par.fs, env);
	// A later pass: what its first column needs from the left -- the outputs of the previous pass's last column, three rows per
	// macro-step -- reaches it exactly like the left neighbour's outputs reach the first lane of any other warp: through exchange slot 0,
	// so the receive path and the steady loop are the same code as in a single-pass problem.  The feeder thread brings the carry rows
	// in with asynchronous 16-byte copies global -> shared (a ring of 16 macro-steps), EIGHT macro-steps ahead: the rows were written by
	// another SM a moment ago and come from the far side of L2 -- about 2000 cycles, four macro-steps; fetched into registers two or three
	// steps ahead they set the pace of the whole pass (about twice the time per row of the same CTA without a carry).
	// At step T it repacks the rows of step T + 1 from the ring into slot 0 of this step's parity, before the barrier.  Every 32 steps
	// it makes sure the previous pass has published what the next 32 issues will read.
	// (Predicated accesses: every thread runs them, one thread's predicate is set -- no divergence region in the steady loop.)
	__shared__ __align__(16) int4 cring[MP ? 16 * 3 : 1];
	const uint32_t cring_a = smem_addr(cring);
	int prog_seen = 0; // what the feeder last read from the previous pass's counter
	const uint32_t xs0[2] = { smem_addr(&xchg[0][0][0]), smem_addr(&xchg[1][0][0]) };
	auto feed_wait = [&](int Tm) {
		const int need = min(3 * Tm + 5, g.nl); // rows below `need` must have left the previous pass
		if (prog_seen < need) {
			while ((prog_seen = *prog_in) < need) __nanosleep(200);
			__threadfence(); // the rows were written before the counter moved
		}
	};
	const int4 *cr = carry + 2;      // feeder: first carry row of the macro-step whose rows are requested next (row 3 Tm + 2) ...
	int cslot = 0;                   // ... and its ring slot, Tm & 15
	int4 *cw = carry + (2 - 3 * (Wp - 1)); // last column: where its rows of macro-step T go (row 3 (T - (Wp - 1)) + 2), before the array while T < Wp - 1
	auto feed_issue = [&]() { // past the last row the array has slack (nasw_host.cu) and the rows are masked
#pragma unroll
		for (int r = 0; r < 3; ++r) cp_async16_if(feeder, cring_a + (uint32_t)(cslot * 3 + r) * 16, cr + r);
		cp_async_commit();
		cr += 3, cslot = (cslot + 1) & 15;
	};
	auto feed_repack = [&](uint32_t slot, int Tm) { // ring rows (H, I, X, S) x 3 -> slot layout H[3], I[3], X[3], S[3]
		const uint32_t a = cring_a + (uint32_t)((Tm & 15) * 3) * 16;
		const int4 v0 = lds128(a), v1 = lds128(a + 16), v2 = lds128(a + 32);
		sts128_if(feeder, slot, make_int4(v0.x, v1.x, v2.x, v0.y)), sts128_if(feeder, slot + 16, make_int4(v1.y, v2.y, v0.z, v1.z));
		sts128_if(feeder, slot + 32, make_int4(v2.z, v0.w, v1.w, v2.w));
	};
	// the last column of a pass that has a successor: every 128th macro-step (and at the end) it publishes the number of finished rows
	// (the fence is not free, and a lag of a hundred rows is nothing against the tens of thousands of a long problem)
	auto carry_publish = [&](int rows_done) {
		__threadfence();
		*prog_out = rows_done;
	};
	if (MP) {
		if (feeder) feed_wait(41);
		for (int k = 0; k < 8; ++k) feed_issue(); // macro-steps 0..7
		cp_async_wait<0>();
		feed_repack(xs0[1], 0); // macro-step 0 reads the slot of parity 1
		__syncthreads();
	}
	const int n_macro = g.nl > 2 ? (g.nl - 2 + 2) / 3 + Wp : 0; // rows 2..nl-1 in triples, plus the skew of the last column
	uint16_t *tbp = TB ? tb + job.tb_off + (int64_t)pass * (3 * (n_macro + 2)) * Wp + x : 0;
	// (T is even at every loop head, so the parity of macro-step T + PH is PH: all exchange slots are static)
#define NSW_V3_RECV(PH, RH) \
		int rI[3], rX[3], rS[3]; \
		_Pragma("unroll") for (int r = 0; r < 3; ++r) { \
			RH[r] = __shfl_up_sync(0xffffffffu, L.oH[r], 1), rI[r] = __shfl_up_sync(0xffffffffu, L.oI[r], 1), rX[r] = __shfl_up_sync(0xffffffffu, L.oX[r], 1); \
			rS[r] = TB ? __shfl_up_sync(0xffffffffu, L.oS[r], 1) : 0; \
		} \
		if (lane == 0) { /* the column to my left lives in the previous warp; slot 0: the constant left boundary, or the previous pass's last column */ \
			const int4 b0 = lds128(xr[PH ^ 1]), b1 = lds128(xr[PH ^ 1] + 16), b2 = lds128(xr[PH ^ 1] + 32); \
			RH[0] = b0.x, RH[1] = b0.y, RH[2] = b0.z, rI[0] = b0.w, rI[1] = b1.x, rI[2] = b1.y, rX[0] = b1.z, rX[1] = b1.w, rX[2] = b2.x; \
			if (TB) rS[0] = b2.y, rS[1] = b2.z, rS[2] = b2.w; \
		}
#define NSW_V3_SEND(PH) \
		if (NW > 1) { \
			if (MP) { /* carry rows of the next macro-step into slot 0, those of the step after the next two on their way */ \
				if (((T + PH) & 31) == 0 && feeder) feed_wait(T + PH + 41); \
				feed_issue(); /* macro-step T + PH + 8 */ \
				cp_async_wait<6>(); /* everything up to macro-step T + PH + 2 has landed */ \
				feed_repack(xs0[PH], T + PH + 1); \
			} \
			if (lane == 31 && warp < NW - 1) { \
				sts128(xw[PH], make_int4(L.oH[0], L.oH[1], L.oH[2], L.oI[0])), sts128(xw[PH] + 16, make_int4(L.oI[1], L.oI[2], L.oX[0], L.oX[1])); \
				sts128(xw[PH] + 32, make_int4(L.oX[2], TB ? L.oS[0] : 0, TB ? L.oS[1] : 0, TB ? L.oS[2] : 0)); \
			} \
			if (!TB && x == Wp - 1) sts32(sf + 4 * PH, trk.stopped ? 1 : 0); \
			__syncthreads(); \
		}
#define NSW_V3_MACRO(PH) { /* general step: ramp-up, ramp-down */ \
		int rH[3]; \
		NSW_V3_RECV(PH, rH) \
		uint32_t wd[3]; \
		const uint32_t done = L.template macro<PH>(g, par, T + PH, rH, rI, rX, rS, env, wd); \
		if (TB) { _Pragma("unroll") for (int r = 0; r < 3; ++r) if (done >> r & 1) tbp[(int64_t)(3 * (T + PH) + r) * Wp] = (uint16_t)wd[r]; } \
		if (MP) { \
			_Pragma("unroll") for (int r = 0; r < 3; ++r) stg128_if(carry_out && (done >> r & 1), cw + r, make_int4(L.oH[r], L.oI[r], L.oX[r], TB ? L.oS[r] : 0)); \
			cw += 3; \
			if (carry_out && done && ((T + PH) & 7) == 7) carry_publish(min(Lane3<TB>::row_of(g, T + PH, 0) + 3, g.nl)); /* ramps: every 8th step */ \
		} \
		if (!TB && warp == NW - 1 && last_pass) { /* the last column sees the complete row maxima; its rows are real when 2 <= i < nl */ \
			(void)done; \
			_Pragma("unroll") for (int r = 0; r < 3; ++r) { \
				const int il = 3 * (T + PH - (Wp - 1)) + 2 + r; \
				if (il >= 2 && il < g.nl) trk.push(ring_w, L.oX[r]); \
			} \
			if (trk.n_ring >= 30) trk.flush(ring_r, lane, g.al * 3, cst.pen, cst.xdrop); } \
		NSW_V3_SEND(PH) }
#define NSW_V3_STEADY(PH) { /* every column has three real rows: nothing to check */ \
		NSW_V3_RECV(PH, hb[PH]) \
		uint32_t wd[3]; \
		L.template macro_steady<PH>(g, par, hb[PH ^ 1], hb[PH], rI, rX, rS, env, wd); \
		if (TB) { if (g.live) { _Pragma("unroll") for (int r = 0; r < 3; ++r) tbs[r * Wp] = (uint16_t)wd[r]; } tbs += 3 * Wp; } \
		if (MP) { \
			_Pragma("unroll") for (int r = 0; r < 3; ++r) stg128_if(carry_out, cw + r, make_int4(L.oH[r], L.oI[r], L.oX[r], TB ? L.oS[r] : 0)); \
			cw += 3; \
			if (((T + PH) & 127) == 127 && carry_out) carry_publish(Lane3<TB>::row_of(g, T + PH, 0) + 3); /* the fence waits for the stores to reach L2: rarely */ \
		} \
		if (!TB && warp == NW - 1 && last_pass) { \
			_Pragma("unroll") for (int r = 0; r < 3; ++r) sts32(ring_w + (trk.n_ring + r) * 128, L.oX[r]); \
			trk.n_ring += 3; \
			if (trk.n_ring == 30) trk.flush(ring_r, lane, g.al * 3, cst.pen, cst.xdrop); } \
		NSW_V3_SEND(PH) }
#define NSW_V3_CHECK_STOP \
		if (!TB) { /* x-drop: the last column's tracker decides; rows after the break row are never looked at */ \
			if (NW > 1) { if (lds32(sf + 4)) break; } \
			else if (trk.stopped) break; \
		}
	int t_lo, t_hi;
	Lane3<TB>::steady_range(g.nl, Wp, t_lo, t_hi);
	int T = 0;
	for (; T < t_lo && T < n_macro; T += 2) { NSW_V3_MACRO(0) NSW_V3_MACRO(1) NSW_V3_CHECK_STOP }
	if (T >= t_lo) {
		int hb[2][3]; // H of the column to the left: this macro-step's and the previous one's, alternating
		L.steady_enter(g, T, hb[1], env);
		uint16_t *tbs = TB ? tbp + (int64_t)3 * T * Wp : 0;
		(void)tbs;
		for (; T < t_hi; T += 2) { NSW_V3_STEADY(0) NSW_V3_STEADY(1) NSW_V3_CHECK_STOP }
		if (T >= t_hi) { // not left through the x-drop break
			L.steady_leave(hb[1]);
			for (; T < n_macro; T += 2) { NSW_V3_MACRO(0) NSW_V3_MACRO(1) NSW_V3_CHECK_STOP }
		}
	}
#undef NSW_V3_RECV
#undef NSW_V3_SEND
#undef NSW_V3_STEADY
#undef NSW_V3_CHECK_STOP
#undef NSW_V3_MACRO
	if (!TB && warp == NW - 1 && last_pass && trk.n_ring > 0) trk.flush(ring_r, lane, g.al * 3, cst.pen, cst.xdrop); // the last, partial batch
	if (TB && g.col == (job.al > 0 ? job.al - 1 : 0)) tb_score = L.score; // the thread that owns column al-1 holds H(nl-1, al-1)
	if (MP && carry_out) carry_publish(g.nl); // whatever is left
	} // passes
	if (TB) {
		const int c_end = job.al > 0 ? job.al - 1 : 0;
		if (x == c_end % Wp && c_end / Wp == unit_pass) out[jid] = make_int4(tb_score, job.nl, job.al, 0);
	} else if (x == Wp - 1 && unit_pass == n_pass - 1) {
		int4 r;
		r.x = trk.max_sc, r.y = trk.max_i + 1;
		r.z = trk.aa_len(job.al);
		r.w = 0;
		out[jid] = r;
	}
}

// ------------------------------------------------------------------ backtrack -> CIGAR
// One warp per problem.  The walk is sequential, but it proceeds a RUN at a time (nasw_core.cuh::backtrack_runs): the 32
// lanes fetch the next 32 cells along the current move direction in one round trip and a ballot tells how far the run
// goes, instead of one dependent L2 access per cell (introns are thousands of cells long).
struct DevScan {
	const uint16_t *base;
	int C, Wp, T, lane; // C == 0: block-wide wavefront layout, word of cell (i, j) at ((i - 2) + 3 j) * Wp + j
	__device__ __forceinline__ uint32_t at(int i, int j) const
	{
		if (C == 0) { // block-wide layout, passes of Wp columns, T rows of Wp words per pass
			const int pass = j / Wp, jc = j - pass * Wp;
			return base[((int64_t)pass * T + (i - 2 + 3 * jc)) * Wp + jc];
		}
		const int pass = j / Wp, jc = j - pass * Wp, ln = jc / C;
		return base[((int64_t)pass * T + (i - 2 + ln)) * Wp + jc];
	}
	__device__ __forceinline__ uint32_t word(int i, int j) const { return at(i, j); }
	__device__ __forceinline__ int lead(int kind, int i, int j, int &n_valid) const
	{
		const int di = kind == 0 ? 3 : kind == 1 ? 0 : kind == 2 ? 3 : 1, dj = kind <= 1 ? 1 : 0;
		const int ii = i - di * lane, jj = j - dj * lane;
		const bool valid = ii >= 2 && jj >= 0;
		bool ok = false;
		if (valid) {
			const uint32_t x = at(ii, jj);
			ok = kind == 0 ? (!(x >> 9 & 1) && (x & 0xf) == 0) : (x >> (kind + 3) & 1);
		}
		const uint32_t vm = __ballot_sync(0xffffffffu, valid), om = __ballot_sync(0xffffffffu, ok);
		n_valid = __popc(vm);
		return om == 0xffffffffu ? 32 : __ffs(~om) - 1;
	}
};

__global__ void __launch_bounds__(NASW_WARPS * 32) nasw_bt_kernel(const DpDev *jobs, const int *order, int n_jobs, const uint16_t *tb, uint32_t *cigar, int4 *out)
{
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int slot = blockIdx.x * NASW_WARPS + warp;
	if (slot >= n_jobs) return;
	const int jid = order[slot];
	const DpDev job = jobs[jid];
	DevScan sc;
	sc.base = tb + job.tb_off, sc.C = job.C, sc.Wp = job.C ? 32 * job.C : job.pad_, sc.lane = lane;
	// rows of traceback words per column pass: column-pass kernels nl - 2 + 32, block-wide kernels 3 (n_macro + 2)
	sc.T = job.nl <= 2 ? 0 : job.C ? job.nl - 2 + 32 : 3 * ((job.nl - 2 + 2) / 3 + job.pad_ + 2);
	const int n = backtrack_runs(sc, job.nl, job.al, cigar + job.cig_off, job.cig_cap, lane == 0);
	if (lane == 0) out[jid].w = n;
}

// ------------------------------------------------------------------ launchers
template <int C, bool MULTI>
static void launch_ext(cudaStream_t st, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out, int *carry)
{
	const int smem = NASW_WARPS * 22 * 32 * C * (int)sizeof(int);
	static SmemLimit lim;
	lim.raise(nasw_ext_kernel<C, MULTI>, smem);
	nasw_ext_kernel<C, MULTI><<<(n + NASW_WARPS - 1) / NASW_WARPS, NASW_WARPS * 32, smem, st>>>(jobs, order, n, rec, aa, cst, out, carry);
}

template <int C, bool MULTI>
static void launch_tb(cudaStream_t st, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out, int *carry,
                      uint16_t *tb)
{
	const int smem = NASW_WARPS * 22 * 32 * C * (int)sizeof(int);
	static SmemLimit lim;
	lim.raise(nasw_tb_kernel<C, MULTI>, smem);
	nasw_tb_kernel<C, MULTI><<<(n + NASW_WARPS - 1) / NASW_WARPS, NASW_WARPS * 32, smem, st>>>(jobs, order, n, rec, aa, cst, out, carry, tb);
}

void nasw_launch_prep(cudaStream_t st, const DpDev *jobs, const PrepChunk *chunks, int n_chunks, const uint8_t *packed, const uint8_t *ss, const NaswConst &cst, int4 *rec)
{
	if (n_chunks > 0) nasw_prep_kernel<<<n_chunks, 256, 0, st>>>(jobs, chunks, n_chunks, packed, ss, cst, rec);
}

// C = 1, 2, 4, 8: single-pass problems (at most 32*C padded columns); C = 16 stands for "8 columns per lane, several passes"
void nasw_launch_ext(cudaStream_t st, int C, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out, int *carry)
{
	if (n <= 0) return;
	switch (C) {
	case 1: launch_ext<1, false>(st, jobs, order, n, rec, aa, cst, out, carry); break;
	case 2: launch_ext<2, false>(st, jobs, order, n, rec, aa, cst, out, carry); break;
	case 4: launch_ext<4, false>(st, jobs, order, n, rec, aa, cst, out, carry); break;
	case 8: launch_ext<8, false>(st, jobs, order, n, rec, aa, cst, out, carry); break;
	default: launch_ext<8, true>(st, jobs, order, n, rec, aa, cst, out, carry); break;
	}
}

void nasw_launch_tb(cudaStream_t st, int C, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out, int *carry,
                    uint16_t *tb)
{
	if (n <= 0) return;
	switch (C) {
	case 1: launch_tb<1, false>(st, jobs, order, n, rec, aa, cst, out, carry, tb); break;
	case 2: launch_tb<2, false>(st, jobs, order, n, rec, aa, cst, out, carry, tb); break;
	case 4: launch_tb<4, false>(st, jobs, order, n, rec, aa, cst, out, carry, tb); break;
	case 8: launch_tb<8, false>(st, jobs, order, n, rec, aa, cst, out, carry, tb); break;
	default: launch_tb<8, true>(st, jobs, order, n, rec, aa, cst, out, carry, tb); break;
	}
}

// warps_per_sm > 0: pad the dynamic shared memory request to nw / warps_per_sm of an SM's shared memory, so that at most that
// many warps of such launches are resident per SM and the hardware dispatches the remaining blocks -- in index order, i.e.
// longest problem first -- as earlier ones retire (list scheduling by decreasing length).  Without the cap every block of a
// wave is resident from the start and the few 100 k-row problems that set the critical path share their issue slots with
// thousands of short ones.  (228 KB per SM, 1 KB reserved per block, static arrays included.)
template <int NW, bool TB, bool MP>
static void launch_v3(cudaStream_t st, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out, uint16_t *tb,
                      int warps_per_sm, int *carry, const int2 *units = 0, int *progress = 0)
{
	int smem = 22 * 32 * NW * (int)sizeof(int);
	if (warps_per_sm > 0) {
		static const int stat = [] { // static shared memory of the kernel: the same on every device of the one architecture built for
			cudaFuncAttributes fa;
			cudaFuncGetAttributes(&fa, nasw_v3_kernel<NW, TB, MP>);
			return ((int)fa.sharedSizeBytes + 15) & ~15;
		}();
		static SmemLimit lim;
		lim.raise(nasw_v3_kernel<NW, TB, MP>, 232448 - stat);
		const int share = (int)((int64_t)233472 * NW / warps_per_sm) - 1024 - stat;
		smem = std::max(smem, std::min(share, 232448 - stat)) & ~15;
	}
	nasw_v3_kernel<NW, TB, MP><<<n, NW * 32, smem, st>>>(jobs, order, n, rec, aa, cst, out, tb, (int4*)carry, units, progress);
}

// block-wide wavefront kernels: nw = warps per problem (1, 2, 4 or 8); multi = some problem of the launch is wider than 256
// columns (nw == 8 only: column passes with a carry)
// multi: some problem of the launch is wider than one CTA (nw == 2 or 8); then n = number of (problem, pass) units, units[] lists
// them pass after pass per problem and progress[] (n zeroed ints) links consecutive passes
void nasw_launch_v3(cudaStream_t st, int nw, bool is_tb, const DpDev *jobs, const int *order, int n, const int4 *rec, const char *aa, const NaswConst &cst, int4 *out,
                    uint16_t *tb, int warps_per_sm, int *carry, bool multi, const int2 *units, int *progress)
{
	if (n <= 0) return;
	switch (nw * 2 + (is_tb ? 1 : 0)) {
	case 2: launch_v3<1, false, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry); break;
	case 3: launch_v3<1, true, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry); break;
	case 4:
		if (multi) launch_v3<2, false, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<2, false, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	case 5:
		if (multi) launch_v3<2, true, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<2, true, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	case 8:
		if (multi) launch_v3<4, false, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<4, false, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	case 9:
		if (multi) launch_v3<4, true, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<4, true, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	case 16:
		if (multi) launch_v3<8, false, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<8, false, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	default:
		if (multi) launch_v3<8, true, true>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry, units, progress);
		else launch_v3<8, true, false>(st, jobs, order, n, rec, aa, cst, out, tb, warps_per_sm, carry);
		break;
	}
}

// ------------------------------------------------------------------ CIGAR packing
// exclusive prefix sum of the CIGAR lengths (out[k].w, zero for extension problems) by one block; offs[n] = total
__global__ void __launch_bounds__(1024) nasw_cigoff_kernel(const DpDev *jobs, int n, const int4 *out, int64_t *offs)
{
	__shared__ int64_t part[1024];
	const int t = threadIdx.x, per = (n + 1023) / 1024, k0 = t * per, k1 = min(n, k0 + per);
	int64_t sum = 0;
	for (int k = k0; k < k1; ++k) sum += jobs[k].cig_cap > 0 ? out[k].w : 0;
	part[t] = sum;
	__syncthreads();
	for (int d = 1; d < 1024; d <<= 1) { // Hillis-Steele inclusive scan of the per-thread sums
		const int64_t v = t >= d ? part[t - d] : 0;
		__syncthreads();
		part[t] += v;
		__syncthreads();
	}
	int64_t run = part[t] - sum;
	for (int k = k0; k < k1; ++k) offs[k] = run, run += jobs[k].cig_cap > 0 ? out[k].w : 0;
	if (t == 1023) offs[n] = part[1023];
}

__global__ void __launch_bounds__(256) nasw_cigpack_kernel(const DpDev *jobs, int n, const int4 *out, const uint32_t *cigar, const int64_t *offs, uint32_t *packed)
{
	const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (k >= n) return;
	const DpDev j = jobs[k];
	if (j.cig_cap <= 0) return;
	const int nc = out[k].w;
	const uint32_t *src = cigar + j.cig_off + j.cig_cap - nc;
	uint32_t *dst = packed + offs[k];
	for (int i = lane; i < nc; i += 32) dst[i] = src[i];
}

void nasw_launch_pack(cudaStream_t st, const DpDev *jobs, int n, const int4 *out, const uint32_t *cigar, int64_t *offs, uint32_t *packed)
{
	if (n <= 0) return;
	nasw_cigoff_kernel<<<1, 1024, 0, st>>>(jobs, n, out, offs);
	nasw_cigpack_kernel<<<(n + 7) / 8, 256, 0, st>>>(jobs, n, out, cigar, offs, packed);
}


__global__ void nasw_spacer_kernel(long long ns)
{
	const long long t0 = (long long)globaltimer_ns();
	while ((long long)globaltimer_ns() - t0 < ns) __nanosleep(1000);
}

void nasw_launch_spacer(cudaStream_t st, int us) { nasw_spacer_kernel<<<1, 1, 0, st>>>((long long)us * 1000); }

void nasw_launch_bt(cudaStream_t st, const DpDev *jobs, const int *order, int n, const uint16_t *tb, uint32_t *cigar, int4 *out)
{
	if (n > 0) nasw_bt_kernel<<<(n + NASW_WARPS - 1) / NASW_WARPS, NASW_WARPS * 32, 0, st>>>(jobs, order, n, tb, cigar, out);
}

} // namespace cuda
} // namespace mpb
