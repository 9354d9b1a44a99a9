// chain_kernels.cu -- minimap2-style anchor chaining on the GPU (replaces reference chain.c:160 mp_chain).
//
//   chain_fill_kernel  one warp per chaining problem.  Anchors are visited in order (the recurrence is sequential
//                      in i), the predecessor scan j = i-1 .. st runs 32 candidates at a time: every lane scores
//                      one candidate (chain.c:112 comput_sc is pure), a warp prefix-max finds the records, two
//                      ballots + chain_core.cuh::resolve_chunk() reproduce the order-dependent max_skip logic,
//                      t[] marks go through memory exactly as in the reference.  Latency / integer bound; the
//                      byte volume is tiny (20 B of scratch per anchor, chain.c:175-178).
//   chain_bt_*_kernel  one warp per problem: backtrack with the reference's unstable sort order (cycle chases and peeling on
//                      lane 0, everything parallel shared by the lanes), compaction; the pre-chain's result by stream compaction.
#include <cuda_runtime.h>
#include "chain_core.cuh"
#include "chain_dev.hpp"
#include "smem_attr.hpp"

namespace mpb {
namespace cuda {

using namespace chn;

constexpr int CHAIN_WARPS = 4;

// The fill walks the anchors in order and looks a short way back, so the warp keeps the 32-anchor block it is in, the one
// before and the one after in registers (lane l holds anchor i0 + l; one coalesced load per 32 anchors, issued a block
// ahead) and hands values around by shuffle; only look-backs of more than a block go to memory.  Without this every
// anchor paid one or two dependent L2 round trips (a[i], a[st], a[hi]) even when it had no predecessor to score, which is
// the common case of the block-level pre-chain.
struct AnchorBlocks {
	uint64_t prev, cur, next;
	int32_t i0; // first anchor of `cur`
	__device__ __forceinline__ void init(const uint64_t *a, int32_t n, int lane)
	{
		i0 = 0, prev = 0;
		cur = lane < n ? a[lane] : 0;
		next = 32 + lane < n ? a[32 + lane] : 0;
	}
	__device__ __forceinline__ void enter(const uint64_t *a, int32_t n, int32_t i, int lane) // i is a multiple of 32, i > 0
	{
		prev = cur, cur = next, i0 = i;
		next = i + 32 + lane < n ? a[i + 32 + lane] : 0;
	}
	// a[idx] for a warp-uniform idx <= i0 + 31
	__device__ __forceinline__ uint64_t at(const uint64_t *a, int32_t idx) const
	{
		if (idx >= i0) return __shfl_sync(0xffffffffu, cur, idx - i0);
		if (idx >= i0 - 32) return __shfl_sync(0xffffffffu, prev, idx - (i0 - 32));
		return a[idx];
	}
	// a[j] for a per-lane j in [i0 - 32, i0 + 31] (every lane calls; lanes with j out of that range get garbage)
	__device__ __forceinline__ uint64_t near(int32_t j) const
	{
		const uint64_t c = __shfl_sync(0xffffffffu, cur, j & 31), p = __shfl_sync(0xffffffffu, prev, j & 31);
		return j >= i0 ? c : p;
	}
};

__global__ void __launch_bounds__(CHAIN_WARPS * 32) chain_fill_kernel(const int32_t *list, const int64_t *a_off, const int32_t *cnt, const uint64_t *a_all, int n_prob, Par par,
                                                                     int32_t *f_all, int32_t *p_all, int32_t *t_all)
{
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int slot = blockIdx.x * CHAIN_WARPS + warp;
	if (slot >= n_prob) return;
	const int prob = list ? list[slot] : slot;
	const int64_t base = a_off[prob];
	const int32_t n = cnt ? cnt[prob] : (int32_t)(a_off[prob + 1] - base);
	const uint64_t *a = a_all + base;
	int32_t *f = f_all + base, *p = p_all + base, *t = t_all + base;
	for (int32_t i = lane; i < n; i += 32) __stcg(t + i, 0);
	__syncwarp();
	AnchorBlocks ab;
	ab.init(a, n, lane);
	int32_t fcur = 0, fprev = 0, pcur = -1, pprev = -1; // f and p of the same two blocks (lane l: anchor i0 + l resp. i0 - 32 + l)
	int32_t st = 0, hi = -1, hf = 0;
	uint64_t a_hi = 0;
	for (int32_t i = 0; i < n; ++i) {
		if (i && (i & 31) == 0) ab.enter(a, n, i, lane), fprev = fcur, pprev = pcur;
		{ // Runs of ISOLATED anchors -- farther than the window from their immediate predecessor, hence from everybody before
		  // them -- need no scan: st = i, the rescue anchor is out of reach, f = kmer, p = -1, and each becomes the rescue
		  // anchor of the next.  The lanes settle the rest of the block's run at once.
			const uint64_t mine = ab.cur;
			uint64_t left = __shfl_up_sync(0xffffffffu, mine, 1);
			const uint64_t last_prev = __shfl_sync(0xffffffffu, ab.prev, 31);
			if (lane == 0) left = last_prev;
			const int32_t idx = ab.i0 + lane;
			const bool iso = idx < n && (idx == 0 || (((int64_t)(mine >> 32) - (int64_t)(left >> 32)) << par.bbit) > par.max_dist_x);
			const uint32_t m = __ballot_sync(0xffffffffu, iso) >> (i & 31);
			const int run = ~m ? __ffs(~m) - 1 : 32; // consecutive isolated anchors from i on (within the block)
			if (run > 0) {
				if (lane >= (i & 31) && lane < (i & 31) + run) {
					__stcg(f + idx, par.kmer), __stcg(p + idx, -1);
					fcur = par.kmer, pcur = -1;
				}
				i += run - 1;
				st = i, hf = par.kmer, hi = i, a_hi = __shfl_sync(0xffffffffu, mine, i & 31);
				continue;
			}
		}
		const uint64_t ai = __shfl_sync(0xffffffffu, ab.cur, i & 31);
		const int64_t xi = (int64_t)(ai >> 32);
		while (st < i && ((xi - (int64_t)(ab.at(a, st) >> 32)) << par.bbit) > par.max_dist_x) ++st;
		int32_t max_f = par.kmer, max_j = -1, n_skip = 0;
		if (hi >= 0 && hi >= st) { // chain.c:185-189: rescue through the best anchor so far
			const int32_t sc = hf + pair_score(par, ai, a_hi);
			if (sc > max_f) max_f = sc, max_j = hi;
		} else hf = 0, hi = -1;
		if (i - st > par.max_iter) st = i - par.max_iter;
		bool any_mark = false; // has any t[] been set to i yet?
		for (int32_t jb = i - 1; jb >= st; jb -= 32) {
			const int32_t j = jb - lane;
			const bool near = jb == i - 1; // first chunk: j in [i - 32, i - 1], all in the register blocks
			bool ok = j >= st;
			int32_t sc = INT32_MIN, pj = -1;
			uint64_t aj = 0;
			int32_t fj = 0;
			if (near) {
				aj = ab.near(j);
				const int32_t fc = __shfl_sync(0xffffffffu, fcur, j & 31), fp = __shfl_sync(0xffffffffu, fprev, j & 31);
				const int32_t pc = __shfl_sync(0xffffffffu, pcur, j & 31), pp = __shfl_sync(0xffffffffu, pprev, j & 31);
				fj = j >= ab.i0 ? fc : fp, pj = j >= ab.i0 ? pc : pp;
			} else if (ok) aj = a[j];
			if (ok) {
				sc = pair_score(par, ai, aj);
				ok = sc != INT32_MIN;
				if (ok) {
					if (!near) fj = __ldcg(f + j), pj = __ldcg(p + j);
					sc += fj;
				}
			}
			if (!ok) pj = -1;
			const bool mark = ok && pj >= 0;
			if (mark) __stcg(t + pj, i);
			any_mark = any_mark || __any_sync(0xffffffffu, mark);
			__syncwarp();
			const bool marked = any_mark && ok && __ldcg(t + j) == i;
			// running maximum in scan order (lane 0 first)
			int32_t pm = ok ? sc : INT32_MIN;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const int32_t o = __shfl_up_sync(0xffffffffu, pm, d);
				if (lane >= d) pm = pm > o ? pm : o;
			}
			int32_t before = __shfl_up_sync(0xffffffffu, pm, 1);
			if (lane == 0) before = INT32_MIN;
			before = before > max_f ? before : max_f;
			const bool rec = ok && sc > before;
			const uint32_t R = __ballot_sync(0xffffffffu, rec), S = __ballot_sync(0xffffffffu, ok && !rec && marked);
			const int brk = resolve_chunk(R, S, par.max_skip, n_skip);
			const uint32_t Rb = brk >= 32 ? R : (R & ((1u << brk) - 1u));
			if (Rb) {
				const int top = 31 - __clz(Rb);
				max_f = __shfl_sync(0xffffffffu, sc, top), max_j = jb - top;
			}
			if (brk < 32) break;
		}
		if (lane == 0) __stcg(f + i, max_f), __stcg(p + i, max_j);
		if (lane == (i & 31)) fcur = max_f, pcur = max_j;
		__syncwarp();
		if (hf < max_f) hf = max_f, hi = i, a_hi = ai;
	}
}

// Warp-cooperative form of flagsort.hpp::flag_sort_by for records in shared memory: identical permutation (every pass
// and every insertion sort acts on the same disjoint range with the same sequential semantics), but the histogram, the
// key-range scan and the many small insertion sorts are spread over the 32 lanes; only the cycle-leader permutation of
// a pass -- the part whose order defines the reference's tie order -- stays on lane 0.
struct WarpSortScratch { uint32_t cnt[256]; uint32_t head[256]; uint32_t tail[256]; int top; };

template <class KeyFn>
__device__ void flag_sort_warp(uint64_t *rec, int n, KeyFn key, FlagRange<uint64_t> *stack, WarpSortScratch *ws, int lane)
{
	if (n <= 64) {
		if (lane == 0) insertion_sort_by(rec, rec + n, key);
		__syncwarp();
		return;
	}
	if (lane == 0) ws->top = 1, stack[0] = FlagRange<uint64_t>{rec, rec + n, 56};
	__syncwarp();
	while (ws->top > 0) {
		const FlagRange<uint64_t> r = stack[ws->top - 1];
		__syncwarp();
		if (lane == 0) ws->top -= 1;
		const int m = (int)(r.end - r.beg);
		uint64_t lo = ~0ULL, hi = 0;
		for (int i = lane; i < m; i += 32) { const uint64_t k = key(r.beg[i]); lo = k < lo ? k : lo, hi = k > hi ? k : hi; }
		for (int d = 16; d; d >>= 1) {
			const uint64_t ol = __shfl_xor_sync(0xffffffffu, lo, d), oh = __shfl_xor_sync(0xffffffffu, hi, d);
			lo = ol < lo ? ol : lo, hi = oh > hi ? oh : hi;
		}
		int shift = r.shift;
		while (shift > 0 && (lo >> shift) == (hi >> shift)) shift -= 8; // passes that cannot move anything
		if (shift == 0 && lo == hi) { __syncwarp(); continue; }
		for (int k = lane; k < 256; k += 32) ws->cnt[k] = 0;
		__syncwarp();
		for (int i = lane; i < m; i += 32) atomicAdd(&ws->cnt[(key(r.beg[i]) >> shift) & 255], 1u);
		__syncwarp();
		if (lane == 0) {
			uint32_t acc = 0;
			for (int k = 0; k < 256; ++k) ws->head[k] = acc, acc += ws->cnt[k], ws->tail[k] = acc;
		}
		__syncwarp();
		{
			// The cycle-leader permutation (ksort.h:133-146).  Its order defines the reference's tie order, so the chase of a
			// cycle stays sequential (lane 0).  What the lanes share is the part that moves nothing: the run of items at the
			// head of bucket k that already carry digit k is skipped 32 at a time (in a chaining problem most scores are equal --
			// the floor score of isolated anchors -- and sit in one huge bucket that is almost entirely in place).
			uint64_t *b = r.beg;
			for (int k = 0; k < 256; ++k) {
				for (;;) {
					const uint32_t h = ws->head[k], e = ws->tail[k];
					if (h >= e) break;
					const uint32_t idx = h + (uint32_t)lane;
					const bool misplaced = idx < e && (int)((key(b[idx]) >> shift) & 255) != k;
					const uint32_t mm = __ballot_sync(0xffffffffu, misplaced);
					__syncwarp();
					if (mm == 0) { // all of the next 32 (or all that are left) are in place
						if (lane == 0) ws->head[k] = h + 32 < e ? h + 32 : e;
						__syncwarp();
						continue;
					}
					if (lane == 0) {
						const uint32_t at = h + (uint32_t)(__ffs(mm) - 1); // items before it are in place: skipped
						uint64_t hand = b[at];
						int d = (int)((key(hand) >> shift) & 255);
						ws->head[k] = at;
						do {
							const uint64_t next = b[ws->head[d]];
							b[ws->head[d]++] = hand;
							hand = next;
							d = (int)((key(hand) >> shift) & 255);
						} while (d != k);
						b[ws->head[k]++] = hand;
					}
					__syncwarp();
				}
			}
		}
		__syncwarp();
		if (shift > 0) {
			for (int k = lane; k < 256; k += 32) { // buckets are disjoint: refine them in parallel
				const uint32_t e = ws->tail[k], bgn = k ? ws->tail[k - 1] : 0;
				if (e - bgn > 64) { const int slot = atomicAdd(&ws->top, 1); stack[slot] = FlagRange<uint64_t>{r.beg + bgn, r.beg + e, shift - 8}; }
				else if (e - bgn > 1) insertion_sort_by(r.beg + bgn, r.beg + e, key);
			}
		}
		__syncwarp();
	}
}

// Result of the block-level pre-chain (map.c:189-192): the reference compacts the accepted chains and then re-sorts the kept
// anchors with a plain 64-bit radix sort whose key is the WHOLE anchor -- i.e. it ends up with the accepted anchors in
// their original sorted order.  So: mark them (v[0..n_v) from the peeling) and stream-compact the sorted input.
template <class T>
__device__ int32_t keep_filter_warp(int32_t n, int32_t n_v, const int32_t *v, T *t, const uint64_t *a, uint64_t *b, int lane)
{
	for (int32_t i = lane; i < n; i += 32) t[i] = 0;
	__syncwarp();
	for (int32_t k = lane; k < n_v; k += 32) t[v[k]] = 1;
	__syncwarp();
	int32_t o = 0;
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		const bool keep = i < n && t[i] != 0;
		const uint32_t m = __ballot_sync(0xffffffffu, keep);
		if (keep) b[o + __popc(m & ((1u << lane) - 1u))] = a[i];
		o += __popc(m);
	}
	return o;
}

// Whole mp_chain for one problem in ONE warp with all per-anchor state in shared memory: scores f (int32), predecessors p
// and scan marks t (int16: fewer than 32768 anchors), sort records (8 B).  Phase 1 is the score fill of chain_fill_kernel
// with shared-memory state (an L2 round trip per dependent access otherwise dominates: ~2 us per anchor), phase 2 the
// backtrack: lanes gather the (score, index) records and clear the marks, the warp-cooperative flag sort orders them with
// the reference's tie order, lane 0 peels chains best-first and compacts; the pre-chain re-sorts the kept anchors.
__global__ void __launch_bounds__(32) chain_smem_kernel(const int32_t *list, int n_list, int cap, const int64_t *a_off, const int32_t *cnt, const uint64_t *a_all,
                                                       Par par, int32_t *v_all, FlagRange<uint64_t> *stack_all, uint64_t *u_all, uint64_t *b_all,
                                                       int32_t *n_u_out, int32_t *n_b_out, int resort)
{
	extern __shared__ uint64_t zs[];
	__shared__ WarpSortScratch ws;
	if ((int)blockIdx.x >= n_list) return;
	const int prob = list[blockIdx.x], lane = threadIdx.x;
	const int64_t base = a_off[prob];
	const int32_t n = cnt ? cnt[prob] : (int32_t)(a_off[prob + 1] - base);
	const uint64_t *a = a_all + base;
	int32_t *f = (int32_t*)(zs + cap);
	int16_t *p = (int16_t*)(f + cap), *t = p + cap;
	for (int32_t i = lane; i < n; i += 32) t[i] = 0;
	__syncwarp();
	// ---- phase 1: fill (chain.c:181-209), identical logic to chain_fill_kernel
	AnchorBlocks ab;
	ab.init(a, n, lane);
	int32_t st = 0, hi = -1, hf = 0;
	uint64_t a_hi = 0;
	for (int32_t i = 0; i < n; ++i) {
		if (i && (i & 31) == 0) ab.enter(a, n, i, lane);
		{ // runs of isolated anchors, see chain_fill_kernel
			const uint64_t mine = ab.cur;
			uint64_t left = __shfl_up_sync(0xffffffffu, mine, 1);
			const uint64_t last_prev = __shfl_sync(0xffffffffu, ab.prev, 31);
			if (lane == 0) left = last_prev;
			const int32_t idx = ab.i0 + lane;
			const bool iso = idx < n && (idx == 0 || (((int64_t)(mine >> 32) - (int64_t)(left >> 32)) << par.bbit) > par.max_dist_x);
			const uint32_t m = __ballot_sync(0xffffffffu, iso) >> (i & 31);
			const int run = ~m ? __ffs(~m) - 1 : 32;
			if (run > 0) {
				if (lane >= (i & 31) && lane < (i & 31) + run) f[idx] = par.kmer, p[idx] = -1;
				__syncwarp();
				i += run - 1;
				st = i, hf = par.kmer, hi = i, a_hi = __shfl_sync(0xffffffffu, mine, i & 31);
				continue;
			}
		}
		const uint64_t ai = __shfl_sync(0xffffffffu, ab.cur, i & 31);
		const int64_t xi = (int64_t)(ai >> 32);
		while (st < i && ((xi - (int64_t)(ab.at(a, st) >> 32)) << par.bbit) > par.max_dist_x) ++st;
		int32_t max_f = par.kmer, max_j = -1, n_skip = 0;
		if (hi >= 0 && hi >= st) {
			const int32_t sc = hf + pair_score(par, ai, a_hi);
			if (sc > max_f) max_f = sc, max_j = hi;
		} else hf = 0, hi = -1;
		if (i - st > par.max_iter) st = i - par.max_iter;
		for (int32_t jb = i - 1; jb >= st; jb -= 32) {
			const int32_t j = jb - lane;
			bool ok = j >= st;
			int32_t sc = INT32_MIN, pj = -1;
			uint64_t aj = 0;
			if (jb == i - 1) aj = ab.near(j); // first chunk: the anchors are in the register blocks
			else if (ok) aj = a[j];
			if (ok) {
				sc = pair_score(par, ai, aj);
				ok = sc != INT32_MIN;
				if (ok) sc += f[j], pj = p[j];
			}
			if (ok && pj >= 0) t[pj] = (int16_t)i;
			__syncwarp();
			const bool marked = ok && t[j] == (int16_t)i;
			int32_t pm = ok ? sc : INT32_MIN;
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const int32_t o = __shfl_up_sync(0xffffffffu, pm, d);
				if (lane >= d) pm = pm > o ? pm : o;
			}
			int32_t before = __shfl_up_sync(0xffffffffu, pm, 1);
			if (lane == 0) before = INT32_MIN;
			before = before > max_f ? before : max_f;
			const bool rec = ok && sc > before;
			const uint32_t R = __ballot_sync(0xffffffffu, rec), S = __ballot_sync(0xffffffffu, ok && !rec && marked);
			const int brk = resolve_chunk(R, S, par.max_skip, n_skip);
			const uint32_t Rb = brk >= 32 ? R : (R & ((1u << brk) - 1u));
			if (Rb) {
				const int top = 31 - __clz(Rb);
				max_f = __shfl_sync(0xffffffffu, sc, top), max_j = jb - top;
			}
			if (brk < 32) break;
		}
		if (lane == 0) f[i] = max_f, p[i] = (int16_t)max_j;
		__syncwarp();
		if (hf < max_f) hf = max_f, hi = i, a_hi = ai;
	}
	// ---- phase 2: backtrack + compaction (chain.c:26-110)
	int32_t n_z = 0;
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		const bool keep = i < n && f[i] >= par.min_sc;
		if (i < n) t[i] = 0;
		const uint32_t m = __ballot_sync(0xffffffffu, keep);
		if (keep) zs[n_z + __popc(m & ((1u << lane) - 1u))] = (uint64_t)(uint32_t)f[i] << 32 | (uint32_t)i;
		n_z += __popc(m);
	}
	__syncwarp();
	int32_t n_u = 0, n_b = 0;
	FlagRange<uint64_t> *stack = stack_all + (int64_t)prob * CHAIN_STACK;
	flag_sort_warp(zs, n_z, [](const uint64_t &e) { return rec_key(e); }, stack, &ws, lane);
	int32_t n_v = 0;
	if (lane == 0 && n > 0) n_u = peel_chains<int16_t, true, int32_t, int16_t>(par, n_z, f, p, t, v_all + base, zs, stack, u_all + base, &n_v);
	n_u = __shfl_sync(0xffffffffu, n_u, 0), n_v = __shfl_sync(0xffffffffu, n_v, 0);
	__syncwarp();
	if (resort) n_b = keep_filter_warp(n, n_v, v_all + base, t, a, b_all + base, lane); // pre-chain: accepted anchors in sorted order
	else {
		if (n > 0) compact_chains(n_u, a, f, v_all + base, zs, stack, u_all + base, b_all + base, &n_b, lane, 32, [] { __syncwarp(); });
		__syncwarp();
		n_b = __shfl_sync(0xffffffffu, n_b, 0);
	}
	if (lane == 0) n_u_out[prob] = n_u, n_b_out[prob] = n_b;
}

// Backtrack + compaction, one WARP per problem, after the global-memory fill.  The peeling is a chain of dependent
// accesses (predecessor -> mark -> score, three passes over every chain), so everything it touches sits in shared memory:
// sort records (8 B), scores as uint16 (2 B), predecessors as int16 (2 B), marks (1 B) -- 13 B per anchor.  A problem
// with a chain score of 65536 or more (never seen; a protein would need > 10^4 residues in one chain) reads its scores from
// global memory instead.  Lanes cooperate on the parallel parts (loading, gathering the (score, index) records in order,
// the flag sort, the compaction copy, re-sorting the kept anchors); lane 0 peels.
__global__ void __launch_bounds__(32) chain_bt_smem_kernel(const int32_t *list, int n_list, int cap, const int64_t *a_off, const int32_t *cnt, const uint64_t *a_all,
                                                          Par par, int32_t *f_all, const int32_t *p_all, int32_t *v_all, FlagRange<uint64_t> *stack_all,
                                                          uint64_t *u_all, uint64_t *b_all, int32_t *n_u_out, int32_t *n_b_out, int resort)
{
	extern __shared__ uint64_t zs[];
	__shared__ WarpSortScratch ws;
	if ((int)blockIdx.x >= n_list) return;
	const int prob = list[blockIdx.x], lane = threadIdx.x;
	const int64_t base = a_off[prob];
	const int32_t n = cnt ? cnt[prob] : (int32_t)(a_off[prob + 1] - base);
	uint16_t *fs = (uint16_t*)(zs + cap);
	int16_t *ps = (int16_t*)(fs + cap);
	int8_t *ts = (int8_t*)(ps + cap);
	int32_t *fg = f_all + base;
	const int32_t *pg = p_all + base;
	int32_t n_z = 0;
	bool wide = false;
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		const int32_t fi = i < n ? fg[i] : 0;
		const bool keep = i < n && fi >= par.min_sc;
		if (i < n) ts[i] = 0, ps[i] = (int16_t)pg[i], fs[i] = (uint16_t)fi;
		wide |= fi > 65535;
		const uint32_t m = __ballot_sync(0xffffffffu, keep);
		if (keep) zs[n_z + __popc(m & ((1u << lane) - 1u))] = (uint64_t)(uint32_t)fi << 32 | (uint32_t)i;
		n_z += __popc(m);
	}
	wide = __any_sync(0xffffffffu, wide);
	__syncwarp();
	int32_t n_u = 0, n_b = 0;
	FlagRange<uint64_t> *stack = stack_all + (int64_t)prob * CHAIN_STACK;
	int32_t *v = v_all + base;
	uint64_t *u = u_all + base, *b = b_all + base;
	flag_sort_warp(zs, n_z, [](const uint64_t &e) { return rec_key(e); }, stack, &ws, lane); // chain ends by score, reference tie order
	int32_t n_v = 0;
	if (lane == 0 && n > 0) {
		if (!wide) n_u = peel_chains<int8_t, true, uint16_t, int16_t>(par, n_z, fs, ps, ts, v, zs, stack, u, &n_v);
		else n_u = peel_chains<int8_t, true, int32_t, int16_t>(par, n_z, fg, ps, ts, v, zs, stack, u, &n_v);
	}
	n_u = __shfl_sync(0xffffffffu, n_u, 0), n_v = __shfl_sync(0xffffffffu, n_v, 0);
	__syncwarp();
	if (resort) n_b = keep_filter_warp(n, n_v, v, ts, a_all + base, b, lane); // pre-chain: accepted anchors in sorted order
	else {
		if (n > 0) {
			if (!wide) compact_chains(n_u, a_all + base, fs, v, zs, stack, u, b, &n_b, lane, 32, [] { __syncwarp(); });
			else compact_chains(n_u, a_all + base, fg, v, zs, stack, u, b, &n_b, lane, 32, [] { __syncwarp(); });
		}
		__syncwarp();
		n_b = __shfl_sync(0xffffffffu, n_b, 0);
	}
	if (lane == 0) n_u_out[prob] = n_u, n_b_out[prob] = n_b;
}

// Same for problems too large for shared memory (more than 16384 anchors: every pre-chain problem of a gigabase genome): one
// WARP per problem, everything in global memory (L2).  The lanes share what is parallel -- gathering the (score, index)
// records, the flag sort's histograms / range scans / skipping of items already in place, the compaction -- and lane 0 does what
// is sequential by definition: the cycle chases of the sort and the best-first peeling, which only visits anchors of chains
// above the floor score (a small fraction of a pre-chain problem).
__global__ void __launch_bounds__(32) chain_bt_global_kernel(const int32_t *list, int n_list, const int64_t *a_off, const int32_t *cnt, const uint64_t *a_all, Par par,
                                                            int32_t *f_all, const int32_t *p_all, int32_t *t_all, int32_t *v_all, uint64_t *z_all,
                                                            FlagRange<uint64_t> *stack_all, uint64_t *u_all, uint64_t *b_all, int32_t *n_u_out, int32_t *n_b_out, int resort)
{
	__shared__ WarpSortScratch ws;
	if ((int)blockIdx.x >= n_list) return;
	const int prob = list[blockIdx.x], lane = threadIdx.x;
	const int64_t base = a_off[prob];
	const int32_t n = cnt ? cnt[prob] : (int32_t)(a_off[prob + 1] - base);
	int32_t *f = f_all + base, *t = t_all + base, *v = v_all + base;
	const int32_t *pp = p_all + base;
	uint64_t *z = z_all + base, *u = u_all + base, *b = b_all + base;
	const uint64_t *a = a_all + base;
	int32_t n_z = 0;
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		const int32_t fi = i < n ? __ldcg(f + i) : 0;
		const bool keep = i < n && fi >= par.min_sc;
		if (i < n) t[i] = 0;
		const uint32_t m = __ballot_sync(0xffffffffu, keep);
		if (keep) z[n_z + __popc(m & ((1u << lane) - 1u))] = (uint64_t)(uint32_t)fi << 32 | (uint32_t)i;
		n_z += __popc(m);
	}
	__syncwarp();
	int32_t n_u = 0, n_b = 0, n_v = 0;
	FlagRange<uint64_t> *stack = stack_all + (int64_t)prob * CHAIN_STACK;
	flag_sort_warp(z, n_z, [](const uint64_t &e) { return rec_key(e); }, stack, &ws, lane);
	if (lane == 0 && n > 0) n_u = peel_chains<int32_t, true, int32_t, int32_t>(par, n_z, f, pp, t, v, z, stack, u, &n_v);
	n_u = __shfl_sync(0xffffffffu, n_u, 0), n_v = __shfl_sync(0xffffffffu, n_v, 0);
	__syncwarp();
	if (resort) n_b = keep_filter_warp(n, n_v, v, t, a, b, lane); // pre-chain: accepted anchors in sorted order
	else {
		if (n > 0) compact_chains(n_u, a, f, v, z, stack, u, b, &n_b, lane, 32, [] { __syncwarp(); });
		__syncwarp();
		n_b = __shfl_sync(0xffffffffu, n_b, 0);
	}
	if (lane == 0) n_u_out[prob] = n_u, n_b_out[prob] = n_b;
}

void chain_launch_fill(cudaStream_t st, const int32_t *list, const int64_t *a_off, const int32_t *cnt, const uint64_t *a, int n_prob, const Par &par, int32_t *f, int32_t *p,
                       int32_t *t)
{
	if (n_prob > 0) chain_fill_kernel<<<(n_prob + CHAIN_WARPS - 1) / CHAIN_WARPS, CHAIN_WARPS * 32, 0, st>>>(list, a_off, cnt, a, n_prob, par, f, p, t);
}

void chain_launch_smem(cudaStream_t st, const int32_t *list, int n_list, int cap, const int64_t *a_off, const int32_t *cnt, const uint64_t *a, const Par &par, int32_t *v,
                       void *stack, uint64_t *u, uint64_t *b, int32_t *n_u, int32_t *n_b, int resort)
{
	if (n_list <= 0) return;
	const int smem = cap * 16 + 16;
	static SmemLimit lim; // raised on demand, per device
	lim.raise(chain_smem_kernel, smem);
	chain_smem_kernel<<<n_list, 32, smem, st>>>(list, n_list, cap, a_off, cnt, a, par, v, (FlagRange<uint64_t>*)stack, u, b, n_u, n_b, resort);
}

void chain_launch_bt_smem(cudaStream_t st, const int32_t *list, int n_list, int cap, const int64_t *a_off, const int32_t *cnt, const uint64_t *a, const Par &par,
                          int32_t *f, const int32_t *p, int32_t *v, void *stack, uint64_t *u, uint64_t *b, int32_t *n_u, int32_t *n_b, int resort)
{
	if (n_list <= 0) return;
	const int smem = cap * 13 + 16;
	static SmemLimit lim; // raised on demand, per device
	lim.raise(chain_bt_smem_kernel, smem);
	chain_bt_smem_kernel<<<n_list, 32, smem, st>>>(list, n_list, cap, a_off, cnt, a, par, f, p, v, (FlagRange<uint64_t>*)stack, u, b, n_u, n_b, resort);
}

void chain_launch_bt(cudaStream_t st, const int32_t *list, int n_list, const int64_t *a_off, const int32_t *cnt, const uint64_t *a, const Par &par, int32_t *f,
                     const int32_t *p, int32_t *t, int32_t *v, void *z, void *stack, uint64_t *u, uint64_t *b, int32_t *n_u, int32_t *n_b, int resort)
{
	if (n_list > 0)
		chain_bt_global_kernel<<<n_list, 32, 0, st>>>(list, n_list, a_off, cnt, a, par, f, p, t, v, (uint64_t*)z, (FlagRange<uint64_t>*)stack, u, b, n_u, n_b, resort);
}

} // namespace cuda
} // namespace mpb
