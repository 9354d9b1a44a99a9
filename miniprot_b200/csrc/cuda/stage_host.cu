// stage_host.cu -- host drivers of the seeding+chaining stage (S1) and the refinement stage (S2): buffer layout
// in HBM, kernel sequence, and the few small device->host hops needed to size the next buffers.
//
// S1 per mini-batch (map.c:155-195):
//   sketch+occupancy kernel -> [D2H: anchors per protein] -> per slice of proteins: expand -> segmented sort -> pre-chain
//   fill/backtrack (kept anchors re-sorted on device) -> main-chain fill/backtrack -> gather -> [D2H: chains + anchors]
// S2 per mini-batch (map.c:41-97):
//   protein 5-mers -> sort -> window count -> [D2H: anchors per window] -> per slice of windows: window emit -> segmented sort ->
//   chain fill/backtrack -> gather -> [D2H] -> host keeps the best chain of each window
// The slices keep the arenas that grow with the anchors within the context's device-memory allowance (slices.hpp, devbuf.hpp
// Ledger).  Every protein and window is independent of the rest of its batch, so the results are those of one pass; with room to
// spare there is one slice, and the launch sequence is that of one pass over the batch.
#include <algorithm>
#include <numeric>
#include "ctx.hpp"
#include "stages_dev.hpp"
#include "chain_dev.hpp"
#include "seed_dev.hpp"
#include "../slices.hpp"

namespace mpb {
namespace cuda {

__global__ void gather_u64_kernel(const uint64_t *src, const int64_t *src_off, const int32_t *cnt, uint64_t *dst, const int64_t *dst_off, int n_seg)
{
	const int s = blockIdx.x;
	if (s >= n_seg) return;
	const uint64_t *from = src + src_off[s];
	uint64_t *to = dst + dst_off[s];
	for (int i = threadIdx.x; i < cnt[s]; i += blockDim.x) to[i] = from[i];
}

static void fill_seed_const(const mp_idx_t *mi, const mp_mapopt_t *opt, SeedConst &c)
{
	memcpy(c.aa13, ns_tab_aa13, 256);
	memcpy(c.codon, ns_tab_codon, 64);
	memcpy(c.codon13, ns_tab_codon13, 64);
	c.kmer = mi->opt.kmer, c.mod_bit = mi->opt.mod_bit, c.max_occ = opt->max_occ, c.n_kb = mi->n_kb;
}

static chn::Par chain_par(int32_t mdx, int32_t mdy, int32_t bw, const mp_mapopt_t *o, int32_t min_cnt, int32_t min_sc, int32_t kmer, int32_t bbit)
{
	chn::Par p;
	p.max_dist_x = mdx, p.max_dist_y = mdy, p.bw = bw, p.max_skip = o->max_chn_max_skip, p.max_iter = o->max_chn_iter, p.min_cnt = min_cnt, p.min_sc = min_sc;
	p.chn_coef_log = o->chn_coef_log, p.is_spliced = !(o->flag & MP_F_NO_SPLICE), p.kmer = kmer, p.bbit = bbit;
	return chn::normalise(p);
}

// simple bump allocator over one grow-only device arena
struct Carver {
	char *base;
	size_t used = 0;
	explicit Carver(void *p) : base((char*)p) {}
	template <class T> T *take(size_t n) { used = (used + 255) & ~(size_t)255; T *r = (T*)(base + used); used += sizeof(T) * n; return r; }
};
template <class F> static size_t carve_size(F f) { Carver c(0); f(c); return c.used + 256; }

// chain scratch of n_prob problems over N anchors (b_c[8]): 72 B per anchor, a stack of CHAIN_STACK * 24 B and a few counters per problem
struct ChainScratch {
	int32_t *f, *p, *t, *v, *d_nu, *d_nb, *d_nu2, *d_nb2, *d_list;
	uint64_t *z, *du, *db, *du2, *db2, *gu, *gb;
	int64_t *d_go_u, *d_go_b;
	void *stack;
	void layout(Carver &c, int n_prob, size_t N)
	{
		f = c.take<int32_t>(N + 1), p = c.take<int32_t>(N + 1), t = c.take<int32_t>(N + 1), v = c.take<int32_t>(N + 1);
		z = c.take<uint64_t>(N + 1);
		d_list = c.take<int32_t>((size_t)n_prob);
		du = c.take<uint64_t>(N + 1), db = c.take<uint64_t>(N + 1), du2 = c.take<uint64_t>(N + 1), db2 = c.take<uint64_t>(N + 1);
		gu = c.take<uint64_t>(N + 1), gb = c.take<uint64_t>(N + 1);
		d_nu = c.take<int32_t>((size_t)n_prob), d_nb = c.take<int32_t>((size_t)n_prob), d_nu2 = c.take<int32_t>((size_t)n_prob), d_nb2 = c.take<int32_t>((size_t)n_prob);
		d_go_u = c.take<int64_t>((size_t)n_prob + 1), d_go_b = c.take<int64_t>((size_t)n_prob + 1);
		stack = c.take<char>((size_t)n_prob * CHAIN_STACK * 24);
	}
	static size_t bytes(int n_prob, size_t N) { ChainScratch s; return carve_size([&](Carver &c) { s.layout(c, n_prob, N); }); }
};

// ---- slices -----------------------------------------------------------------------------------------------------------------
// Arena bytes of a slice: per anchor the anchors and the sort's ping-pong buffer (b_c[1] / b_c[2] or b_c[5] / b_c[6], 16 B) and, when
// it is chained, the chain scratch (b_c[8], 72 B); per problem its chain stack, counters and sort descriptors; per slice the
// alignment of the carved pieces and the arenas' rounding.
static const int64_t kAnchorBytesChain = 88, kAnchorBytesSeed = 16, kProbBytes = (int64_t)CHAIN_STACK * 24 + 128, kSliceFixed = (int64_t)64 << 10;

static inline size_t anchor_arena(size_t N) { return sizeof(uint64_t) * (N + 2); }

// Cuts the items [0, n) (cnt[i] anchors each) of a stage whose sliced arenas are `mine`: one slice, without asking the device, when
// the budget is automatic and the whole batch fits what they hold (`whole`: each arena's need for one pass); else greedy slices
// within the room the ledger gives them, less the quarter reserve() may add, and the largest slice (with that quarter) is claimed
// until the stage ends (the caller holds a ClaimScope).  Returns that room, or -1 for the first case.
static int64_t plan_items(mpb_ctx_s *ctx, std::initializer_list<DevBuf*> mine, std::initializer_list<size_t> whole, int n, const int64_t *cnt, int64_t per_anchor,
                          SlicePlan &p, int64_t &n_slices)
{
	int64_t room = -1;
	if (ctx->mem.budget == 0 && Ledger::fits(mine, whole)) {
		p.cut.assign(1, 0), p.cut.push_back(n), p.n_over = 0;
	} else {
		std::vector<int64_t> bytes((size_t)n);
		for (int i = 0; i < n; ++i) bytes[(size_t)i] = cnt[i] * per_anchor + kProbBytes;
		room = ctx->mem.plan(mine, [&](int64_t r) {
			plan_slices(n, bytes.data(), cnt, kSliceFixed, r / 5 * 4, kSliceMaxCount, p);
			int64_t most = 0;
			for (int k = 0; k < p.n_slices(); ++k) {
				int64_t s = kSliceFixed;
				for (int i = p.cut[(size_t)k]; i < p.cut[(size_t)k + 1]; ++i) s += bytes[(size_t)i];
				most = std::max(most, s);
			}
			return most / 4 * 5;
		});
	}
	n_slices += p.n_slices(), ctx->mem.n_over_budget += p.n_over;
	return room;
}

// chain n_prob problems whose sorted anchors sit in d_a at d_off[]; returns per-problem chains and compacted anchors
// on the host.  pre != null runs the block-level pre-chain first (map.c:186-192).
static void chain_problems(mpb_ctx_s *ctx, int n_prob, const std::vector<int64_t> &h_off, const int64_t *d_off, uint64_t *d_a, const chn::Par *pre, const chn::Par &mainp,
                           std::vector<int32_t> &n_u, std::vector<int32_t> &n_b, std::vector<uint64_t> &u, std::vector<uint64_t> &bb)
{
	cudaStream_t st = ctx->stream;
	const size_t N = (size_t)h_off[(size_t)n_prob];
	n_u.assign((size_t)n_prob, 0), n_b.assign((size_t)n_prob, 0), u.clear(), bb.clear();
	if (n_prob == 0) return;
	ChainScratch cs;
	ctx->b_c[8].reserve(ChainScratch::bytes(n_prob, N));
	Carver cv(ctx->b_c[8].p);
	cs.layout(cv, n_prob, N);
	int32_t *f = cs.f, *p = cs.p, *t = cs.t, *v = cs.v, *d_nu = cs.d_nu, *d_nb = cs.d_nb, *d_nu2 = cs.d_nu2, *d_nb2 = cs.d_nb2, *d_list = cs.d_list;
	uint64_t *z = cs.z, *du = cs.du, *db = cs.db, *du2 = cs.du2, *db2 = cs.db2, *gu = cs.gu, *gb = cs.gb;
	int64_t *d_go_u = cs.d_go_u, *d_go_b = cs.d_go_b;
	void *stack = cs.stack;
	// Size classes (from the offsets: an upper bound for a main chain that follows a pre-chain), run concurrently on side
	// streams:  0: <= 2048 anchors   fill + backtrack fused in one warp with ALL state in shared memory (32 KB, 7 warps per SM)
	//           1..NC-1: up to 16384 anchors in steps of ~1 K   global-memory fill (every problem its own warp, ~1000 in
	//                flight) followed by the shared-memory backtrack (13 B per anchor of the class capacity: the finer the
	//                classes, the more problems fit an SM's shared memory together)
	//           NC: larger   global-memory fill + single-thread global backtrack
	static const int NC = 11;
	static const int caps[NC] = { 2048, 3072, 4096, 5120, 6144, 7168, 8192, 10240, 12288, 14000, 16384 };
	static const int fused_max = getenv("MPB_CHAIN_FUSED_MAX") ? atoi(getenv("MPB_CHAIN_FUSED_MAX")) : 2048;
	std::vector<int32_t> lists[NC + 1], flat, sizes((size_t)n_prob);
	size_t lfirst[NC + 1];
	for (int i = 0; i < n_prob; ++i) sizes[(size_t)i] = (int32_t)(h_off[(size_t)i + 1] - h_off[(size_t)i]);
	auto classify = [&]() { // sizes[] -> per-class problem lists on the device
		flat.clear();
		for (int c = 0; c <= NC; ++c) lists[c].clear();
		for (int i = 0; i < n_prob; ++i) {
			const int32_t n = sizes[(size_t)i];
			int c = 0;
			while (c < NC && n > caps[c]) ++c;
			lists[c].push_back(i);
		}
		for (int c = 0; c <= NC; ++c) lfirst[c] = flat.size(), flat.insert(flat.end(), lists[c].begin(), lists[c].end());
		MPB_CUDA_OK(cudaMemcpyAsync(d_list, flat.data(), sizeof(int32_t) * flat.size(), cudaMemcpyHostToDevice, st));
	};
	classify();
	auto chain_once = [&](const int32_t *cnt, const uint64_t *in, const chn::Par &par, uint64_t *uo, uint64_t *bo, int32_t *nuo, int32_t *nbo, int resort) {
		MPB_CUDA_OK(cudaEventRecord(ctx->ev_fork, st));
		for (int c = NC; c >= 0; --c) { // largest problems first
			if (lists[c].empty()) continue;
			cudaStream_t ss = ctx->side[c];
			const int32_t *lst = d_list + lfirst[c];
			const int nl = (int)lists[c].size();
			MPB_CUDA_OK(cudaStreamWaitEvent(ss, ctx->ev_fork, 0));
			if (c < NC && caps[c] <= fused_max) {
				chain_launch_smem(ss, lst, nl, caps[c], d_off, cnt, in, par, v, stack, uo, bo, nuo, nbo, resort);
				ctx->stats.kernel_launches += 1;
			} else {
				chain_launch_fill(ss, lst, d_off, cnt, in, nl, par, f, p, t);
				if (c < NC) chain_launch_bt_smem(ss, lst, nl, caps[c], d_off, cnt, in, par, f, p, v, stack, uo, bo, nuo, nbo, resort);
				else chain_launch_bt(ss, lst, nl, d_off, cnt, in, par, f, p, t, v, z, stack, uo, bo, nuo, nbo, resort);
				ctx->stats.kernel_launches += 2;
			}
			MPB_CUDA_OK(cudaEventRecord(ctx->ev_join[c], ss));
			MPB_CUDA_OK(cudaStreamWaitEvent(st, ctx->ev_join[c], 0));
		}
	};
	ctx->time_begin();
	const uint64_t *in = d_a;
	const int32_t *cnt = 0;
	if (pre) {
		chain_once(0, d_a, *pre, du, db, d_nu, d_nb, 1);
		in = db, cnt = d_nb;
		// the pre-chain usually keeps a small fraction of the anchors: re-classify by the true sizes (a 4 B/problem copy)
		MPB_CUDA_OK(cudaMemcpyAsync(sizes.data(), d_nb, sizeof(int32_t) * (size_t)n_prob, cudaMemcpyDeviceToHost, st));
		MPB_CUDA_OK(cudaStreamSynchronize(st));
		classify();
	}
	chain_once(cnt, in, mainp, du2, db2, d_nu2, d_nb2, 0);
	MPB_CUDA_OK(cudaMemcpyAsync(n_u.data(), d_nu2, sizeof(int32_t) * (size_t)n_prob, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaMemcpyAsync(n_b.data(), d_nb2, sizeof(int32_t) * (size_t)n_prob, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	std::vector<int64_t> go_u((size_t)n_prob + 1, 0), go_b((size_t)n_prob + 1, 0);
	for (int i = 0; i < n_prob; ++i) go_u[(size_t)i + 1] = go_u[(size_t)i] + n_u[(size_t)i], go_b[(size_t)i + 1] = go_b[(size_t)i] + n_b[(size_t)i];
	MPB_CUDA_OK(cudaMemcpyAsync(d_go_u, go_u.data(), sizeof(int64_t) * go_u.size(), cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(d_go_b, go_b.data(), sizeof(int64_t) * go_b.size(), cudaMemcpyHostToDevice, st));
	gather_u64_kernel<<<n_prob, 128, 0, st>>>(du2, d_off, d_nu2, gu, d_go_u, n_prob);
	gather_u64_kernel<<<n_prob, 128, 0, st>>>(db2, d_off, d_nb2, gb, d_go_b, n_prob);
	ctx->stats.kernel_launches += 2;
	u.resize((size_t)go_u.back()), bb.resize((size_t)go_b.back());
	if (!u.empty()) MPB_CUDA_OK(cudaMemcpyAsync(u.data(), gu, sizeof(uint64_t) * u.size(), cudaMemcpyDeviceToHost, st));
	if (!bb.empty()) MPB_CUDA_OK(cudaMemcpyAsync(bb.data(), gb, sizeof(uint64_t) * bb.size(), cudaMemcpyDeviceToHost, st));
	ctx->stats.ms_chain += ctx->time_end();
	MPB_CUDA_OK(cudaGetLastError());
	ctx->stats.d2h_bytes += (int64_t)(sizeof(uint64_t) * (u.size() + bb.size()) + 8 * (size_t)n_prob);
	ctx->stats.n_chain_problems += n_prob * (pre ? 2 : 1);
}

// stage-level entry for tests/benchmarks: chain host-provided sorted anchors (mpb_chain_batch)
void chain_batch_run(mpb_ctx_s *ctx, const chn::Par &par, int n_prob, const int64_t *a_off, const uint64_t *a, std::vector<int32_t> &n_u, std::vector<int32_t> &n_b,
                     std::vector<uint64_t> &u, std::vector<uint64_t> &bb)
{
	cudaStream_t st = ctx->stream;
	Busy busy({ &ctx->b_c[1], &ctx->b_c[7], &ctx->b_c[8] });
	std::vector<int64_t> off(a_off, a_off + n_prob + 1);
	const size_t N = (size_t)off[(size_t)n_prob];
	ctx->b_c[1].reserve(sizeof(uint64_t) * (N + 2));
	ctx->b_c[7].reserve(sizeof(int64_t) * ((size_t)n_prob + 2));
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_c[1].p, a, sizeof(uint64_t) * N, cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_c[7].p, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice, st));
	ctx->stats.h2d_bytes += (int64_t)(sizeof(uint64_t) * N);
	chain_problems(ctx, n_prob, off, ctx->b_c[7].as<int64_t>(), ctx->b_c[1].as<uint64_t>(), 0, chn::normalise(par), n_u, n_b, u, bb);
}

// Seeding of a batch (map.c:155-177 per query): sketch, adaptive occupancy cut-off [D2H: anchors per query], then per slice of
// queries the expansion of the index buckets and the sort, handed to fn(q0, q1, a_off, d_a_off, d_a): a_off[q1 - q0 + 1] delimits
// each query's sorted anchors (from 0) inside d_a (ctx->b_c[1]), d_a_off is the same table on the device.  chain: fn chains the
// slice (the plan leaves room for the chain scratch).
template <class F>
static void seed_run(mpb_ctx_s *ctx, const mp_idx_t *mi, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa, bool chain, F fn)
{
	cudaStream_t st = ctx->stream;
	const int n_q = b.n;
	const size_t R = (size_t)aa_off[(size_t)n_q];
	Busy busy({ &ctx->b_aa, &ctx->b_c[0], &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[3], &ctx->b_c[8] });
	ClaimScope claim(ctx->mem);
	SeedConst cst;
	mp_mapopt_t tmp;
	memset(&tmp, 0, sizeof(tmp));
	tmp.max_occ = max_occ;
	fill_seed_const(mi, &tmp, cst);
	int32_t *d_aa_off, *sd_pos, *d_nsd;
	uint32_t *sd_hash;
	int64_t *sd_cnt, *sd_aoff, *d_tot, *d_a_off;
	auto layout = [&](Carver &c) {
		d_aa_off = c.take<int32_t>((size_t)n_q + 1), sd_hash = c.take<uint32_t>(R + 1), sd_pos = c.take<int32_t>(R + 1);
		sd_cnt = c.take<int64_t>(R + 1), sd_aoff = c.take<int64_t>(R + 1), d_nsd = c.take<int32_t>((size_t)n_q), d_tot = c.take<int64_t>((size_t)n_q);
		d_a_off = c.take<int64_t>((size_t)n_q + 1);
	};
	ctx->b_c[0].reserve(carve_size(layout));
	Carver cv(ctx->b_c[0].p);
	layout(cv);
	MPB_CUDA_OK(cudaMemcpyAsync(d_aa_off, aa_off.data(), sizeof(int32_t) * ((size_t)n_q + 1), cudaMemcpyHostToDevice, st));
	ctx->time_begin();
	seed_launch_sketch(st, d_aa, d_aa_off, n_q, cst, ctx->d_ki, sd_hash, sd_pos, sd_cnt, sd_aoff, d_nsd, d_tot);
	std::vector<int64_t> tot((size_t)n_q);
	MPB_CUDA_OK(cudaMemcpyAsync(tot.data(), d_tot, sizeof(int64_t) * (size_t)n_q, cudaMemcpyDeviceToHost, st));
	ctx->stats.ms_seed += ctx->time_end();
	ctx->stats.kernel_launches += 1;
	const size_t N_all = (size_t)std::accumulate(tot.begin(), tot.end(), (int64_t)0);
	SlicePlan plan;
	const int64_t room = plan_items(ctx, { &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[8] },
	                                { anchor_arena(N_all), anchor_arena(N_all), chain ? ChainScratch::bytes(n_q, N_all) : 0 }, n_q, tot.data(),
	                                chain ? kAnchorBytesChain : kAnchorBytesSeed, plan, ctx->mem.n_slices_seed);
	std::vector<int64_t> a_off;
	for (int k = 0; k < plan.n_slices(); ++k) {
		const int q0 = plan.cut[(size_t)k], n = plan.cut[(size_t)k + 1] - q0;
		a_off.assign((size_t)n + 1, 0);
		for (int q = 0; q < n; ++q) a_off[(size_t)q + 1] = a_off[(size_t)q] + tot[(size_t)(q0 + q)];
		const size_t N = (size_t)a_off[(size_t)n];
		if (room >= 0) ctx->mem.trim({ &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[8] }, { anchor_arena(N), anchor_arena(N), chain ? ChainScratch::bytes(n, N) : 0 }, room);
		ctx->time_begin();
		MPB_CUDA_OK(cudaMemcpyAsync(d_a_off, a_off.data(), sizeof(int64_t) * a_off.size(), cudaMemcpyHostToDevice, st));
		ctx->b_c[1].reserve(anchor_arena(N));
		ctx->b_c[2].reserve(anchor_arena(N));
		uint64_t *d_a = ctx->b_c[1].as<uint64_t>(), *d_tmp = ctx->b_c[2].as<uint64_t>();
		seed_launch_expand(st, d_aa_off + q0, n, ctx->d_ki, ctx->d_kb, sd_hash, sd_pos, sd_cnt, sd_aoff, d_nsd + q0, d_a_off, d_a);
		seg_sort_u64(ctx, st, d_a, d_tmp, n, a_off.data(), a_off.data() + 1);
		ctx->stats.ms_seed += ctx->time_end();
		ctx->stats.kernel_launches += 2;
		ctx->stats.n_anchors += (int64_t)N;
		fn(q0, q0 + n, a_off, (const int64_t*)d_a_off, d_a);
	}
}

// sorted anchors of a slice -> appended to a host array (seed_off[q0] is set; seed_off[q0 + 1 ..] are)
static void append_anchors(mpb_ctx_s *ctx, int q0, const std::vector<int64_t> &a_off, const uint64_t *d_a, std::vector<int64_t> &off, std::vector<uint64_t> &a)
{
	const int n = (int)a_off.size() - 1;
	const size_t at = a.size();
	a.resize(at + (size_t)a_off[(size_t)n]);
	if (a.size() > at) MPB_CUDA_OK(cudaMemcpyAsync(a.data() + at, d_a, sizeof(uint64_t) * (a.size() - at), cudaMemcpyDeviceToHost, ctx->stream));
	MPB_CUDA_OK(cudaStreamSynchronize(ctx->stream));
	ctx->stats.d2h_bytes += (int64_t)(sizeof(uint64_t) * (a.size() - at));
	for (int q = 0; q < n; ++q) off[(size_t)(q0 + q) + 1] = off[(size_t)q0] + a_off[(size_t)q + 1];
}

// stage-level entry for tests/benchmarks: seeding only (mpb_seed_batch)
void seed_batch_run(mpb_ctx_s *ctx, const mp_idx_t *mi, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa,
                    std::vector<int64_t> &a_off, std::vector<uint64_t> &a)
{
	a_off.assign((size_t)b.n + 1, 0), a.clear();
	if (b.n == 0) return;
	seed_run(ctx, mi, max_occ, b, aa_off, d_aa, false, [&](int q0, int, const std::vector<int64_t> &so, const int64_t *, uint64_t *d_a) {
		append_anchors(ctx, q0, so, d_a, a_off, a);
	});
}

// map.c:186-195: pre-chain and main chain of the sorted seeds of queries [q0, q0 + n) (d_a at a_off, from 0), appended to out
static void chain_seeds(mpb_ctx_s *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, int q0, const std::vector<int64_t> &a_off, const int64_t *d_a_off, uint64_t *d_a,
                        ChainSet &out)
{
	const int n = (int)a_off.size() - 1;
	const int32_t w = 1 << mi->opt.bbit, spl = !(opt->flag & MP_F_NO_SPLICE);
	const chn::Par pre = chain_par(w, w, w, opt, 2, 0, mi->opt.kmer, mi->opt.bbit);
	const chn::Par mainp = chain_par(opt->max_intron, opt->max_gap, opt->bw, opt, opt->min_chn_cnt, opt->min_chn_sc, mi->opt.kmer, mi->opt.bbit);
	std::vector<int32_t> n_u, n_b;
	std::vector<uint64_t> u, bb;
	chain_problems(ctx, n, a_off, d_a_off, d_a, (!(opt->flag & MP_F_NO_PRE_CHAIN) && spl) ? &pre : 0, mainp, n_u, n_b, u, bb);
	for (int q = 0; q < n; ++q) {
		const size_t g = (size_t)(q0 + q);
		out.u_off[g + 1] = out.u_off[g] + n_u[(size_t)q], out.a_off[g + 1] = out.a_off[g] + n_b[(size_t)q];
	}
	if (out.u.empty()) out.u.swap(u); else out.u.insert(out.u.end(), u.begin(), u.end());
	if (out.a.empty()) out.a.swap(bb); else out.a.insert(out.a.end(), bb.begin(), bb.end());
}

void seed_chain_run(mpb_ctx_s *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa, ChainSet &out)
{
	const int n_q = b.n;
	out.u_off.assign((size_t)n_q + 1, 0), out.a_off.assign((size_t)n_q + 1, 0), out.u.clear(), out.a.clear();
	if (n_q == 0) return;
	if (out.want_seeds) out.seed_off.assign((size_t)n_q + 1, 0), out.seed.clear();
	seed_run(ctx, mi, opt->max_occ, b, aa_off, d_aa, true, [&](int q0, int, const std::vector<int64_t> &a_off, const int64_t *d_a_off, uint64_t *d_a) {
		if (out.want_seeds) append_anchors(ctx, q0, a_off, d_a, out.seed_off, out.seed); // --dbg-anchor: the sorted seeds, before chaining reuses the buffers
		chain_seeds(ctx, mi, opt, q0, a_off, d_a_off, d_a, out);
	});
}

// Seeding of a batch of locus sets (map_sets): query q against contigs [ctg_off[q], ctg_off[q+1]) of the locus view vi only, exactly
// what the reference seeds from an index of a genome made of those ranges alone.  The units of all of a query's strands are contiguous,
// so that one segment of join pairs holds the (bucket, block) pairs of the query's whole index.  There is no k-mer table; per batch:
//   protein seeds (prot_kmer_kernel with the mod filter) -> sort per protein -> ORF scan of both strands of every range, keeping the
//   k-mers whose bucket the protein has (count [D2H]); then per slice of pairs (20 B per join pair: the pairs, their distinct keys and
//   blocks): emit -> sort + unique per locus: its (bucket, block) pairs, as index.c:71-90 holds them -> bucket sizes, adaptive
//   occupancy cut-off, anchors per pair [D2H]; and per slice of those pairs by anchors: seed_expand_kernel -> sort per query, handed
//   to fn as seed_run does.
template <class F>
static void seed_loci_run(mpb_ctx_s *ctx, const mp_idx_t *vi, const int32_t *ctg_off, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off,
                          const char *d_aa, bool chain, F fn)
{
	cudaStream_t st = ctx->stream;
	const int n_q = b.n;
	const size_t R = (size_t)aa_off[(size_t)n_q];
	Busy busy({ &ctx->b_aa, &ctx->b_c[0], &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[3], &ctx->b_c[4], &ctx->b_c[5], &ctx->b_c[6], &ctx->b_c[8] });
	ClaimScope claim(ctx->mem);
	SeedConst cst;
	mp_mapopt_t tmp;
	memset(&tmp, 0, sizeof(tmp));
	tmp.max_occ = max_occ;
	fill_seed_const(vi, &tmp, cst);
	std::vector<LocusStrand> strands((size_t)ctg_off[n_q] * 2);
	std::vector<LocusUnit> units;
	std::vector<size_t> unit_first((size_t)n_q + 1, 0);
	for (int q = 0; q < n_q; ++q) {
		for (int k = ctg_off[q]; k < ctg_off[q + 1]; ++k) {
			const mp_ctg_t *c = &vi->nt->ctg[k];
			for (int s = 0; s < 2; ++s) {
				LocusStrand &ls = strands[(size_t)k * 2 + s];
				ls.g_start = s ? c->off + c->len - 1 : c->off, ls.dir = s ? -1 : 1, ls.comp = s, ls.len = c->len, ls.boff = vi->bo[k * 2 + s], ls.qid = q;
				const int64_t step = (int64_t)WIN_TILE * 16;
				for (int64_t p = 0; p < c->len; p += step) units.push_back(LocusUnit{ k * 2 + s, 0, p, std::min(p + step, (int64_t)c->len) });
			}
		}
		unit_first[(size_t)q + 1] = units.size();
	}
	const int n_units = (int)units.size();
	int32_t *d_aa_off, *d_npk, *sd_pos;
	uint32_t *sd_idx;
	uint64_t *d_pk, *d_pk_tmp;
	int64_t *sd_lo, *sd_cnt, *sd_aoff, *d_unit_off, *d_unit_n, *d_seg, *d_nu, *d_tot, *d_a_off;
	LocusUnit *d_units;
	LocusStrand *d_strands;
	auto layout = [&](Carver &c) {
		d_aa_off = c.take<int32_t>((size_t)n_q + 1), d_npk = c.take<int32_t>((size_t)n_q), d_pk = c.take<uint64_t>(R + 1), d_pk_tmp = c.take<uint64_t>(R + 1);
		sd_idx = c.take<uint32_t>(R + 1), sd_pos = c.take<int32_t>(R + 1), sd_lo = c.take<int64_t>(R + 1), sd_cnt = c.take<int64_t>(R + 1), sd_aoff = c.take<int64_t>(R + 1);
		d_units = c.take<LocusUnit>((size_t)n_units + 1), d_strands = c.take<LocusStrand>(strands.size());
		d_unit_off = c.take<int64_t>((size_t)n_units + 1), d_unit_n = c.take<int64_t>((size_t)n_units + 1);
		d_seg = c.take<int64_t>((size_t)n_q + 1), d_nu = c.take<int64_t>((size_t)n_q), d_tot = c.take<int64_t>((size_t)n_q), d_a_off = c.take<int64_t>((size_t)n_q + 1);
	};
	ctx->b_c[0].reserve(carve_size(layout));
	Carver cv(ctx->b_c[0].p);
	layout(cv);
	MPB_CUDA_OK(cudaMemcpyAsync(d_aa_off, aa_off.data(), sizeof(int32_t) * ((size_t)n_q + 1), cudaMemcpyHostToDevice, st));
	if (n_units) MPB_CUDA_OK(cudaMemcpyAsync(d_units, units.data(), sizeof(LocusUnit) * units.size(), cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(d_strands, strands.data(), sizeof(LocusStrand) * strands.size(), cudaMemcpyHostToDevice, st));
	ctx->stats.h2d_bytes += (int64_t)(sizeof(LocusUnit) * units.size() + sizeof(LocusStrand) * strands.size());
	ctx->time_begin();
	// protein seeds, sorted per protein
	seed_launch_prot_kmer(st, d_aa, d_aa_off, n_q, cst, cst.kmer, cst.mod_bit, d_pk, d_npk);
	std::vector<int32_t> n_pk((size_t)n_q);
	MPB_CUDA_OK(cudaMemcpyAsync(n_pk.data(), d_npk, sizeof(int32_t) * (size_t)n_q, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	{
		std::vector<int64_t> sb((size_t)n_q), se((size_t)n_q);
		for (int q = 0; q < n_q; ++q) sb[(size_t)q] = aa_off[(size_t)q], se[(size_t)q] = aa_off[(size_t)q] + n_pk[(size_t)q];
		seg_sort_u64(ctx, st, d_pk, d_pk_tmp, n_q, sb.data(), se.data());
	}
	// the join's count pass over every locus
	locus_launch_join(st, false, d_units, n_units, d_strands, ctx->d_seq, cst, vi->opt.min_aa_len, vi->opt.bbit, d_pk, d_aa_off, d_npk, 0, d_unit_n, 0);
	std::vector<int64_t> unit_n((size_t)n_units + 1, 0), m_q((size_t)n_q, 0);
	if (n_units) MPB_CUDA_OK(cudaMemcpyAsync(unit_n.data(), d_unit_n, sizeof(int64_t) * (size_t)n_units, cudaMemcpyDeviceToHost, st));
	ctx->stats.ms_seed += ctx->time_end();
	ctx->stats.kernel_launches += 2;
	for (int q = 0; q < n_q; ++q)
		for (size_t u = unit_first[(size_t)q]; u < unit_first[(size_t)q + 1]; ++u) m_q[(size_t)q] += unit_n[u];
	const size_t M_all = (size_t)std::accumulate(m_q.begin(), m_q.end(), (int64_t)0);
	// slices of pairs by join pairs: a quarter of the room, the rest is for the anchors of the slices inside
	SlicePlan outer;
	const int64_t room_p = plan_items(ctx, { &ctx->b_c[4], &ctx->b_c[5], &ctx->b_c[6] }, { anchor_arena(M_all), anchor_arena(M_all), sizeof(uint32_t) * (M_all + 2) }, n_q,
	                                  m_q.data(), 20 * 4, outer, ctx->mem.n_slices_loci);
	const int64_t per_anchor = chain ? kAnchorBytesChain : kAnchorBytesSeed;
	std::vector<int64_t> unit_off, seg, tot, a_off;
	for (int k = 0; k < outer.n_slices(); ++k) {
		const int p0 = outer.cut[(size_t)k], np = outer.cut[(size_t)k + 1] - p0;
		const size_t u0 = unit_first[(size_t)p0], nu = unit_first[(size_t)(p0 + np)] - u0;
		unit_off.assign(nu + 1, 0), seg.assign((size_t)np + 1, 0);
		for (size_t u = 0; u < nu; ++u) unit_off[u + 1] = unit_off[u] + unit_n[u0 + u];
		for (int q = 0; q <= np; ++q) seg[(size_t)q] = unit_off[unit_first[(size_t)(p0 + q)] - u0];
		const size_t M = (size_t)seg[(size_t)np];
		if (room_p >= 0) ctx->mem.trim({ &ctx->b_c[4], &ctx->b_c[5], &ctx->b_c[6] }, { anchor_arena(M), anchor_arena(M), sizeof(uint32_t) * (M + 2) }, room_p);
		ctx->time_begin();
		MPB_CUDA_OK(cudaMemcpyAsync(d_unit_off, unit_off.data(), sizeof(int64_t) * unit_off.size(), cudaMemcpyHostToDevice, st));
		MPB_CUDA_OK(cudaMemcpyAsync(d_seg, seg.data(), sizeof(int64_t) * seg.size(), cudaMemcpyHostToDevice, st));
		ctx->b_c[4].reserve(anchor_arena(M)), ctx->b_c[5].reserve(anchor_arena(M)), ctx->b_c[6].reserve(sizeof(uint32_t) * (M + 2));
		uint64_t *d_pairs = ctx->b_c[4].as<uint64_t>(), *d_uniq = ctx->b_c[5].as<uint64_t>();
		uint32_t *d_blk = ctx->b_c[6].as<uint32_t>();
		locus_launch_join(st, true, d_units + u0, (int)nu, d_strands, ctx->d_seq, cst, vi->opt.min_aa_len, vi->opt.bbit, d_pk, d_aa_off, d_npk, d_unit_off, 0, d_pairs);
		seg_sort_u64(ctx, st, d_pairs, d_uniq, np, seg.data(), seg.data() + 1);
		locus_launch_unique(st, d_pairs, d_seg, np, d_uniq, d_blk, d_nu + p0);
		// bucket sizes, occupancy cut-off
		locus_launch_occ(st, d_pk, d_aa_off + p0, d_npk + p0, np, d_uniq, d_seg, d_nu + p0, max_occ, sd_idx, sd_pos, sd_lo, sd_cnt, sd_aoff, d_tot + p0);
		tot.assign((size_t)np, 0);
		MPB_CUDA_OK(cudaMemcpyAsync(tot.data(), d_tot + p0, sizeof(int64_t) * (size_t)np, cudaMemcpyDeviceToHost, st));
		ctx->stats.ms_seed += ctx->time_end();
		ctx->stats.kernel_launches += 3;
		// expansion, by slices of anchors
		const size_t N_all = (size_t)std::accumulate(tot.begin(), tot.end(), (int64_t)0);
		SlicePlan inner;
		const int64_t room = plan_items(ctx, { &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[8] },
		                                { anchor_arena(N_all), anchor_arena(N_all), chain ? ChainScratch::bytes(np, N_all) : 0 }, np, tot.data(), per_anchor, inner,
		                                ctx->mem.n_slices_loci);
		ctx->mem.n_slices_loci -= 1; // an outer slice counts as its inner slices
		for (int j = 0; j < inner.n_slices(); ++j) {
			const int r0 = inner.cut[(size_t)j], n = inner.cut[(size_t)j + 1] - r0;
			a_off.assign((size_t)n + 1, 0);
			for (int q = 0; q < n; ++q) a_off[(size_t)q + 1] = a_off[(size_t)q] + tot[(size_t)(r0 + q)];
			const size_t N = (size_t)a_off[(size_t)n];
			if (room >= 0) ctx->mem.trim({ &ctx->b_c[1], &ctx->b_c[2], &ctx->b_c[8] }, { anchor_arena(N), anchor_arena(N), chain ? ChainScratch::bytes(n, N) : 0 }, room);
			ctx->time_begin();
			MPB_CUDA_OK(cudaMemcpyAsync(d_a_off, a_off.data(), sizeof(int64_t) * a_off.size(), cudaMemcpyHostToDevice, st));
			ctx->b_c[1].reserve(anchor_arena(N));
			ctx->b_c[2].reserve(anchor_arena(N));
			uint64_t *d_a = ctx->b_c[1].as<uint64_t>(), *d_tmp = ctx->b_c[2].as<uint64_t>();
			const int q0 = p0 + r0;
			seed_launch_expand(st, d_aa_off + q0, n, sd_lo, d_blk, sd_idx, sd_pos, sd_cnt, sd_aoff, d_npk + q0, d_a_off, d_a);
			seg_sort_u64(ctx, st, d_a, d_tmp, n, a_off.data(), a_off.data() + 1);
			ctx->stats.ms_seed += ctx->time_end();
			MPB_CUDA_OK(cudaGetLastError());
			ctx->stats.kernel_launches += 1;
			ctx->stats.n_anchors += (int64_t)N;
			fn(q0, q0 + n, a_off, (const int64_t*)d_a_off, d_a);
		}
	}
}

void seed_chain_loci_run(mpb_ctx_s *ctx, const mp_idx_t *vi, const int32_t *ctg_off, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off,
                         const char *d_aa, ChainSet &out)
{
	const int n_q = b.n;
	out.u_off.assign((size_t)n_q + 1, 0), out.a_off.assign((size_t)n_q + 1, 0), out.u.clear(), out.a.clear();
	if (n_q == 0) return;
	seed_loci_run(ctx, vi, ctg_off, opt->max_occ, b, aa_off, d_aa, true, [&](int q0, int, const std::vector<int64_t> &a_off, const int64_t *d_a_off, uint64_t *d_a) {
		chain_seeds(ctx, vi, opt, q0, a_off, d_a_off, d_a, out);
	});
}

// stage-level entry for tests: locus seeding only (mpb_seed_loci_batch, mpb_seed_locus_sets_batch)
void seed_loci_batch_run(mpb_ctx_s *ctx, const mp_idx_t *vi, const int32_t *ctg_off, int32_t max_occ, const Batch &b, const std::vector<int32_t> &aa_off,
                         const char *d_aa, std::vector<int64_t> &a_off, std::vector<uint64_t> &a)
{
	a_off.assign((size_t)b.n + 1, 0), a.clear();
	if (b.n == 0) return;
	seed_loci_run(ctx, vi, ctg_off, max_occ, b, aa_off, d_aa, false, [&](int q0, int, const std::vector<int64_t> &so, const int64_t *, uint64_t *d_a) {
		append_anchors(ctx, q0, so, d_a, a_off, a);
	});
}

void refine_run(mpb_ctx_s *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<int32_t> &aa_off, const char *d_aa,
                const std::vector<RefineJob> &jobs, RefineSet &out)
{
	cudaStream_t st = ctx->stream;
	const int n_q = b.n, n_j = (int)jobs.size();
	const size_t R = (size_t)aa_off[(size_t)n_q];
	out.off.assign((size_t)n_j + 1, 0), out.a.clear(), out.sc.assign((size_t)n_j, 0);
	if (n_j == 0) return;
	if (mi->opt.min_aa_len > WIN_MAX_MIN_AA) { fprintf(stderr, "[miniprot_b200] min ORF length %d > %d is not supported by the window kernel\n", mi->opt.min_aa_len, WIN_MAX_MIN_AA); abort(); }
	Busy busy({ &ctx->b_aa, &ctx->b_c[3], &ctx->b_c[4], &ctx->b_c[5], &ctx->b_c[6], &ctx->b_c[8] });
	ClaimScope claim(ctx->mem);
	SeedConst cst;
	fill_seed_const(mi, opt, cst);
	const int k2 = opt->kmer2;
	// protein k-mers, sorted per protein
	std::vector<int32_t> n_pk((size_t)n_q);
	std::vector<int64_t> seg_b((size_t)n_q), seg_e((size_t)n_q);
	std::vector<WinJob> wj((size_t)n_j);
	int64_t grp_tot = 0;
	int32_t *d_aa_off, *d_npk, *d_grp;
	uint64_t *d_pk, *d_pk_tmp;
	int64_t *d_seg_b, *d_seg_e, *d_na, *d_a_off;
	WinJob *d_wj;
	for (int j = 0; j < n_j; ++j) grp_tot += b.len[jobs[(size_t)j].qid] + 1;
	auto layout = [&](Carver &c) {
		d_aa_off = c.take<int32_t>((size_t)n_q + 1), d_npk = c.take<int32_t>((size_t)n_q), d_pk = c.take<uint64_t>(R + 1), d_pk_tmp = c.take<uint64_t>(R + 1);
		d_seg_b = c.take<int64_t>((size_t)n_q), d_seg_e = c.take<int64_t>((size_t)n_q), d_wj = c.take<WinJob>((size_t)n_j), d_grp = c.take<int32_t>((size_t)grp_tot + 1);
		d_na = c.take<int64_t>((size_t)n_j), d_a_off = c.take<int64_t>((size_t)n_j + 1);
	};
	ctx->b_c[4].reserve(carve_size(layout));
	Carver cv(ctx->b_c[4].p);
	layout(cv);
	MPB_CUDA_OK(cudaMemcpyAsync(d_aa_off, aa_off.data(), sizeof(int32_t) * ((size_t)n_q + 1), cudaMemcpyHostToDevice, st));
	ctx->time_begin();
	seed_launch_prot_kmer(st, d_aa, d_aa_off, n_q, cst, k2, 0, d_pk, d_npk);
	MPB_CUDA_OK(cudaMemcpyAsync(n_pk.data(), d_npk, sizeof(int32_t) * (size_t)n_q, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	for (int q = 0; q < n_q; ++q) seg_b[(size_t)q] = aa_off[(size_t)q], seg_e[(size_t)q] = aa_off[(size_t)q] + n_pk[(size_t)q];
	MPB_CUDA_OK(cudaMemcpyAsync(d_seg_b, seg_b.data(), sizeof(int64_t) * (size_t)n_q, cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(d_seg_e, seg_e.data(), sizeof(int64_t) * (size_t)n_q, cudaMemcpyHostToDevice, st));
	seg_sort_u64(ctx, st, d_pk, d_pk_tmp, n_q, seg_b.data(), seg_e.data());
	int64_t go = 0;
	for (int j = 0; j < n_j; ++j) {
		const RefineJob &r = jobs[(size_t)j];
		const mp_ctg_t *c = &mi->nt->ctg[r.vid >> 1];
		WinJob &w = wj[(size_t)j];
		const bool rev = r.vid & 1;
		w.g_start = rev ? c->off + c->len - 1 - r.as : c->off + r.as, w.dir = rev ? -1 : 1, w.comp = rev ? 1 : 0;
		w.len = r.ae - r.as, w.qid = r.qid, w.pad_ = 0, w.grp_off = go;
		go += b.len[r.qid] + 1;
	}
	MPB_CUDA_OK(cudaMemcpyAsync(d_wj, wj.data(), sizeof(WinJob) * (size_t)n_j, cudaMemcpyHostToDevice, st));
	win_launch_count(st, d_wj, n_j, ctx->d_seq, cst, k2, mi->opt.min_aa_len, opt->max_ava, d_pk, d_aa_off, d_npk, d_grp, d_na);
	std::vector<int64_t> na((size_t)n_j), a_off;
	MPB_CUDA_OK(cudaMemcpyAsync(na.data(), d_na, sizeof(int64_t) * (size_t)n_j, cudaMemcpyDeviceToHost, st));
	ctx->stats.ms_refine += ctx->time_end();
	ctx->stats.kernel_launches += 3;
	ctx->stats.n_refine_regions += n_j;
	const chn::Par par = chain_par(opt->max_intron, opt->max_gap, opt->bw, opt, opt->min_chn_cnt, opt->min_chn_sc, k2, 0);
	const size_t N_all = (size_t)std::accumulate(na.begin(), na.end(), (int64_t)0);
	SlicePlan plan;
	const int64_t room = plan_items(ctx, { &ctx->b_c[5], &ctx->b_c[6], &ctx->b_c[8] }, { anchor_arena(N_all), anchor_arena(N_all), ChainScratch::bytes(n_j, N_all) }, n_j,
	                                na.data(), kAnchorBytesChain, plan, ctx->mem.n_slices_refine);
	std::vector<int32_t> n_u, n_b;
	std::vector<uint64_t> u, bb;
	for (int k = 0; k < plan.n_slices(); ++k) {
		const int j0 = plan.cut[(size_t)k], n = plan.cut[(size_t)k + 1] - j0;
		a_off.assign((size_t)n + 1, 0);
		for (int j = 0; j < n; ++j) a_off[(size_t)j + 1] = a_off[(size_t)j] + na[(size_t)(j0 + j)];
		const size_t N = (size_t)a_off[(size_t)n];
		if (room >= 0) ctx->mem.trim({ &ctx->b_c[5], &ctx->b_c[6], &ctx->b_c[8] }, { anchor_arena(N), anchor_arena(N), ChainScratch::bytes(n, N) }, room);
		ctx->time_begin();
		MPB_CUDA_OK(cudaMemcpyAsync(d_a_off, a_off.data(), sizeof(int64_t) * a_off.size(), cudaMemcpyHostToDevice, st));
		ctx->b_c[5].reserve(anchor_arena(N));
		ctx->b_c[6].reserve(anchor_arena(N));
		uint64_t *d_a = ctx->b_c[5].as<uint64_t>(), *d_tmp = ctx->b_c[6].as<uint64_t>();
		win_launch_emit(st, d_wj + j0, n, ctx->d_seq, cst, k2, mi->opt.min_aa_len, d_pk, d_aa_off, d_npk, d_grp, d_a_off, d_a);
		seg_sort_u64(ctx, st, d_a, d_tmp, n, a_off.data(), a_off.data() + 1);
		ctx->stats.ms_refine += ctx->time_end();
		ctx->stats.kernel_launches += 2;
		chain_problems(ctx, n, a_off, d_a_off, d_a, 0, par, n_u, n_b, u, bb);
		// keep the best-scoring chain of each window (first maximum, map.c:88-96)
		size_t uo = 0, bo = 0;
		for (int j = 0; j < n; ++j) {
			const int32_t nu = n_u[(size_t)j];
			if (nu > 0) {
				int32_t best = 0, mx = (int32_t)(u[uo] >> 32);
				for (int32_t i = 1; i < nu; ++i) if (mx < (int32_t)(u[uo + (size_t)i] >> 32)) mx = (int32_t)(u[uo + (size_t)i] >> 32), best = i;
				size_t kk = 0;
				for (int32_t i = 0; i < best; ++i) kk += (uint32_t)u[uo + (size_t)i];
				const uint32_t cnt = (uint32_t)u[uo + (size_t)best];
				out.a.insert(out.a.end(), bb.begin() + (ptrdiff_t)(bo + kk), bb.begin() + (ptrdiff_t)(bo + kk + cnt));
				out.sc[(size_t)(j0 + j)] = mx;
			}
			out.off[(size_t)(j0 + j) + 1] = (int64_t)out.a.size();
			uo += (size_t)nu, bo += (size_t)n_b[(size_t)j];
		}
	}
}

} // namespace cuda
} // namespace mpb
