// idx_build.cu -- the k-mer index built on the GPU (SURVEY 8f #1; replaces index.c:52-136 + sketch.c:40-117 for this step).
//
// The reference sketches every contig strand on a host thread (ORFs of >= min_aa_len codons in three frames, the hashed
// 6-mers of the reduced alphabet that pass the mod filter, as hash >> mod_bit << 32 | block id), sorts and dedups each
// strand's list and counting-sorts the lists into ki / kb.  What that produces is simply the set of distinct
// (bucket, block) pairs in ascending order; block ids grow with the strand number, so no per-strand pass is needed:
//   1. idx_count_kernel   the ORF scan of win_scan.cuh over every contig strand, a CTA per range of 16 tiles: one atomic
//                         per k-mer on the bucket counters (8 M buckets at the defaults)
//   2. exclusive scan     bucket starts (device-wide scan below: block sums, recursion, second pass)
// Steps 3-5 run once per pass over a range [lo, hi) of buckets.  The output is bucket-major, so each pass appends its piece of kb and
// ki; with room for every pair there is one pass over [0, n_bucket) (plan_bucket_passes in slices.hpp and the ledger decide):
//   3. idx_fill_kernel    the same scan again, (bucket << 32 | block) of the range's buckets written at bucket start - start[lo]
//                         + atomic cursor
//   4. bucket sort        buckets of <= 32 pairs by a warp (bitonic network over shuffles), larger ones by the segmented
//                         sort of seg_sort.cu: the pass's pairs are now sorted
//   5. unique + compact   flag = differs from the left neighbour; scan of the flags; kb (after the earlier passes' pairs) = low
//                         halves of the flagged keys, ki[bucket] = earlier passes' pairs + scan value at the bucket's start
// The genome is read from the 4-bit packed store in HBM (0.5 B per base and scan, one more fill scan per extra pass), the pairs are
// written twice (8 B) and read by the sort; everything else is atomics on an 32 MB table that lives in L2.  ki / kb stay resident for
// mapping and are copied to the host once for the ABI (mp_idx_dump, mp_idx_print_stat read them).
#include <algorithm>
#include <vector>
#include "ctx.hpp"
#include "seed_dev.hpp"
#include "stages_dev.hpp"
#include "win_scan.cuh"
#include "../internal.hpp"
#include "../slices.hpp"

namespace mpb {
namespace cuda {

constexpr int IDX_TILES_PER_CTA = 16;

struct IdxUnit { int32_t sc, pad_; int64_t pos_lo, pos_hi; }; // contig strand, positions whose tiles this CTA scans

struct IdxStrand { int64_t g_start; int32_t dir, comp; int64_t len; uint32_t boff, pad_; };

template <class Fn>
__device__ __forceinline__ void idx_scan_unit(const IdxUnit &u, const IdxStrand *strands, const uint8_t *packed, const SeedConst &cst, int min_aa_len, uint8_t *sm, Fn fn)
{
	const IdxStrand s = strands[u.sc];
	WinJob job;
	job.g_start = s.g_start, job.dir = s.dir, job.comp = s.comp, job.len = s.len, job.qid = 0, job.pad_ = 0, job.grp_off = 0;
	scan_window(packed, job, cst, cst.kmer, min_aa_len, sm, sm + WIN_SMEM_SPAN, [&](uint32_t h, int64_t e) { fn(h, e, s.boff); }, u.pos_lo, u.pos_hi);
}

__global__ void __launch_bounds__(SEED_THREADS) idx_count_kernel(const IdxUnit *units, const IdxStrand *strands, const uint8_t *packed, SeedConst cst, int min_aa_len,
                                                                 uint32_t *cnt)
{
	extern __shared__ uint8_t sm[];
	const uint32_t mask_mod = (1u << cst.mod_bit) - 1;
	idx_scan_unit(units[blockIdx.x], strands, packed, cst, min_aa_len, sm, [&](uint32_t h, int64_t, uint32_t) {
		if ((h & mask_mod) == 0) atomicAdd(&cnt[h >> cst.mod_bit], 1u);
	});
}

// the pairs of buckets [lo, hi), at start[b] - base (base = start[lo])
__global__ void __launch_bounds__(SEED_THREADS) idx_fill_kernel(const IdxUnit *units, const IdxStrand *strands, const uint8_t *packed, SeedConst cst, int min_aa_len,
                                                                int bbit, const int64_t *start, uint32_t lo, uint32_t hi, int64_t base, uint32_t *cur, uint64_t *keys)
{
	extern __shared__ uint8_t sm[];
	const uint32_t mask_mod = (1u << cst.mod_bit) - 1;
	idx_scan_unit(units[blockIdx.x], strands, packed, cst, min_aa_len, sm, [&](uint32_t h, int64_t e, uint32_t boff) {
		if ((h & mask_mod) != 0) return;
		const uint32_t b = h >> cst.mod_bit;
		if (b < lo || b >= hi) return;
		keys[start[b] - base + atomicAdd(&cur[b], 1u)] = (uint64_t)b << 32 | (uint32_t)((e >> bbit) + boff); // sketch.c:58: block of the codon's last base
	});
}

// ---- device-wide exclusive scan (int64 sums) of f(0), f(1), .. f(n-1); out[n] = total ------------------------------------------
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 16, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct LoadU32 { const uint32_t *p; __device__ int64_t operator()(int64_t i) const { return p[i]; } };
struct LoadI64 { const int64_t *p; __device__ int64_t operator()(int64_t i) const { return p[i]; } };
struct LoadFirst { const uint64_t *k; __device__ int64_t operator()(int64_t i) const { return i == 0 || k[i] != k[i - 1]; } }; // first of a run of equal keys

__device__ __forceinline__ int64_t block_excl_scan(int64_t v, int64_t *total) // exclusive scan of one value per thread across the CTA
{
	__shared__ int64_t ws[SCAN_THREADS / 32];
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	int64_t x = v;
	for (int d = 1; d < 32; d <<= 1) { const int64_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
	__syncthreads();
	if (lane == 31) ws[w] = x;
	__syncthreads();
	int64_t base = 0, tot = 0;
	for (int k = 0; k < SCAN_THREADS / 32; ++k) { if (k < w) base += ws[k]; tot += ws[k]; }
	*total = tot;
	return base + x - v;
}

template <class Load>
__global__ void __launch_bounds__(SCAN_THREADS) scan_sums_kernel(Load f, int64_t n, int64_t *sums)
{
	const int64_t i0 = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
	int64_t v = 0;
	for (int k = 0; k < SCAN_ITEMS; ++k) if (i0 + k < n) v += f(i0 + k);
	int64_t tot;
	block_excl_scan(v, &tot);
	if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

template <class Load>
__global__ void __launch_bounds__(SCAN_THREADS) scan_write_kernel(Load f, int64_t n, const int64_t *sums_excl, int64_t *out)
{
	const int64_t i0 = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
	int64_t x[SCAN_ITEMS], v = 0;
	for (int k = 0; k < SCAN_ITEMS; ++k) x[k] = i0 + k < n ? f(i0 + k) : 0, v += x[k];
	int64_t tot;
	int64_t run = block_excl_scan(v, &tot) + (sums_excl ? sums_excl[blockIdx.x] : 0);
	for (int k = 0; k < SCAN_ITEMS; ++k) {
		if (i0 + k < n) out[i0 + k] = run;
		run += x[k];
	}
	if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = (sums_excl ? sums_excl[blockIdx.x] : 0) + tot; // the total
}

// out[0..n] = exclusive scan of f; scratch grows as needed
template <class Load>
static void device_excl_scan(mpb_ctx_s *c, cudaStream_t st, Load f, int64_t n, int64_t *out, int depth = 0)
{
	const int64_t n_blk = (n + SCAN_TILE - 1) / SCAN_TILE;
	if (n_blk <= 1) {
		scan_write_kernel<<<1, SCAN_THREADS, 0, st>>>(f, n, (const int64_t*)0, out);
		c->stats.kernel_launches += 1;
		return;
	}
	DevBuf &sb = c->b_c[10 + depth];
	sb.reserve(sizeof(int64_t) * (size_t)(2 * n_blk + 2));
	int64_t *sums = sb.as<int64_t>(), *sums_ex = sums + n_blk;
	scan_sums_kernel<<<(unsigned)n_blk, SCAN_THREADS, 0, st>>>(f, n, sums);
	device_excl_scan(c, st, LoadI64{ sums }, n_blk, sums_ex, depth + 1);
	scan_write_kernel<<<(unsigned)n_blk, SCAN_THREADS, 0, st>>>(f, n, sums_ex, out);
	c->stats.kernel_launches += 2;
}

// ---- buckets of up to 32 pairs: one warp each, bitonic network over shuffles -----------------------------------------------------
__global__ void __launch_bounds__(256) idx_sort_small_kernel(const int64_t *start, uint32_t lo, uint32_t hi, int64_t base, uint64_t *keys)
{
	const int lane = threadIdx.x & 31;
	const uint32_t w0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
	for (uint32_t b = lo + w0; b < hi; b += nw) {
		const int64_t s = start[b] - base;
		const int n = (int)(start[b + 1] - start[b]);
		if (n < 2 || n > 32) continue;
		uint64_t v = lane < n ? keys[s + lane] : ~0ULL;
		for (int k = 2; k <= 32; k <<= 1)
			for (int j = k >> 1; j > 0; j >>= 1) {
				const uint64_t o = __shfl_xor_sync(0xffffffffu, v, j);
				const bool up = (lane & k) == 0, low = (lane & j) == 0;
				v = (low == up) ? (v < o ? v : o) : (v > o ? v : o);
			}
		if (lane < n) keys[s + lane] = v;
	}
}

__global__ void __launch_bounds__(256) idx_compact_kernel(const uint64_t *keys, int64_t n, const int64_t *rank, uint32_t *kb)
{
	const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n && (i == 0 || keys[i] != keys[i - 1])) kb[rank[i]] = (uint32_t)keys[i];
}

// ki[lo..hi]: kb_base (the distinct pairs of the earlier passes) + rank at the bucket's start.  start[hi] - base = n, rank[n] = the
// pass's distinct pairs, so ki[hi] is where the next pass starts, and after the last pass ki[n_bucket] = n_kb, the sentinel the
// lookup kernels expect.
__global__ void __launch_bounds__(256) idx_ki_kernel(const int64_t *start, uint32_t lo, uint32_t hi, int64_t base, const int64_t *rank, int64_t kb_base, int64_t *ki)
{
	const uint32_t b = lo + blockIdx.x * blockDim.x + threadIdx.x;
	if (b <= hi) ki[b] = kb_base + rank[start[b] - base];
}

// Scratch of a pass: per pair the keys, the sort's ping-pong buffer and the rank (b_c[4] / b_c[5] / b_c[6], 8 B each); per pass the
// rounding of those three arenas and of the sort's segment table (b_c[3], 4 KB each).  The segment table itself and the rank scan's
// block sums (under 1 B per pair) grow into the fifth of the room the plan leaves.  The bucket counters and starts (b_c[2] / b_c[7],
// 12 B per bucket) and the work units are busy arenas held before the plan: the ledger leaves them out of the room.
static const int64_t kIdxPairBytes = 3 * 8, kIdxPassFixed = 4 * 4096;

// nt (host, packed genome already read) -> ki / kb on the device of `c` and on the host; 0 on success
int idx_build_device(mpb_ctx_s *c, mp_idx_t *mi)
{
	const mp_ntdb_t *nt = mi->nt;
	const mp_idxopt_t *io = &mi->opt;
	if (io->min_aa_len > WIN_MAX_MIN_AA || io->min_aa_len < io->kmer || io->kmer * 4 > 28) return -1; // outside what the tile halos cover: the caller builds on the host
	MPB_CUDA_OK(cudaSetDevice(c->device));
	cudaStream_t st = c->stream;
	const uint32_t n_bucket = idx_n_bucket(io);
	const size_t seq_bytes = (size_t)((nt->l_seq + 1) >> 1);
	c->own_seq.reserve(seq_bytes + 16);
	MPB_CUDA_OK(cudaMemcpyAsync(c->own_seq.p, nt->seq, seq_bytes, cudaMemcpyHostToDevice, st));
	// work units
	std::vector<IdxStrand> strands((size_t)nt->n_ctg * 2);
	std::vector<IdxUnit> units;
	for (int32_t j = 0; j < nt->n_ctg * 2; ++j) {
		const mp_ctg_t *ct = &nt->ctg[j >> 1];
		IdxStrand &s = strands[(size_t)j];
		s.g_start = (j & 1) ? ct->off + ct->len - 1 : ct->off, s.dir = (j & 1) ? -1 : 1, s.comp = j & 1, s.len = ct->len, s.boff = mi->bo[j], s.pad_ = 0;
		const int64_t step = (int64_t)WIN_TILE * IDX_TILES_PER_CTA;
		for (int64_t p = 0; p < ct->len; p += step) units.push_back(IdxUnit{ j, 0, p, std::min(p + step, (int64_t)ct->len) });
	}
	if (units.empty()) return -1;
	SeedConst cst;
	memset(&cst, 0, sizeof(cst));
	memcpy(cst.aa13, ns_tab_aa13, 256), memcpy(cst.codon, ns_tab_codon, 64), memcpy(cst.codon13, ns_tab_codon13, 64);
	cst.kmer = io->kmer, cst.mod_bit = io->mod_bit;
	c->b_c[0].reserve(sizeof(IdxUnit) * units.size()), c->b_c[1].reserve(sizeof(IdxStrand) * strands.size());
	c->b_c[2].reserve(sizeof(uint32_t) * ((size_t)n_bucket + 1)), c->b_c[7].reserve(sizeof(int64_t) * ((size_t)n_bucket + 2));
	MPB_CUDA_OK(cudaMemcpyAsync(c->b_c[0].p, units.data(), sizeof(IdxUnit) * units.size(), cudaMemcpyHostToDevice, st));
	MPB_CUDA_OK(cudaMemcpyAsync(c->b_c[1].p, strands.data(), sizeof(IdxStrand) * strands.size(), cudaMemcpyHostToDevice, st));
	const IdxUnit *d_units = c->b_c[0].as<IdxUnit>();
	const IdxStrand *d_str = c->b_c[1].as<IdxStrand>();
	uint32_t *d_cnt = c->b_c[2].as<uint32_t>();
	int64_t *d_start = c->b_c[7].as<int64_t>(); // (b_c[3] belongs to seg_sort_u64)
	const uint8_t *d_seq = c->own_seq.as<uint8_t>();
	const size_t smem = 2 * WIN_SMEM_SPAN;
	// 1. count, 2. bucket starts
	MPB_CUDA_OK(cudaMemsetAsync(d_cnt, 0, sizeof(uint32_t) * ((size_t)n_bucket + 1), st));
	idx_count_kernel<<<(unsigned)units.size(), SEED_THREADS, smem, st>>>(d_units, d_str, d_seq, cst, io->min_aa_len, d_cnt);
	c->stats.kernel_launches += 1;
	device_excl_scan(c, st, LoadU32{ d_cnt }, (int64_t)n_bucket, d_start);
	std::vector<uint32_t> h_cnt((size_t)n_bucket);
	int64_t n_pairs = 0;
	MPB_CUDA_OK(cudaMemcpyAsync(h_cnt.data(), d_cnt, sizeof(uint32_t) * (size_t)n_bucket, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaMemcpyAsync(&n_pairs, d_start + n_bucket, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	// the resident tables, held before the plan so that automatic mode's allowance sees them: kb for every pair (n_kb <= n_pairs is
	// only known after the last pass)
	c->own_ki.reserve(sizeof(int64_t) * ((size_t)n_bucket + 1));
	c->own_kb.reserve(sizeof(uint32_t) * (size_t)(n_pairs + 1));
	int64_t *d_ki = c->own_ki.as<int64_t>();
	uint32_t *d_kb = c->own_kb.as<uint32_t>();
	// bucket ranges whose scratch fits the room the ledger gives it, less the quarter reserve() may add; the largest pass (with that
	// quarter) is claimed until the build ends
	ClaimScope claim(c->mem);
	SlicePlan plan;
	std::vector<int64_t> pass_pairs;
	int64_t most = 0;
	c->mem.plan({ &c->b_c[4], &c->b_c[5], &c->b_c[6] }, [&](int64_t room) {
		plan_bucket_passes(n_bucket, h_cnt.data(), kIdxPairBytes, kIdxPassFixed, room / 5 * 4, kIdxMaxPasses, plan);
		pass_pairs.assign((size_t)plan.n_slices(), 0), most = 0;
		for (int k = 0; k < plan.n_slices(); ++k) {
			for (int32_t b = plan.cut[(size_t)k]; b < plan.cut[(size_t)k + 1]; ++b) pass_pairs[(size_t)k] += h_cnt[(size_t)b];
			most = std::max(most, pass_pairs[(size_t)k]);
		}
		return (kIdxPassFixed + most * kIdxPairBytes) / 4 * 5;
	});
	c->mem.n_index_passes += plan.n_slices(), c->mem.n_over_budget += plan.n_over;
	c->b_c[4].reserve(sizeof(uint64_t) * (size_t)(most + 2)), c->b_c[5].reserve(sizeof(uint64_t) * (size_t)(most + 2)), c->b_c[6].reserve(sizeof(int64_t) * (size_t)(most + 2));
	uint64_t *d_keys = c->b_c[4].as<uint64_t>(), *d_tmp = c->b_c[5].as<uint64_t>();
	int64_t *d_rank = c->b_c[6].as<int64_t>();
	int n_sm = 0;
	MPB_CUDA_OK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, c->device));
	int64_t base = 0, n_kb = 0; // pairs and distinct pairs of the earlier passes
	for (int k = 0; k < plan.n_slices(); ++k) {
		const uint32_t lo = (uint32_t)plan.cut[(size_t)k], hi = (uint32_t)plan.cut[(size_t)k + 1];
		const int64_t n = pass_pairs[(size_t)k];
		// 3. fill
		MPB_CUDA_OK(cudaMemsetAsync(d_cnt + lo, 0, sizeof(uint32_t) * (size_t)(hi - lo), st));
		if (n > 0) {
			idx_fill_kernel<<<(unsigned)units.size(), SEED_THREADS, smem, st>>>(d_units, d_str, d_seq, cst, io->min_aa_len, io->bbit, d_start, lo, hi, base, d_cnt, d_keys);
			// 4. sort inside the buckets
			idx_sort_small_kernel<<<n_sm * 8, 256, 0, st>>>(d_start, lo, hi, base, d_keys); // grid-stride over the buckets: eight CTAs per SM
			c->stats.kernel_launches += 2;
			std::vector<int64_t> sb, se;
			int64_t acc = 0;
			for (uint32_t b = lo; b < hi; ++b) {
				if (h_cnt[b] > 32) sb.push_back(acc), se.push_back(acc + h_cnt[b]);
				acc += h_cnt[b];
			}
			if (!sb.empty()) seg_sort_u64(c, st, d_keys, d_tmp, (int)sb.size(), sb.data(), se.data());
		}
		// 5. distinct pairs -> kb, bucket starts -> ki
		device_excl_scan(c, st, LoadFirst{ d_keys }, n, d_rank);
		if (n > 0) idx_compact_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_keys, n, d_rank, d_kb + n_kb), c->stats.kernel_launches += 1;
		idx_ki_kernel<<<(hi - lo + 256) / 256, 256, 0, st>>>(d_start, lo, hi, base, d_rank, n_kb, d_ki);
		c->stats.kernel_launches += 1;
		int64_t n_kb_pass = 0;
		MPB_CUDA_OK(cudaMemcpyAsync(&n_kb_pass, d_rank + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
		MPB_CUDA_OK(cudaStreamSynchronize(st));
		base += n, n_kb += n_kb_pass;
	}
	mi->n_kb = n_kb;
	mi->ki = (int64_t*)malloc(sizeof(int64_t) * (size_t)n_bucket);
	mi->kb = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(n_kb ? n_kb : 1));
	MPB_CUDA_OK(cudaMemcpyAsync(mi->ki, c->own_ki.p, sizeof(int64_t) * (size_t)n_bucket, cudaMemcpyDeviceToHost, st));
	if (n_kb) MPB_CUDA_OK(cudaMemcpyAsync(mi->kb, c->own_kb.p, sizeof(uint32_t) * (size_t)n_kb, cudaMemcpyDeviceToHost, st));
	MPB_CUDA_OK(cudaStreamSynchronize(st));
	c->stats.h2d_bytes += (int64_t)seq_bytes, c->stats.d2h_bytes += (int64_t)(sizeof(int64_t) * n_bucket + sizeof(uint32_t) * (size_t)n_kb);
	// the build's scratch (24 B per pair in one pass: 45 GB for a 3 Gbp genome) is not an arena of the mapping stages: give it back
	for (int k : { 2, 4, 5, 6, 7 }) c->b_c[k].release();
	return 0;
}

} // namespace cuda
} // namespace mpb
