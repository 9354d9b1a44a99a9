// seed_kernels.cu -- k-mer extraction, index lookup and window k-mer join on the GPU.
//
// Replaces, per mini-batch instead of per protein:
//   seed_sketch_kernel   sketch.c:18 mp_sketch_prot (k=6, mod sampling) + map.c:126-141 mp_cal_max_occ + the
//                        bucket-size pass of map.c:163-167.  One CTA per protein, one thread per residue
//                        position; the two box-plot quantiles are order statistics found by bisection on the
//                        value (no sort), in FP64 exactly like the reference.
//   seed_expand_kernel   map.c:169-175: CSR gather kb[ki[h] .. ki[h+1]) -> anchors block<<32 | qpos; one warp per
//                        seed, coalesced 128-byte reads of kb.  HBM-bound: 4 B read + 8 B written per anchor.
//   prot_kmer_kernel     sketch.c:18 with k=5, mod 0 (all k-mers) for the refinement join.
//   win_count_kernel /   map.c:41-79: the window's ORF k-mers (sketch.c:40-100 semantics: stop-to-stop runs of
//   win_emit_kernel      >= min_aa_len codons, three frames) are matched against the protein's sorted 5-mer list;
//                        groups with n1*n2 <= max_ava emit anchors ntpos<<32 | aapos.  The genome window is read
//                        straight from the 4-bit packed store (0.5 B/nt), strand-aware.
#include <cuda_runtime.h>
#include "seed_dev.hpp"
#include "win_scan.cuh"

namespace mpb {
namespace cuda {

// k-mer of reduced-alphabet residues ending at position i; false if any residue is stop/unknown or i < k-1
__device__ __forceinline__ bool prot_kmer_at(const char *s, int i, int k, const SeedConst &c, uint32_t &packed)
{
	if (i < k - 1) return false;
	uint32_t x = 0;
	for (int d = k - 1; d >= 0; --d) {
		const uint32_t r = c.aa13[(uint8_t)s[i - d]];
		if (r >= 14) return false;
		x = x << 4 | r;
	}
	packed = x;
	return true;
}

// block-wide count of elements <= v
__device__ int64_t block_count_le(const int64_t *cnt, int n, int64_t v, int64_t *red)
{
	int64_t c = 0;
	for (int i = threadIdx.x; i < n; i += blockDim.x) c += cnt[i] <= v;
	for (int d = 16; d; d >>= 1) c += __shfl_down_sync(0xffffffffu, c, d);
	__syncthreads();
	if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
	__syncthreads();
	int64_t tot = 0;
	for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
	return tot;
}

// k-th smallest (0-based) of cnt[0..n): smallest v with #(cnt <= v) >= k+1
__device__ int64_t block_kth(const int64_t *cnt, int n, int64_t k, int64_t vmax, int64_t *red)
{
	int64_t lo = 0, hi = vmax;
	while (lo < hi) {
		const int64_t mid = lo + (hi - lo) / 2;
		if (block_count_le(cnt, n, mid, red) >= k + 1) hi = mid; else lo = mid + 1;
	}
	return lo;
}

// map.c:158-167 over the bucket sizes cnt[0..n) (all <= vmax) of one protein's seeds: the adaptive occupancy cut-off (map.c:126-141),
// then the exclusive scan of the sizes that pass it into aoff[] (-1 marks a dropped bucket).  Returns the number of anchors.
__device__ __forceinline__ int64_t occ_cut_scan(const int64_t *cnt, int n, int32_t max_occ, int64_t vmax, int64_t *aoff, int64_t *red, int64_t &scan_carry)
{
	if (n >= 8) { // map.c:158-161 + 126-141
		const int64_t q25 = block_kth(cnt, n, (int64_t)(n * .25 + .499), vmax, red);
		const int64_t q75 = block_kth(cnt, n, (int64_t)(n * .75 + .499), vmax, red);
		const int32_t cap = (int32_t)((double)(uint64_t)q75 + (double)(uint64_t)(q75 - q25) * 1.5 + 10.);
		if (cap < max_occ) max_occ = cap;
	}
	// exclusive scan of the effective bucket sizes (0 for buckets above the cap)
	if (threadIdx.x == 0) scan_carry = 0;
	__syncthreads();
	for (int i0 = 0; i0 < n; i0 += blockDim.x) {
		const int i = i0 + threadIdx.x;
		int64_t v = (i < n && cnt[i] <= max_occ) ? cnt[i] : 0, inc = v;
		for (int d = 1; d < 32; d <<= 1) { const int64_t o = __shfl_up_sync(0xffffffffu, inc, d); if ((int)(threadIdx.x & 31) >= d) inc += o; }
		if ((threadIdx.x & 31) == 31) red[threadIdx.x >> 5] = inc;
		__syncthreads();
		int64_t wbase = scan_carry;
		for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wbase += red[w];
		if (i < n) aoff[i] = cnt[i] <= max_occ ? wbase + inc - v : -1;
		__syncthreads();
		if (threadIdx.x == blockDim.x - 1) scan_carry = wbase + inc;
		__syncthreads();
	}
	return scan_carry;
}

__global__ void __launch_bounds__(SEED_THREADS) seed_sketch_kernel(const char *aa, const int32_t *aa_off, int n_q, SeedConst cst, const int64_t *ki,
                                                                   uint32_t *sd_hash, int32_t *sd_pos, int64_t *sd_cnt, int64_t *sd_aoff,
                                                                   int32_t *n_sd_out, int64_t *tot_out)
{
	__shared__ int n_sd_s;
	__shared__ int64_t red[SEED_THREADS / 32];
	__shared__ int64_t scan_carry;
	const int q = blockIdx.x;
	if (q >= n_q) return;
	const int32_t base = aa_off[q], L = aa_off[q + 1] - base;
	const char *s = aa + base;
	if (threadIdx.x == 0) n_sd_s = 0;
	__syncthreads();
	const uint32_t mask = (1u << cst.kmer * 4) - 1, mod = (1u << cst.mod_bit) - 1;
	for (int i = threadIdx.x; i < L; i += blockDim.x) {
		uint32_t x;
		if (!prot_kmer_at(s, i, cst.kmer, cst, x)) continue;
		const uint32_t h = hash32_mask_dev(x, mask);
		if (h & mod) continue;
		const uint32_t b = h >> cst.mod_bit;
		const int slot = atomicAdd(&n_sd_s, 1);
		sd_hash[base + slot] = b, sd_pos[base + slot] = i;
		sd_cnt[base + slot] = ki[b + 1] - ki[b]; // ki carries a sentinel n_kb after the last bucket
	}
	__syncthreads();
	const int n = n_sd_s;
	const int64_t tot = occ_cut_scan(sd_cnt + base, n, cst.max_occ, cst.n_kb, sd_aoff + base, red, scan_carry);
	if (threadIdx.x == 0) n_sd_out[q] = n, tot_out[q] = tot;
}

__global__ void __launch_bounds__(SEED_THREADS) seed_expand_kernel(const int32_t *aa_off, int n_q, const int64_t *ki, const uint32_t *kb, const uint32_t *sd_hash,
                                                                   const int32_t *sd_pos, const int64_t *sd_cnt, const int64_t *sd_aoff, const int32_t *n_sd,
                                                                   const int64_t *a_off, uint64_t *a)
{
	const int q = blockIdx.x;
	if (q >= n_q) return;
	const int32_t base = aa_off[q];
	const int n = n_sd[q], warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warp = blockDim.x >> 5;
	uint64_t *out = a + a_off[q];
	for (int s = warp; s < n; s += n_warp) {
		const int64_t o = sd_aoff[base + s];
		if (o < 0) continue;
		const int64_t st = ki[sd_hash[base + s]], c = sd_cnt[base + s];
		const uint64_t pos = (uint32_t)sd_pos[base + s];
		for (int64_t k = lane; k < c; k += 32) out[o + k] = (uint64_t)kb[st + k] << 32 | pos;
	}
}

// the k-mers of every protein whose hash passes the mod filter (sketch.c:18; mod_bit 0: all of them): key = hash>>mod_bit<<32 | pos,
// written at aa_off[q] + slot; n_out[q] = count
__global__ void __launch_bounds__(SEED_THREADS) prot_kmer_kernel(const char *aa, const int32_t *aa_off, int n_q, SeedConst cst, int kmer, int mod_bit, uint64_t *keys,
                                                                 int32_t *n_out)
{
	__shared__ int n_s;
	const int q = blockIdx.x;
	if (q >= n_q) return;
	const int32_t base = aa_off[q], L = aa_off[q + 1] - base;
	if (threadIdx.x == 0) n_s = 0;
	__syncthreads();
	const uint32_t mask = (1u << kmer * 4) - 1, mod = (1u << mod_bit) - 1;
	for (int i = threadIdx.x; i < L; i += blockDim.x) {
		uint32_t x;
		if (!prot_kmer_at(aa + base, i, kmer, cst, x)) continue;
		const uint32_t h = hash32_mask_dev(x, mask);
		if (h & mod) continue;
		const int slot = atomicAdd(&n_s, 1);
		keys[base + slot] = (uint64_t)(h >> mod_bit) << 32 | (uint32_t)i;
	}
	__syncthreads();
	if (threadIdx.x == 0) n_out[q] = n_s;
}

// first index in the sorted protein k-mer list whose hash is >= h
__device__ __forceinline__ int lower_hash(const uint64_t *pk, int n, uint32_t h)
{
	int lo = 0, hi = n;
	while (lo < hi) { const int mid = (lo + hi) >> 1; if ((uint32_t)(pk[mid] >> 32) < h) lo = mid + 1; else hi = mid; }
	return lo;
}

__global__ void __launch_bounds__(SEED_THREADS) win_count_kernel(const WinJob *jobs, int n_jobs, const uint8_t *packed, SeedConst cst, int kmer, int min_aa_len,
                                                                 int max_ava, const uint64_t *pk_all, const int32_t *aa_off, const int32_t *n_pk, int32_t *grp_cnt_all,
                                                                 int64_t *n_a_out)
{
	extern __shared__ uint8_t sm[];
	__shared__ unsigned long long tot_s;
	const int jb = blockIdx.x;
	if (jb >= n_jobs) return;
	const WinJob job = jobs[jb];
	const uint64_t *pk = pk_all + aa_off[job.qid];
	const int npk = n_pk[job.qid];
	int32_t *grp = grp_cnt_all + job.grp_off; // one counter per protein k-mer slot (indexed by the group's first slot)
	for (int i = threadIdx.x; i < npk; i += blockDim.x) grp[i] = 0;
	if (threadIdx.x == 0) tot_s = 0;
	__syncthreads();
	uint8_t *codes = sm, *good = sm + WIN_SMEM_SPAN;
	scan_window(packed, job, cst, kmer, min_aa_len, codes, good, [&](uint32_t h, int64_t) {
		const int lo = lower_hash(pk, npk, h);
		if (lo < npk && (uint32_t)(pk[lo] >> 32) == h) atomicAdd(&grp[lo], 1);
	});
	__syncthreads();
	// n_a = sum over groups of n1*n2 where allowed (map.c:53-64)
	unsigned long long loc = 0;
	for (int i = threadIdx.x; i < npk; i += blockDim.x) {
		const int n1 = grp[i];
		if (n1 == 0) continue;
		const uint32_t h = (uint32_t)(pk[i] >> 32);
		int n2 = 1;
		while (i + n2 < npk && (uint32_t)(pk[i + n2] >> 32) == h) ++n2;
		if ((int64_t)n1 * n2 <= max_ava) loc += (unsigned long long)n1 * n2;
		else grp[i] = -1; // too repetitive: dropped
	}
	atomicAdd(&tot_s, loc);
	__syncthreads();
	if (threadIdx.x == 0) n_a_out[jb] = (int64_t)tot_s;
}

__global__ void __launch_bounds__(SEED_THREADS) win_emit_kernel(const WinJob *jobs, int n_jobs, const uint8_t *packed, SeedConst cst, int kmer, int min_aa_len,
                                                                const uint64_t *pk_all, const int32_t *aa_off, const int32_t *n_pk, const int32_t *grp_cnt_all,
                                                                const int64_t *a_off, uint64_t *a)
{
	extern __shared__ uint8_t sm[];
	__shared__ unsigned long long slot_s;
	const int jb = blockIdx.x;
	if (jb >= n_jobs) return;
	const WinJob job = jobs[jb];
	const uint64_t *pk = pk_all + aa_off[job.qid];
	const int npk = n_pk[job.qid];
	const int32_t *grp = grp_cnt_all + job.grp_off;
	uint64_t *out = a + a_off[jb];
	if (threadIdx.x == 0) slot_s = 0;
	__syncthreads();
	uint8_t *codes = sm, *good = sm + WIN_SMEM_SPAN;
	scan_window(packed, job, cst, kmer, min_aa_len, codes, good, [&](uint32_t h, int64_t e) {
		const int lo = lower_hash(pk, npk, h);
		if (lo >= npk || (uint32_t)(pk[lo] >> 32) != h || grp[lo] <= 0) return;
		int n2 = 1;
		while (lo + n2 < npk && (uint32_t)(pk[lo + n2] >> 32) == h) ++n2;
		const unsigned long long s = atomicAdd(&slot_s, (unsigned long long)n2);
		for (int k = 0; k < n2; ++k) out[s + k] = (uint64_t)e << 32 | (uint32_t)pk[lo + k];
	});
}

// ---- locus seeding: what the reference seeds from an index of one locus, without a k-mer table -----------------------------
// The ORF scan of the index build runs over both strands of the locus; a k-mer is kept when its bucket is one of the protein's
// seed buckets (binary search in the protein's sorted seeds).  Count pass, then emit pass: bucket<<32 | block, the block numbered
// from the strand's first block boff.  Ranges of tiles of one strand per CTA, as in the index build.
template <bool EMIT>
__global__ void __launch_bounds__(SEED_THREADS) locus_join_kernel(const LocusUnit *units, const LocusStrand *strands, const uint8_t *packed, SeedConst cst, int min_aa_len,
                                                                  int bbit, const uint64_t *pk_all, const int32_t *aa_off, const int32_t *n_pk, const int64_t *unit_off,
                                                                  int64_t *unit_n, uint64_t *out)
{
	extern __shared__ uint8_t sm[];
	__shared__ unsigned long long n_s;
	const LocusUnit u = units[blockIdx.x];
	const LocusStrand s = strands[u.strand];
	const uint64_t *pk = pk_all + aa_off[s.qid];
	const int npk = n_pk[s.qid];
	if (npk == 0) { // nothing to join with
		if (!EMIT && threadIdx.x == 0) unit_n[blockIdx.x] = 0;
		return;
	}
	if (threadIdx.x == 0) n_s = 0;
	__syncthreads();
	WinJob job;
	job.g_start = s.g_start, job.dir = s.dir, job.comp = s.comp, job.len = s.len, job.qid = s.qid, job.pad_ = 0, job.grp_off = 0;
	const uint32_t mod = (1u << cst.mod_bit) - 1;
	uint64_t *o = EMIT ? out + unit_off[blockIdx.x] : 0;
	scan_window(packed, job, cst, cst.kmer, min_aa_len, sm, sm + WIN_SMEM_SPAN, [&](uint32_t h, int64_t e) {
		if (h & mod) return;
		const uint32_t b = h >> cst.mod_bit;
		const int lo = lower_hash(pk, npk, b);
		if (lo >= npk || (uint32_t)(pk[lo] >> 32) != b) return;
		const unsigned long long k = atomicAdd(&n_s, 1ULL);
		if (EMIT) o[k] = (uint64_t)b << 32 | (uint32_t)((e >> bbit) + s.boff); // sketch.c:58: block of the codon's last base
	}, u.pos_lo, u.pos_hi);
	if (!EMIT && threadIdx.x == 0) unit_n[blockIdx.x] = (int64_t)n_s; // (scan_window ends with a barrier)
}

// the distinct keys of each sorted segment keys[seg[q], seg[q+1]) -- a locus's (bucket, block) pairs, what index.c:71-90 holds for
// it -- to the same place in blk (their block halves only) and uniq (whole keys); n_u[q] = how many.  One CTA per segment.
__global__ void __launch_bounds__(SEED_THREADS) locus_unique_kernel(const uint64_t *keys, const int64_t *seg, int n_q, uint64_t *uniq, uint32_t *blk, int64_t *n_u)
{
	__shared__ int64_t red[SEED_THREADS / 32];
	__shared__ int64_t carry;
	const int q = blockIdx.x;
	if (q >= n_q) return;
	const int64_t b = seg[q], n = seg[q + 1] - b;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (threadIdx.x == 0) carry = 0;
	__syncthreads();
	for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {
		const int64_t i = i0 + threadIdx.x;
		const bool first = i < n && (i == 0 || keys[b + i] != keys[b + i - 1]);
		const uint32_t m = __ballot_sync(0xffffffffu, first);
		if (lane == 0) red[warp] = __popc(m);
		__syncthreads();
		int64_t base = carry, tot = 0;
		for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { if (w < warp) base += red[w]; tot += red[w]; }
		if (first) {
			const int64_t k = b + base + __popc(m & ((1u << lane) - 1));
			uniq[k] = keys[b + i], blk[k] = (uint32_t)keys[b + i];
		}
		__syncthreads();
		if (threadIdx.x == 0) carry += tot;
		__syncthreads();
	}
	if (threadIdx.x == 0) n_u[q] = carry;
}

// first index in the sorted keys u[0..n) that is >= x
__device__ __forceinline__ int64_t lower_u64(const uint64_t *u, int64_t n, uint64_t x)
{
	int64_t lo = 0, hi = n;
	while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (u[mid] < x) lo = mid + 1; else hi = mid; }
	return lo;
}

// per protein (one CTA): the size of each seed's bucket in the locus's distinct pairs and where it starts, the adaptive occupancy
// cut-off and the anchor offsets (occ_cut_scan, as seed_sketch_kernel does with the k-mer table), and the per-seed inputs of
// seed_expand_kernel: its "ki" is sd_lo indexed by sd_idx (the seed's own slot), its "kb" the block halves of the distinct pairs
__global__ void __launch_bounds__(SEED_THREADS) locus_occ_kernel(const uint64_t *pk_all, const int32_t *aa_off, const int32_t *n_pk, int n_q, const uint64_t *uniq,
                                                                 const int64_t *seg, const int64_t *n_u, int32_t max_occ, uint32_t *sd_idx, int32_t *sd_pos,
                                                                 int64_t *sd_lo, int64_t *sd_cnt, int64_t *sd_aoff, int64_t *tot_out)
{
	__shared__ int64_t red[SEED_THREADS / 32];
	__shared__ int64_t scan_carry;
	const int q = blockIdx.x;
	if (q >= n_q) return;
	const int32_t base = aa_off[q];
	const int n = n_pk[q];
	const uint64_t *u = uniq + seg[q];
	const int64_t nu = n_u[q];
	for (int i = threadIdx.x; i < n; i += blockDim.x) {
		const uint64_t key = pk_all[base + i], b = key >> 32;
		const int64_t lo = lower_u64(u, nu, b << 32), hi = lower_u64(u, nu, (b + 1) << 32);
		sd_idx[base + i] = (uint32_t)(base + i), sd_pos[base + i] = (int32_t)(uint32_t)key;
		sd_lo[base + i] = seg[q] + lo, sd_cnt[base + i] = hi - lo;
	}
	__syncthreads();
	const int64_t tot = occ_cut_scan(sd_cnt + base, n, max_occ, nu, sd_aoff + base, red, scan_carry);
	if (threadIdx.x == 0) tot_out[q] = tot;
}

// ---- launchers ----------------------------------------------------------------------------------------------
void seed_launch_sketch(cudaStream_t st, const char *aa, const int32_t *aa_off, int n_q, const SeedConst &cst, const int64_t *ki, uint32_t *sd_hash, int32_t *sd_pos,
                        int64_t *sd_cnt, int64_t *sd_aoff, int32_t *n_sd, int64_t *tot)
{
	if (n_q > 0) seed_sketch_kernel<<<n_q, SEED_THREADS, 0, st>>>(aa, aa_off, n_q, cst, ki, sd_hash, sd_pos, sd_cnt, sd_aoff, n_sd, tot);
}
void seed_launch_expand(cudaStream_t st, const int32_t *aa_off, int n_q, const int64_t *ki, const uint32_t *kb, const uint32_t *sd_hash, const int32_t *sd_pos,
                        const int64_t *sd_cnt, const int64_t *sd_aoff, const int32_t *n_sd, const int64_t *a_off, uint64_t *a)
{
	if (n_q > 0) seed_expand_kernel<<<n_q, SEED_THREADS, 0, st>>>(aa_off, n_q, ki, kb, sd_hash, sd_pos, sd_cnt, sd_aoff, n_sd, a_off, a);
}
void seed_launch_prot_kmer(cudaStream_t st, const char *aa, const int32_t *aa_off, int n_q, const SeedConst &cst, int kmer, int mod_bit, uint64_t *keys, int32_t *n_out)
{
	if (n_q > 0) prot_kmer_kernel<<<n_q, SEED_THREADS, 0, st>>>(aa, aa_off, n_q, cst, kmer, mod_bit, keys, n_out);
}
void locus_launch_join(cudaStream_t st, bool emit, const LocusUnit *units, int n_units, const LocusStrand *strands, const uint8_t *packed, const SeedConst &cst,
                       int min_aa_len, int bbit, const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, const int64_t *unit_off, int64_t *unit_n, uint64_t *out)
{
	if (n_units <= 0) return;
	if (emit) locus_join_kernel<true><<<n_units, SEED_THREADS, 2 * WIN_SMEM_SPAN, st>>>(units, strands, packed, cst, min_aa_len, bbit, pk, aa_off, n_pk, unit_off, unit_n, out);
	else locus_join_kernel<false><<<n_units, SEED_THREADS, 2 * WIN_SMEM_SPAN, st>>>(units, strands, packed, cst, min_aa_len, bbit, pk, aa_off, n_pk, unit_off, unit_n, out);
}
void locus_launch_unique(cudaStream_t st, const uint64_t *keys, const int64_t *seg, int n_q, uint64_t *uniq, uint32_t *blk, int64_t *n_u)
{
	if (n_q > 0) locus_unique_kernel<<<n_q, SEED_THREADS, 0, st>>>(keys, seg, n_q, uniq, blk, n_u);
}
void locus_launch_occ(cudaStream_t st, const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, int n_q, const uint64_t *uniq, const int64_t *seg, const int64_t *n_u,
                      int32_t max_occ, uint32_t *sd_idx, int32_t *sd_pos, int64_t *sd_lo, int64_t *sd_cnt, int64_t *sd_aoff, int64_t *tot)
{
	if (n_q > 0) locus_occ_kernel<<<n_q, SEED_THREADS, 0, st>>>(pk, aa_off, n_pk, n_q, uniq, seg, n_u, max_occ, sd_idx, sd_pos, sd_lo, sd_cnt, sd_aoff, tot);
}
void win_launch_count(cudaStream_t st, const WinJob *jobs, int n_jobs, const uint8_t *packed, const SeedConst &cst, int kmer, int min_aa_len, int max_ava,
                      const uint64_t *pk, const int32_t *aa_off, const int32_t *n_pk, int32_t *grp, int64_t *n_a)
{
	if (n_jobs > 0) win_count_kernel<<<n_jobs, SEED_THREADS, 2 * WIN_SMEM_SPAN, st>>>(jobs, n_jobs, packed, cst, kmer, min_aa_len, max_ava, pk, aa_off, n_pk, grp, n_a);
}
void win_launch_emit(cudaStream_t st, const WinJob *jobs, int n_jobs, const uint8_t *packed, const SeedConst &cst, int kmer, int min_aa_len, const uint64_t *pk,
                     const int32_t *aa_off, const int32_t *n_pk, const int32_t *grp, const int64_t *a_off, uint64_t *a)
{
	if (n_jobs > 0) win_emit_kernel<<<n_jobs, SEED_THREADS, 2 * WIN_SMEM_SPAN, st>>>(jobs, n_jobs, packed, cst, kmer, min_aa_len, pk, aa_off, n_pk, grp, a_off, a);
}

} // namespace cuda
} // namespace mpb
