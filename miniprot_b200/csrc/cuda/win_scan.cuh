// win_scan.cuh -- the six-frame ORF k-mer scan of a genome slice (sketch.c:40-100), shared by the refinement join
// (seed_kernels.cu) and the index build (idx_build.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "seed_dev.hpp"

namespace mpb {
namespace cuda {

__device__ __forceinline__ uint32_t hash32_mask_dev(uint32_t x, uint32_t mask) // sketch.c:7-16
{
	x = (x + ~(x << 15)) & mask;
	x ^= x >> 10;
	x = (x + (x << 3)) & mask;
	x ^= x >> 6;
	x = (x + ~(x << 11)) & mask;
	x ^= x >> 16;
	return x;
}

// ---- genome window scan -------------------------------------------------------------------------------------

// nucleotide code at window position k of a refinement job (strand aware)
__device__ __forceinline__ int win_code(const uint8_t *packed, const WinJob &j, int64_t k)
{
	const int64_t g = j.g_start + (int64_t)j.dir * k;
	int b = packed[g >> 1] >> ((g & 1) * 4) & 0xf;
	if (j.comp) b = b < 4 ? 3 - b : b;
	return b;
}

// Bit strings of one reading frame of a tile, one 32-bit word per lane (bit b of lane w = codon 32 w + b of the frame;
// lanes >= n_words hold 0).  shl/shr shift the whole string by s >= 0 bits towards higher / lower codon indices.
__device__ __forceinline__ uint32_t bits_shl(uint32_t v, int s, int lane)
{
	const int q = s >> 5, r = s & 31;
	uint32_t a = __shfl_up_sync(0xffffffffu, v, q), b = __shfl_up_sync(0xffffffffu, v, q + 1);
	if (lane < q) a = 0;
	if (lane < q + 1) b = 0;
	return r ? (a << r | b >> (32 - r)) : a;
}
__device__ __forceinline__ uint32_t bits_shr(uint32_t v, int s, int lane)
{
	const int q = s >> 5, r = s & 31;
	uint32_t a = __shfl_down_sync(0xffffffffu, v, q), b = __shfl_down_sync(0xffffffffu, v, q + 1);
	if (lane + q > 31) a = 0;
	if (lane + q + 1 > 31) b = 0;
	return r ? (a >> r | b << (32 - r)) : a;
}
// bits at which a run of >= n consecutive ones ENDS (n >= 1), by doubling
__device__ __forceinline__ uint32_t bits_run_ends(uint32_t g, int n, int lane)
{
	uint32_t r = g;
	int len = 1;
	while (len * 2 <= n) r &= bits_shl(r, len, lane), len *= 2;
	if (len < n) r &= bits_shl(r, n - len, lane);
	return r;
}
// bits i for which some bit of e in [i, i + n - 1] is set
__device__ __forceinline__ uint32_t bits_spread_down(uint32_t e, int n, int lane)
{
	uint32_t r = e;
	int len = 1;
	while (len * 2 <= n) r |= bits_shr(r, len, lane), len *= 2;
	if (len < n) r |= bits_shr(r, n - len, lane);
	return r;
}

constexpr int WIN_WORDS = (WIN_SMEM_SPAN / 3 + 1 + 31) / 32; // words per frame bit string of a tile

// For every window position e that ends a k-mer inside an ORF of >= min_aa_len codons call fn(hash, e)
// (sketch.c:40-100: stop-to-stop runs of good codons in the three frames).
// Tile = WIN_TILE positions + halos; smem: codes[].  "A good codon ends here" is kept as one bit string per frame; the
// positions that qualify -- inside a run of >= min_aa_len good codons, with >= kmer of them ending here -- come out of a few
// shift/and/or steps on those strings (one warp per frame) instead of a 2 x min_aa_len loop per position.
// Only the tiles that start in [pos_lo, pos_hi) are scanned (pos_lo a multiple of WIN_TILE): the index build gives every CTA a
// range of a contig strand, the refinement join the whole window.
template <class Fn>
__device__ void scan_window(const uint8_t *packed, const WinJob &job, const SeedConst &cst, int kmer, int min_aa_len, uint8_t *codes, uint8_t * /*unused*/, Fn fn,
                            int64_t pos_lo = 0, int64_t pos_hi = INT64_MAX)
{
	__shared__ uint32_t ok[3][WIN_WORDS];
	const int64_t L = job.len;
	// the left halo covers the look-back of both run tests: min_aa_len codons for the ORF, kmer codons for the k-mer (the
	// refinement's kmer2 may exceed min_aa_len)
	const int halo_l = 3 * ((min_aa_len > kmer ? min_aa_len : kmer) + 1), halo_r = 3 * min_aa_len;
	const uint32_t mask = (1u << kmer * 4) - 1;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
	for (int64_t t0 = pos_lo; t0 < L && t0 < pos_hi; t0 += WIN_TILE) {
		const int64_t lo = t0 - halo_l, hi = (t0 + WIN_TILE + halo_r < L ? t0 + WIN_TILE + halo_r : L); // smem covers [lo, hi)
		const int span = (int)(hi - lo);
		for (int x = threadIdx.x; x < span; x += blockDim.x) {
			const int64_t k = lo + x;
			codes[x] = k >= 0 ? (uint8_t)win_code(packed, job, k) : 4;
		}
		__syncthreads();
		for (int idx = warp; idx < 3 * WIN_WORDS; idx += n_warps) { // good-codon bits, 32 codons of one frame per ballot
			const int f = idx / WIN_WORDS, w = idx - f * WIN_WORDS, x = 3 * (32 * w + lane) + f;
			bool g = false;
			if (x < span && x >= 2 && lo + x >= 2) {
				const int a = codes[x - 2], b = codes[x - 1], c = codes[x];
				g = a < 4 && b < 4 && c < 4 && cst.codon[a << 4 | b << 2 | c] < 20;
			}
			const uint32_t m = __ballot_sync(0xffffffffu, g);
			if (lane == 0) ok[f][w] = m;
		}
		__syncthreads();
		if (warp < 3) {
			const uint32_t g = lane < WIN_WORDS ? ok[warp][lane] : 0;
			const uint32_t in_orf = bits_spread_down(bits_run_ends(g, min_aa_len, lane), min_aa_len, lane);
			const uint32_t v = in_orf & bits_run_ends(g, kmer, lane);  // an ORF shorter than kmer has no k-mer end
			if (lane < WIN_WORDS) ok[warp][lane] = v;
		}
		__syncthreads();
		const int64_t t1 = t0 + WIN_TILE < L ? t0 + WIN_TILE : L;
		for (int64_t e = t0 + threadIdx.x; e < t1; e += blockDim.x) {
			const int x = (int)(e - lo), i = x / 3, f = x - 3 * i;
			if (!(ok[f][i >> 5] >> (i & 31) & 1)) continue;
			uint32_t w = 0;
			for (int d = kmer - 1; d >= 0; --d) {
				const int y = x - 3 * d;
				w = w << 4 | cst.codon13[codes[y - 2] << 4 | codes[y - 1] << 2 | codes[y]];
			}
			fn(hash32_mask_dev(w, mask), e);
		}
		__syncthreads();
	}
}


} // namespace cuda
} // namespace mpb
