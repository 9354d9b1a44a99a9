// slices.hpp -- how a stage cuts the items of a batch (proteins, locus pairs, refinement windows, DP problems) into consecutive slices
// whose device arenas fit a byte allowance, how the index build cuts its buckets into passes, and the parser of MPB_DEVICE_MEM.  Pure
// host code: the CPU tests check it directly.
//
// Every item of a stage is independent of the rest of its batch (DESIGN §2), so running the slices one after the other and
// appending their results in item order gives the same bytes as one pass over the whole batch.
#pragma once
#include <stdint.h>
#include <vector>

namespace mpb {

// Slices of items [0, n): item i costs bytes[i] of arena and count[i] elements of the arrays the kernels index with 32-bit
// counts (count may be null: no such cap); a slice also costs `fixed` bytes.  Greedy prefixes in input order: a slice takes items
// while fixed + its bytes <= allowance and its count < max_count, and at least one item.  cut[0] = 0 < cut[1] < ... < cut[k] = n
// delimit the k slices; n_over counts the slices of one item that do not fit on their own (they run anyway, alone).
struct SlicePlan {
	std::vector<int32_t> cut;
	int32_t n_over = 0;
	int32_t n_slices() const { return cut.empty() ? 0 : (int32_t)cut.size() - 1; }
};

static const int64_t kSliceMaxCount = (int64_t)1 << 31;

inline void plan_slices(int32_t n, const int64_t *bytes, const int64_t *count, int64_t fixed, int64_t allowance, int64_t max_count, SlicePlan &p)
{
	p.cut.assign(1, 0), p.n_over = 0;
	int32_t lo = 0;
	while (lo < n) {
		int64_t b = fixed, c = 0;
		int32_t hi = lo;
		while (hi < n) {
			const int64_t nb = b + bytes[hi], nc = c + (count ? count[hi] : 0);
			if (hi > lo && (nb > allowance || nc >= max_count)) break;
			b = nb, c = nc, ++hi;
		}
		if (hi == lo + 1 && (b > allowance || c >= max_count)) ++p.n_over;
		p.cut.push_back(hi);
		lo = hi;
	}
}

// The index build's passes (cuda/idx_build.cu): its output is bucket-major, so consecutive bucket ranges give consecutive pieces of
// kb / ki and the passes just append.  kIdxMaxPasses bounds the genome scans a budget far below the build's need may cost: a pass
// always holds at least ceil(total / max_passes) pairs, where one pass per bucket could mean millions of scans.
static const int32_t kIdxMaxPasses = 64;

// Passes over buckets [0, n_bucket) (cnt[b] pairs each, per_pair bytes of scratch per pair, `fixed` per pass), in the SlicePlan's
// cut[]: greedy contiguous ranges within the allowance, each of at least one bucket and of fewer than kSliceMaxCount pairs (the sort
// of seg_sort.cu keeps its segment sizes and unit numbers in 32 bits).  A pass below ceil(total / max_passes) pairs takes the next
// bucket even past the allowance, and the empty buckets after the last pair join the last pass, so there are at most max_passes
// passes (unless that pair limit cuts them shorter).  n_over counts the passes over the allowance: a bucket too large on its own,
// or a range the pass minimum forced.  Walks cnt directly: at -k 7 -M 0 there are 2^28 buckets.
inline void plan_bucket_passes(uint32_t n_bucket, const uint32_t *cnt, int64_t per_pair, int64_t fixed, int64_t allowance, int32_t max_passes, SlicePlan &p)
{
	int64_t total = 0;
	for (uint32_t b = 0; b < n_bucket; ++b) total += cnt[b];
	const int64_t min_pairs = (total + (max_passes > 1 ? max_passes : 1) - 1) / (max_passes > 1 ? max_passes : 1);
	p.cut.assign(1, 0), p.n_over = 0;
	int64_t done = 0;
	uint32_t lo = 0;
	while (lo < n_bucket) {
		int64_t c = 0;
		uint32_t hi = lo;
		for (; hi < n_bucket; ++hi) {
			const int64_t nc = c + cnt[hi];
			if (hi > lo && done + c < total && (nc >= kSliceMaxCount || (c >= min_pairs && fixed + nc * per_pair > allowance))) break;
			c = nc;
		}
		if (fixed + c * per_pair > allowance || c >= kSliceMaxCount) ++p.n_over;
		p.cut.push_back((int32_t)hi);
		lo = hi, done += c;
	}
}

// MPB_DEVICE_MEM=<n>[k|m|g] (binary units, either case): the byte count, 0 for "0" (automatic), -1 when the text is not of that form
// or does not fit in 63 bits.
inline int64_t parse_mem_size(const char *s)
{
	if (!s || !*s) return -1;
	uint64_t v = 0;
	const char *q = s;
	for (; *q >= '0' && *q <= '9'; ++q) {
		v = v * 10 + (uint64_t)(*q - '0');
		if (v > ((uint64_t)1 << 62)) return -1;
	}
	if (q == s) return -1;
	int shift = 0;
	if (*q) {
		const char c = *q | 0x20;
		shift = c == 'k' ? 10 : c == 'm' ? 20 : c == 'g' ? 30 : -1;
		if (shift < 0 || q[1]) return -1;
	}
	if (shift && v > (((uint64_t)1 << 62) >> shift)) return -1;
	return (int64_t)(v << shift);
}

} // namespace mpb
