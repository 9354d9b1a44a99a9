// slices.hpp -- how a stage cuts the items of a batch (proteins, locus pairs, refinement windows, DP problems) into consecutive slices
// whose device arenas fit a byte allowance, and the parser of MPB_DEVICE_MEM.  Pure host code: the CPU tests check it directly.
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
