// seg_sort.cu -- segmented ascending sort of 64-bit keys: the anchors of every protein (map.c:177), the k-mers of every protein
// and the anchors of every refinement window (sketch.c:95, map.c:55-76).  The reference sorts each list with radix_sort_mp64
// (ksort.h:112-162), a full-key sort: any correct sort gives the same array.
//
// Hand-written for the shapes of this path (a few thousand segments of a few hundred to a few hundred thousand keys, segment
// bounds known on the host):
//   seg_tile_sort_kernel   one CTA per TILE of a segment: the tile is loaded into shared memory once, sorted there by a bitonic
//                          network (no atomics, no histogram: the keys are unique and the network is oblivious) and written back
//                          once -- 16 bytes of HBM traffic per key.  Segments of up to 1024 keys use a 1024-key tile (256 threads),
//                          larger ones 8192-key tiles (1024 threads).  A C2 protein (5 k anchors) is ONE tile.
//   seg_merge_kernel       segments of more than one tile (gigabase genomes: 50-150 k anchors per protein): log2(tiles) passes, each
//                          merging neighbouring sorted runs; a CTA produces 2048 consecutive output keys: two merge-path searches
//                          in global memory bound its inputs, the inputs are staged in shared memory, every thread merges eight
//                          keys, the chunk leaves coalesced.  16 bytes per key and pass.
// A block finds its (segment, tile / chunk) by a binary search in a small table of per-segment first-unit numbers built on the host.
#include <algorithm>
#include <vector>
#include "ctx.hpp"
#include "seed_dev.hpp"
#include "smem_attr.hpp"

namespace mpb {
namespace cuda {

struct SegDesc { int64_t begin; int32_t n; int32_t first_unit; };

constexpr int SORT_SMALL = 1024, SORT_TILE = 8192, MERGE_CHUNK = 2048;

__device__ __forceinline__ int seg_of_unit(const SegDesc *segs, int n_segs, int unit)
{
	int lo = 0, hi = n_segs - 1; // last segment whose first_unit <= unit
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (segs[mid].first_unit <= unit) lo = mid; else hi = mid - 1;
	}
	return lo;
}

template <int TILE, int THREADS>
__global__ void __launch_bounds__(THREADS) seg_tile_sort_kernel(const SegDesc *segs, int n_segs, const uint64_t *src, uint64_t *dst)
{
	extern __shared__ uint64_t sk[];
	const SegDesc sd = segs[seg_of_unit(segs, n_segs, (int)blockIdx.x)];
	const int t = (int)blockIdx.x - sd.first_unit;
	const int64_t base = sd.begin + (int64_t)t * TILE;
	const int n = min(TILE, sd.n - t * TILE);
	// the network only needs a power of two that covers the tile's keys
	int N = 32;
	while (N < n) N <<= 1;
	for (int i = threadIdx.x; i < N; i += THREADS) sk[i] = i < n ? src[base + i] : ~0ULL;
	__syncthreads();
	for (int k = 2; k <= N; k <<= 1)
		for (int j = k >> 1; j > 0; j >>= 1) {
			for (int q = threadIdx.x; q < N / 2; q += THREADS) {
				const int i = 2 * q - (q & (j - 1)), p = i + j; // i has bit j clear: the pair (i, i ^ j)
				const uint64_t a = sk[i], b = sk[p];
				const bool up = (i & k) == 0;
				if ((a > b) == up) sk[i] = b, sk[p] = a;
			}
			__syncthreads();
		}
	for (int i = threadIdx.x; i < n; i += THREADS) dst[base + i] = sk[i];
}

// merge path: how many keys of A precede output position d of merge(A, B) (ties: A first)
__device__ __forceinline__ int merge_split(const uint64_t *A, int na, const uint64_t *B, int nb, int d)
{
	int lo = d > nb ? d - nb : 0, hi = d < na ? d : na;
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (A[mid] <= B[d - 1 - mid]) lo = mid + 1; else hi = mid;
	}
	return lo;
}

// one pass: inside every segment, sorted runs of L keys (the last one shorter) are merged two by two into runs of 2 L
__global__ void __launch_bounds__(256) seg_merge_kernel(const SegDesc *segs, int n_segs, const uint64_t *src, uint64_t *dst, int64_t L)
{
	__shared__ uint64_t in[MERGE_CHUNK], outb[MERGE_CHUNK];
	__shared__ int sp[2];
	const SegDesc sd = segs[seg_of_unit(segs, n_segs, (int)blockIdx.x)];
	const int64_t out0 = (int64_t)((int)blockIdx.x - sd.first_unit) * MERGE_CHUNK; // position in the segment
	const int64_t pair0 = out0 / (2 * L) * (2 * L);                              // start of the pair of runs this chunk belongs to
	const int na = (int)min(L, (int64_t)sd.n - pair0), nb = (int)min(L, max((int64_t)0, (int64_t)sd.n - pair0 - L));
	const uint64_t *A = src + sd.begin + pair0, *B = A + na;
	const int d0 = (int)(out0 - pair0), d1 = min(d0 + MERGE_CHUNK, na + nb), n_out = d1 - d0;
	uint64_t *O = dst + sd.begin + out0;
	if (nb == 0) { // a run without a partner moves on unchanged
		for (int i = threadIdx.x; i < n_out; i += 256) O[i] = A[d0 + i];
		return;
	}
	if (threadIdx.x < 2) sp[threadIdx.x] = merge_split(A, na, B, nb, threadIdx.x ? d1 : d0);
	__syncthreads();
	const int a0 = sp[0], a1 = sp[1], b0 = d0 - a0, b1 = d1 - a1, ca = a1 - a0, cb = b1 - b0; // ca + cb == n_out
	for (int i = threadIdx.x; i < n_out; i += 256) in[i] = i < ca ? A[a0 + i] : B[b0 + i - ca];
	__syncthreads();
	const uint64_t *SA = in, *SB = in + ca;
	const int e0 = min((int)threadIdx.x * 8, n_out), e1 = min(e0 + 8, n_out);
	int ia = merge_split(SA, ca, SB, cb, e0), ib = e0 - ia;
	for (int e = e0; e < e1; ++e) {
		const bool take_a = ib >= cb || (ia < ca && SA[ia] <= SB[ib]);
		outb[e] = take_a ? SA[ia++] : SB[ib++];
	}
	__syncthreads();
	for (int i = threadIdx.x; i < n_out; i += 256) O[i] = outb[i];
}

// keys[h_begin[s] .. h_end[s]) sorted in place for every segment s; tmp = scratch of the same size as keys
void seg_sort_u64(mpb_ctx_s *ctx, cudaStream_t st, uint64_t *keys, uint64_t *tmp, int n_seg, const int64_t *h_begin, const int64_t *h_end)
{
	// unit tables: segments of <= 1024 keys (one small tile), of one large tile, of several tiles (tile units), and the same several-tile
	// segments again with their merge chunks as units
	std::vector<SegDesc> small, single, mtile, mchunk;
	int u_small = 0, u_single = 0, u_mtile = 0, u_mchunk = 0;
	int64_t max_n = 0;
	for (int s = 0; s < n_seg; ++s) {
		const int64_t n = h_end[s] - h_begin[s];
		if (n <= 1) continue;
		if (n <= SORT_SMALL) small.push_back(SegDesc{ h_begin[s], (int32_t)n, u_small }), ++u_small;
		else if (n <= SORT_TILE) single.push_back(SegDesc{ h_begin[s], (int32_t)n, u_single }), ++u_single;
		else {
			mtile.push_back(SegDesc{ h_begin[s], (int32_t)n, u_mtile }), u_mtile += (int)((n + SORT_TILE - 1) / SORT_TILE);
			mchunk.push_back(SegDesc{ h_begin[s], (int32_t)n, u_mchunk }), u_mchunk += (int)((n + MERGE_CHUNK - 1) / MERGE_CHUNK);
			max_n = std::max(max_n, n);
		}
	}
	const size_t n_desc = small.size() + single.size() + mtile.size() + mchunk.size();
	if (n_desc == 0) return;
	std::vector<SegDesc> all;
	all.reserve(n_desc);
	for (const std::vector<SegDesc> *v : { &small, &single, &mtile, &mchunk }) all.insert(all.end(), v->begin(), v->end());
	ctx->b_c[3].reserve(sizeof(SegDesc) * (n_desc + 1));
	MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_c[3].p, all.data(), sizeof(SegDesc) * all.size(), cudaMemcpyHostToDevice, st));
	// (a copy from pageable memory has left the host buffer when the call returns)
	const SegDesc *d_small = ctx->b_c[3].as<SegDesc>(), *d_single = d_small + small.size(), *d_mtile = d_single + single.size(), *d_mchunk = d_mtile + mtile.size();
	static SmemLimit lim;
	lim.raise(seg_tile_sort_kernel<SORT_TILE, 1024>, SORT_TILE * 8);
	if (u_small) seg_tile_sort_kernel<SORT_SMALL, 256><<<u_small, 256, SORT_SMALL * 8, st>>>(d_small, (int)small.size(), keys, keys), ctx->stats.kernel_launches += 1;
	if (u_single) seg_tile_sort_kernel<SORT_TILE, 1024><<<u_single, 1024, SORT_TILE * 8, st>>>(d_single, (int)single.size(), keys, keys), ctx->stats.kernel_launches += 1;
	if (u_mtile) {
		int n_pass = 0;
		for (int64_t L = SORT_TILE; L < max_n; L <<= 1) ++n_pass;
		// the runs ping-pong between the two buffers and must come home with the last pass: with an odd number of passes the tiles are
		// sorted INTO tmp
		uint64_t *src = (n_pass & 1) ? tmp : keys, *dst = (n_pass & 1) ? keys : tmp;
		seg_tile_sort_kernel<SORT_TILE, 1024><<<u_mtile, 1024, SORT_TILE * 8, st>>>(d_mtile, (int)mtile.size(), keys, src);
		ctx->stats.kernel_launches += 1;
		for (int64_t L = SORT_TILE; L < max_n; L <<= 1) {
			seg_merge_kernel<<<u_mchunk, 256, 0, st>>>(d_mchunk, (int)mchunk.size(), src, dst, L);
			std::swap(src, dst);
			ctx->stats.kernel_launches += 1;
		}
	}
}

} // namespace cuda
} // namespace mpb
