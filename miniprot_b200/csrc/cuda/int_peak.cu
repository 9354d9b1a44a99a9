// int_peak.cu -- measured integer-issue peak of the device for the operations the nasw kernels are made of (SURVEY 8d: "integer
// peak must be measured on the box with a max/add micro-benchmark, 32-bit and packed-16x2 variants").
//
// Every thread runs 8 independent dependency chains of ONE operation (fused add-max VIADDMNMX, three-way max VIMNMX3, their
// packed int16x2 forms), all SMs filled with 8 CTAs of 256 threads, no memory traffic.  The rate
// is reported in elementary integer operations per second: an add-max or a three-way max counts 2, the packed forms 4 (two lanes).
#include <cuda_runtime.h>
#include <stdint.h>
#include "ctx.hpp"

namespace mpb {
namespace cuda {

template <int V>
__device__ __forceinline__ uint32_t peak_op(uint32_t a, uint32_t b, uint32_t c)
{
	if (V == 0) return (uint32_t)__viaddmax_s32((int)a, (int)b, (int)c);
	if (V == 1) return (uint32_t)__vimax3_s32((int)a, (int)b, (int)c);
	if (V == 2) return __viaddmax_s16x2(a, b, c);
	if (V == 3) return __vimax3_s16x2(a, b, c);
	return __viaddmax_s16x2_relu(a, b, c);
}

template <int V>
__global__ void __launch_bounds__(256) int_peak_kernel(uint32_t *out, int iters, uint32_t seed)
{
	uint32_t x[8], b = seed * 2654435761u + threadIdx.x, c = seed ^ (blockIdx.x * 40503u);
#pragma unroll
	for (int k = 0; k < 8; ++k) x[k] = seed + k * 77u + threadIdx.x;
	for (int i = 0; i < iters; ++i) {
#pragma unroll
		for (int u = 0; u < 4; ++u) {
#pragma unroll
			for (int k = 0; k < 8; ++k) x[k] = peak_op<V>(x[k], b, c);
		}
	}
	uint32_t s = 0;
#pragma unroll
	for (int k = 0; k < 8; ++k) s ^= x[k];
	if (s == 0x12345678u) out[blockIdx.x * blockDim.x + threadIdx.x] = s; // keeps the chains alive
}

template <int V>
static double run_peak(cudaStream_t st, uint32_t *scratch, int n_sm)
{
	const int iters = 4096, grid = n_sm * 8;
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0), cudaEventCreate(&e1);
	int_peak_kernel<V><<<grid, 256, 0, st>>>(scratch, 64, 1u); // warm-up
	double best = 0;
	for (int rep = 0; rep < 3; ++rep) {
		cudaEventRecord(e0, st);
		int_peak_kernel<V><<<grid, 256, 0, st>>>(scratch, iters, 3u + rep);
		cudaEventRecord(e1, st);
		cudaEventSynchronize(e1);
		float ms = 0;
		cudaEventElapsedTime(&ms, e0, e1);
		const double instr = (double)grid * 256 * iters * 32; // thread-level instructions of the measured operation
		const double rate = instr / (ms * 1e-3);
		if (rate > best) best = rate;
	}
	cudaEventDestroy(e0), cudaEventDestroy(e1);
	return best;
}

} // namespace cuda
} // namespace mpb

extern "C" int mpb_int_peak(mpb_ctx_t *c, int variant, double *thread_instr_per_s, double *int_ops_per_s)
{
	using namespace mpb::cuda;
	if (!c || variant < 0 || variant > 4) return -1;
	std::lock_guard<std::mutex> lk(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	cudaDeviceProp pr;
	MPB_CUDA_OK(cudaGetDeviceProperties(&pr, c->device));
	c->b_c[15].reserve((size_t)pr.multiProcessorCount * 8 * 256 * 4 + 256);
	uint32_t *scr = c->b_c[15].as<uint32_t>();
	double r = 0;
	switch (variant) {
	case 0: r = run_peak<0>(c->stream, scr, pr.multiProcessorCount); break;
	case 1: r = run_peak<1>(c->stream, scr, pr.multiProcessorCount); break;
	case 2: r = run_peak<2>(c->stream, scr, pr.multiProcessorCount); break;
	case 3: r = run_peak<3>(c->stream, scr, pr.multiProcessorCount); break;
	default: r = run_peak<4>(c->stream, scr, pr.multiProcessorCount); break;
	}
	MPB_CUDA_OK(cudaGetLastError());
	static const int ops[5] = { 2, 2, 4, 4, 4 };
	*thread_instr_per_s = r, *int_ops_per_s = r * ops[variant];
	return 0;
}
