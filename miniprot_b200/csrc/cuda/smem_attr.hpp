// smem_attr.hpp -- the dynamic shared-memory limit of a kernel, per device.
// cudaFuncSetAttribute applies to the CURRENT device only, so a launcher that needs more than the 48 KB default must have set the
// limit on every device it launches on.  One SmemLimit per kernel remembers, per device, the largest limit set so far; raising it
// is serialised, checking it is one atomic load.  Every entry point of the library makes the context's device current first.
#pragma once
#include <atomic>
#include <mutex>
#include <cuda_runtime.h>

namespace mpb {
namespace cuda {

class SmemLimit {
public:
	template <class K>
	void raise(K *kernel, int bytes)
	{
		int dev = 0;
		cudaGetDevice(&dev);
		if (dev < 0 || dev >= MAX_DEV) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); return; }
		if (set_[dev].load(std::memory_order_acquire) >= bytes) return;
		std::lock_guard<std::mutex> lk(mu_);
		if (set_[dev].load(std::memory_order_relaxed) >= bytes) return;
		cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
		set_[dev].store(bytes, std::memory_order_release);
	}

private:
	static const int MAX_DEV = 64;
	std::atomic<int> set_[MAX_DEV] = {};
	std::mutex mu_;
};

} // namespace cuda
} // namespace mpb
