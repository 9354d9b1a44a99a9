// devbuf.hpp -- tiny helpers for device memory and error checking (host side of the CUDA backend), and the ledger that keeps a
// context's working arenas within its device-memory budget.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>
#include <functional>
#include <initializer_list>
#include <vector>

#define MPB_CUDA_OK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
	fprintf(stderr, "[miniprot_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(e_), __FILE__, __LINE__, cudaGetErrorString(e_)); abort(); } } while (0)

namespace mpb {
namespace cuda {

struct Ledger;

// Grow-only device buffer: the arenas of a context live as long as the context, so steady-state batches
// allocate nothing (cudaMalloc is a device-wide synchronisation point).  A working arena (led != null) reports its capacity to its
// context's ledger, which may release it while no stage uses it (busy == 0).
struct DevBuf {
	void *p = 0;
	size_t cap = 0;
	Ledger *led = 0;
	int busy = 0;
	void reserve(size_t bytes);
	void release();
	template <class T> T *as() const { return (T*)p; }
};

// Pinned host staging buffer (grow-only).
struct PinBuf {
	void *p = 0;
	size_t cap = 0;
	void reserve(size_t bytes)
	{
		if (bytes <= cap) return;
		if (p) MPB_CUDA_OK(cudaFreeHost(p));
		cap = bytes + bytes / 4 + 4096;
		MPB_CUDA_OK(cudaMallocHost(&p, cap));
	}
	void release() { if (p) cudaFreeHost(p); p = 0, cap = 0; }
	template <class T> T *as() const { return (T*)p; }
};

// The working arenas of one context and how many bytes they may hold at once: the explicit budget, or (budget 0, automatic) what
// they hold plus the device's free memory less a headroom of a sixteenth of the device (at least kHeadroom), asked of the device
// only when an arena has to grow.  The headroom is for what the CUDA runtime allocates outside the arenas while the stages run
// (kernel local memory, modules loaded at their first launch): with 1 GiB the full C3 set fills an 80 GB device until a launch
// fails for want of memory.  Contexts on one
// device in one process plan and grow under a lock per device, and a plan claims the bytes its arenas will grow by until they have
// grown or the stage ends: the automatic allowance of the other contexts leaves the claimed memory out, so two mapper threads do
// not spend the same free memory.
struct Ledger {
	static const int64_t kHeadroom = (int64_t)1 << 30;
	int device = 0;
	int64_t budget = 0;
	int64_t held = 0, peak = 0, allowance_last = 0;
	int64_t claim = 0; // bytes this context's current plan will still grow its arenas by
	int64_t n_slices_seed = 0, n_slices_loci = 0, n_slices_refine = 0, n_subwaves = 0;
	int64_t n_released = 0, bytes_released = 0, n_over_budget = 0;
	int64_t n_index_passes = 0; // passes of the k-mer index builds (idx_build.cu)
	std::vector<DevBuf*> bufs;

	void add(DevBuf &b) { b.led = this, bufs.push_back(&b); }
	// Under the device lock: the room of a stage's arenas `mine` (which it sizes per slice) -- the allowance less what the context's
	// other busy arenas hold; idle arenas are released when the space is needed -- handed to f, which plans within it and returns the
	// most `mine` will hold; what that exceeds their present capacity is claimed.  Returns the room.
	int64_t plan(std::initializer_list<DevBuf*> mine, const std::function<int64_t(int64_t)> &f);
	void end_claim(); // the stage is done: nothing more of its plan will grow
	// does every arena of `mine` already hold its share of `need` (no growth, no device query)?
	static bool fits(std::initializer_list<DevBuf*> mine, std::initializer_list<size_t> need);
	// Before a slice fills the arenas of `mine` (none holds live data): release those larger than their need when keeping them would
	// not leave the others room within `room`, so that a large slice of an earlier batch does not crowd out this one's other arenas.
	void trim(std::initializer_list<DevBuf*> mine, std::initializer_list<size_t> need, int64_t room);
	// release idle arenas, largest first, until held <= target (never `keep` nor a busy one)
	void release_idle(int64_t target, const DevBuf *keep);
	void grow(DevBuf &b, size_t bytes);
	void reset_counters() { n_slices_seed = n_slices_loci = n_slices_refine = n_subwaves = n_released = bytes_released = n_over_budget = n_index_passes = 0, peak = held; }
};

// a stage's claim ends with it
struct ClaimScope {
	Ledger &l;
	explicit ClaimScope(Ledger &x) : l(x) {}
	~ClaimScope() { l.end_claim(); }
};

// arenas a stage uses: they are not released under it
struct Busy {
	std::vector<DevBuf*> v;
	Busy(std::initializer_list<DevBuf*> l) : v(l) { for (DevBuf *b : v) ++b->busy; }
	Busy(DevBuf *a, int n) { for (int i = 0; i < n; ++i) v.push_back(a + i), ++a[i].busy; }
	~Busy() { for (DevBuf *b : v) --b->busy; }
};

inline void DevBuf::reserve(size_t bytes)
{
	if (bytes <= cap) return;
	if (led) { led->grow(*this, bytes); return; }
	if (p) MPB_CUDA_OK(cudaFree(p));
	cap = bytes + bytes / 4 + 4096;
	MPB_CUDA_OK(cudaMalloc(&p, cap));
}

} // namespace cuda
} // namespace mpb
