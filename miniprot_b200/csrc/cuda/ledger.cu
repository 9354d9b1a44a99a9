// ledger.cu -- the device-memory ledger of a context (devbuf.hpp): what its working arenas hold, how much they may hold, and which
// idle arenas give way when one has to grow past that.
#include <algorithm>
#include <functional>
#include <mutex>
#include "devbuf.hpp"

namespace mpb {
namespace cuda {

namespace {
// per device: the lock under which the contexts of this process plan and grow, and the bytes they have planned to grow by but not
// allocated yet (the sum of their claims)
std::mutex &device_mutex(int device)
{
	static std::mutex mu[64];
	return mu[(unsigned)device % 64];
}
int64_t &device_claimed(int device)
{
	static int64_t claimed[64];
	return claimed[(unsigned)device % 64];
}

// automatic mode: what the arenas hold, plus the free memory of the device that no other context of the process has claimed, less
// the headroom
int64_t allowance_locked(Ledger &L)
{
	if (L.budget > 0) return L.allowance_last = L.budget;
	size_t free_b = 0, total_b = 0;
	MPB_CUDA_OK(cudaSetDevice(L.device));
	MPB_CUDA_OK(cudaMemGetInfo(&free_b, &total_b));
	const int64_t a = L.held + (int64_t)free_b - (device_claimed(L.device) - L.claim) - std::max(Ledger::kHeadroom, (int64_t)total_b / 16);
	return L.allowance_last = a > 0 ? a : 0;
}

void set_claim_locked(Ledger &L, int64_t bytes)
{
	device_claimed(L.device) += bytes - L.claim;
	L.claim = bytes;
}
} // namespace

void DevBuf::release()
{
	if (p) cudaFree(p);
	if (led) led->held -= (int64_t)cap;
	p = 0, cap = 0;
}

int64_t Ledger::plan(std::initializer_list<DevBuf*> mine, const std::function<int64_t(int64_t)> &f)
{
	std::lock_guard<std::mutex> lk(device_mutex(device));
	int64_t other = 0, own = 0;
	for (DevBuf *b : bufs) {
		if (std::find(mine.begin(), mine.end(), b) != mine.end()) own += (int64_t)b->cap;
		else if (b->busy) other += (int64_t)b->cap;
	}
	const int64_t room = allowance_locked(*this) - other;
	set_claim_locked(*this, std::max<int64_t>(f(room) - own, 0));
	return room;
}

void Ledger::end_claim()
{
	std::lock_guard<std::mutex> lk(device_mutex(device));
	set_claim_locked(*this, 0);
}

bool Ledger::fits(std::initializer_list<DevBuf*> mine, std::initializer_list<size_t> need)
{
	const size_t *n = need.begin();
	for (DevBuf *b : mine) if (*n++ > b->cap) return false;
	return true;
}

void Ledger::trim(std::initializer_list<DevBuf*> mine, std::initializer_list<size_t> need, int64_t room)
{
	int64_t tot = 0;
	const size_t *n = need.begin();
	for (DevBuf *b : mine) tot += (int64_t)std::max(b->cap, *n++);
	if (tot <= room) return;
	n = need.begin();
	for (DevBuf *b : mine) {
		const size_t want = *n++;
		if (b->cap > want + want / 4 + 4096) n_released += 1, bytes_released += (int64_t)b->cap, b->release();
	}
}

void Ledger::release_idle(int64_t target, const DevBuf *keep)
{
	while (held > target) {
		DevBuf *big = 0;
		for (DevBuf *b : bufs)
			if (b != keep && !b->busy && b->cap && (!big || b->cap > big->cap)) big = b;
		if (!big) return;
		n_released += 1, bytes_released += (int64_t)big->cap;
		big->release();
	}
}

// Growth of a working arena: in automatic mode the new capacity gets a quarter of slack (fewer regrowths).  When the growth would pass
// the allowance, idle arenas of other stages are released, largest first, and failing that the slack is dropped.  A slice planned within the allowance
// then stays within it; an item that does not fit alone grows past it (and may fail in cudaMalloc, as without a budget).
void Ledger::grow(DevBuf &b, size_t bytes)
{
	std::lock_guard<std::mutex> lk(device_mutex(device));
	const int64_t allow = allowance_locked(*this);
	// (under an explicit budget the stages plan their slices to fill it, and slack would crowd out the smaller arenas they did not plan)
	size_t want = bytes + (budget > 0 ? 0 : bytes / 4) + 4096;
	const int64_t rest = held - (int64_t)b.cap;
	if (rest + (int64_t)want > allow) {
		release_idle(allow - (int64_t)want + (int64_t)b.cap, &b);
		const int64_t rest2 = held - (int64_t)b.cap;
		if (rest2 + (int64_t)want > allow) want = std::max(bytes, (size_t)std::max<int64_t>(allow - rest2, 0));
		if (rest2 + (int64_t)want > allow) n_over_budget += 1; // past the allowance all the same: counted like an item that does not fit
	}
	const int64_t old = (int64_t)b.cap;
	if (b.p) MPB_CUDA_OK(cudaFree(b.p));
	held -= old, b.p = 0, b.cap = 0;
	MPB_CUDA_OK(cudaMalloc(&b.p, want));
	b.cap = want, held += (int64_t)want;
	peak = std::max(peak, held);
	set_claim_locked(*this, std::max<int64_t>(claim - ((int64_t)want - old), 0)); // (what was claimed is now held)
}

} // namespace cuda
} // namespace mpb
