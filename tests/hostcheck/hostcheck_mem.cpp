// hostcheck_mem.cpp -- the slice planner and the MPB_DEVICE_MEM parser of the device-memory budget (miniprot_b200/csrc/slices.hpp),
// exported for the CPU tests.
#include <string.h>
#include "slices.hpp"

extern "C" {

// cut[] receives the n_slices + 1 boundaries (room for n + 1); returns the number of slices, *n_over the slices of one item over
// the allowance.  count may be null.
int32_t hc_plan_slices(int32_t n, const int64_t *bytes, const int64_t *count, int64_t fixed, int64_t allowance, int64_t max_count, int32_t *cut, int32_t *n_over)
{
	mpb::SlicePlan p;
	mpb::plan_slices(n, bytes, count, fixed, allowance, max_count, p);
	memcpy(cut, p.cut.data(), sizeof(int32_t) * p.cut.size());
	*n_over = p.n_over;
	return p.n_slices();
}

int64_t hc_slice_max_count(void) { return mpb::kSliceMaxCount; }

int64_t hc_parse_mem_size(const char *s) { return mpb::parse_mem_size(s); }

} // extern "C"
