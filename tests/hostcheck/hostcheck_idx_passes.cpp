// hostcheck_idx_passes.cpp -- the pass planner of the device index build (plan_bucket_passes, miniprot_b200/csrc/slices.hpp),
// exported for the CPU tests.
#include <string.h>
#include "slices.hpp"

extern "C" {

// cut[] receives the n_passes + 1 bucket boundaries (room for n_bucket + 1); returns the number of passes, *n_over the passes over
// the allowance.
int32_t hc_plan_bucket_passes(uint32_t n_bucket, const uint32_t *cnt, int64_t per_pair, int64_t fixed, int64_t allowance, int32_t max_passes, int32_t *cut,
                              int32_t *n_over)
{
	mpb::SlicePlan p;
	mpb::plan_bucket_passes(n_bucket, cnt, per_pair, fixed, allowance, max_passes, p);
	memcpy(cut, p.cut.data(), sizeof(int32_t) * p.cut.size());
	*n_over = p.n_over;
	return p.n_slices();
}

int32_t hc_idx_max_passes(void) { return mpb::kIdxMaxPasses; }

int64_t hc_pass_max_pairs(void) { return mpb::kSliceMaxCount; }

} // extern "C"
