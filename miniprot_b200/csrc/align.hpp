// align.hpp -- per-region alignment plan (host state machine around the GPU nasw stage); see align.cpp.
#pragma once
#include "internal.hpp"

namespace mpb {

void make_ns_opt(const mp_mapopt_t *mo, ns_opt_t *no);
void cigar_push(std::vector<uint32_t> &c, uint32_t op, int32_t len);

struct Fill {             // one anchor-to-anchor (or extension-span) global alignment
	int32_t ne0 = 0, ne1 = 0; // nucleotide span relative to vs0
	int32_t ae0 = 0, ae1 = 0; // residue span
	int32_t job = -1;         // index into the wave's job list, or -1
	int32_t score = 0;        // score of the ungapped shortcut
	bool ungapped = false;
};

struct RegionPlan {
	mp_reg1_t *r = 0;
	int32_t qid = 0, qlen = 0;
	int64_t as = 0, ae = 0;   // DP window on the strand
	int64_t vs0 = 0;          // region start before extension (anchor coordinates are relative to it)
	int64_t vs1 = 0;          // end (exclusive) of the first pinned anchor
	int32_t as1 = 0;          // its residue end (exclusive)
	int64_t ve_pin = 0;       // end of the last pinned anchor
	int32_t qe_pin = 0;
	bool has_right = false;
	bool whole = false;       // --dbg-aflt (align.c:248,303): no seed filter, one global DP from the extended start to the region's end
	bool failed = false;      // a DP problem of this region could not be run (extension over more than 32767 residues, or a whole-region
	                          // traceback larger than the free device memory): the region is dropped
	int32_t jobL = -1, jobL2 = -1, jobR = -1, jobR2 = -1;
	int32_t l_nt = 0, l_aa = 0, r_nt = 0, r_aa = 0; // accepted extension results
	Fill left_fill, right_fill; // wave 2
	std::vector<Fill> fills;    // wave 1: between pinned anchors, in order

	Fill make_fill(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, int32_t ne0, int32_t ne1, int32_t ae0, int32_t ae1,
	               std::vector<DpJob> &jobs) const;
	// returns false when the region has no pinned anchor and is dropped; whole = --dbg-aflt (MP_DBG_MORE_DP)
	bool plan(const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t qid, int32_t qlen, const char *aa, mp_reg1_t *r, int32_t extl0, int32_t extr0, bool whole,
	          std::vector<DpJob> &jobs);
	// wave-1 job indices were taken in a list that is appended to the wave's list at position d
	void rebase_wave1(int32_t d)
	{
		if (jobL >= 0) jobL += d;
		if (jobR >= 0) jobR += d;
		for (Fill &f : fills) if (f.job >= 0) f.job += d;
	}
	void after_wave1(const mp_mapopt_t *opt, const DpSet &w1, std::vector<DpJob> &retry);
	void after_retry(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, const DpSet &w1r, std::vector<DpJob> &jobs2);
	void finish(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, const DpSet &w1, const DpSet &w2);
};

} // namespace mpb
