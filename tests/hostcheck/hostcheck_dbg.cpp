// tests/hostcheck/hostcheck_dbg.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The oracle backend of hostcheck.cpp (compiled into this translation unit) with the seeds of --dbg-anchor: when the dispatcher
// asks for them (ChainSet::want_seeds), the sorted, max_occ-filtered anchors of each protein are returned next to the chains, as
// the CUDA backend returns them.  Exports the reference's mp_map_file() with this backend behind it, so that the reference CLI
// (main.c) or a test that drives the library like main.c does (tests/dbg_lib.py) sees every dump line of the --dbg-* switches.
// Built under tests/_build/dbg/ by tests/build_hostcheck_dbg.py; never shipped.
#define mp_map_file hc_oracle_mp_map_file // hostcheck.cpp's own entry, without the seeds, keeps out of the way
#include "hostcheck.cpp"
#undef mp_map_file

namespace {

struct SeedingOracle : Stages {
	OracleStages inner;
	void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override
	{
		inner.seed_chain(mi, opt, b, out);
		if (!out.want_seeds) return;
		ora_tab_t tab = product_tables();
		out.seed_off.assign(1, 0), out.seed.clear();
		for (int32_t q = 0; q < b.n; ++q) { // map.c:155-177, the input of the chaining above
			int64_t n_a = 0;
			uint64_t *a = ora_seed_anchors(&tab, mi->ki, mi->n_kb, mi->kb, mi->opt.kmer, mi->opt.mod_bit, opt->max_occ, b.seq[q], b.len[q], &n_a);
			if (a) out.seed.insert(out.seed.end(), a, a + n_a);
			out.seed_off.push_back((int64_t)out.seed.size());
			free(a);
		}
	}
	void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) override
	{
		inner.refine(mi, opt, b, jobs, out);
	}
	void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) override { inner.nasw(mi, base, b, jobs, out); }
};

} // namespace

extern "C" int32_t mp_map_file(const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, int)
{
	SeedingOracle st;
	return map_file(&st, mi, fn, opt, stdout);
}
