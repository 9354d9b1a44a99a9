// tests/hostcheck/hostcheck_multi.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The multi-context file driver (map_file_multi, csrc/pipeline.cpp) with n independent oracle backends behind it, for the CPU
// tests of tests/test_host_multi.py.  The oracle backend is the one of hostcheck.cpp, compiled into this translation unit (its
// OracleStages lives in an anonymous namespace there).  Built under tests/_build/ by tests/build_hostcheck_multi.py; never shipped.
#include <chrono>
#include <memory>
#include <thread>
#include "hostcheck.cpp"

namespace {

// One oracle backend, optionally slowed down: with HC_UNIT_DELAY=<seed> every batch waits 0..15 ms, drawn from the seed and the
// batch's first protein name, before its first stage.  With several mappers the work units then finish out of input order, which
// the writer of map_file_multi must undo.
struct DelayedOracle : Stages {
	OracleStages inner;
	void batch_begin(const Batch &b) override
	{
		if (const char *e = getenv("HC_UNIT_DELAY")) {
			if (b.n > 0) {
				uint64_t h = (uint64_t)strtoull(e, 0, 10) * 0x9e3779b97f4a7c15ULL + 1;
				for (const char *p = b.name ? b.name[0] : b.seq[0]; *p; ++p) h = (h ^ (uint8_t)*p) * 0x100000001b3ULL;
				std::this_thread::sleep_for(std::chrono::milliseconds((h >> 29) % 16));
			}
		}
		inner.batch_begin(b);
	}
	void batch_end() override { inner.batch_end(); }
	void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override { inner.seed_chain(mi, opt, b, out); }
	void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) override
	{
		inner.refine(mi, opt, b, jobs, out);
	}
	void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) override { inner.nasw(mi, base, b, jobs, out); }
};

} // namespace

extern "C" {

// map a protein FASTA against a genome FASTA through map_file_multi over n_mappers oracle backends (one mapper thread each) and
// write the output to out_path; returns what map_file_multi returns (-1 for a protein file that cannot be opened)
int hc_map_file_multi(const char *genome, const char *prot, const char *out_path, uint32_t flag, int64_t mini_batch, int32_t n_mappers)
{
	mp_idxopt_t io;
	mp_mapopt_t mo;
	mp_verbose = 1;
	mp_start();
	mp_idxopt_init(&io);
	mp_mapopt_init(&mo);
	mo.flag |= flag;
	if (mini_batch > 0) mo.mini_batch_size = mini_batch;
	if (getenv("HC_GFF_DELIM")) mo.gff_delim = getenv("HC_GFF_DELIM")[0]; // --gff-delim
	mp_idx_t *mi = mp_idx_load(genome, &io, 4);
	if (!mi) return -1;
	FILE *fp = fopen(out_path, "wb");
	if (!fp) return -2;
	std::vector<std::unique_ptr<DelayedOracle>> own;
	std::vector<Stages*> st;
	for (int32_t k = 0; k < n_mappers; ++k) own.emplace_back(new DelayedOracle), st.push_back(own.back().get());
	int32_t rc = map_file_multi(st.data(), n_mappers, mi, prot, &mo, fp);
	fclose(fp);
	mp_idx_destroy(mi);
	return rc;
}

} // extern "C"
