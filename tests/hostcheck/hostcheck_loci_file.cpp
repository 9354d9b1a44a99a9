// tests/hostcheck/hostcheck_loci_file.cpp -- TEST INFRASTRUCTURE ONLY.
//
// The locus file driver (loci_file_read + map_loci_file, csrc/pipeline.cpp) over the oracle stages and the locus seeding oracle of
// hostcheck_loci.cpp (compiled into this translation unit).  Lets tests/test_host_loci_file.py check the parsing, the refusals, the
// units, the output formats and the coordinate translation of mpb_map_loci_file* without a GPU.  Built under tests/_build/loci_file/
// by tests/build_hostcheck_loci_file.py; never shipped.
#include "hostcheck_loci.cpp"

extern "C" {

// mpb_map_loci_file_multi_path with n_backends oracle backends (one mapper thread each when n_backends > 1)
int32_t hc_map_loci_file(const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, int32_t n_backends, const char *out_path)
{
	if (!mi || !opt || n_backends < 1) return -1;
	LociFile in;
	int32_t rc = loci_file_read(mi, prot_fn, loci_fn, in);
	if (rc != 0) return rc;
	FILE *fp = fopen(out_path, "wb");
	if (!fp) return -2;
	std::vector<LociOracle> st((size_t)n_backends);
	std::vector<Stages*> sp;
	for (LociOracle &s : st) sp.push_back(&s);
	rc = map_loci_file(sp.data(), n_backends, mi, in, opt, fp);
	fclose(fp);
	return rc;
}

} // extern "C"
