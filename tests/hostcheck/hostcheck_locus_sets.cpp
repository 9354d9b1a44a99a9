// tests/hostcheck/hostcheck_locus_sets.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Locus sets (map_locus_sets, and loci_file_read + map_loci_file with sets, csrc/pipeline.cpp) over the oracle stages of
// hostcheck_loci_file.cpp (compiled into this translation unit) plus an oracle of the set seeding stage: the index of the genome made
// of a query's view contigs, as the reference builds it from a FASTA of those records -- ora_sketch_nt4 over both strands of every
// record, sorted, distinct (bucket, block) pairs -- the protein's seeds looked up in it, the adaptive occupancy cut-off of
// map.c:126-161, then the chains of OracleStages::seed_chain.  Lets tests/test_host_locus_sets.py check the host orchestration, the
// canonical genome of a set, the per-region coordinate move and the set file driver without a GPU.  Built under
// tests/_build/locus_sets/ by tests/build_hostcheck_locus_sets.py; never shipped.
#include "hostcheck_loci_file.cpp"

namespace {

// the anchors of one protein against contigs [c0, c1) of a locus view together, with the view's block ids; sorted
std::vector<uint64_t> set_anchors(const ora_tab_t *tab, const mp_idx_t *vi, int32_t c0, int32_t c1, int32_t max_occ_cap, const char *seq, int32_t len)
{
	const mp_idxopt_t &io = vi->opt;
	std::vector<uint64_t> pairs;
	for (int32_t k = c0; k < c1; ++k) {
		const int64_t L = vi->nt->ctg[k].len;
		std::vector<uint64_t> buf((size_t)L + 1);
		std::vector<uint8_t> nt((size_t)L + 1);
		for (int s = 0; s < 2; ++s) {
			const int64_t l = nt_fetch(vi->nt, k, 0, L, s, nt.data());
			const int64_t n = ora_sketch_nt4(tab, nt.data(), l, io.min_aa_len, io.kmer, io.mod_bit, io.bbit, vi->bo[k * 2 + s], buf.data());
			pairs.insert(pairs.end(), buf.begin(), buf.begin() + n);
		}
	}
	std::sort(pairs.begin(), pairs.end());
	pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end()); // index.c:71-90 keeps one entry per (bucket, block)
	std::vector<uint64_t> sd((size_t)len + 1);
	const int32_t n_sd = ora_sketch_prot(tab, seq, len, io.kmer, io.mod_bit, sd.data());
	std::sort(sd.begin(), sd.begin() + n_sd);
	auto lo = [&](uint64_t b) { return std::lower_bound(pairs.begin(), pairs.end(), b << 32) - pairs.begin(); };
	std::vector<uint64_t> cnt((size_t)n_sd);
	for (int32_t i = 0; i < n_sd; ++i) cnt[(size_t)i] = (uint64_t)(lo((sd[(size_t)i] >> 32) + 1) - lo(sd[(size_t)i] >> 32));
	int32_t max_occ = max_occ_cap;
	if (n_sd >= 8) { // map.c:158-161 + 126-141
		std::vector<uint64_t> c(cnt);
		std::sort(c.begin(), c.end());
		const uint64_t q25 = c[(size_t)(int64_t)(n_sd * .25 + .499)], q75 = c[(size_t)(int64_t)(n_sd * .75 + .499)];
		const int32_t r = (int32_t)(q75 + (q75 - q25) * 1.5 + 10.);
		if (r < max_occ) max_occ = r;
	}
	std::vector<uint64_t> a;
	for (int32_t i = 0; i < n_sd; ++i) {
		if (cnt[(size_t)i] > (uint64_t)max_occ) continue;
		for (int64_t j = lo(sd[(size_t)i] >> 32), e = j + (int64_t)cnt[(size_t)i]; j < e; ++j) a.push_back((uint64_t)(uint32_t)pairs[(size_t)j] << 32 | (uint32_t)sd[(size_t)i]);
	}
	std::sort(a.begin(), a.end());
	return a;
}

struct SetsOracle : LociOracle {
	bool locus_sets() override { return true; }
	void seed_chain_locus_sets(const mp_idx_t *vi, const int32_t *ctg_off, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override
	{
		ora_tab_t tab = product_tables();
		const int32_t w = 1 << vi->opt.bbit, spl = !(opt->flag & MP_F_NO_SPLICE);
		out.u_off.assign(1, 0), out.a_off.assign(1, 0);
		for (int32_t q = 0; q < b.n; ++q) { // the chaining of OracleStages::seed_chain (map.c:186-195)
			std::vector<uint64_t> av = set_anchors(&tab, vi, ctg_off[q], ctg_off[q + 1], opt->max_occ, b.seq[q], b.len[q]);
			int64_t n_a = (int64_t)av.size();
			uint64_t *a = (uint64_t*)malloc(sizeof(uint64_t) * (av.size() + 1));
			if (n_a) memcpy(a, av.data(), sizeof(uint64_t) * av.size());
			int32_t n_u = 0;
			uint64_t *u = 0;
			if (!(opt->flag & MP_F_NO_PRE_CHAIN) && spl) {
				ora_chain_par_t p = chain_par(w, w, w, opt, 2, 0, vi->opt.kmer, vi->opt.bbit);
				uint64_t *a2 = ora_chain(&p, n_a, a, &n_u, &u);
				free(a);
				a = a2, n_a = 0;
				for (int32_t i = 0; i < n_u; ++i) n_a += (uint32_t)u[i];
				free(u);
				u = 0;
				if (a) ora_sort64(a, a + n_a);
			}
			ora_chain_par_t p = chain_par(opt->max_intron, opt->max_gap, opt->bw, opt, opt->min_chn_cnt, opt->min_chn_sc, vi->opt.kmer, vi->opt.bbit);
			uint64_t *c = ora_chain(&p, n_a, a, &n_u, &u);
			free(a);
			int64_t nc = 0;
			for (int32_t i = 0; i < n_u; ++i) nc += (uint32_t)u[i];
			out.u.insert(out.u.end(), u, u + n_u);
			if (c) out.a.insert(out.a.end(), c, c + nc);
			out.u_off.push_back((int64_t)out.u.size()), out.a_off.push_back((int64_t)out.a.size());
			free(u); free(c);
		}
	}
};

} // namespace

extern "C" {

// mpb_map_locus_sets with the oracle stages behind it
int hc_map_locus_sets(const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names,
                      int32_t n_sets, const int64_t *set_off, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	SetsOracle st;
	return map_locus_sets(&st, mi, opt, n_seq, seqs, lens, names, n_sets, set_off, loci, n_reg_out, reg_out);
}

// mpb_map_locus_sets_file_multi_path with n_backends oracle backends (one mapper thread each when n_backends > 1); sets = 0 reads the
// file as mpb_map_loci_file does, one set per pair, on the same backends
int32_t hc_map_locus_sets_file(const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, int32_t n_backends, const char *out_path,
                               int32_t sets)
{
	if (!mi || !opt || n_backends < 1) return -1;
	LociFile in;
	int32_t rc = loci_file_read(mi, prot_fn, loci_fn, in, sets != 0);
	if (rc != 0) return rc;
	FILE *fp = fopen(out_path, "wb");
	if (!fp) return -2;
	std::vector<SetsOracle> st((size_t)n_backends);
	std::vector<Stages*> sp;
	for (SetsOracle &s : st) sp.push_back(&s);
	rc = map_loci_file(sp.data(), n_backends, mi, in, opt, fp);
	fclose(fp);
	return rc;
}

} // extern "C"
