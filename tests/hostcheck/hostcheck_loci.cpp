// tests/hostcheck/hostcheck_loci.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Locus mode (map_loci, csrc/pipeline.cpp) with the oracle backend of hostcheck.cpp (compiled into this translation unit) plus an
// oracle of the locus seeding stage: the locus's index as the reference builds it from a one-record FASTA -- ora_sketch_nt4 over
// both strands, sorted, distinct (bucket, block) pairs -- the protein's seeds looked up in it, the adaptive occupancy cut-off of
// map.c:126-161 as ora_seed_anchors applies it, then the chains of OracleStages::seed_chain.  Lets tests/test_host_loci.py check the
// host orchestration and the coordinate translation of locus mode without a GPU.  Built under tests/_build/loci/ by
// tests/build_hostcheck_loci.py; never shipped.
#include <algorithm>
#define mp_map_file hc_oracle_mp_map_file // hostcheck.cpp's CLI entry is not needed here
#include "hostcheck.cpp"
#undef mp_map_file

namespace {

// the anchors of one protein against contig q of a locus view, with the view's block ids; malloc'ed, sorted, *n_a the count
uint64_t *locus_anchors(const ora_tab_t *tab, const mp_idx_t *vi, int32_t q, int32_t max_occ_cap, const char *seq, int32_t len, int64_t *n_a)
{
	const mp_idxopt_t &io = vi->opt;
	const int64_t L = vi->nt->ctg[q].len;
	std::vector<uint64_t> pairs, buf((size_t)L + 1);
	std::vector<uint8_t> nt((size_t)L + 1);
	for (int s = 0; s < 2; ++s) {
		const int64_t l = nt_fetch(vi->nt, q, 0, L, s, nt.data());
		const int64_t n = ora_sketch_nt4(tab, nt.data(), l, io.min_aa_len, io.kmer, io.mod_bit, io.bbit, vi->bo[q * 2 + s], buf.data());
		pairs.insert(pairs.end(), buf.begin(), buf.begin() + n);
	}
	std::sort(pairs.begin(), pairs.end());
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
	uint64_t *out = (uint64_t*)malloc(sizeof(uint64_t) * (a.size() + 1));
	if (!a.empty()) memcpy(out, a.data(), sizeof(uint64_t) * a.size());
	*n_a = (int64_t)a.size();
	return out;
}

struct LociOracle : Stages {
	OracleStages inner;
	bool loci_view(const mp_idx_t *, const mp_idx_t *) override { return true; } // the view's contigs are read straight from its genome
	void seed_chain_loci(const mp_idx_t *vi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override
	{
		ora_tab_t tab = product_tables();
		const int32_t w = 1 << vi->opt.bbit, spl = !(opt->flag & MP_F_NO_SPLICE);
		out.u_off.assign(1, 0), out.a_off.assign(1, 0);
		for (int32_t q = 0; q < b.n; ++q) { // the chaining of OracleStages::seed_chain (map.c:186-195)
			int64_t n_a = 0;
			uint64_t *a = locus_anchors(&tab, vi, q, opt->max_occ, b.seq[q], b.len[q], &n_a);
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
	void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override { inner.seed_chain(mi, opt, b, out); }
	void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) override
	{
		inner.refine(mi, opt, b, jobs, out);
	}
	void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) override { inner.nasw(mi, base, b, jobs, out); }
};

} // namespace

extern "C" {

// mpb_map_loci with the oracle stages behind it
int hc_map_loci(const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names, int32_t n_loci,
                const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	LociOracle st;
	return map_loci(&st, mi, opt, n_seq, seqs, lens, names, n_loci, loci, n_reg_out, reg_out);
}

// one PAF line (format.c:333), appended to a malloc'ed buffer: mpb_format_paf of the product library
int64_t hc_format_paf(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq, const mp_reg1_t *r, char **buf, int64_t *len,
                      int64_t *cap)
{
	Str s;
	s.s = *buf, s.l = *len, s.m = *cap;
	format_hit(s, mi, opt, qname, qlen, qseq, r);
	*buf = s.s, *len = s.l, *cap = s.m;
	return s.l;
}

} // extern "C"
