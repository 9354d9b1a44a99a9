// align.cpp -- host side of the per-region alignment: which DP problems exist, in which wave, and what
// to do with their answers (reference align.c).  The DP itself is the GPU nasw stage; nothing here
// touches a DP matrix.
//
//   plan_region()   align.c:239-323  seed filter, window, wave-1 problems (left ext, right ext, fills)
//   after_wave1()   align.c:290-296 / 324-330  conditional retries with io_end (wave 1')
//   after_retry()   align.c:297-301 / 331      wave-2 problems: the two spans found by the extensions
//   finish_region() align.c:331-339  CIGAR assembly + mp_extra_* statistics
#include <assert.h>
#include <stdio.h>
#include <atomic>
#include "internal.hpp"
#include "align.hpp"

namespace mpb {

// align.c:6-31: flag (bit 31) the anchors that sit inside "tight" runs -- consecutive anchors in the
// same frame, close on both sequences -- trimmed at both ends; only flagged anchors pin the DP.
static void mark_tight_anchors(int32_t n, uint64_t *a, int32_t max_aa_dist, int32_t min_cnt, int32_t kmer2, int32_t trim)
{
	for (int32_t i = 0; i < n; ++i) {
		int32_t j = i + 1;
		for (; j < n; ++j) {
			const int32_t x0 = (int32_t)(a[j - 1] >> 32), y0 = (int32_t)a[j - 1], x1 = (int32_t)(a[j] >> 32), y1 = (int32_t)a[j];
			if ((x1 - x0) % 3 != 0 || x1 - x0 > max_aa_dist * 3 || y1 - y0 > max_aa_dist) break;
		}
		if (j - i < min_cnt) continue;
		int32_t k, t = (int32_t)a[j - 1];
		for (k = j - 2; k >= i; --k) if (t - (int32_t)a[k] >= trim) break;
		t = (int32_t)a[i] + 1 - kmer2;
		for (; i < k; ++i) if ((int32_t)a[i] + 1 - t >= trim) break;
		for (; i <= k; ++i) a[i] |= 1ULL << 31;
		i = j - 1;
	}
}

static inline uint8_t codon_aa(uint8_t n1, uint8_t n2, uint8_t n3)
{
	return (n1 > 3 || n2 > 3 || n3 > 3) ? ns_tab_aa20[(uint8_t)'X'] : ns_tab_codon[n1 << 4 | n2 << 2 | n3];
}

void make_ns_opt(const mp_mapopt_t *mo, ns_opt_t *no) // align.c:50-60
{
	ns_opt_init(no);
	no->go = mo->go, no->ge = mo->ge, no->io = mo->io, no->fs = mo->fs, no->xdrop = mo->xdrop, no->sc = mo->mat;
	no->ie_coef = mo->ie_coef;
	no->end_bonus = mo->end_bonus;
	no->sp_null_bonus = mo->sp_null_bonus;
	ns_opt_set_sp(no, mo->sp_model);
	for (int i = 0; i < 6; ++i) no->sp[i] = (int32_t)(no->sp[i] * mo->sp_scale + .499f);
}

void cigar_push(std::vector<uint32_t> &c, uint32_t op, int32_t len) // nasw.h:141-151
{
	if (c.empty() || op != (c.back() & 0xf) || op == NS_CIGAR_F || op == NS_CIGAR_G) c.push_back((uint32_t)len << 4 | op);
	else c.back() += (uint32_t)len << 4;
}

// One anchor-to-anchor segment (align.c:62-80): either the ungapped shortcut, resolved right here, or a DP job.
Fill RegionPlan::make_fill(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, int32_t ne0, int32_t ne1, int32_t ae0, int32_t ae1,
                           std::vector<DpJob> &jobs) const
{
	Fill f;
	f.ne0 = ne0, f.ne1 = ne1, f.ae0 = ae0, f.ae1 = ae1;
	const int32_t nlen = ne1 - ne0, alen = ae1 - ae0;
	if (nlen == alen * 3 && alen <= opt->kmer2) { // align.c:65-67 + 33-43
		int32_t sc = 0;
		const int64_t g = vs0 + ne0;
		// NB: the reference's loop counter runs over nucleotides but is bounded by the residue count
		// (align.c:36: "for (i = 0, j = 0; i < alen; i += 3, ++j)"), so only the first ceil(alen/3)
		// codons contribute to AS:i.  Reproduced on purpose: AS:i is part of the PAF.
		for (int32_t j = 0; j * 3 < alen; ++j) {
			const uint8_t na = codon_aa(nt_at_v(mi->nt, r->vid, g + j * 3), nt_at_v(mi->nt, r->vid, g + j * 3 + 1), nt_at_v(mi->nt, r->vid, g + j * 3 + 2));
			sc += opt->mat[na * opt->asize + ns_tab_aa20[(uint8_t)aa[ae0 + j]]];
		}
		f.score = sc, f.ungapped = true;
	} else {
		DpJob j;
		j.qid = qid, j.vid = r->vid, j.win_st = as, j.nt_st = vs0 + ne0, j.nl = nlen, j.aa_st = ae0, j.al = alen, j.flag = NS_F_CIGAR, j.io = opt->io;
		f.job = (int32_t)jobs.size();
		jobs.push_back(j);
	}
	return f;
}

bool RegionPlan::plan(const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t qid_, int32_t qlen_, const char *aa, mp_reg1_t *r_, int32_t extl0, int32_t extr0,
                      std::vector<DpJob> &jobs)
{
	r = r_, qid = qid_, qlen = qlen_;
	jobL = jobL2 = jobR = jobR2 = -1;
	fills.clear();
	mark_tight_anchors(r->cnt, r->a, 6, 3, opt->kmer2, opt->kmer2 + 1);
	int32_t i0 = 0;
	while (i0 < r->cnt && !(r->a[i0] >> 31 & 1)) ++i0;
	if (i0 == r->cnt) { r->cnt = 0; return false; } // align.c:252-255: nothing to pin the alignment
	int32_t extl = opt->max_ext, extr = opt->max_ext;
	if (r->qs >= 10) extl = opt->max_intron / 2;
	if (qlen - r->qe >= 10) extr = opt->max_intron / 2;
	if (extl0 > 0) extl = extl < extl0 ? extl : extl0;
	if (extr0 > 0) extr = extr < extr0 ? extr : extr0;
	const int64_t ctg_len = mi->nt->ctg[r->vid >> 1].len;
	as = r->vs > extl ? r->vs - extl : 0;
	ae = r->ve + extr < ctg_len ? r->ve + extr : ctg_len;
	vs0 = r->vs;
	// left extension from the first pinned anchor (align.c:280-288)
	vs1 = vs0 + (int64_t)(r->a[i0] >> 32) + 1;
	as1 = (int32_t)(r->a[i0] & 0x7fffffffU) + 1;
	{
		DpJob j;
		j.qid = qid, j.vid = r->vid, j.win_st = as, j.nt_st = as, j.nl = (int32_t)(vs1 - as), j.aa_st = 0, j.al = as1, j.flag = NS_F_EXT_LEFT, j.io = opt->io;
		jobL = (int32_t)jobs.size();
		jobs.push_back(j);
	}
	int32_t ne0 = (int32_t)(r->a[i0] >> 32) + 1, ae0 = as1;
	for (int32_t i = i0 + 1; i < r->cnt; ++i) { // align.c:306-312
		if (!(r->a[i] >> 31 & 1)) continue;
		const int32_t ne1 = (int32_t)(r->a[i] >> 32) + 1, ae1 = (int32_t)(r->a[i] & 0x7fffffffU) + 1;
		fills.push_back(make_fill(mi, opt, aa, ne0, ne1, ae0, ae1, jobs));
		ne0 = ne1, ae0 = ae1;
	}
	ve_pin = ne0 + vs0, qe_pin = ae0;
	// align.c:316.  With fewer than 3 bases left the reference's extension loop never runs and it stops at an assertion
	// (nasw-sse.c:443); such a hit simply ends at the last pinned anchor here.
	has_right = qe_pin < qlen && ve_pin < ae && ae - ve_pin >= 3;
	if (has_right) {
		DpJob j;
		j.qid = qid, j.vid = r->vid, j.win_st = as, j.nt_st = ve_pin, j.nl = (int32_t)(ae - ve_pin), j.aa_st = qe_pin, j.al = qlen - qe_pin, j.flag = NS_F_EXT_RIGHT, j.io = opt->io;
		jobR = (int32_t)jobs.size();
		jobs.push_back(j);
	}
	return true;
}

void RegionPlan::after_wave1(const mp_mapopt_t *opt, const DpSet &w1, std::vector<DpJob> &retry)
{
	l_nt = w1.nt_len[(size_t)jobL], l_aa = w1.aa_len[(size_t)jobL];
	if (l_nt < 0 || (has_right && w1.nt_len[(size_t)jobR] < 0)) { // the stage refused the problem
		static std::atomic<bool> warned{false}; // several contexts plan on different host threads
		if (!warned.exchange(true)) fprintf(stderr, "[WARNING] an extension over more than 32767 residues is not supported; such hits are dropped\n");
		failed = true;
		return;
	}
	if (l_aa != as1 && l_nt < opt->max_ext && opt->io > opt->io_end) { // align.c:290-296: 5'-end exon
		const int64_t as_alt = vs1 - as > opt->max_ext ? vs1 - opt->max_ext : as;
		DpJob j;
		j.qid = qid, j.vid = r->vid, j.win_st = as, j.nt_st = as_alt, j.nl = (int32_t)(vs1 - as_alt), j.aa_st = 0, j.al = as1, j.flag = NS_F_EXT_LEFT, j.io = opt->io_end;
		jobL2 = (int32_t)retry.size();
		retry.push_back(j);
	}
	if (has_right) {
		r_nt = w1.nt_len[(size_t)jobR], r_aa = w1.aa_len[(size_t)jobR];
		if (r_aa < qlen - qe_pin && r_nt < opt->max_ext && opt->io > opt->io_end) { // align.c:324-330: 3'-end exon
			const int32_t l_ext = ae - ve_pin < opt->max_ext ? (int32_t)(ae - ve_pin) : opt->max_ext;
			DpJob j;
			j.qid = qid, j.vid = r->vid, j.win_st = as, j.nt_st = ve_pin, j.nl = l_ext, j.aa_st = qe_pin, j.al = qlen - qe_pin, j.flag = NS_F_EXT_RIGHT, j.io = opt->io_end;
			jobR2 = (int32_t)retry.size();
			retry.push_back(j);
		}
	}
}

void RegionPlan::after_retry(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, const DpSet &w1r, std::vector<DpJob> &jobs2)
{
	if (failed) return;
	if (jobL2 >= 0 && w1r.aa_len[(size_t)jobL2] == as1) l_nt = w1r.nt_len[(size_t)jobL2], l_aa = w1r.aa_len[(size_t)jobL2];
	if (jobR2 >= 0 && w1r.aa_len[(size_t)jobR2] == qlen - qe_pin) r_nt = w1r.nt_len[(size_t)jobR2], r_aa = w1r.aa_len[(size_t)jobR2];
	r->vs = vs1 - l_nt;
	r->qs = as1 - l_aa;
	// the span found by the left extension, aligned globally to get its CIGAR (first pass of the loop at align.c:306)
	left_fill = make_fill(mi, opt, aa, (int32_t)(r->vs - vs0), (int32_t)(vs1 - vs0), r->qs, as1, jobs2);
	if (has_right) // align.c:331
		right_fill = make_fill(mi, opt, aa, (int32_t)(ve_pin - vs0), (int32_t)(ve_pin - vs0) + r_nt, qe_pin, qe_pin + r_aa, jobs2);
}

// align.c:209-237
static int32_t dist_to_stop(const mp_idx_t *mi, const mp_reg1_t *r, int64_t ae)
{
	for (int64_t j = r->ve; j + 2 < ae; j += 3)
		if (codon_aa(nt_at_v(mi->nt, r->vid, j), nt_at_v(mi->nt, r->vid, j + 1), nt_at_v(mi->nt, r->vid, j + 2)) == 20) return (int32_t)(j - r->ve);
	return -1;
}

static int32_t dist_to_start(const mp_idx_t *mi, const mp_reg1_t *r, int64_t as, int64_t ae)
{
	for (int64_t j = r->vs; j >= as && j + 2 < ae; j -= 3) {
		const uint8_t a = codon_aa(nt_at_v(mi->nt, r->vid, j), nt_at_v(mi->nt, r->vid, j + 1), nt_at_v(mi->nt, r->vid, j + 2));
		if (a == 20) break;
		if (a == 12) return (int32_t)(r->vs - j); // 'M'
	}
	return -1;
}

// align.c:82-201: walk the CIGAR once; totals into r->p, one mp_feat_t per exon (+ stop codon)
static void fill_statistics(const mp_idx_t *mi, mp_reg1_t *r, const mp_mapopt_t *opt, int64_t ae, const char *aa /* from r->qs */, int32_t qlen)
{
	mp_extra_t *e = r->p;
	const uint8_t aa_stop = ns_tab_aa20[(uint8_t)'*'];
	const int64_t l_nt = ae - r->vs;
	auto nt = [&](int64_t i) -> uint8_t { return nt_at_v(mi->nt, r->vid, r->vs + i); };
	const bool has_stop = (r->qe == qlen && e->dist_stop == 0);
	int32_t n_intron = 0;
	for (int32_t k = 0; k < e->n_cigar; ++k) {
		const uint32_t op = e->cigar[k] & 0xf;
		n_intron += (op == NS_CIGAR_N || op == NS_CIGAR_U || op == NS_CIGAR_V);
	}
	r->n_exon = n_intron + 1;
	r->n_feat = r->n_exon + (has_stop ? 1 : 0);
	r->feat = (mp_feat_t*)calloc((size_t)r->n_feat, sizeof(mp_feat_t));
	e->blen = e->n_iden = e->n_plus = e->n_fs = e->n_stop = e->dp_max = 0;
	int32_t nl = 0, al = 0, ft = 0;
	int32_t blen0 = 0, iden0 = 0, score0 = 0, fs0 = 0, stop0 = 0, phase0 = 0, qs0 = r->qs;
	int64_t vs_exon = r->vs;
	char acc0[2] = { 0, 0 };
	auto score_codon = [&](uint8_t n1, uint8_t n2, uint8_t n3, char res) {
		const uint8_t na = codon_aa(n1, n2, n3), ra = ns_tab_aa20[(uint8_t)res];
		const int32_t s = opt->mat[na * opt->asize + ra];
		e->n_stop += (na == aa_stop), e->n_iden += (na == ra), e->n_plus += (s > 0), e->dp_max += s;
	};
	auto close_exon = [&](mp_feat_t *f) {
		f->type = MP_FEAT_CDS;
		f->vs = vs_exon, f->qs = qs0, f->qe = r->qs + al, f->phase = (int16_t)phase0;
		f->blen = e->blen - blen0, f->n_iden = e->n_iden - iden0, f->n_fs = e->n_fs - fs0, f->n_stop = e->n_stop - stop0, f->score = e->dp_max - score0;
		if (ft > 1) f->acceptor[0] = acc0[0], f->acceptor[1] = acc0[1];
	};
	for (int32_t k = 0; k < e->n_cigar; ++k) {
		const int32_t op = (int32_t)(e->cigar[k] & 0xf), len = (int32_t)(e->cigar[k] >> 4), len3 = len * 3;
		if (op == NS_CIGAR_M) {
			for (int32_t l = 0; l < len; ++l) score_codon(nt(nl + l * 3), nt(nl + l * 3 + 1), nt(nl + l * 3 + 2), aa[al + l]);
			nl += len3, al += len, e->blen += len3;
		} else if (op == NS_CIGAR_I) {
			e->dp_max -= opt->go + opt->ge * len;
			al += len, e->blen += len3;
		} else if (op == NS_CIGAR_D) {
			for (int32_t l = 0; l < len; ++l) e->n_stop += (codon_aa(nt(nl + l * 3), nt(nl + l * 3 + 1), nt(nl + l * 3 + 2)) == aa_stop);
			e->dp_max -= opt->go + opt->ge * len;
			nl += len3, e->blen += len3;
		} else if (op == NS_CIGAR_F) {
			e->dp_max -= opt->fs;
			nl += len, e->blen += len, e->n_fs++;
		} else if (op == NS_CIGAR_G) {
			e->dp_max -= opt->fs;
			nl += len, ++al, e->blen += 3, e->n_fs++;
		} else if (op == NS_CIGAR_N || op == NS_CIGAR_U || op == NS_CIGAR_V) {
			if (op == NS_CIGAR_U) score_codon(nt(nl), nt(nl + len - 2), nt(nl + len - 1), aa[al]), e->blen += 3;
			else if (op == NS_CIGAR_V) score_codon(nt(nl), nt(nl + 1), nt(nl + len - 1), aa[al]), e->blen += 3;
			mp_feat_t *f = &r->feat[ft++];
			close_exon(f);
			const int32_t head = op == NS_CIGAR_N ? 0 : op == NS_CIGAR_U ? 1 : 2; // codon bases left of the intron
			f->ve = r->vs + nl + head;
			vs_exon = r->vs + nl + len - (head ? 3 - head : 0);
			phase0 = head ? 3 - head : 0;
			f->donor[0] = f->ve - r->vs < l_nt ? ns_tab_nt_i2c[nt(f->ve - r->vs)] : '.';
			f->donor[1] = f->ve - r->vs + 1 < l_nt ? ns_tab_nt_i2c[nt(f->ve - r->vs + 1)] : '.';
			qs0 = f->qe, fs0 = e->n_fs, stop0 = e->n_stop, score0 = e->dp_max, blen0 = e->blen, iden0 = e->n_iden;
			acc0[0] = vs_exon - r->vs >= 2 ? ns_tab_nt_i2c[nt(vs_exon - r->vs - 2)] : '.';
			acc0[1] = vs_exon - r->vs >= 1 ? ns_tab_nt_i2c[nt(vs_exon - r->vs - 1)] : '.';
			nl += len, al += (op != NS_CIGAR_N);
		}
	}
	{
		mp_feat_t *f = &r->feat[ft++];
		close_exon(f);
		f->ve = r->vs + nl;
	}
	if (has_stop) {
		mp_feat_t *f = &r->feat[ft++];
		f->type = MP_FEAT_STOP;
		f->vs = r->ve, f->ve = r->ve + 3, f->qs = f->qe = r->qe + al, f->phase = 0, f->n_fs = 0, f->blen = 3, f->n_iden = 0;
	}
	if (nl != r->ve - r->vs || al != r->qe - r->qs) { // cannot happen without --spsc (align.c:193-200)
		fprintf(stderr, "[ERROR] inconsistent CIGAR (%d!=%d or %d!=%d)\n", nl, (int)(r->ve - r->vs), al, r->qe - r->qs);
		free(r->p); free(r->feat);
		r->p = 0, r->feat = 0;
	}
}

void RegionPlan::finish(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *aa, const DpSet &w1, const DpSet &w2)
{
	if (failed) { r->p = 0; return; }
	std::vector<uint32_t> cg;
	int32_t score = 0;
	auto take = [&](const Fill &f, const DpSet &src) {
		if (f.ungapped) cigar_push(cg, NS_CIGAR_M, f.ae1 - f.ae0), score += f.score;
		else {
			for (int64_t k = src.cig_off[(size_t)f.job]; k < src.cig_off[(size_t)f.job + 1]; ++k) cigar_push(cg, src.cig[(size_t)k] & 0xf, (int32_t)(src.cig[(size_t)k] >> 4));
			score += src.score[(size_t)f.job];
		}
	};
	take(left_fill, w2);
	for (size_t i = 0; i < fills.size(); ++i) take(fills[i], w1);
	r->ve = ve_pin, r->qe = qe_pin;
	if (has_right) {
		take(right_fill, w2);
		r->ve += r_nt, r->qe += r_aa;
	}
	// align.c:203-212,336-339
	r->p = (mp_extra_t*)calloc(1, sizeof(mp_extra_t) + sizeof(uint32_t) * cg.size());
	r->p->dp_score = score;
	r->p->n_cigar = r->p->m_cigar = (int32_t)cg.size();
	if (!cg.empty()) memcpy(r->p->cigar, cg.data(), sizeof(uint32_t) * cg.size());
	r->p->dist_stop = dist_to_stop(mi, r, ae);
	r->p->dist_start = dist_to_start(mi, r, as, ae);
	fill_statistics(mi, r, opt, ae, aa + r->qs, qlen);
}

} // namespace mpb
