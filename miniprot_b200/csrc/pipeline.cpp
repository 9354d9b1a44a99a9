// pipeline.cpp -- the GPU batch dispatcher that replaces the reference's per-query worker
// (map.c:264 worker_for -> map.c:143 mp_map), and the file-level driver around it (map.c:273-343).
//
// The reference maps one protein at a time, start to finish, on one CPU thread.  Here a whole mini-batch
// moves through the same steps together, so that each compute step is ONE device stage over all proteins:
//
//   S1  seed_chain   sketch + index lookup + anchor sort + pre-chain + chain          (map.c:155-195)
//   H1  regions      chains -> regions, order, primary/secondary, ext budgets          (map.c:196-208)
//   S2  refine       per region: window 5-mers x protein 5-mers -> base-level chain   (map.c:32-111)
//   H2  re-rank, seed filter, DP work list                                              (map.c:217-226, align.c)
//   S3  nasw waves   wave 1 (extensions + inner fills), 1' (io_end retries), 2 (spans) (align.c:280-333)
//   H3  statistics, final ranking                                                       (map.c:233-236)
//
// Results per protein are identical to mp_map() (no state crosses proteins: SURVEY 8b "determinism contract").
#include <stdio.h>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <errno.h>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include "internal.hpp"
#include "align.hpp"
#include "fastx.hpp"
#include "parfor.hpp"

namespace mpb {

namespace {

struct QueryState {
	mp_reg1_t *reg = 0;
	int32_t n_reg = 0;
	std::vector<uint64_t> anchors; // collated refined anchors of all regions (map.c:217 mp_collate_a)
	std::vector<uint64_t> ext;
};

template <class... T> void put_fmt(Str &s, const char *fmt, T... v)
{
	char line[1024];
	const int l = snprintf(line, sizeof(line), fmt, v...);
	if (l < (int)sizeof(line)) s.put(line, l);
	else {
		std::vector<char> big((size_t)l + 1);
		snprintf(big.data(), big.size(), fmt, v...);
		s.put(big.data(), l);
	}
}

// map.c:179-184: the seeds of one protein, with contig, strand and offset of their block
void dump_seeds(Str &s, const mp_idx_t *mi, int64_t n, const uint64_t *a)
{
	for (int64_t k = 0; k < n; ++k) {
		const uint64_t blk = a[k] >> 32;
		const int32_t v = idx_block2vid(mi, (uint32_t)blk);
		put_fmt(s, "X\t%ld\t%s\t%c\t%ld\t%d\n", (long)blk, mi->nt->ctg[v >> 1].name, "+-"[v & 1], (long)((blk - mi->bo[v]) << mi->opt.bbit), (int32_t)(uint32_t)a[k]);
	}
}

// map.c:113-124 (mp_dbg_chain, label Y1): every anchor counted by a first-round region, offset from the block of its strand.  A chain
// cut at a contig boundary still counts the anchors of the side it lost, and they print with the kept strand's first block: the
// difference may be negative, and is computed as the reference's 64-bit wrap-around.
void dump_chains(Str &s, const mp_idx_t *mi, int32_t n_reg, const mp_reg1_t *reg, const uint64_t *a)
{
	for (int32_t i = 0; i < n_reg; ++i) {
		const mp_reg1_t *r = &reg[i];
		for (int32_t k = 0; k < r->cnt; ++k) {
			const uint64_t ak = a[r->off + k];
			const int64_t off = (int64_t)(((ak >> 32) - (uint64_t)mi->bo[r->vid]) << mi->opt.bbit);
			put_fmt(s, "Y1\t%d\t%ld\t%s\t%c\t%ld\t%d\n", i, (long)(ak >> 32), mi->nt->ctg[r->vid >> 1].name, "+-"[r->vid & 1], (long)off, (int32_t)(uint32_t)ak);
		}
	}
}

} // namespace

bool bad_dbg_flags(const mp_mapopt_t *opt)
{
	if (!(mp_dbg_flag & MP_DBG_NO_REFINE) || (opt->flag & MP_F_NO_ALIGN)) return false;
	fprintf(stderr, "[miniprot_b200] --dbg-no-refine is supported with -A only (the reference aligns regions without refined anchors and crashes)\n");
	return true;
}

void map_batch(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, int32_t *n_reg_out, mp_reg1_t **reg_out, int32_t qr_tid)
{
	const int32_t n = b.n, kmer = mi->opt.kmer;
	// one reading of the switches for the whole batch.  The entry points refuse --dbg-no-refine without -A (bad_dbg_flags); should
	// that case get here anyway, the regions are refined as usual rather than aligned without anchors.
	const int32_t dbg = mp_dbg_flag;
	const bool qr = (dbg & MP_DBG_QNAME) && qr_tid >= 0, no_refine = (dbg & MP_DBG_NO_REFINE) && (opt->flag & MP_F_NO_ALIGN);
	const bool dumps = qr || (dbg & (MP_DBG_ANCHOR | MP_DBG_CHAIN));
	std::vector<QueryState> qs((size_t)n);
	auto t_prev = std::chrono::steady_clock::now();
	auto lap = [&](int phase) {
		const auto now = std::chrono::steady_clock::now();
		st->note_wall(phase, std::chrono::duration<double, std::milli>(now - t_prev).count());
		t_prev = now;
	};

	// ---- S1
	st->batch_begin(b);
	ChainSet cs;
	cs.want_seeds = (dbg & MP_DBG_ANCHOR) != 0;
	st->seed_chain(mi, opt, b, cs);
	const bool x_lines = cs.want_seeds && cs.seed_off.size() == (size_t)n + 1;
	if (cs.want_seeds && !x_lines && n > 0) { // a backend that does not keep the seeding contract: no X lines rather than a bad read
		static std::atomic<bool> warned{false};
		if (!warned.exchange(true)) fprintf(stderr, "[WARNING] the seeding stage returned no seeds: --dbg-anchor prints nothing\n");
	}
	lap(0);

	// ---- H1 + S2 work list
	// (the host phases are independent per protein: contiguous ranges of proteins on the worker pool, per-range results
	// concatenated in order; so are the dump lines of the --dbg-* switches, formatted per range and written in order)
	std::vector<RefineJob> rjobs;
	std::vector<int32_t> rjob_first((size_t)n + 1, 0);
	{
		std::vector<std::vector<RefineJob>> part(64);
		std::vector<Str> dump(dumps ? 64 : 0);
		const int n_part = par_ranges(n, 64, [&](int lo, int hi, int c) {
			std::vector<RefineJob> &out = part[(size_t)c];
			for (int32_t q = lo; q < hi; ++q) {
				QueryState &Q = qs[(size_t)q];
				const int32_t n_u = (int32_t)(cs.u_off[(size_t)q + 1] - cs.u_off[(size_t)q]);
				const uint64_t *u = cs.u.data() + cs.u_off[(size_t)q], *a = cs.a.data() + cs.a_off[(size_t)q];
				if (qr) put_fmt(dump[(size_t)c], "QR\t%s\t%d\t%d\n", b.name && b.name[q] ? b.name[q] : "*", b.len[q], qr_tid); // map.c:268
				if (x_lines) dump_seeds(dump[(size_t)c], mi, cs.seed_off[(size_t)q + 1] - cs.seed_off[(size_t)q], cs.seed.data() + cs.seed_off[(size_t)q]);
				Q.reg = regs_from_chains(mi, n_u, u, a, &Q.n_reg);
				regs_sort(&Q.n_reg, Q.reg);
				regs_set_parent(opt->mask_level, opt->mask_len, Q.n_reg, Q.reg, kmer, 0);
				regs_select_sub(opt->pri_ratio * opt->pri_ratio, kmer * 2, opt->best_n, &Q.n_reg, Q.reg);
				if (dbg & MP_DBG_CHAIN) dump_chains(dump[(size_t)c], mi, Q.n_reg, Q.reg, a);
				if (no_refine) continue;
				regs_max_ext(0, Q.n_reg, Q.reg, a, 100, opt->max_ext, Q.ext);
				for (int32_t i = 0; i < Q.n_reg; ++i) { // window of map.c:41-42
					const mp_reg1_t *r = &Q.reg[i];
					const int64_t ctg_len = mi->nt->ctg[r->vid >> 1].len;
					const int32_t extl = (int32_t)(Q.ext[(size_t)i] >> 32), extr = (int32_t)Q.ext[(size_t)i];
					RefineJob j;
					j.qid = q, j.vid = r->vid;
					j.as = r->vs > extl ? r->vs - extl : 0;
					j.ae = r->ve + extr < ctg_len ? r->ve + extr : ctg_len;
					out.push_back(j);
				}
			}
		});
		for (int c = 0; c < n_part; ++c) rjobs.insert(rjobs.end(), part[(size_t)c].begin(), part[(size_t)c].end());
		for (int32_t q = 0; q < n; ++q) rjob_first[(size_t)q + 1] = rjob_first[(size_t)q] + qs[(size_t)q].n_reg;
		if (dumps) { // one block per batch: the dumps of contexts that map other units concurrently do not interleave with it
			flockfile(stderr);
			for (int c = 0; c < n_part; ++c) {
				if (dump[(size_t)c].l) fwrite(dump[(size_t)c].s, 1, (size_t)dump[(size_t)c].l, stderr);
				free(dump[(size_t)c].s);
			}
			funlockfile(stderr);
		}
	}
	cs = ChainSet(); // first-round anchors are not needed any more
	lap(1);

	// ---- S2 (none with --dbg-no-refine -A: the first-round regions are the result, map.c:205)
	RefineSet rs;
	if (!no_refine) st->refine(mi, opt, b, rjobs, rs);
	lap(2);

	// ---- H2: adopt refined chains (map.c:83-109), re-rank (map.c:217-221)
	const int32_t k2 = opt->kmer2;
	if (!no_refine) par_ranges(n, 64, [&](int q_lo, int q_hi, int) {
	for (int32_t q = q_lo; q < q_hi; ++q) {
		QueryState &Q = qs[(size_t)q];
		int32_t kept = 0;
		std::vector<int64_t> offs;
		Q.anchors.clear();
		for (int32_t i = 0; i < Q.n_reg; ++i) {
			const size_t jb = (size_t)(rjob_first[(size_t)q] + i);
			const int64_t na = rs.off[jb + 1] - rs.off[jb];
			if (na == 0) continue;
			mp_reg1_t r = Q.reg[i];
			const uint64_t *ra = rs.a.data() + rs.off[jb];
			const int64_t as = rjobs[jb].as;
			r.chn_sc = rs.sc[jb];
			r.cnt = (int32_t)na, r.off = (int32_t)Q.anchors.size();
			r.qs = (int32_t)(uint32_t)ra[0] - (k2 - 1);
			r.qe = (int32_t)(uint32_t)ra[na - 1] + 1;
			r.vs = as + (int64_t)(ra[0] >> 32) + 1 - 3 * k2;
			r.ve = as + (int64_t)(ra[na - 1] >> 32) + 1;
			for (int64_t t = 0; t < na; ++t)
				Q.anchors.push_back(((ra[t] >> 32) + (uint64_t)(as - r.vs)) << 32 | (ra[t] & 0xffffffffULL));
			r.chn_sc_ungap = chain_score_ungapped(r.cnt, Q.anchors.data() + r.off, k2);
			Q.reg[kept++] = r;
		}
		Q.n_reg = kept;
		for (int32_t i = 0; i < Q.n_reg; ++i) Q.reg[i].a = Q.anchors.data() + Q.reg[i].off;
		regs_sort(&Q.n_reg, Q.reg);
		regs_set_parent(opt->mask_level, opt->mask_len, Q.n_reg, Q.reg, kmer, 0);
		regs_select_sub(opt->pri_ratio * opt->pri_ratio, kmer * 2, opt->best_n, &Q.n_reg, Q.reg);
	}
	});
	rs = RefineSet();

	// ---- S3: alignment in three waves
	if (!(opt->flag & MP_F_NO_ALIGN)) {
		ns_opt_t nso;
		make_ns_opt(opt, &nso);
		std::vector<RegionPlan> plans;
		std::vector<DpJob> w1, w1r, w2;
		DpSet o1, o1r, o2;
		{
			std::vector<std::vector<RegionPlan>> pplan(64);
			std::vector<std::vector<DpJob>> pjobs(64);
			const int n_part = par_ranges(n, 64, [&](int q_lo, int q_hi, int c) {
				for (int32_t q = q_lo; q < q_hi; ++q) {
					QueryState &Q = qs[(size_t)q];
					regs_max_ext(mi->nt, Q.n_reg, Q.reg, Q.anchors.data(), 100, opt->max_intron / 2, Q.ext);
					for (int32_t i = 0; i < Q.n_reg; ++i) {
						RegionPlan p;
						if (p.plan(mi, opt, q, b.len[q], b.seq[q], &Q.reg[i], (int32_t)(Q.ext[(size_t)i] >> 32), (int32_t)Q.ext[(size_t)i], (dbg & MP_DBG_MORE_DP) != 0,
						           pjobs[(size_t)c]))
							pplan[(size_t)c].push_back(std::move(p));
					}
				}
			});
			for (int c = 0; c < n_part; ++c) {
				const int32_t base = (int32_t)w1.size();
				w1.insert(w1.end(), pjobs[(size_t)c].begin(), pjobs[(size_t)c].end());
				for (RegionPlan &p : pplan[(size_t)c]) {
					p.rebase_wave1(base);
					plans.push_back(std::move(p));
				}
			}
		}
		lap(3);
		static const bool trace = getenv("MPB_TRACE") != 0;
		double tt[6] = { mp_realtime() };
		st->nasw(mi, &nso, b, w1, o1);
		tt[1] = mp_realtime();
		for (RegionPlan &p : plans) p.after_wave1(opt, o1, w1r);
		tt[2] = mp_realtime();
		st->nasw(mi, &nso, b, w1r, o1r);
		tt[3] = mp_realtime();
		for (RegionPlan &p : plans) p.after_retry(mi, opt, b.seq[p.qid], o1r, w2);
		tt[4] = mp_realtime();
		st->nasw(mi, &nso, b, w2, o2);
		tt[5] = mp_realtime();
		if (trace)
			fprintf(stderr, "[mpb-trace] S3: wave1 %.2f ms, host %.2f, retries %.2f, host %.2f, wave2 %.2f\n", (tt[1] - tt[0]) * 1e3, (tt[2] - tt[1]) * 1e3, (tt[3] - tt[2]) * 1e3,
			        (tt[4] - tt[3]) * 1e3, (tt[5] - tt[4]) * 1e3);
		lap(4);
		par_ranges((int)plans.size(), 256, [&](int lo, int hi, int) {
			for (int k = lo; k < hi; ++k) plans[(size_t)k].finish(mi, opt, b.seq[plans[(size_t)k].qid], o1, o2);
		});
		// ---- H3 (map.c:228-236)
		par_ranges(n, 64, [&](int q_lo, int q_hi, int) {
			for (int32_t q = q_lo; q < q_hi; ++q) {
				QueryState &Q = qs[(size_t)q];
				int32_t k = 0;
				for (int32_t i = 0; i < Q.n_reg; ++i) if (Q.reg[i].p) Q.reg[k++] = Q.reg[i];
				Q.n_reg = k;
				regs_sort(&Q.n_reg, Q.reg);
				regs_select_multi_exon(Q.n_reg, Q.reg, opt->io);
				regs_set_parent(opt->mask_level, opt->mask_len, Q.n_reg, Q.reg, kmer, 0);
				regs_select_sub(opt->pri_ratio, kmer * 2, opt->best_n, &Q.n_reg, Q.reg);
			}
		});
	}
	for (int32_t q = 0; q < n; ++q) {
		QueryState &Q = qs[(size_t)q];
		for (int32_t i = 0; i < Q.n_reg; ++i) Q.reg[i].a = 0; // the anchor store dies with this call
		n_reg_out[q] = Q.n_reg, reg_out[q] = Q.reg;
	}
	st->batch_end();
	lap(5);
}

// The end, on the strand of hit r of set s (in contig coordinates), of the set's range that holds the hit: en on +, len(cid) - st on -.
// The ranges of a set are disjoint and sorted, and a hit lies in one of them: the last one that starts at or before the hit's start.
static int64_t range_end(const mp_idx_t *mi, const LocusSets &ls, int32_t s, const mp_reg1_t *r)
{
	const int32_t cid = (int32_t)(r->vid >> 1), rev = r->vid & 1;
	const int64_t clen = mi->nt->ctg[cid].len, pos = rev ? clen - r->vs - 1 : r->vs; // a base of the hit on the + strand
	const mpb_locus_t *b = ls.rng.data() + ls.off[(size_t)s], *e = ls.rng.data() + ls.off[(size_t)s + 1];
	const mpb_locus_t *l = std::upper_bound(b, e, std::make_pair(cid, pos), [](const std::pair<int32_t, int64_t> &x, const mpb_locus_t &y) {
		return x.first < y.cid || (x.first == y.cid && x.second < y.st);
	}) - 1;
	return rev ? clen - l->st : l->en;
}

// map.c:293-326: per protein, hits in rank order subject to --outn / --outs / --outc; unmapped line with -u.  Every printed hit
// gets the next number of a counter that runs over the whole file (the MP%06d ids of GFF / GTF, map.c:306): the hits each
// protein will print are counted first, so that formatting -- independent per protein -- can run on the worker pool, each range
// into its own buffer, written in order.  sets (locus mode): query q is the protein of set s0 + q, whose hits are in contig
// coordinates but must not read the genome past the end of their range (format_output's nt_lim), as the reference given the set alone.
static void write_batch(FILE *out, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const int32_t *n_reg, mp_reg1_t *const *reg, int64_t *id_counter,
                        const LocusSets *sets = 0, int32_t s0 = 0)
{
	auto printed = [&](int32_t q, int32_t j, int32_t best) {
		const mp_reg1_t *r = &reg[q][j];
		const int32_t sc = r->p ? r->p->dp_max : r->chn_sc;
		if (sc <= 0 || sc < (double)best * opt->out_sim) return false;
		if (r->qe - r->qs < (double)b.len[q] * opt->out_cov) return false;
		return true;
	};
	std::vector<int64_t> id0((size_t)b.n + 1, *id_counter);
	for (int32_t q = 0; q < b.n; ++q) {
		int64_t k = 0;
		const int32_t best = n_reg[q] > 0 ? (reg[q][0].p ? reg[q][0].p->dp_max : reg[q][0].chn_sc) : -1;
		for (int32_t j = 0; j < n_reg[q] && j < opt->out_n; ++j) k += printed(q, j, best);
		id0[(size_t)q + 1] = id0[(size_t)q] + k;
	}
	*id_counter = id0[(size_t)b.n];
	std::vector<Str> part(64);
	const int n_part = par_ranges(b.n, 64, [&](int q_lo, int q_hi, int c) {
		Str &buf = part[(size_t)c];
		for (int32_t q = q_lo; q < q_hi; ++q) {
			int32_t best = -1, n_out = 0;
			if (n_reg[q] > 0) best = reg[q][0].p ? reg[q][0].p->dp_max : reg[q][0].chn_sc;
			for (int32_t j = 0; j < n_reg[q] && j < opt->out_n; ++j) {
				if (!printed(q, j, best)) continue;
				++n_out;
				const int64_t nt_lim = sets ? range_end(mi, *sets, s0 + q, &reg[q][j]) : -1;
				format_output(buf, mi, opt, b.name[q], b.len[q], b.seq[q], &reg[q][j], id0[(size_t)q] + n_out, j + 1, nt_lim);
			}
			if (n_out == 0) format_output(buf, mi, opt, b.name[q], b.len[q], b.seq[q], 0, 0, 0);
		}
	});
	for (int c = 0; c < n_part; ++c) {
		if (part[(size_t)c].l) fwrite(part[(size_t)c].s, 1, (size_t)part[(size_t)c].l, out);
		free(part[(size_t)c].s);
	}
}

namespace {

// One unit of a file driver's input, with everything that must live from the reader to the writer
struct Unit {
	std::vector<std::string> names, seqs; // the records (FASTA input only; the pointers below point into them)
	std::vector<const char*> sp, np;      // the Batch view
	std::vector<int32_t> len;
	const LocusSets *sets = 0;            // locus mode: query q is the protein of set s0 + q
	int32_t s0 = 0;
	std::vector<int32_t> n_reg;
	std::vector<mp_reg1_t*> reg;
	int rc = 0;
	Batch view() const
	{
		Batch b;
		b.n = (int32_t)len.size(), b.seq = sp.data(), b.len = len.data(), b.name = np.data();
		return b;
	}
};
typedef std::unique_ptr<Unit> UnitPtr;

// bseq.c:53-74: records until the unit holds unit_size residues; null at the end of the input
UnitPtr read_batch(FastxReader &rd, int64_t unit_size, bool &more)
{
	UnitPtr u(new Unit);
	std::string name, seq;
	int64_t residues = 0;
	while (residues < unit_size && (more = rd.next(name, seq))) {
		residues += (int64_t)seq.size();
		u->names.push_back(name), u->seqs.push_back(seq);
	}
	if (u->seqs.empty()) return nullptr;
	const size_t n = u->seqs.size();
	for (size_t i = 0; i < n; ++i) u->sp.push_back(u->seqs[i].c_str()), u->np.push_back(u->names[i].c_str()), u->len.push_back((int32_t)u->seqs[i].size());
	u->n_reg.assign(n, 0), u->reg.assign(n, (mp_reg1_t*)0);
	return u;
}

// map.c:273-343 (worker_pipeline under kt_pipeline with three steps), over n backends: one reader thread cuts the input into units
// (read(more) returns the next unit, or null at the end, and clears `more` once the input is exhausted), one mapper thread per backend
// maps the next unit each (map(st[k], k, unit)), and the calling thread writes the units strictly in input order and owns the hit
// counter.  At most 2n + 1 units are read but not yet written: with one backend, reading unit k+1 and writing unit k-1 overlap the
// mapping of unit k, as in the reference.  The host phases of the mappers share one worker pool and take turns on it (parfor.hpp);
// the device stages overlap.  With one backend, an input that fits one unit has nothing to overlap and starts no thread, and
// MPB_FILE_PIPELINE=0 runs the three steps one after another on the calling thread for any input (A/B, debugging).  Returns the first
// non-zero return code of a unit, else 0.
template <class Read, class Map>
int32_t run_units(Stages *const *st, int n, const mp_idx_t *mi, const mp_mapopt_t *opt, FILE *out, const char *label, const char *noun, Read read, Map map)
{
	if (opt->flag & MP_F_GFF) fputs("##gff-version 3\n", out); // map.c:338
	static const bool trace = getenv("MPB_TRACE") != 0;
	int64_t id_counter = 0;
	int32_t rc = 0;
	auto map_step = [&](int k, Unit &u) {
		map(st[k], k, u);
		if (mp_verbose < 3) return;
		if (n > 1) fprintf(stderr, "[M::%s::%.3f*%.2f] mapped %d %s (context %d)\n", label, mp_realtime(), mp_cputime() / mp_realtime(), (int)u.len.size(), noun, k);
		else fprintf(stderr, "[M::%s::%.3f*%.2f] mapped %d %s\n", label, mp_realtime(), mp_cputime() / mp_realtime(), (int)u.len.size(), noun);
	};
	auto write_step = [&](int64_t i, Unit &u) {
		if (u.rc != 0 && rc == 0) rc = u.rc;
		const double t0 = mp_realtime();
		write_batch(out, mi, opt, u.view(), u.n_reg.data(), u.reg.data(), &id_counter, u.sets, u.s0);
		const double t1 = mp_realtime();
		mpb_regs_free((int32_t)u.reg.size(), u.n_reg.data(), u.reg.data());
		if (trace)
			fprintf(stderr, "[mpb-trace] output: unit %ld, %d %s formatted + written in %.2f ms, released in %.2f ms\n", (long)i, (int)u.len.size(), noun, (t1 - t0) * 1e3,
			        (mp_realtime() - t1) * 1e3);
	};
	bool more = true;
	UnitPtr first = read(more);
	if (!first) return 0;
	const char *e = getenv("MPB_FILE_PIPELINE");
	if (n == 1 && (!more || (e && atoi(e) == 0))) {
		int64_t i = 0;
		for (UnitPtr u = std::move(first); u; u = more ? read(more) : nullptr) {
			map_step(0, *u);
			write_step(i++, *u);
		}
		return rc;
	}

	const int64_t max_in_flight = 2 * (int64_t)n + 1;
	std::mutex mu;
	std::condition_variable cv;
	std::deque<std::pair<int64_t, UnitPtr>> todo; // read, not yet taken by a mapper
	std::map<int64_t, UnitPtr> mapped;              // mapped, not yet written
	int64_t n_read = 1, n_written = 0;              // units
	bool eof = !more;
	todo.emplace_back(0, std::move(first));
	std::thread reader([&] {
		for (bool last = eof; !last;) {
			{
				std::unique_lock<std::mutex> lk(mu);
				cv.wait(lk, [&] { return n_read - n_written < max_in_flight; });
			}
			UnitPtr u = read(more);
			last = !u || !more;
			std::lock_guard<std::mutex> lk(mu);
			if (u) todo.emplace_back(n_read++, std::move(u));
			eof = last;
			cv.notify_all();
		}
	});
	std::vector<std::thread> mappers;
	for (int k = 0; k < n; ++k)
		mappers.emplace_back([&, k] {
			st[k]->thread_init();
			for (;;) {
				std::pair<int64_t, UnitPtr> u;
				{
					std::unique_lock<std::mutex> lk(mu);
					cv.wait(lk, [&] { return !todo.empty() || eof; });
					if (todo.empty()) return;
					u = std::move(todo.front());
					todo.pop_front();
				}
				map_step(k, *u.second);
				std::lock_guard<std::mutex> lk(mu);
				mapped.emplace(u.first, std::move(u.second));
				cv.notify_all();
			}
		});
	for (int64_t i = 0;; ++i) {
		UnitPtr u;
		{
			std::unique_lock<std::mutex> lk(mu);
			cv.wait(lk, [&] { return mapped.count(i) || (eof && i == n_read); });
			auto it = mapped.find(i);
			if (it == mapped.end()) break; // everything read has been written
			u = std::move(it->second);
			mapped.erase(it);
		}
		write_step(i, *u);
		u.reset();
		std::lock_guard<std::mutex> lk(mu);
		n_written = i + 1;
		cv.notify_all();
	}
	reader.join();
	for (std::thread &t : mappers) t.join();
	return rc;
}

} // namespace

int32_t map_file_multi(Stages *const *st, int n, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out)
{
	if (n < 1) return -1;
	if (bad_dbg_flags(opt)) return -3;
	FastxReader rd(fn);
	if (!rd.fp) return -1;
	const int64_t unit_size = std::max<int64_t>(1, opt->mini_batch_size / n);
	return run_units(st, n, mi, opt, out, "map_file", "sequences", [&](bool &more) { return read_batch(rd, unit_size, more); },
	                 [&](Stages *s, int k, Unit &u) { map_batch(s, mi, opt, u.view(), u.n_reg.data(), u.reg.data(), k); });
}

// ---------------------------------------------------------------- locus mode

LocusView::LocusView(const mp_idx_t *mi, int32_t n, const mpb_locus_t *rng) : ctg((size_t)n), bo((size_t)n * 2 + 1)
{
	memset(&idx, 0, sizeof(idx));
	memset(&nt, 0, sizeof(nt));
	const int32_t bbit = mi->opt.bbit;
	int64_t acc = 0;
	for (int32_t k = 0; k < n; ++k) {
		const mp_ctg_t *c = &mi->nt->ctg[rng[k].cid];
		mp_ctg_t &v = ctg[(size_t)k];
		v.off = c->off + rng[k].st, v.len = rng[k].en - rng[k].st, v.name = c->name;
		const int64_t nb = (v.len + (1 << bbit) - 1) >> bbit; // index.c:11-26
		bo[(size_t)k * 2] = (uint32_t)acc, acc += nb;
		bo[(size_t)k * 2 + 1] = (uint32_t)acc, acc += nb;
	}
	bo[(size_t)n * 2] = (uint32_t)acc;
	nt.n_ctg = nt.m_ctg = n, nt.l_seq = nt.m_seq = mi->nt->l_seq, nt.seq = mi->nt->seq, nt.ctg = ctg.data();
	idx.opt = mi->opt, idx.n_block = (uint32_t)acc, idx.nt = &nt, idx.bo = bo.data();
}

int check_loci(const mp_idx_t *mi, int32_t n_seq, int32_t n_loci, const mpb_locus_t *loci)
{
	if (!mi || !mi->nt || n_seq < 0 || n_loci < 0 || (n_loci > 0 && !loci)) return -1;
	for (int32_t k = 0; k < n_loci; ++k) {
		const mpb_locus_t &l = loci[k];
		if (l.qid < 0 || l.qid >= n_seq || l.cid < 0 || l.cid >= mi->nt->n_ctg || l.st < 0 || l.en > mi->nt->ctg[l.cid].len || l.st >= l.en) return -1;
	}
	if (mi->nt->spsc) {
		fprintf(stderr, "[miniprot_b200] locus mode does not take --spsc splice scores\n");
		return -3;
	}
	if (mp_dbg_flag & ~MP_DBG_NO_KALLOC) {
		fprintf(stderr, "[miniprot_b200] locus mode does not take the --dbg-* switches (mp_dbg_flag = %#x)\n", (unsigned)mp_dbg_flag);
		return -3;
	}
	return 0;
}

void LocusSets::add(const mpb_locus_t *loci, int64_t n)
{
	const size_t first = rng.size();
	rng.insert(rng.end(), loci, loci + n);
	std::sort(rng.begin() + (ptrdiff_t)first, rng.end(), [](const mpb_locus_t &x, const mpb_locus_t &y) { return x.cid < y.cid || (x.cid == y.cid && x.st < y.st); });
	size_t k = first;
	for (size_t i = first; i < rng.size(); ++i) {
		if (k > first && rng[k - 1].cid == rng[i].cid && rng[i].st <= rng[k - 1].en) rng[k - 1].en = std::max(rng[k - 1].en, rng[i].en); // overlap or abut
		else rng[k++] = rng[i];
	}
	rng.resize(k);
	off.push_back((int64_t)k);
}

int locus_sets_make(const mp_idx_t *mi, int32_t n_seq, int32_t n_sets, const int64_t *set_off, const mpb_locus_t *loci, LocusSets &out)
{
	if (n_sets < 0 || (n_sets > 0 && (!set_off || set_off[0] != 0 || !loci))) return -1;
	for (int32_t s = 0; s < n_sets; ++s)
		if (set_off[s + 1] <= set_off[s] || set_off[s + 1] > INT32_MAX) return -1; // an empty set, or more loci than one call takes
	for (int32_t s = 0; s < n_sets; ++s)
		for (int64_t k = set_off[s] + 1; k < set_off[s + 1]; ++k)
			if (loci[k].qid != loci[set_off[s]].qid) return -1;
	const int rc = check_loci(mi, n_seq, n_sets > 0 ? (int32_t)set_off[n_sets] : 0, loci);
	if (rc != 0) return rc;
	out = LocusSets();
	for (int32_t s = 0; s < n_sets; ++s) out.add(loci + set_off[s], set_off[s + 1] - set_off[s]);
	return 0;
}

namespace {

// map_batch's stages in locus mode: S1 is the backend's set seeding over the query -> view-contig ranges ctg_off, everything else
// passes through
struct LociStages : Stages {
	Stages *in;
	const int32_t *ctg_off = 0;
	explicit LociStages(Stages *s) : in(s) {}
	void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override { in->seed_chain_locus_sets(mi, ctg_off, opt, b, out); }
	void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) override { in->refine(mi, opt, b, jobs, out); }
	void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) override { in->nasw(mi, base, b, jobs, out); }
	void batch_begin(const Batch &b) override { in->batch_begin(b); }
	void batch_end() override { in->batch_end(); }
	void note_wall(int phase, double ms) override { in->note_wall(phase, ms); }
	void thread_init() override { in->thread_init(); }
};

// -3 with a message when a set of [s_lo, s_hi) has several ranges and the backend cannot seed a query against several contigs
int check_set_seeding(Stages *st, const LocusSets &ls, int32_t s_lo, int32_t s_hi)
{
	for (int32_t s = s_lo; s < s_hi; ++s)
		if (ls.n_rng(s) > 1 && !st->locus_sets()) {
			fprintf(stderr, "[miniprot_b200] this backend cannot seed a protein against several loci at once\n");
			return -3;
		}
	return 0;
}

} // namespace

int map_sets(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *const *seqs, const int32_t *lens, const char *const *names, const LocusSets &ls,
             int32_t s_lo, int32_t s_hi, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	for (int32_t s = s_lo; s < s_hi; ++s) n_reg_out[s - s_lo] = 0, reg_out[s - s_lo] = 0;
	if (s_lo >= s_hi) return 0;
	if (check_set_seeding(st, ls, s_lo, s_hi) != 0) return -3;
	LociStages lst(st);
	for (int32_t i0 = s_lo; i0 < s_hi;) {
		// a batch holds whole sets until it has mini_batch_size residues (bseq.c:53-74), and fewer than 2^31 blocks
		int32_t i1 = i0;
		int64_t residues = 0, blocks = 0;
		while (i1 < s_hi && residues < opt->mini_batch_size) {
			int64_t nb = 0;
			for (int64_t k = ls.off[(size_t)i1]; k < ls.off[(size_t)i1 + 1]; ++k) nb += 2 * ((ls.rng[(size_t)k].en - ls.rng[(size_t)k].st + (1 << mi->opt.bbit) - 1) >> mi->opt.bbit);
			if (i1 > i0 && blocks + nb >= (int64_t)1 << 31) break;
			residues += lens[ls.rng[(size_t)ls.off[(size_t)i1]].qid], blocks += nb, ++i1;
		}
		const int32_t n = i1 - i0;
		const int64_t r0 = ls.off[(size_t)i0];
		const mpb_locus_t *rng = ls.rng.data() + r0; // contig k of the view is range rng[k]
		LocusView v(mi, (int32_t)(ls.off[(size_t)i1] - r0), rng);
		std::vector<int32_t> ctg_off((size_t)n + 1);
		std::vector<const char*> sp((size_t)n), np((size_t)n);
		std::vector<int32_t> lp((size_t)n);
		for (int32_t q = 0; q <= n; ++q) ctg_off[(size_t)q] = (int32_t)(ls.off[(size_t)(i0 + q)] - r0);
		for (int32_t q = 0; q < n; ++q) {
			const int32_t p = rng[ctg_off[(size_t)q]].qid;
			sp[(size_t)q] = seqs[p], lp[(size_t)q] = lens[p], np[(size_t)q] = names ? names[p] : 0;
		}
		Batch b;
		b.n = n, b.seq = sp.data(), b.len = lp.data(), b.name = np.data();
		if (!st->loci_view(mi, &v.idx)) {
			fprintf(stderr, "[miniprot_b200] this backend has no locus seeding stage\n");
			return -3;
		}
		lst.ctg_off = ctg_off.data();
		int32_t *nr = n_reg_out + (i0 - s_lo);
		mp_reg1_t **rr = reg_out + (i0 - s_lo);
		map_batch(&lst, &v.idx, opt, b, nr, rr);
		st->loci_view(0, 0);
		// view strand -> contig strand: + adds st, - adds len(cid) - en of the range the region lies on
		for (int32_t q = 0; q < n; ++q)
			for (int32_t j = 0; j < nr[q]; ++j) {
				mp_reg1_t *r = &rr[q][j];
				const mpb_locus_t &l = rng[r->vid >> 1];
				const uint32_t rev = r->vid & 1;
				const int64_t sh = rev ? mi->nt->ctg[l.cid].len - l.en : l.st;
				r->vid = (uint32_t)l.cid << 1 | rev, r->vs += sh, r->ve += sh;
				for (int32_t f = 0; f < r->n_feat; ++f) r->feat[f].vs += sh, r->feat[f].ve += sh;
			}
		i0 = i1;
	}
	return 0;
}

int map_locus_sets(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names,
                   int32_t n_sets, const int64_t *set_off, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	LocusSets ls;
	const int rc = locus_sets_make(mi, n_seq, n_sets, set_off, loci, ls);
	return rc != 0 ? rc : map_sets(st, mi, opt, seqs, lens, names, ls, 0, n_sets, n_reg_out, reg_out);
}

int map_loci(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, const char *const *names,
             int32_t n_loci, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	const int rc = check_loci(mi, n_seq, n_loci, loci);
	if (rc != 0) return rc;
	LocusSets ls;
	for (int32_t k = 0; k < n_loci; ++k) ls.add(loci + k, 1);
	return map_sets(st, mi, opt, seqs, lens, names, ls, 0, n_loci, n_reg_out, reg_out);
}

// ---------------------------------------------------------------- locus mode: the file driver

void LociFile::add_protein(const std::string &name, const std::string &seq)
{
	auto it = qid.find(name);
	if (it != qid.end()) { // the last record of a name is the one its loci are aligned to
		seqs[(size_t)it->second] = seq;
		return;
	}
	qid.emplace(name, (int32_t)names.size());
	names.push_back(name), seqs.push_back(seq);
}

int loci_file_read(const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, LociFile &in, bool by_set)
{
	if (!mi || !mi->nt || !prot_fn || !loci_fn) return -1;
	{
		FastxReader rd(prot_fn);
		if (!rd.fp) {
			fprintf(stderr, "[miniprot_b200] %s: cannot open the protein file\n", prot_fn);
			return -1;
		}
		std::string name, seq;
		while (rd.next(name, seq)) in.add_protein(name, seq);
	}
	in.sp.resize(in.seqs.size()), in.np.resize(in.seqs.size()), in.len.resize(in.seqs.size());
	for (size_t i = 0; i < in.seqs.size(); ++i) in.sp[i] = in.seqs[i].c_str(), in.np[i] = in.names[i].c_str(), in.len[i] = (int32_t)in.seqs[i].size();
	std::unordered_map<std::string, int32_t> cid;
	for (int32_t i = 0; i < mi->nt->n_ctg; ++i) cid[mi->nt->ctg[i].name] = i;
	FILE *fp = fopen(loci_fn, "r");
	if (!fp) {
		fprintf(stderr, "[miniprot_b200] %s: cannot open the loci file\n", loci_fn);
		return -1;
	}
	char *line = 0;
	size_t cap = 0;
	int rc = 0;
	std::map<std::pair<int32_t, std::string>, int32_t> set_of; // by_set: (protein, label or "") -> set number, in order of first line
	std::vector<int32_t> line_set;
	for (long ln = 1; getline(&line, &cap, fp) >= 0; ++ln) {
		std::vector<char*> t; // whitespace-separated fields
		for (char *q = line; *q;) {
			while (*q && isspace((unsigned char)*q)) ++q;
			if (!*q) break;
			t.push_back(q);
			while (*q && !isspace((unsigned char)*q)) ++q;
			if (*q) *q++ = 0;
		}
		if (t.empty() || t[0][0] == '#') continue;
		int64_t v[2] = { 0, 0 };
		bool num = t.size() >= 4;
		for (int k = 0; k < 2 && num; ++k) {
			char *end;
			errno = 0;
			v[k] = strtoll(t[2 + (size_t)k], &end, 10);
			num = *end == 0 && errno == 0;
		}
		const char *why = 0;
		if (!num) why = "expected `protein contig start end` with integer start and end";
		else if (!in.qid.count(t[0])) why = "unknown protein";
		else if (!cid.count(t[1])) why = "unknown contig";
		else if (v[0] < 0 || v[0] >= v[1] || v[1] > mi->nt->ctg[cid[t[1]]].len) why = "the range is not 0 <= start < end <= contig length";
		if (why) {
			fprintf(stderr, "[miniprot_b200] %s:%ld: %s\n", loci_fn, ln, why);
			rc = -1;
			break;
		}
		mpb_locus_t l;
		l.qid = in.qid[t[0]], l.cid = cid[t[1]], l.st = v[0], l.en = v[1];
		in.loci.push_back(l);
		if (by_set) line_set.push_back(set_of.emplace(std::make_pair(l.qid, std::string(t.size() >= 5 ? t[4] : "")), (int32_t)set_of.size()).first->second);
	}
	free(line);
	fclose(fp);
	if (rc != 0) return rc;
	rc = check_loci(mi, (int32_t)in.seqs.size(), (int32_t)in.loci.size(), in.loci.data());
	if (rc != 0) return rc;
	in.by_set = by_set, in.sets = LocusSets();
	if (!by_set) {
		for (const mpb_locus_t &l : in.loci) in.sets.add(&l, 1);
		return 0;
	}
	std::vector<std::vector<mpb_locus_t>> lines(set_of.size()); // the loci of each set, in file order
	for (size_t k = 0; k < in.loci.size(); ++k) lines[(size_t)line_set[k]].push_back(in.loci[k]);
	for (const std::vector<mpb_locus_t> &x : lines) in.sets.add(x.data(), (int64_t)x.size());
	return 0;
}

// run_units over the sets of a loci file, which are in memory already: units of whole sets, at most mini_batch_size / n residues (at
// least one set), each aligned with map_sets.  Hits do not depend on unit boundaries (map_sets), so neither does the output.
int32_t map_loci_file(Stages *const *st, int n, const mp_idx_t *mi, const LociFile &in, const mp_mapopt_t *opt, FILE *out)
{
	if (n < 1) return -1;
	const LocusSets &ls = in.sets;
	const int32_t n_sets = ls.n();
	for (int k = 0; k < n; ++k) {
		if (!st[k]->loci_view(0, 0)) {
			fprintf(stderr, "[miniprot_b200] this backend has no locus seeding stage\n");
			return -3;
		}
		if (check_set_seeding(st[k], ls, 0, n_sets) != 0) return -3;
	}
	const int64_t unit_size = std::max<int64_t>(1, opt->mini_batch_size / n);
	int32_t s = 0;
	auto read = [&](bool &more) {
		UnitPtr u;
		if (s < n_sets) {
			u.reset(new Unit);
			u->sets = &ls, u->s0 = s;
			for (int64_t residues = 0; s < n_sets && residues < unit_size; ++s) {
				const size_t q = (size_t)ls.rng[(size_t)ls.off[(size_t)s]].qid;
				residues += in.len[q];
				u->sp.push_back(in.sp[q]), u->np.push_back(in.np[q]), u->len.push_back(in.len[q]);
			}
			u->n_reg.assign(u->len.size(), 0), u->reg.assign(u->len.size(), (mp_reg1_t*)0);
		}
		more = s < n_sets;
		return u;
	};
	return run_units(st, n, mi, opt, out, in.by_set ? "map_locus_sets_file" : "map_loci_file", in.by_set ? "sets" : "pairs", read, [&](Stages *k, int, Unit &u) {
		u.rc = map_sets(k, mi, opt, in.sp.data(), in.len.data(), in.np.data(), ls, u.s0, u.s0 + (int32_t)u.len.size(), u.n_reg.data(), u.reg.data());
	});
}

} // namespace mpb

// what the caller of mp_map does per protein (map.c:314-318): the hits are libc-allocated like the reference's
void mpb_regs_free(int32_t n, const int32_t *n_reg, mp_reg1_t **reg)
{
	for (int32_t i = 0; i < n; ++i) {
		for (int32_t j = 0; j < n_reg[i]; ++j) free(reg[i][j].feat), free(reg[i][j].p);
		free(reg[i]);
	}
}
