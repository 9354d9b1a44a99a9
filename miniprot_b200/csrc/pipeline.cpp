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
#include <chrono>
#include <condition_variable>
#include <deque>
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

} // namespace

void map_batch(Stages *st, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	const int32_t n = b.n, kmer = mi->opt.kmer;
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
	st->seed_chain(mi, opt, b, cs);
	lap(0);

	// ---- H1 + S2 work list
	// (the host phases are independent per protein: contiguous ranges of proteins on the worker pool, per-range results
	// concatenated in order)
	std::vector<RefineJob> rjobs;
	std::vector<int32_t> rjob_first((size_t)n + 1, 0);
	{
		std::vector<std::vector<RefineJob>> part(64);
		const int n_part = par_ranges(n, 64, [&](int lo, int hi, int c) {
			std::vector<RefineJob> &out = part[(size_t)c];
			for (int32_t q = lo; q < hi; ++q) {
				QueryState &Q = qs[(size_t)q];
				const int32_t n_u = (int32_t)(cs.u_off[(size_t)q + 1] - cs.u_off[(size_t)q]);
				const uint64_t *u = cs.u.data() + cs.u_off[(size_t)q], *a = cs.a.data() + cs.a_off[(size_t)q];
				Q.reg = regs_from_chains(mi, n_u, u, a, &Q.n_reg);
				regs_sort(&Q.n_reg, Q.reg);
				regs_set_parent(opt->mask_level, opt->mask_len, Q.n_reg, Q.reg, kmer, 0);
				regs_select_sub(opt->pri_ratio * opt->pri_ratio, kmer * 2, opt->best_n, &Q.n_reg, Q.reg);
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
	}
	cs = ChainSet(); // first-round anchors are not needed any more
	lap(1);

	// ---- S2
	RefineSet rs;
	st->refine(mi, opt, b, rjobs, rs);
	lap(2);

	// ---- H2: adopt refined chains (map.c:83-109), re-rank (map.c:217-221)
	const int32_t k2 = opt->kmer2;
	par_ranges(n, 64, [&](int q_lo, int q_hi, int) {
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
						if (p.plan(mi, opt, q, b.len[q], b.seq[q], &Q.reg[i], (int32_t)(Q.ext[(size_t)i] >> 32), (int32_t)Q.ext[(size_t)i], pjobs[(size_t)c]))
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

// map.c:293-326: per protein, hits in rank order subject to --outn / --outs / --outc; unmapped line with -u.  Every printed hit
// gets the next number of a counter that runs over the whole file (the MP%06d ids of GFF / GTF, map.c:306): the hits each
// protein will print are counted first, so that formatting -- independent per protein -- can run on the worker pool, each range
// into its own buffer, written in order.
static void write_batch(FILE *out, const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const int32_t *n_reg, mp_reg1_t *const *reg, int64_t *id_counter)
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
				format_output(buf, mi, opt, b.name[q], b.len[q], b.seq[q], &reg[q][j], id0[(size_t)q] + n_out, j + 1);
			}
			if (n_out == 0) format_output(buf, mi, opt, b.name[q], b.len[q], b.seq[q], 0, 0, 0);
		}
	});
	for (int c = 0; c < n_part; ++c) {
		if (part[(size_t)c].l) fwrite(part[(size_t)c].s, 1, (size_t)part[(size_t)c].l, out);
		free(part[(size_t)c].s);
	}
}

// One mini-batch of the query file with everything that must live from the reader to the writer.
struct FileBatch {
	std::vector<std::string> names, seqs;
	std::vector<const char*> sp, np;
	std::vector<int32_t> len, n_reg;
	std::vector<mp_reg1_t*> reg;
	Batch view() const
	{
		Batch b;
		b.n = (int32_t)seqs.size(), b.seq = sp.data(), b.len = len.data(), b.name = np.data();
		return b;
	}
	void release() // hits are libc-allocated like the reference's (map.c:314-318)
	{
		for (size_t i = 0; i < reg.size(); ++i) {
			for (int32_t j = 0; j < n_reg[i]; ++j) free(reg[i][j].feat), free(reg[i][j].p);
			free(reg[i]);
		}
		reg.clear();
	}
};

// bseq.c:53-74: records until the batch holds mini_batch_size residues; null at the end of the input
static std::unique_ptr<FileBatch> read_batch(FastxReader &rd, int64_t mini_batch_size, bool &more)
{
	std::unique_ptr<FileBatch> fb(new FileBatch);
	std::string name, seq;
	int64_t residues = 0;
	while (residues < mini_batch_size && (more = rd.next(name, seq))) {
		residues += (int64_t)seq.size();
		fb->names.push_back(name), fb->seqs.push_back(seq);
	}
	if (fb->seqs.empty()) return nullptr;
	const size_t n = fb->seqs.size();
	fb->sp.resize(n), fb->np.resize(n), fb->len.resize(n), fb->n_reg.assign(n, 0), fb->reg.assign(n, (mp_reg1_t*)0);
	for (size_t i = 0; i < n; ++i) fb->sp[i] = fb->seqs[i].c_str(), fb->np[i] = fb->names[i].c_str(), fb->len[i] = (int32_t)fb->seqs[i].size();
	return fb;
}

// A one-slot hand-over between two steps of the file pipeline: put() waits while the slot is taken, take() returns null once
// the producer has closed an empty slot.
class Handoff {
public:
	void put(std::unique_ptr<FileBatch> fb)
	{
		std::unique_lock<std::mutex> lk(mu_);
		cv_.wait(lk, [&] { return !slot_; });
		slot_ = std::move(fb);
		cv_.notify_all();
	}
	void close()
	{
		std::lock_guard<std::mutex> lk(mu_);
		closed_ = true;
		cv_.notify_all();
	}
	std::unique_ptr<FileBatch> take()
	{
		std::unique_lock<std::mutex> lk(mu_);
		cv_.wait(lk, [&] { return slot_ || closed_; });
		std::unique_ptr<FileBatch> fb = std::move(slot_);
		cv_.notify_all();
		return fb;
	}

private:
	std::mutex mu_;
	std::condition_variable cv_;
	std::unique_ptr<FileBatch> slot_;
	bool closed_ = false;
};

// map.c:273-343 (worker_pipeline under kt_pipeline with three steps): step 0 reads and parses the next mini-batch, step 1 maps
// it (the GPU batch dispatcher above), step 2 formats and writes the hits -- in the order of the input, by one thread, which
// also owns the hit counter.  As in the reference, step 0 of batch n+1 and step 2 of batch n-1 run while batch n is mapped:
// one reader thread, the calling thread as the mapper (it owns the device), one writer thread, a one-slot hand-over between
// neighbours.  An input that fits one mini-batch has nothing to overlap and starts no thread; MPB_FILE_PIPELINE=0 runs the three
// steps one after another on the calling thread for any input (A/B, debugging).
int32_t map_file(Stages *st, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out)
{
	FastxReader rd(fn);
	if (!rd.fp) return -1;
	int64_t id_counter = 0;
	if (opt->flag & MP_F_GFF) fputs("##gff-version 3\n", out); // map.c:338
	auto map_step = [&](FileBatch &fb) {
		map_batch(st, mi, opt, fb.view(), fb.n_reg.data(), fb.reg.data());
		if (mp_verbose >= 3)
			fprintf(stderr, "[M::%s::%.3f*%.2f] mapped %d sequences\n", "map_file", mp_realtime(), mp_cputime() / mp_realtime(), (int)fb.seqs.size());
	};
	static const bool trace = getenv("MPB_TRACE") != 0;
	auto write_step = [&](FileBatch &fb) {
		const double t0 = mp_realtime();
		write_batch(out, mi, opt, fb.view(), fb.n_reg.data(), fb.reg.data(), &id_counter);
		const double t1 = mp_realtime();
		fb.release();
		if (trace) fprintf(stderr, "[mpb-trace] output: %d proteins formatted + written in %.2f ms, released in %.2f ms\n", (int)fb.seqs.size(), (t1 - t0) * 1e3, (mp_realtime() - t1) * 1e3);
	};
	const char *e = getenv("MPB_FILE_PIPELINE");
	bool more = true;
	std::unique_ptr<FileBatch> first = read_batch(rd, opt->mini_batch_size, more);
	if (!first) return 0;
	if ((e && atoi(e) == 0) || !more) { // the whole input is one mini-batch (nothing to overlap: no threads), or the serial form was asked for
		for (std::unique_ptr<FileBatch> fb = std::move(first); fb; fb = more ? read_batch(rd, opt->mini_batch_size, more) : std::unique_ptr<FileBatch>()) {
			map_step(*fb);
			write_step(*fb);
		}
		return 0;
	}
	Handoff to_map, to_write;
	std::thread reader([&] {
		while (more) {
			std::unique_ptr<FileBatch> fb = read_batch(rd, opt->mini_batch_size, more);
			if (!fb) break;
			to_map.put(std::move(fb));
		}
		to_map.close();
	});
	std::thread writer([&] {
		while (std::unique_ptr<FileBatch> fb = to_write.take()) write_step(*fb);
	});
	for (std::unique_ptr<FileBatch> fb = std::move(first); fb; fb = to_map.take()) {
		map_step(*fb);
		to_write.put(std::move(fb));
	}
	to_write.close();
	reader.join();
	writer.join();
	return 0;
}

// map_file over n backends (contexts, possibly on several devices): one reader thread cuts the input into work units of at most
// mini_batch_size / n residues (at least one protein; results do not depend on batch boundaries), n mapper threads -- one per
// backend -- take the next unit each, and one writer thread emits the units strictly in input order and owns the hit counter, as
// in map_file.  At most 2n units are between the reader and the writer, so memory stays bounded whatever the input.
// The host phases of the mappers share one worker pool and take turns on it (parfor.hpp), the device stages overlap.
int32_t map_file_multi(Stages *const *st, int n, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out)
{
	if (n < 1) return -1;
	if (n == 1) return map_file(st[0], mi, fn, opt, out);
	FastxReader rd(fn);
	if (!rd.fp) return -1;
	if (opt->flag & MP_F_GFF) fputs("##gff-version 3\n", out); // map.c:338
	const int64_t unit_size = std::max<int64_t>(1, opt->mini_batch_size / n);
	const int64_t max_in_flight = 2 * (int64_t)n;
	static const bool trace = getenv("MPB_TRACE") != 0;

	std::mutex mu;
	std::condition_variable cv;
	std::deque<std::pair<int64_t, std::unique_ptr<FileBatch>>> todo; // read, not yet taken by a mapper
	std::map<int64_t, std::unique_ptr<FileBatch>> mapped;              // mapped, not yet written
	int64_t n_read = 0, n_written = 0;                                   // units
	bool eof = false;

	std::thread reader([&] {
		bool more = true;
		while (more) {
			{
				std::unique_lock<std::mutex> lk(mu);
				cv.wait(lk, [&] { return n_read - n_written < max_in_flight; });
			}
			std::unique_ptr<FileBatch> fb = read_batch(rd, unit_size, more);
			const bool last = !fb || !more;
			std::lock_guard<std::mutex> lk(mu);
			if (fb) todo.emplace_back(n_read++, std::move(fb));
			if (last) eof = true;
			cv.notify_all();
		}
	});
	std::vector<std::thread> mappers;
	for (int k = 0; k < n; ++k)
		mappers.emplace_back([&, k] {
			st[k]->thread_init();
			for (;;) {
				std::pair<int64_t, std::unique_ptr<FileBatch>> u;
				{
					std::unique_lock<std::mutex> lk(mu);
					cv.wait(lk, [&] { return !todo.empty() || eof; });
					if (todo.empty()) return;
					u = std::move(todo.front());
					todo.pop_front();
				}
				FileBatch &fb = *u.second;
				map_batch(st[k], mi, opt, fb.view(), fb.n_reg.data(), fb.reg.data());
				if (mp_verbose >= 3)
					fprintf(stderr, "[M::%s::%.3f*%.2f] mapped %d sequences (context %d)\n", "map_file_multi", mp_realtime(), mp_cputime() / mp_realtime(), (int)fb.seqs.size(), k);
				std::lock_guard<std::mutex> lk(mu);
				mapped.emplace(u.first, std::move(u.second));
				cv.notify_all();
			}
		});
	std::thread writer([&] {
		int64_t id_counter = 0;
		for (;;) {
			std::unique_ptr<FileBatch> fb;
			{
				std::unique_lock<std::mutex> lk(mu);
				cv.wait(lk, [&] { return mapped.count(n_written) || (eof && n_written == n_read); });
				auto it = mapped.find(n_written);
				if (it == mapped.end()) return; // everything read has been written
				fb = std::move(it->second);
				mapped.erase(it);
			}
			const double t0 = mp_realtime();
			write_batch(out, mi, opt, fb->view(), fb->n_reg.data(), fb->reg.data(), &id_counter);
			fb->release();
			if (trace) fprintf(stderr, "[mpb-trace] output: unit %ld, %d proteins formatted + written in %.2f ms\n", (long)n_written, (int)fb->seqs.size(), (mp_realtime() - t0) * 1e3);
			std::lock_guard<std::mutex> lk(mu);
			++n_written;
			cv.notify_all();
		}
	});
	reader.join();
	for (std::thread &t : mappers) t.join();
	writer.join();
	return 0;
}

} // namespace mpb
