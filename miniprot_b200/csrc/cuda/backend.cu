// backend.cu -- the CUDA implementation of the stage interface (mpb::Stages) and the C ABI of the batch API.
// This is the ONLY implementation of the stages in the product: there is no CPU fallback.
#include <algorithm>
#include <stdio.h>
#include <condition_variable>
#include <mutex>
#include <sched.h>
#include "ctx.hpp"
#include "stages_dev.hpp"
#include "seed_dev.hpp"
#include "../align.hpp"

using namespace mpb;
using namespace mpb::cuda;

namespace {

// device job from a pipeline job: where DP row 0 sits in the packed genome and which way rows walk
DpDev make_dev_job(const mp_idx_t *mi, const DpJob &j, int32_t aa_base)
{
	DpDev d;
	memset(&d, 0, sizeof(d));
	const mp_ctg_t *c = &mi->nt->ctg[j.vid >> 1];
	const bool rev = j.vid & 1, left = j.flag & NS_F_EXT_LEFT;
	if (!left) {
		d.g_start = rev ? c->off + c->len - 1 - j.nt_st : c->off + j.nt_st;
		d.dir = rev ? -1 : 1;
	} else { // rows run from the anchor outwards, i.e. against the strand
		d.g_start = rev ? c->off + c->len - j.nt_st - j.nl : c->off + j.nt_st + j.nl - 1;
		d.dir = rev ? 1 : -1;
	}
	d.comp = rev ? 1 : 0;
	d.nl = j.nl, d.al = j.al, d.aa_off = aa_base + j.aa_st, d.flag = j.flag, d.io = j.io;
	d.ss_off = -1, d.ss_excl = -1;
	if (mi->nt->spsc) { // --spsc: the dense table is indexed like the genome, the - strand in its second half
		d.ss_off = rev ? mi->nt->l_seq : 0;
		if (j.win_st >= 0) d.ss_excl = d.ss_off + (rev ? c->off + c->len - 1 - j.win_st : c->off + j.win_st);
	}
	return d;
}

// one thread per (position, byte) entry of the sparse --spsc arrays
__global__ void spsc_scatter_kernel(const uint64_t *e, int64_t n, uint8_t *ss)
{
	const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (k < n) ss[e[k] >> 8] = (uint8_t)(e[k] & 0xff);
}

// mi->nt->spsc (sorted (pos, byte) arrays per contig and strand, ntseq.c:234-296) -> dense byte table in HBM.  Where several
// entries share a position the reference keeps the largest byte while it fills a window (ntseq.c:146-152); the arrays are
// sorted on the whole word, so that is the last entry of the position.
void build_spsc_table(mpb_ctx_s *c, const mp_idx_t *mi)
{
	const mp_ntdb_t *nt = mi->nt;
	const size_t bytes = (size_t)nt->l_seq * 2;
	c->own_ss.reserve(bytes + 16);
	MPB_CUDA_OK(cudaMemsetAsync(c->own_ss.p, 0xff, bytes + 16, c->stream));
	std::vector<uint64_t> e;
	const size_t piece = (size_t)4 << 20;
	auto flush = [&]() {
		if (e.empty()) return;
		c->b_c[14].reserve(sizeof(uint64_t) * piece);
		MPB_CUDA_OK(cudaMemcpyAsync(c->b_c[14].p, e.data(), sizeof(uint64_t) * e.size(), cudaMemcpyHostToDevice, c->stream));
		spsc_scatter_kernel<<<(unsigned)((e.size() + 255) / 256), 256, 0, c->stream>>>(c->b_c[14].as<uint64_t>(), (int64_t)e.size(), c->own_ss.as<uint8_t>());
		MPB_CUDA_OK(cudaStreamSynchronize(c->stream)); // e is reused
		c->stats.h2d_bytes += (int64_t)(sizeof(uint64_t) * e.size()), c->stats.kernel_launches += 1;
		e.clear();
	};
	for (int32_t j = 0; j < nt->n_ctg * 2; ++j) {
		const mp_spsc_t *s = &nt->spsc[j];
		const mp_ctg_t *ct = &nt->ctg[j >> 1];
		for (uint32_t k = 0; k < s->n; ++k) {
			if (k + 1 < s->n && s->a[k + 1] >> 8 == s->a[k] >> 8) continue;
			const int64_t pos = (int64_t)(s->a[k] >> 8);
			const int64_t idx = (j & 1) ? nt->l_seq + ct->off + ct->len - 1 - pos : ct->off + pos;
			e.push_back((uint64_t)idx << 8 | (s->a[k] & 0xff));
			if (e.size() == piece) flush();
		}
	}
	flush();
	MPB_CUDA_OK(cudaStreamSynchronize(c->stream));
	c->d_ss = c->own_ss.as<uint8_t>(), c->ss_src = nt->spsc, c->ss_l_seq = nt->l_seq;
}

int acquire_index(mpb_ctx_s *c, const mp_idx_t *mi);
int acquire_genome(mpb_ctx_s *c, const mp_idx_t *mi);
void pin_to_device_node(int device);

struct CudaStages : Stages {
	mpb_ctx_s *ctx;
	explicit CudaStages(mpb_ctx_s *c) : ctx(c) {}

	// locus mode (loci_view): the stages called with `view` read the resident genome of `view_of`; the k-mer tables are not needed
	const mp_idx_t *view = 0, *view_of = 0;
	bool loci_view(const mp_idx_t *mi, const mp_idx_t *v) override
	{
		view_of = mi, view = v;
		return true;
	}
	void need_index(const mp_idx_t *mi)
	{
		if (mi && mi == view) {
			if (acquire_genome(ctx, view_of) != 0) { fprintf(stderr, "[miniprot_b200] genome upload failed\n"); abort(); }
			return;
		}
		if (ctx->mi != mi || !ctx->d_seq || !ctx->d_ki) {
			if (acquire_index(ctx, mi) != 0) { fprintf(stderr, "[miniprot_b200] index upload failed\n"); abort(); }
		}
	}
	void thread_init() override
	{
		MPB_CUDA_OK(cudaSetDevice(ctx->device));
		pin_to_device_node(ctx->device);
	}
	// residues of the whole batch, concatenated, resident for the duration of the call
	const Batch *cur_batch = 0; // residues of this batch are already resident (between batch_begin and batch_end)
	std::vector<int32_t> cur_off;
	const char *upload_residues(const Batch &b, std::vector<int32_t> &off)
	{
		if (&b == cur_batch) {
			off = cur_off;
			return ctx->b_aa.as<char>();
		}
		off.assign((size_t)b.n + 1, 0);
		for (int32_t i = 0; i < b.n; ++i) off[(size_t)i + 1] = off[(size_t)i] + b.len[i];
		const size_t tot = (size_t)off[(size_t)b.n];
		ctx->b_aa.reserve(tot + 16);
		ctx->h_c[0].reserve(tot + 16);
		char *h = ctx->h_c[0].as<char>();
		for (int32_t i = 0; i < b.n; ++i) memcpy(h + off[(size_t)i], b.seq[i], (size_t)b.len[i]);
		MPB_CUDA_OK(cudaMemcpyAsync(ctx->b_aa.p, h, tot, cudaMemcpyHostToDevice, ctx->stream));
		MPB_CUDA_OK(cudaStreamSynchronize(ctx->stream)); // staging buffer is reused
		ctx->stats.h2d_bytes += (int64_t)tot;
		return ctx->b_aa.as<char>();
	}
	void batch_begin(const Batch &b) override
	{
		cur_batch = 0;
		upload_residues(b, cur_off);
		cur_batch = &b;
	}
	void batch_end() override { cur_batch = 0; }

	void note_wall(int phase, double ms) override { if (phase >= 0 && phase < 6) ctx->stats.ms_wall[phase] += ms; }
	void seed_chain(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override
	{
		need_index(mi);
		std::vector<int32_t> off;
		const char *d_aa = upload_residues(b, off);
		seed_chain_run(ctx, mi, opt, b, off, d_aa, out);
	}
	void seed_chain_loci(const mp_idx_t *vi, const mp_mapopt_t *opt, const Batch &b, ChainSet &out) override
	{
		need_index(vi);
		std::vector<int32_t> off;
		const char *d_aa = upload_residues(b, off);
		seed_chain_loci_run(ctx, vi, opt, b, off, d_aa, out);
	}
	void refine(const mp_idx_t *mi, const mp_mapopt_t *opt, const Batch &b, const std::vector<RefineJob> &jobs, RefineSet &out) override
	{
		need_index(mi);
		std::vector<int32_t> off;
		const char *d_aa = upload_residues(b, off);
		refine_run(ctx, mi, opt, b, off, d_aa, jobs, out);
	}
	void nasw(const mp_idx_t *mi, const ns_opt_t *base, const Batch &b, const std::vector<DpJob> &jobs, DpSet &out) override
	{
		need_index(mi);
		std::vector<int32_t> off;
		const char *d_aa = upload_residues(b, off);
		std::vector<DpDev> dj(jobs.size());
		for (size_t k = 0; k < jobs.size(); ++k) dj[k] = make_dev_job(mi, jobs[k], off[(size_t)jobs[k].qid]);
		if (mi->nt->spsc && ctx->ss_src != mi->nt->spsc) build_spsc_table(ctx, mi);
		nasw_run(ctx, ctx->d_seq, mi->nt->spsc ? ctx->d_ss : 0, d_aa, base, dj, out);
	}
};

// Scoring parameters the kernels cannot reproduce bit for bit are refused (loudly) instead of mapped approximately:
//  * gap open 0 (-O 0).  The reference's lazy-F loop ends when "I - ge <= max(H, I) - go - ge" holds in every SIMD lane
//    (nasw-sse.c:411, :530).  With go > 0 that is only true where the insertion did not raise H, so stopping loses nothing and
//    the result is the textbook recurrence, which is what the kernels compute.  With go == 0 it is true at once: only the
//    first column of each of the eight stripe segments ever sees the insertion carried over from the segment before, and the
//    scores depend on the SSE layout (found by tools/fuzz_emu.py: reference and recurrence differ on ~1 % of random problems).
//  * nasw-sse.c:426 is served from a step table; a coefficient whose steps do not fit it.
bool bad_scoring(int go, float ie_coef)
{
	if (go < 1) {
		fprintf(stderr, "[miniprot_b200] gap open penalty %d: values below 1 are not supported (with -O 0 the reference's result depends on its SIMD stripe layout)\n", go);
		return true;
	}
	if (nasw_check_ie_coef(ie_coef) == 0) return false;
	fprintf(stderr, "[miniprot_b200] ie_coef = %g: the extension length penalty has more than %d steps and is not supported\n", (double)ie_coef, nsw::PEN_STEPS);
	return true;
}
// ... and an index whose minimum ORF length (-L) exceeds what the halos of the window kernel's tiles cover (win_scan.cuh)
bool bad_index(const mp_idx_t *mi)
{
	if (mi->opt.min_aa_len <= WIN_MAX_MIN_AA) return false;
	fprintf(stderr, "[miniprot_b200] min ORF length %d: values above %d are not supported by the window kernels\n", mi->opt.min_aa_len, WIN_MAX_MIN_AA);
	return true;
}

// Host threads of a rank stay on the NUMA node its GPU hangs off (pinned staging buffers, the worker pool of the host phases
// and the driver's own threads then never cross the socket interconnect; with one rank per GPU on a two-socket box the ranks
// of the far socket otherwise straggle).  MPB_AFFINITY=0 leaves the affinity of the calling thread alone.
void pin_to_device_node(int device)
{
	if (const char *e = getenv("MPB_AFFINITY")) if (atoi(e) == 0) return;
	char bus[64];
	if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) return;
	for (char *q = bus; *q; ++q) if (*q >= 'A' && *q <= 'F') *q = (char)(*q - 'A' + 'a');
	char path[256];
	snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
	FILE *fp = fopen(path, "r");
	if (!fp) return;
	int node = -1;
	if (fscanf(fp, "%d", &node) != 1) node = -1;
	fclose(fp);
	if (node < 0) return;
	snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
	fp = fopen(path, "r");
	if (!fp) return;
	char list[4096];
	const size_t got = fread(list, 1, sizeof(list) - 1, fp);
	fclose(fp);
	list[got] = 0;
	cpu_set_t cur, want;
	CPU_ZERO(&want);
	if (sched_getaffinity(0, sizeof(cur), &cur) != 0) return;
	int n_set = 0;
	for (char *q = list; *q;) { // "0-31,64-95"
		char *end;
		long a = strtol(q, &end, 10), b = a;
		if (end == q) break;
		if (*end == '-') b = strtol(end + 1, &end, 10);
		for (long c = a; c <= b && c < CPU_SETSIZE; ++c) if (CPU_ISSET((int)c, &cur)) CPU_SET((int)c, &want), ++n_set;
		q = *end == ',' ? end + 1 : end;
		if (*end != ',') break;
	}
	if (n_set > 0) sched_setaffinity(0, sizeof(want), &want);
}

// Locks, always taken in this order: a context's own mutex (mpb_ctx_s::mu, at the ABI boundary), then g_idx_mu (every change of
// which index a context holds, so that one context can read another's while it shares it), then g_default_mu (the context list).
std::mutex g_default_mu;
std::mutex g_idx_mu;
mpb_ctx_t *g_default_ctx = 0;
std::vector<mpb_ctx_s*> g_all_ctx;

// (the --spsc table goes with the index: it is keyed by the address of mi->nt->spsc, which the next index may reuse)
void forget_index(mpb_ctx_s *c) { c->mi = 0, c->d_seq = 0, c->d_ki = 0, c->d_kb = 0, c->idx_owner = 0, c->ss_src = 0, c->d_ss = 0; }

// an index is identified by its address, so a context must forget it when the host object dies (the next
// mp_idx_t may be allocated at the same address)
void on_idx_destroy(const mp_idx_t *mi)
{
	std::lock_guard<std::mutex> lk(g_default_mu);
	for (mpb_ctx_s *c : g_all_ctx)
		if (c->mi == mi) forget_index(c);
}

// c is about to overwrite or free its own index buffers: the contexts that adopted them forget the index (they share it again, or
// upload it, when they next need it).  Under g_idx_mu.
void forget_adopters(mpb_ctx_s *c)
{
	std::lock_guard<std::mutex> lk(g_default_mu);
	for (mpb_ctx_s *o : g_all_ctx)
		if (o != c && o->idx_owner == c) forget_index(o);
}

// Create a context; pin = keep the calling thread on the device's NUMA node (what mpb_ctx_create does for a process per GPU).
mpb_ctx_s *ctx_new(int device, bool pin);

} // namespace

namespace {

mpb_ctx_s *ctx_new(int device, bool pin)
{
	int n_dev = 0;
	if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
		fprintf(stderr, "[miniprot_b200] no CUDA device: the mapping stages exist only as sm_90a kernels (no CPU fallback)\n");
		return 0;
	}
	if (device < 0 || device >= n_dev) { fprintf(stderr, "[miniprot_b200] bad device %d (have %d)\n", device, n_dev); return 0; }
	MPB_CUDA_OK(cudaSetDevice(device));
	if (pin) pin_to_device_node(device);
	mpb_ctx_s *c = new mpb_ctx_s();
	c->device = device;
	MPB_CUDA_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	MPB_CUDA_OK(cudaEventCreate(&c->ev0));
	MPB_CUDA_OK(cudaEventCreate(&c->ev1));
	MPB_CUDA_OK(cudaEventCreate(&c->ev_bench[0]));
	MPB_CUDA_OK(cudaEventCreate(&c->ev_bench[1]));
	MPB_CUDA_OK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
	MPB_CUDA_OK(cudaEventCreateWithFlags(&c->ev_fork2, cudaEventDisableTiming));
	int prio_lo = 0, prio_hi = 0;
	MPB_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
	for (int i = 0; i < mpb_ctx_s::N_SIDE; ++i) {
		// (numerically lower = more urgent) widest extension class first, then the other extension classes, then the rest
		const int prio = i < 13 ? prio_hi : prio_lo; // extension classes of a DP wave (stream ids 0..12) before everything else
		MPB_CUDA_OK(cudaStreamCreateWithPriority(&c->side[i], cudaStreamNonBlocking, prio));
		MPB_CUDA_OK(cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming));
		MPB_CUDA_OK(cudaEventCreate(&c->ev_k0[i]));
		MPB_CUDA_OK(cudaEventCreate(&c->ev_k1[i]));
		MPB_CUDA_OK(cudaEventCreate(&c->ev_km[i]));
	}
	MPB_CUDA_OK(cudaEventCreate(&c->ev_w0));
	MPB_CUDA_OK(cudaEventCreate(&c->ev_w1));
	MPB_CUDA_OK(cudaEventCreate(&c->ev_p0));
	memset(&c->stats, 0, sizeof(c->stats));
	c->stages = new CudaStages(c);
	{
		std::lock_guard<std::mutex> lk(g_default_mu);
		g_all_ctx.push_back(c);
		g_idx_destroy_hook = on_idx_destroy;
	}
	if (ns_tab_aa20[(uint8_t)'X'] != 21) mp_start();
	return c;
}

void upload_meta(mpb_ctx_s *c, const mp_idx_t *mi)
{
	const int32_t n_ctg = mi->nt->n_ctg;
	c->own_bo.reserve(sizeof(uint32_t) * (size_t)(2 * n_ctg + 1));
	MPB_CUDA_OK(cudaMemcpy(c->own_bo.p, mi->bo, sizeof(uint32_t) * (size_t)(2 * n_ctg + 1), cudaMemcpyHostToDevice));
	std::vector<int64_t> ctg((size_t)n_ctg * 2);
	for (int32_t i = 0; i < n_ctg; ++i) ctg[(size_t)i * 2] = mi->nt->ctg[i].off, ctg[(size_t)i * 2 + 1] = mi->nt->ctg[i].len;
	c->own_ctg.reserve(sizeof(int64_t) * ctg.size() + 16);
	MPB_CUDA_OK(cudaMemcpy(c->own_ctg.p, ctg.data(), sizeof(int64_t) * ctg.size(), cudaMemcpyHostToDevice));
	c->d_bo = c->own_bo.as<uint32_t>(), c->d_ctg = c->own_ctg.as<int64_t>();
}

// mpb_idx_upload without the locks (the caller holds c->mu and g_idx_mu)
int idx_upload_unlocked(mpb_ctx_s *c, const mp_idx_t *mi)
{
	if (!mi->ki || !mi->kb) return c->mi == mi && c->d_ki ? 0 : -1; // loaded straight into HBM: no host tables to upload from (see mpb_idx_share)
	MPB_CUDA_OK(cudaSetDevice(c->device));
	forget_adopters(c);
	const size_t nb = idx_n_bucket(&mi->opt), seq_bytes = (size_t)((mi->nt->l_seq + 1) >> 1);
	c->own_ki.reserve(sizeof(int64_t) * (nb + 1));
	c->own_kb.reserve(sizeof(uint32_t) * (size_t)(mi->n_kb + 1));
	c->own_seq.reserve(seq_bytes + 16);
	MPB_CUDA_OK(cudaMemcpy(c->own_ki.p, mi->ki, sizeof(int64_t) * nb, cudaMemcpyHostToDevice));
	MPB_CUDA_OK(cudaMemcpy(c->own_ki.as<int64_t>() + nb, &mi->n_kb, sizeof(int64_t), cudaMemcpyHostToDevice)); // sentinel: end of the last bucket
	MPB_CUDA_OK(cudaMemcpy(c->own_kb.p, mi->kb, sizeof(uint32_t) * (size_t)mi->n_kb, cudaMemcpyHostToDevice));
	MPB_CUDA_OK(cudaMemcpy(c->own_seq.p, mi->nt->seq, seq_bytes, cudaMemcpyHostToDevice));
	c->d_ki = c->own_ki.as<int64_t>(), c->d_kb = c->own_kb.as<uint32_t>(), c->d_seq = c->own_seq.as<uint8_t>();
	upload_meta(c, mi);
	c->mi = mi, c->own_index = true, c->idx_owner = 0;
	c->stats.h2d_bytes += (int64_t)(sizeof(int64_t) * nb + sizeof(uint32_t) * (size_t)mi->n_kb + seq_bytes);
	return 0;
}

// mpb_idx_share without the locks (the caller holds dst->mu and g_idx_mu; src's index cannot change meanwhile)
int idx_share_unlocked(mpb_ctx_s *dst, mpb_ctx_s *src)
{
	const mp_idx_t *mi = src->mi;
	if (!mi || !src->d_ki || !src->d_kb || !src->d_seq) return -1;
	if (dst == src) return 0;
	MPB_CUDA_OK(cudaSetDevice(dst->device));
	if (dst->device == src->device) { // adopt: nothing is copied
		dst->d_ki = src->d_ki, dst->d_kb = src->d_kb, dst->d_seq = src->d_seq;
		upload_meta(dst, mi);
		dst->mi = mi, dst->own_index = false;
		dst->idx_owner = src->own_index ? src : src->idx_owner; // null: the buffers came from outside (mpb_idx_attach_device)
		return 0;
	}
	// another device: a copy of the three arrays in dst's own buffers, straight from src's (works with or without peer access)
	forget_adopters(dst);
	const size_t nb = idx_n_bucket(&mi->opt), seq_bytes = (size_t)((mi->nt->l_seq + 1) >> 1);
	dst->own_ki.reserve(sizeof(int64_t) * (nb + 1));
	dst->own_kb.reserve(sizeof(uint32_t) * (size_t)(mi->n_kb + 1));
	dst->own_seq.reserve(seq_bytes + 16);
	MPB_CUDA_OK(cudaMemcpyPeerAsync(dst->own_ki.p, dst->device, src->d_ki, src->device, sizeof(int64_t) * (nb + 1), dst->stream)); // with the sentinel
	if (mi->n_kb) MPB_CUDA_OK(cudaMemcpyPeerAsync(dst->own_kb.p, dst->device, src->d_kb, src->device, sizeof(uint32_t) * (size_t)mi->n_kb, dst->stream));
	MPB_CUDA_OK(cudaMemcpyPeerAsync(dst->own_seq.p, dst->device, src->d_seq, src->device, seq_bytes, dst->stream));
	MPB_CUDA_OK(cudaStreamSynchronize(dst->stream));
	dst->d_ki = dst->own_ki.as<int64_t>(), dst->d_kb = dst->own_kb.as<uint32_t>(), dst->d_seq = dst->own_seq.as<uint8_t>();
	upload_meta(dst, mi);
	dst->mi = mi, dst->own_index = true, dst->idx_owner = 0;
	return 0;
}

// CudaStages::need_index: the index from another context that holds it (one on the same device first: nothing is copied), else
// from the host tables.  An index loaded with mpb_idx_load_device has no host tables, so it can only be shared.
int acquire_index(mpb_ctx_s *c, const mp_idx_t *mi)
{
	std::lock_guard<std::mutex> il(g_idx_mu);
	if (c->mi == mi && c->d_seq && c->d_ki) return 0;
	mpb_ctx_s *src = 0;
	{
		std::lock_guard<std::mutex> lk(g_default_mu);
		for (mpb_ctx_s *o : g_all_ctx)
			if (o != c && o->mi == mi && o->d_ki && o->d_kb && o->d_seq && (!src || (o->device == c->device && src->device != c->device))) src = o;
	}
	return src ? idx_share_unlocked(c, src) : idx_upload_unlocked(c, mi);
}

// CudaStages::need_index in locus mode: mi's genome resident in c.  Nothing is uploaded when c holds mi (with or without its k-mer
// tables); otherwise only the packed genome and the contig table are, never the k-mer tables (mi may have none: mpb_idx_load_meta).
int acquire_genome(mpb_ctx_s *c, const mp_idx_t *mi)
{
	std::lock_guard<std::mutex> il(g_idx_mu);
	if (c->mi == mi && c->d_seq) return 0;
	if (!mi || !mi->nt || !mi->nt->seq) return -1;
	MPB_CUDA_OK(cudaSetDevice(c->device));
	forget_adopters(c);
	forget_index(c);
	const size_t seq_bytes = (size_t)((mi->nt->l_seq + 1) >> 1);
	c->own_seq.reserve(seq_bytes + 16);
	MPB_CUDA_OK(cudaMemcpy(c->own_seq.p, mi->nt->seq, seq_bytes, cudaMemcpyHostToDevice));
	c->d_seq = c->own_seq.as<uint8_t>();
	upload_meta(c, mi);
	c->mi = mi, c->own_index = true;
	c->stats.h2d_bytes += (int64_t)seq_bytes;
	return 0;
}

// MPB_DEVICES=<device>[,<device>...] (repeats allowed: "0,0" = two contexts on device 0), read once; empty when unset
const std::vector<int> &pool_devices()
{
	static const std::vector<int> dev = [] {
		std::vector<int> d;
		const char *e = getenv("MPB_DEVICES");
		if (!e || !*e) return d;
		for (const char *q = e; *q;) {
			char *end;
			const long v = strtol(q, &end, 10);
			if (end == q || v < 0 || (*end && *end != ',')) {
				fprintf(stderr, "[miniprot_b200] MPB_DEVICES=%s: expected a comma-separated list of device numbers\n", e);
				abort();
			}
			d.push_back((int)v);
			q = *end == ',' ? end + 1 : end;
		}
		return d;
	}();
	return dev;
}

// The contexts of MPB_DEVICES: mp_map_file maps over all of them, mp_map and ns_global_gs16b take an idle one.  Context 0 is the
// default context.  Lives as long as the process.
class CtxPool {
public:
	static CtxPool *get() // null when MPB_DEVICES is unset
	{
		static CtxPool *p = pool_devices().empty() ? 0 : new CtxPool();
		return p;
	}
	std::vector<mpb_ctx_s*> ctx;
	mpb_ctx_s *acquire()
	{
		std::unique_lock<std::mutex> lk(mu_);
		cv_.wait(lk, [&] { return std::find(busy_.begin(), busy_.end(), (char)0) != busy_.end(); });
		const size_t k = (size_t)(std::find(busy_.begin(), busy_.end(), (char)0) - busy_.begin());
		busy_[k] = 1;
		return ctx[k];
	}
	void release(mpb_ctx_s *c)
	{
		std::lock_guard<std::mutex> lk(mu_);
		for (size_t k = 0; k < ctx.size(); ++k) if (ctx[k] == c) busy_[k] = 0;
		cv_.notify_one();
	}

private:
	CtxPool()
	{
		const std::vector<int> &dev = pool_devices();
		ctx.push_back(mpb_ctx_default());
		for (size_t k = 1; k < dev.size(); ++k) {
			mpb_ctx_s *c = ctx_new(dev[k], false); // the mapper threads keep to the node of their device themselves
			if (!c) { fprintf(stderr, "[miniprot_b200] MPB_DEVICES: cannot create a context on device %d\n", dev[k]); abort(); }
			ctx.push_back(c);
		}
		busy_.assign(ctx.size(), 0);
	}
	std::mutex mu_;
	std::condition_variable cv_;
	std::vector<char> busy_;
};

// one protein on a pool context when MPB_DEVICES is set, else on the default context (whose mutex makes concurrent callers take turns)
struct AnyCtx {
	CtxPool *pool = CtxPool::get();
	mpb_ctx_s *c = pool ? pool->acquire() : mpb_ctx_default();
	~AnyCtx() { if (pool) pool->release(c); }
};

// The contexts of one call of a file entry point
struct FileCtx {
	std::vector<mpb_ctx_s*> ctx, by_addr;
	std::vector<std::unique_lock<std::mutex>> held;
	std::vector<Stages*> st; // after hold(): the contexts' stages, in the caller's order
	// false unless the n contexts are non-null and distinct: a context maps one unit at a time
	bool distinct(mpb_ctx_t *const *c, int32_t n)
	{
		if (!c || n < 1) return false;
		ctx.assign(c, c + n), by_addr = ctx;
		std::sort(by_addr.begin(), by_addr.end());
		return by_addr[0] && std::adjacent_find(by_addr.begin(), by_addr.end()) == by_addr.end();
	}
	// After distinct(): holds the contexts' mutexes in address order until destruction (two such calls never wait for each other in a
	// cycle), makes mi resident in every context before the mappers start -- the whole index (shared between contexts where one holds
	// it), or only its genome when genome_only (locus mode) -- and makes the first context's device current.  -1 with a message when
	// mi cannot be made resident.
	int hold(const mp_idx_t *mi, bool genome_only)
	{
		for (mpb_ctx_s *c : by_addr) held.emplace_back(c->mu);
		for (mpb_ctx_s *c : ctx) {
			if (genome_only ? acquire_genome(c, mi) != 0 : acquire_index(c, mi) != 0) {
				fprintf(stderr, genome_only ? "[miniprot_b200] the index has no genome on the host and is not resident in the context\n"
				                            : "[miniprot_b200] the index is neither resident in a context nor on the host\n");
				return -1;
			}
			st.push_back(c->stages);
		}
		MPB_CUDA_OK(cudaSetDevice(ctx[0]->device));
		return 0;
	}
};

} // namespace

extern "C" {

mpb_ctx_t *mpb_ctx_create(int device) { return ctx_new(device, true); }

// A context that adopted another's index buffers (mpb_idx_share on one device) must not be in use while their owner is destroyed
// or replaces its index.  When that happens the adopter forgets the index, so it never reads freed memory: its next mapping call
// shares the index again from a context that holds it, or uploads it from the host tables.
void mpb_ctx_destroy(mpb_ctx_t *c)
{
	if (!c) return;
	std::unique_lock<std::mutex> cl(c->mu);
	{
		std::lock_guard<std::mutex> il(g_idx_mu);
		forget_adopters(c);
		std::lock_guard<std::mutex> lk(g_default_mu);
		for (size_t i = 0; i < g_all_ctx.size(); ++i) if (g_all_ctx[i] == c) { g_all_ctx.erase(g_all_ctx.begin() + (ptrdiff_t)i); break; }
	}
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->stream);
	DevBuf *bufs[] = { &c->own_ki, &c->own_kb, &c->own_seq, &c->own_bo, &c->own_ctg, &c->b_jobs, &c->b_order, &c->b_chunks, &c->b_rw, &c->b_aa, &c->b_out,
	                   &c->b_carry, &c->b_tb, &c->b_cigar, &c->b_cigpack, &c->b_cigoff, &c->b_packed, &c->b_units };
	for (DevBuf *b : bufs) b->release();
	for (DevBuf &b : c->b_c) b.release();
	c->h_out.release(), c->h_cigar.release();
	for (PinBuf &b : c->h_c) b.release();
	cudaEventDestroy(c->ev0), cudaEventDestroy(c->ev1), cudaEventDestroy(c->ev_fork), cudaEventDestroy(c->ev_fork2);
	cudaEventDestroy(c->ev_bench[0]), cudaEventDestroy(c->ev_bench[1]);
	for (int i = 0; i < mpb_ctx_s::N_SIDE; ++i) cudaStreamDestroy(c->side[i]), cudaEventDestroy(c->ev_join[i]), cudaEventDestroy(c->ev_k0[i]), cudaEventDestroy(c->ev_k1[i]), cudaEventDestroy(c->ev_km[i]);
	cudaEventDestroy(c->ev_w0), cudaEventDestroy(c->ev_w1), cudaEventDestroy(c->ev_p0);
	cudaStreamDestroy(c->stream);
	delete c->stages;
	cl.unlock();
	delete c;
}

// LOCAL_RANK or device 0; with MPB_DEVICES set, the first device of that list (the default context is context 0 of the pool, and the
// calling thread is left where it is: the mapper threads keep to their devices' nodes themselves)
mpb_ctx_t *mpb_ctx_default(void)
{
	static std::mutex once_mu; // not g_default_mu: mpb_ctx_create takes that one itself
	std::lock_guard<std::mutex> lk(once_mu);
	if (!g_default_ctx) {
		int dev = 0;
		if (const char *e = getenv("LOCAL_RANK")) dev = atoi(e);
		const std::vector<int> &pool = pool_devices();
		g_default_ctx = pool.empty() ? mpb_ctx_create(dev) : ctx_new(pool[0], false);
		if (!g_default_ctx) { fprintf(stderr, "[miniprot_b200] cannot run without a GPU\n"); abort(); }
	}
	return g_default_ctx;
}

int mpb_idx_upload(mpb_ctx_t *c, const mp_idx_t *mi)
{
	if (!c || !mi) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	std::lock_guard<std::mutex> il(g_idx_mu);
	return idx_upload_unlocked(c, mi);
}

int mpb_idx_share(mpb_ctx_t *dst, mpb_ctx_t *src)
{
	if (!dst || !src) return -1;
	std::lock_guard<std::mutex> cl(dst->mu);
	std::lock_guard<std::mutex> il(g_idx_mu);
	return idx_share_unlocked(dst, src);
}

// FASTA -> index with the k-mer tables built on the device (idx_build.cu); called by mp_idx_load through g_idx_build_hook once the
// genome is packed.  The tables stay resident in the default context, so the mapping calls that follow find the index uploaded.
// Returns non-zero when there is no device or the options are outside what the device scan covers: the caller then builds on the host.
static int build_index_on_device(mp_idx_t *mi)
{
	if (const char *e = getenv("MPB_IDX_BUILD")) if (strcmp(e, "host") == 0) return -1;
	int n_dev = 0;
	if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0) { cudaGetLastError(); return -1; }
	mpb_ctx_t *c = mpb_ctx_default();
	std::lock_guard<std::mutex> cl(c->mu);
	std::lock_guard<std::mutex> il(g_idx_mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	const double t0 = mp_realtime();
	forget_adopters(c);
	if (c->own_index) forget_index(c); // the build reuses the context's own buffers
	if (idx_build_device(c, mi) != 0) return -1;
	c->d_ki = c->own_ki.as<int64_t>(), c->d_kb = c->own_kb.as<uint32_t>(), c->d_seq = c->own_seq.as<uint8_t>();
	upload_meta(c, mi);
	c->mi = mi, c->own_index = true, c->idx_owner = 0;
	if (mp_verbose >= 3) fprintf(stderr, "[M::%s@%.3f] built the k-mer tables on the device in %.3f s: %ld kmer-block pairs\n", __func__, mp_realtime(), mp_realtime() - t0, (long)mi->n_kb);
	return 0;
}
namespace { struct IdxBuildHook { IdxBuildHook() { mpb::g_idx_build_hook = build_index_on_device; } } g_idx_build_hook_init; }

// .mpi file -> HBM (SURVEY 8f #3): the k-mer tables ki / kb -- 85-90 % of the file, needed on the device only -- never get a
// host copy: the file is read in 32 MB pieces into two pinned buffers and each piece leaves for the device while the next
// one is being read.  The genome section is kept on the host as well (statistics, cs tags, output formats read it).  The
// returned index has ki == kb == NULL; everything of the library works with it except mp_idx_dump / mp_idx_print_stat.
mp_idx_t *mpb_idx_load_device(mpb_ctx_t *c, const char *fn)
{
	if (!c || !fn) return 0;
	std::lock_guard<std::mutex> cl(c->mu);
	std::lock_guard<std::mutex> il(g_idx_mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	FILE *fp = fopen(fn, "rb");
	if (!fp) return 0;
	mp_idx_t *mi = idx_restore_head(fp);
	if (!mi) { fclose(fp); return 0; }
	forget_adopters(c);
	if (c->own_index) forget_index(c); // its buffers are refilled below
	const size_t nb = idx_n_bucket(&mi->opt), seq_bytes = (size_t)((mi->nt->l_seq + 1) >> 1);
	c->own_ki.reserve(sizeof(int64_t) * (nb + 1));
	c->own_kb.reserve(sizeof(uint32_t) * (size_t)(mi->n_kb + 1));
	c->own_seq.reserve(seq_bytes + 16);
	MPB_CUDA_OK(cudaMemcpyAsync(c->own_seq.p, mi->nt->seq, seq_bytes, cudaMemcpyHostToDevice, c->stream));
	const size_t piece = (size_t)32 << 20;
	c->h_c[1].reserve(piece), c->h_c[2].reserve(piece);
	cudaEvent_t done[2];
	MPB_CUDA_OK(cudaEventCreateWithFlags(&done[0], cudaEventDisableTiming));
	MPB_CUDA_OK(cudaEventCreateWithFlags(&done[1], cudaEventDisableTiming));
	bool ok = true;
	int turn = 0;
	auto stream_section = [&](char *dst, size_t bytes) {
		for (size_t off = 0; off < bytes && ok; off += piece, turn ^= 1) {
			const size_t n = std::min(piece, bytes - off);
			PinBuf &pb = c->h_c[1 + turn];
			MPB_CUDA_OK(cudaEventSynchronize(done[turn])); // the copy that last used this buffer has left
			ok = fread(pb.p, 1, n, fp) == n;
			if (!ok) break;
			MPB_CUDA_OK(cudaMemcpyAsync(dst + off, pb.p, n, cudaMemcpyHostToDevice, c->stream));
			MPB_CUDA_OK(cudaEventRecord(done[turn], c->stream));
		}
	};
	stream_section((char*)c->own_ki.p, sizeof(int64_t) * nb);
	stream_section((char*)c->own_kb.p, sizeof(uint32_t) * (size_t)mi->n_kb);
	fclose(fp);
	if (ok) MPB_CUDA_OK(cudaMemcpyAsync(c->own_ki.as<int64_t>() + nb, &mi->n_kb, sizeof(int64_t), cudaMemcpyHostToDevice, c->stream)); // sentinel
	MPB_CUDA_OK(cudaStreamSynchronize(c->stream));
	cudaEventDestroy(done[0]), cudaEventDestroy(done[1]);
	if (!ok) { mp_idx_destroy(mi); return 0; }
	c->d_ki = c->own_ki.as<int64_t>(), c->d_kb = c->own_kb.as<uint32_t>(), c->d_seq = c->own_seq.as<uint8_t>();
	upload_meta(c, mi);
	c->mi = mi, c->own_index = true, c->idx_owner = 0;
	c->stats.h2d_bytes += (int64_t)(sizeof(int64_t) * nb + sizeof(uint32_t) * (size_t)mi->n_kb + seq_bytes);
	if (mp_verbose >= 3) fprintf(stderr, "[M::%s@%.3f] loaded the index into device memory\n", __func__, mp_realtime());
	return mi;
}

// the head of a .mpi file only (options, contig table, genome): what a rank needs on the host when the k-mer tables reach its GPU
// through the NCCL broadcast (mpb_idx_attach_device)
mp_idx_t *mpb_idx_load_meta(const char *fn)
{
	FILE *fp = fn ? fopen(fn, "rb") : 0;
	if (!fp) return 0;
	mp_idx_t *mi = idx_restore_head(fp);
	fclose(fp);
	return mi;
}

// device addresses of the resident index of a context (the source buffers of the broadcast on the rank that loaded the file)
int mpb_idx_device_ptrs(mpb_ctx_t *c, void **d_ki, void **d_kb, void **d_seq)
{
	if (!c) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	if (!c->d_ki) return -1;
	*d_ki = c->d_ki, *d_kb = c->d_kb, *d_seq = c->d_seq;
	return 0;
}

int mpb_idx_attach_device(mpb_ctx_t *c, const mp_idx_t *mi, void *d_ki, void *d_kb, void *d_seq)
{
	if (!c || !mi || !d_ki || !d_kb || !d_seq) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	std::lock_guard<std::mutex> il(g_idx_mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	c->d_ki = (int64_t*)d_ki, c->d_kb = (uint32_t*)d_kb, c->d_seq = (uint8_t*)d_seq;
	upload_meta(c, mi);
	c->mi = mi, c->own_index = false, c->idx_owner = 0;
	return 0;
}

// mpb_map_batch; qr_tid < 0: no QR lines of --dbg-qname (mp_map, which the reference calls after printing them in worker_for)
static int map_batch_on(mpb_ctx_t *c, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens,
                        const char *const *names, int32_t *n_reg_out, mp_reg1_t **reg_out, int32_t qr_tid)
{
	if (!c) return -1;
	if (bad_scoring(opt->go, opt->ie_coef) || bad_index(mi) || bad_dbg_flags(opt)) return -3;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	Batch b;
	b.n = n_seq, b.seq = seqs, b.len = lens, b.name = names;
	map_batch(c->stages, mi, opt, b, n_reg_out, reg_out, qr_tid);
	return 0;
}

int mpb_map_batch(mpb_ctx_t *c, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens,
                  const char *const *names, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	return map_batch_on(c, mi, opt, n_seq, seqs, lens, names, n_reg_out, reg_out, 0);
}

int mpb_map_loci(mpb_ctx_t *c, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens,
                 const char *const *names, int32_t n_loci, const mpb_locus_t *loci, int32_t *n_reg_out, mp_reg1_t **reg_out)
{
	if (!c || !opt) return -1;
	const int rc = check_loci(mi, n_seq, n_loci, loci);
	if (rc != 0) return rc;
	if (bad_scoring(opt->go, opt->ie_coef) || bad_index(mi)) return -3;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	return map_loci(c->stages, mi, opt, n_seq, seqs, lens, names, n_loci, loci, n_reg_out, reg_out);
}

int mpb_seed_loci_batch(mpb_ctx_t *c, const mp_idx_t *mi, int32_t max_occ, int32_t n_seq, const char *const *seqs, const int32_t *lens, int32_t n_loci,
                        const mpb_locus_t *loci, int64_t *a_off, uint64_t **a)
{
	if (!c) return -1;
	const int rc = check_loci(mi, n_seq, n_loci, loci);
	if (rc != 0) return rc;
	if (bad_index(mi)) return -3;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	LocusView v(mi, n_loci, loci);
	std::vector<const char*> sp((size_t)n_loci);
	std::vector<int32_t> lp((size_t)n_loci);
	for (int32_t k = 0; k < n_loci; ++k) sp[(size_t)k] = seqs[loci[k].qid], lp[(size_t)k] = lens[loci[k].qid];
	Batch b;
	b.n = n_loci, b.seq = sp.data(), b.len = lp.data(), b.name = 0;
	std::vector<int64_t> ao((size_t)n_loci + 1, 0);
	std::vector<uint64_t> av;
	if (n_loci > 0) {
		CudaStages *cs = static_cast<CudaStages*>(c->stages);
		cs->loci_view(mi, &v.idx);
		cs->need_index(&v.idx);
		std::vector<int32_t> off;
		const char *d_aa = cs->upload_residues(b, off);
		seed_loci_batch_run(c, &v.idx, max_occ, b, off, d_aa, ao, av);
		cs->loci_view(0, 0);
	}
	for (int32_t k = 0; k <= n_loci; ++k) a_off[k] = ao[(size_t)k];
	for (int32_t k = 0; k < n_loci; ++k) // view block ids -> those of an index of the locus alone
		for (int64_t j = ao[(size_t)k]; j < ao[(size_t)k + 1]; ++j) av[(size_t)j] -= (uint64_t)v.bo[(size_t)k * 2] << 32;
	*a = (uint64_t*)malloc(sizeof(uint64_t) * (av.size() + 1));
	if (!av.empty()) memcpy(*a, av.data(), sizeof(uint64_t) * av.size());
	return 0;
}

int32_t mpb_map_file(mpb_ctx_t *c, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out)
{
	return mpb_map_file_multi(&c, 1, mi, fn, opt, out);
}

int32_t mpb_map_file_path(mpb_ctx_t *c, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, const char *out_path)
{
	return mpb_map_file_multi_path(&c, 1, mi, fn, opt, out_path);
}

int32_t mpb_map_file_multi(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out)
{
	FileCtx fc;
	if (!fc.distinct(ctx, n_ctx)) return -1;
	if (bad_scoring(opt->go, opt->ie_coef) || bad_index(mi) || bad_dbg_flags(opt)) return -3;
	if (fc.hold(mi, false) != 0) return -1;
	return map_file_multi(fc.st.data(), n_ctx, mi, fn, opt, out);
}

int32_t mpb_map_file_multi_path(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, const char *out_path)
{
	FILE *fp = fopen(out_path, "wb");
	if (!fp) return -2;
	int32_t rc = mpb_map_file_multi(ctx, n_ctx, mi, fn, opt, fp);
	fclose(fp);
	return rc;
}

// the locus file driver on n_ctx contexts, into `out` or, when that is null, into a file created at out_path once the input is valid
static int32_t map_loci_file_on(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt,
                                FILE *out, const char *out_path)
{
	FileCtx fc;
	if (!fc.distinct(ctx, n_ctx) || !opt || !mi) return -1;
	LociFile in;
	int32_t rc = loci_file_read(mi, prot_fn, loci_fn, in);
	if (rc != 0) return rc;
	if (bad_scoring(opt->go, opt->ie_coef) || bad_index(mi)) return -3;
	FILE *fp = out ? out : fopen(out_path, "wb");
	if (!fp) return -2;
	rc = fc.hold(mi, true);
	if (rc == 0) rc = map_loci_file(fc.st.data(), n_ctx, mi, in, opt, fp);
	if (!out) fclose(fp);
	return rc;
}

int32_t mpb_map_loci_file(mpb_ctx_t *c, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, FILE *out)
{
	return out ? map_loci_file_on(&c, 1, mi, prot_fn, loci_fn, opt, out, 0) : -1;
}

int32_t mpb_map_loci_file_path(mpb_ctx_t *c, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, const char *out_path)
{
	return out_path ? map_loci_file_on(&c, 1, mi, prot_fn, loci_fn, opt, 0, out_path) : -1;
}

int32_t mpb_map_loci_file_multi(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, FILE *out)
{
	return out ? map_loci_file_on(ctx, n_ctx, mi, prot_fn, loci_fn, opt, out, 0) : -1;
}

int32_t mpb_map_loci_file_multi_path(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt,
                                     const char *out_path)
{
	return out_path ? map_loci_file_on(ctx, n_ctx, mi, prot_fn, loci_fn, opt, 0, out_path) : -1;
}

mp_reg1_t *mp_map(const mp_idx_t *mi, int qlen, const char *seq, int *n_reg, mp_tbuf_t *, const mp_mapopt_t *opt, const char *qname)
{
	mp_reg1_t *reg = 0;
	int32_t len = qlen, nr = 0;
	AnyCtx a;
	map_batch_on(a.c, mi, opt, 1, &seq, &len, &qname, &nr, &reg, -1);
	*n_reg = nr;
	return reg;
}

int32_t mp_map_file(const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, int)
{
	CtxPool *p = CtxPool::get();
	mpb_ctx_s *c = p ? 0 : mpb_ctx_default();
	return mpb_map_file_multi(p ? p->ctx.data() : &c, p ? (int32_t)p->ctx.size() : 1, mi, fn, opt, stdout);
}

int64_t mpb_format_paf(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq, const mp_reg1_t *r, char **buf,
                       int64_t *len, int64_t *cap)
{
	Str s;
	s.s = *buf, s.l = *len, s.m = *cap;
	format_hit(s, mi, opt, qname, qlen, qseq, r);
	*buf = s.s, *len = s.l, *cap = s.m;
	return s.l;
}

int mpb_nasw_batch(mpb_ctx_t *c, const ns_opt_t *opt, int32_t n, const mpb_dp_problem_t *prob, mpb_dp_result_t *rst)
{
	if (!c) return -1;
	if (bad_scoring(opt->go, opt->ie_coef)) return -3;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	// pack the host sequences the way the genome is stored, so that the same kernels serve both paths
	int64_t nt_tot = 0, aa_tot = 0;
	bool any_ss = false;
	for (int32_t i = 0; i < n; ++i) {
		if (prob[i].ss) any_ss = true;
		nt_tot += prob[i].nl + 2, aa_tot += prob[i].al;
	}
	std::vector<uint8_t> ssb;
	if (any_ss) ssb.assign((size_t)nt_tot + 16, 0xff);
	std::vector<uint8_t> packed((size_t)(nt_tot / 2 + 2), 0);
	std::vector<char> aa((size_t)aa_tot + 1);
	std::vector<DpDev> jobs((size_t)n);
	int64_t g = 0, a = 0;
	for (int32_t i = 0; i < n; ++i) {
		const mpb_dp_problem_t &p = prob[i];
		for (int32_t k = 0; k < p.nl; ++k) packed[(size_t)((g + k) >> 1)] |= (uint8_t)(ns_tab_nt4[p.nt[k]] << (((g + k) & 1) * 4));
		memcpy(aa.data() + a, p.aa, (size_t)p.al);
		DpDev &d = jobs[(size_t)i];
		memset(&d, 0, sizeof(d));
		const bool left = p.flag & NS_F_EXT_LEFT;
		d.g_start = left ? g + p.nl - 1 : g, d.dir = left ? -1 : 1, d.comp = 0;
		d.nl = p.nl, d.al = p.al, d.aa_off = (int32_t)a, d.flag = p.flag, d.io = p.io;
		d.ss_off = -1, d.ss_excl = -1;
		if (p.ss) memcpy(ssb.data() + g, p.ss, (size_t)p.nl), d.ss_off = 0; // splice bytes travel laid out like the packed bases
		g += p.nl + 2, a += p.al;
	}
	c->b_packed.reserve(packed.size() + 16);
	c->b_aa.reserve(aa.size() + 16);
	MPB_CUDA_OK(cudaMemcpyAsync(c->b_packed.p, packed.data(), packed.size(), cudaMemcpyHostToDevice, c->stream));
	MPB_CUDA_OK(cudaMemcpyAsync(c->b_aa.p, aa.data(), aa.size(), cudaMemcpyHostToDevice, c->stream));
	if (any_ss) {
		c->b_c[15].reserve(ssb.size());
		MPB_CUDA_OK(cudaMemcpyAsync(c->b_c[15].p, ssb.data(), ssb.size(), cudaMemcpyHostToDevice, c->stream));
	}
	MPB_CUDA_OK(cudaStreamSynchronize(c->stream));
	c->stats.h2d_bytes += (int64_t)(packed.size() + aa.size() + ssb.size());
	DpSet out;
	nasw_run(c, c->b_packed.as<uint8_t>(), any_ss ? c->b_c[15].as<uint8_t>() : 0, c->b_aa.as<char>(), opt, jobs, out);
	for (int32_t i = 0; i < n; ++i) {
		rst[i].score = out.score[(size_t)i], rst[i].nt_len = out.nt_len[(size_t)i], rst[i].aa_len = out.aa_len[(size_t)i];
		const int64_t nc = out.cig_off[(size_t)i + 1] - out.cig_off[(size_t)i];
		rst[i].n_cigar = (int32_t)nc, rst[i].cigar = 0;
		if (nc > 0) {
			rst[i].cigar = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)nc);
			memcpy(rst[i].cigar, out.cig.data() + out.cig_off[(size_t)i], sizeof(uint32_t) * (size_t)nc);
		}
	}
	return 0;
}

int mpb_chain_batch(mpb_ctx_t *c, const mpb_chain_par_t *par, int32_t n, const int64_t *a_off, const uint64_t *a, int64_t *u_off, uint64_t **u, int64_t *b_off,
                    uint64_t **b)
{
	if (!c) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	chn::Par p;
	p.max_dist_x = par->max_dist_x, p.max_dist_y = par->max_dist_y, p.bw = par->bw, p.max_skip = par->max_skip, p.max_iter = par->max_iter;
	p.min_cnt = par->min_cnt, p.min_sc = par->min_sc, p.chn_coef_log = par->chn_coef_log, p.is_spliced = par->is_spliced, p.kmer = par->kmer, p.bbit = par->bbit;
	std::vector<int32_t> nu, nb;
	std::vector<uint64_t> uu, bb;
	chain_batch_run(c, p, n, a_off, a, nu, nb, uu, bb);
	u_off[0] = b_off[0] = 0;
	for (int32_t i = 0; i < n; ++i) u_off[i + 1] = u_off[i] + nu[(size_t)i], b_off[i + 1] = b_off[i] + nb[(size_t)i];
	*u = (uint64_t*)malloc(sizeof(uint64_t) * (uu.size() + 1)), *b = (uint64_t*)malloc(sizeof(uint64_t) * (bb.size() + 1));
	if (!uu.empty()) memcpy(*u, uu.data(), sizeof(uint64_t) * uu.size());
	if (!bb.empty()) memcpy(*b, bb.data(), sizeof(uint64_t) * bb.size());
	return 0;
}

int mpb_seed_batch(mpb_ctx_t *c, const mp_idx_t *mi, int32_t max_occ, int32_t n_seq, const char *const *seqs, const int32_t *lens, int64_t *a_off, uint64_t **a)
{
	if (c == 0 || mi == 0 || n_seq < 0) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	Batch b;
	b.n = n_seq, b.seq = seqs, b.len = lens, b.name = 0;
	CudaStages *cs = static_cast<CudaStages*>(c->stages);
	cs->need_index(mi);
	std::vector<int32_t> off;
	const char *d_aa = cs->upload_residues(b, off);
	std::vector<int64_t> ao;
	std::vector<uint64_t> av;
	seed_batch_run(c, mi, max_occ, b, off, d_aa, ao, av);
	for (int32_t i = 0; i <= n_seq; ++i) a_off[i] = ao[(size_t)i];
	*a = (uint64_t*)malloc(sizeof(uint64_t) * (av.size() + 1));
	if (!av.empty()) memcpy(*a, av.data(), sizeof(uint64_t) * av.size());
	return 0;
}

int mpb_refine_batch(mpb_ctx_t *c, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens, int32_t n_win,
                     const mpb_window_t *win, int64_t *a_off, uint64_t **a, int32_t *sc)
{
	if (c == 0 || mi == 0 || opt == 0 || n_seq < 0 || n_win < 0) return -1;
	if (bad_index(mi)) return -3;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	Batch b;
	b.n = n_seq, b.seq = seqs, b.len = lens, b.name = 0;
	std::vector<RefineJob> jobs((size_t)n_win);
	for (int32_t k = 0; k < n_win; ++k) {
		if (win[k].qid < 0 || win[k].qid >= n_seq) return -1;
		jobs[(size_t)k].qid = win[k].qid, jobs[(size_t)k].vid = win[k].vid, jobs[(size_t)k].as = win[k].as, jobs[(size_t)k].ae = win[k].ae;
	}
	RefineSet rs;
	c->stages->refine(mi, opt, b, jobs, rs);
	a_off[0] = 0;
	for (int32_t k = 0; k < n_win; ++k) a_off[k + 1] = rs.off[(size_t)k + 1], sc[k] = rs.sc[(size_t)k];
	*a = (uint64_t*)malloc(sizeof(uint64_t) * (rs.a.size() + 1));
	if (!rs.a.empty()) memcpy(*a, rs.a.data(), sizeof(uint64_t) * rs.a.size());
	return 0;
}

// stage-level entry for tests: the segmented sort alone (seg_sort.cu), on host keys, in place
int mpb_sort_segments(mpb_ctx_t *c, int32_t n_seg, const int64_t *off, uint64_t *keys)
{
	if (!c || n_seg < 0) return -1;
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	const size_t N = n_seg ? (size_t)off[n_seg] : 0;
	if (N == 0) return 0;
	c->b_c[1].reserve(sizeof(uint64_t) * (N + 2)), c->b_c[2].reserve(sizeof(uint64_t) * (N + 2));
	MPB_CUDA_OK(cudaMemcpyAsync(c->b_c[1].p, keys, sizeof(uint64_t) * N, cudaMemcpyHostToDevice, c->stream));
	seg_sort_u64(c, c->stream, c->b_c[1].as<uint64_t>(), c->b_c[2].as<uint64_t>(), n_seg, off, off + 1);
	MPB_CUDA_OK(cudaMemcpyAsync(keys, c->b_c[1].p, sizeof(uint64_t) * N, cudaMemcpyDeviceToHost, c->stream));
	MPB_CUDA_OK(cudaStreamSynchronize(c->stream));
	MPB_CUDA_OK(cudaGetLastError());
	return 0;
}

void mpb_free(void *p) { free(p); }

// CUDA-event bracket on the context's stream (bench.py times its K steps with these); each context has its own pair of events, on
// its own device
void mpb_event_begin(mpb_ctx_t *c)
{
	std::lock_guard<std::mutex> cl(c->mu);
	MPB_CUDA_OK(cudaSetDevice(c->device));
	MPB_CUDA_OK(cudaStreamSynchronize(c->stream));
	MPB_CUDA_OK(cudaEventRecord(c->ev_bench[0], c->stream));
}
double mpb_event_end_ms(mpb_ctx_t *c)
{
	std::lock_guard<std::mutex> cl(c->mu);
	float ms = 0;
	MPB_CUDA_OK(cudaSetDevice(c->device));
	MPB_CUDA_OK(cudaEventRecord(c->ev_bench[1], c->stream));
	MPB_CUDA_OK(cudaEventSynchronize(c->ev_bench[1]));
	MPB_CUDA_OK(cudaEventElapsedTime(&ms, c->ev_bench[0], c->ev_bench[1]));
	return ms;
}

void ns_global_gs16b(void *, const char *ns, int32_t nl, const char *as, int32_t al, const ns_opt_t *opt, const uint8_t *ss, ns_rst_t *r)
{
	mpb_dp_problem_t p;
	mpb_dp_result_t o;
	p.nt = (const uint8_t*)ns, p.aa = as, p.ss = ss, p.nl = nl, p.al = al, p.flag = opt->flag, p.io = opt->io;
	AnyCtx a;
	if (mpb_nasw_batch(a.c, opt, 1, &p, &o) != 0) abort();
	r->score = o.score, r->nt_len = o.nt_len, r->aa_len = o.aa_len;
	r->n_cigar = r->m_cigar = o.n_cigar, r->cigar = o.cigar;
	if (!(opt->flag & (NS_F_EXT_LEFT | NS_F_EXT_RIGHT))) r->nt_len = nl, r->aa_len = al;
}

void ns_global_gs16(void *km, const char *ns, int32_t nl, const char *as, int32_t al, const ns_opt_t *opt, ns_rst_t *r)
{
	ns_global_gs16b(km, ns, nl, as, al, opt, 0, r);
}

void mpb_get_stats(const mpb_ctx_t *c, mpb_stats_t *st)
{
	std::lock_guard<std::mutex> cl(c->mu);
	*st = c->stats;
}
void mpb_reset_stats(mpb_ctx_t *c)
{
	std::lock_guard<std::mutex> cl(c->mu);
	memset(&c->stats, 0, sizeof(c->stats));
}

} // extern "C"
