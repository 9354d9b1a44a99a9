// index.cpp -- the read-only k-mer index: build (host, one-time), .mpi dump/restore, block lookup.
//
// Data contract (reference miniprot.h:100-106, index.c:11-26,71-95; consumed unchanged by the GPU stages):
//   bo[c*2+s]   first block id of strand s of contig c; a block is 1<<bbit bases; bo[2*n_ctg] = n_block
//   ki[h]       start of bucket h in kb[], h in [0, 2^(4k-mod_bit)); no sentinel: the last bucket ends at n_kb
//   kb[]        block ids; inside a bucket grouped by contig*2+strand in ascending order, ascending within a group
// Index construction (SURVEY 8f #1): the FASTA is read and packed here; ki / kb are built on the GPU (cuda/idx_build.cu) or,
// without a device, on host threads, one task per contig strand like the reference (index.c:52-69,123).  Identical ki/kb either way.
#include <stdio.h>
#include <algorithm>
#include <atomic>
#include <thread>
#include "internal.hpp"

namespace mpb {

void (*g_idx_destroy_hook)(const mp_idx_t *) = 0;
int (*g_idx_build_hook)(mp_idx_t *) = 0; // the device builder (cuda/idx_build.cu), set when the CUDA backend is linked in

uint32_t hash32_mask(uint32_t x, uint32_t mask) // invertible mixer on 4k-bit keys (sketch.c:7-16)
{
	x = (x + ~(x << 15)) & mask;
	x ^= x >> 10;
	x = (x + (x << 3)) & mask;
	x ^= x >> 6;
	x = (x + ~(x << 11)) & mask;
	x ^= x >> 16;
	return x;
}

void sort_u64(uint64_t *beg, uint64_t *end) { std::sort(beg, end); }

void sort_128x(mp128_t *beg, mp128_t *end)
{
	std::vector<FlagRange<mp128_t>> stack(end - beg > 64 ? 8 * 256 + 8 : 1);
	flag_sort_by(beg, end, [](const mp128_t &r) { return r.x; }, stack.data());
}

namespace {

// emit every sampled k-mer of the stop-free codon run [st,en) (sketch.c:40-60)
void emit_orf(const uint8_t *seq, int64_t st, int64_t en, int32_t kmer, int32_t mod_bit, int32_t bbit, int64_t boff, std::vector<uint64_t> &out)
{
	const uint32_t mask = (1U << kmer * 4) - 1, mod = (1U << mod_bit) - 1;
	uint32_t win = 0;
	int32_t have = 0;
	for (int64_t i = st; i < en; i += 3) {
		win = (win << 4 | ns_tab_codon13[seq[i] << 4 | seq[i + 1] << 2 | seq[i + 2]]) & mask;
		if (++have < kmer) continue;
		uint32_t h = hash32_mask(win, mask);
		if ((h & mod) == 0) out.push_back((uint64_t)(h >> mod_bit) << 32 | (uint64_t)(((i + 2) >> bbit) + boff));
	}
}

} // namespace

void sketch_strand(const uint8_t *seq, int64_t len, int32_t min_aa_len, int32_t kmer, int32_t mod_bit, int32_t bbit, int64_t boff,
                   std::vector<uint64_t> &out)
{
	int64_t last_end[3] = { -1, -1, -1 }, n_codon[3] = { 0, 0, 0 };
	uint32_t cod = 0;
	int32_t clean = 0;
	out.clear();
	auto close = [&](int f) {
		if (n_codon[f] >= min_aa_len) emit_orf(seq, last_end[f] + 1 - n_codon[f] * 3, last_end[f] + 1, kmer, mod_bit, bbit, boff, out);
		n_codon[f] = 0, last_end[f] = -1;
	};
	for (int64_t i = 0; i < len; ++i) {
		const int f = (int)((i + 1) % 3);
		if (seq[i] >= 4) { close(0); close(1); close(2); clean = 0, cod = 0; continue; }
		cod = (cod << 2 | seq[i]) & 0x3f;
		if (++clean < 3) continue;
		if (ns_tab_codon[cod] >= 20) close(f);
		else last_end[f] = i, ++n_codon[f];
	}
	close(0); close(1); close(2);
	if (out.size() <= 1) return;
	std::sort(out.begin(), out.end());
	out.erase(std::unique(out.begin(), out.end()), out.end());
}

int32_t idx_block2vid(const mp_idx_t *mi, uint32_t b) // index.c:28-44
{
	const int32_t n = mi->nt->n_ctg * 2;
	if (b >= mi->bo[n]) return -1;
	int32_t lo = 0, hi = n - 1;
	while (lo <= hi) {
		int32_t mid = (lo + hi) / 2;
		if (mi->bo[mid] <= b && b < mi->bo[mid + 1]) return mid;
		if (b < mi->bo[mid]) hi = mid - 1; else lo = mid + 1;
	}
	return -2;
}

static uint32_t *block_offsets(const mp_ntdb_t *db, int32_t bbit, uint32_t *n_block) // index.c:11-26
{
	uint32_t *bo = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(db->n_ctg * 2 + 1));
	int64_t acc = 0;
	for (int32_t i = 0; i < db->n_ctg; ++i) {
		const int64_t nb = (db->ctg[i].len + (1 << bbit) - 1) >> bbit;
		bo[i * 2] = (uint32_t)acc, acc += nb;
		bo[i * 2 + 1] = (uint32_t)acc, acc += nb;
	}
	bo[db->n_ctg * 2] = *n_block = (uint32_t)acc;
	return bo;
}

static mp_idx_t *idx_build(const char *fn, const mp_idxopt_t *io, int32_t n_threads)
{
	mp_ntdb_t *nt = ntdb_read_fasta(fn);
	if (!nt) return 0;
	mp_idx_t *mi = (mp_idx_t*)calloc(1, sizeof(mp_idx_t));
	mi->opt = *io, mi->nt = nt;
	mi->bo = block_offsets(nt, io->bbit, &mi->n_block);
	// the k-mer tables are built on the GPU when there is one (SURVEY 8f #1); the host threads below serve boxes without a device
	// (preparing a .mpi file on a login node) and MPB_IDX_BUILD=host
	if (g_idx_build_hook && g_idx_build_hook(mi) == 0) return mi;
	const int32_t n_task = nt->n_ctg * 2;
	std::vector<std::vector<uint64_t>> sk((size_t)n_task);
	std::atomic<int32_t> next(0);
	auto work = [&]() {
		std::vector<uint8_t> buf;
		for (int32_t j; (j = next.fetch_add(1)) < n_task;) {
			buf.resize((size_t)nt->ctg[j >> 1].len + 1);
			int64_t len = nt_fetch(nt, j >> 1, 0, -1, j & 1, buf.data());
			sketch_strand(buf.data(), len, io->min_aa_len, io->kmer, io->mod_bit, io->bbit, mi->bo[j], sk[(size_t)j]);
		}
	};
	{
		std::vector<std::thread> pool;
		const int32_t nt_use = std::max(1, std::min(n_threads, n_task));
		for (int32_t t = 1; t < nt_use; ++t) pool.emplace_back(work);
		work();
		for (auto &t : pool) t.join();
	}
	// counting sort of (bucket, block) pairs into ki/kb, tasks in order (index.c:71-95)
	const uint32_t n_bucket = idx_n_bucket(io);
	mi->ki = (int64_t*)calloc(n_bucket, sizeof(int64_t));
	for (auto &v : sk) for (uint64_t x : v) ++mi->ki[x >> 32];
	int64_t acc = 0;
	for (uint32_t h = 0; h < n_bucket; ++h) { int64_t c = mi->ki[h]; mi->ki[h] = acc; acc += c; }
	mi->n_kb = acc;
	mi->kb = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(acc ? acc : 1));
	{
		std::vector<int64_t> cur(mi->ki, mi->ki + n_bucket);
		for (auto &v : sk) for (uint64_t x : v) mi->kb[cur[x >> 32]++] = (uint32_t)x;
	}
	if (mp_verbose >= 3)
		fprintf(stderr, "[M::%s@%.3f] %u blocks, %ld kmer-block pairs\n", __func__, mp_realtime(), mi->n_block, (long)mi->n_kb);
	return mi;
}

} // namespace mpb

using namespace mpb;

extern "C" {

void mp_idx_destroy(mp_idx_t *mi)
{
	if (!mi) return;
	if (mpb::g_idx_destroy_hook) mpb::g_idx_destroy_hook(mi); // GPU contexts drop their resident copy of this index
	ntdb_destroy(mi->nt);
	free(mi->ki); free(mi->bo); free(mi->kb);
	free(mi);
}

int mp_idx_dump(const char *fn, const mp_idx_t *mi) // index.c:189-202
{
	if (!mi->ki || !mi->kb) return -1; // an index that was loaded straight into HBM (mpb_idx_load_device) has no host copy of ki / kb
	FILE *fp = strcmp(fn, "-") == 0 ? stdout : fopen(fn, "wb");
	if (!fp) return -1;
	fwrite(MP_IDX_MAGIC, 1, 4, fp);
	fwrite(&mi->opt, sizeof(mi->opt), 1, fp);
	fwrite(&mi->n_kb, 8, 1, fp);
	ntdb_dump(fp, mi->nt);
	fwrite(mi->ki, 8, idx_n_bucket(&mi->opt), fp);
	fwrite(mi->kb, 4, (size_t)mi->n_kb, fp);
	if (fp != stdout) fclose(fp);
	return 0;
}

} // extern "C"

// Head of a .mpi file (index.c:204-220): magic, index options, n_kb and the genome section; on return fp stands at the first
// byte of ki (8 * n_bucket bytes, followed by 4 * n_kb bytes of kb).  The result has no ki / kb yet.
mp_idx_t *mpb::idx_restore_head(FILE *fp)
{
	char magic[4];
	if (fread(magic, 1, 4, fp) != 4 || memcmp(magic, MP_IDX_MAGIC, 4) != 0) return 0;
	mp_idx_t *mi = (mp_idx_t*)calloc(1, sizeof(mp_idx_t));
	bool ok = fread(&mi->opt, sizeof(mi->opt), 1, fp) == 1 && fread(&mi->n_kb, 8, 1, fp) == 1;
	if (ok) {
		ns_make_tables((int)mi->opt.trans_code);
		mi->nt = ntdb_restore(fp);
		ok = mi->nt != 0;
	}
	if (!ok) { mp_idx_destroy(mi); return 0; }
	mi->bo = block_offsets(mi->nt, mi->opt.bbit, &mi->n_block);
	return mi;
}

extern "C" {

mp_idx_t *mp_idx_restore(const char *fn) // index.c:204-229
{
	FILE *fp = strcmp(fn, "-") == 0 ? stdin : fopen(fn, "rb");
	if (!fp) return 0;
	mp_idx_t *mi = idx_restore_head(fp);
	if (!mi) { if (fp != stdin) fclose(fp); return 0; }
	bool ok = true;
	{
		const uint32_t nb = idx_n_bucket(&mi->opt);
		mi->ki = (int64_t*)malloc(sizeof(int64_t) * nb);
		mi->kb = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(mi->n_kb ? mi->n_kb : 1));
		ok = fread(mi->ki, 8, nb, fp) == nb && fread(mi->kb, 4, (size_t)mi->n_kb, fp) == (size_t)mi->n_kb;
	}
	if (fp != stdin) fclose(fp);
	if (!ok) { mp_idx_destroy(mi); return 0; }
	if (mp_verbose >= 3) fprintf(stderr, "[M::%s@%.3f] loaded the index\n", __func__, mp_realtime());
	return mi;
}

mp_idx_t *mp_idx_load(const char *fn, const mp_idxopt_t *io, int32_t n_threads) // index.c:165-187,231-237
{
	if (strcmp(fn, "-") != 0) {
		FILE *fp = fopen(fn, "rb");
		char magic[4];
		if (!fp) return 0;
		size_t got = fread(magic, 1, 4, fp);
		fclose(fp);
		if (got == 4 && memcmp(magic, MP_IDX_MAGIC, 3) == 0 && magic[3] <= MP_IDX_MAGIC[3]) return mp_idx_restore(fn);
	}
	return idx_build(fn, io, n_threads);
}

// An index for locus mode only: the genome, contig table and block offsets of a FASTA (io's options, mp_idxopt_init's without io), or
// the head of a .mpi file (options as stored, io ignored).  No k-mer table is built or read: ki == kb == NULL, n_kb == 0.
mp_idx_t *mpb_idx_load_genome(const char *fn, const mp_idxopt_t *io)
{
	if (!fn) return 0;
	FILE *fp = fopen(fn, "rb");
	if (!fp) return 0;
	char magic[4];
	const size_t got = fread(magic, 1, 4, fp);
	if (got == 4 && memcmp(magic, MP_IDX_MAGIC, 3) == 0 && magic[3] <= MP_IDX_MAGIC[3]) {
		rewind(fp);
		mp_idx_t *mi = idx_restore_head(fp);
		fclose(fp);
		if (mi) mi->n_kb = 0;
		return mi;
	}
	fclose(fp);
	mp_ntdb_t *nt = ntdb_read_fasta(fn);
	if (!nt) return 0;
	mp_idx_t *mi = (mp_idx_t*)calloc(1, sizeof(mp_idx_t));
	if (io) mi->opt = *io;
	else mp_idxopt_init(&mi->opt);
	mi->nt = nt;
	mi->bo = block_offsets(nt, mi->opt.bbit, &mi->n_block);
	return mi;
}

void mp_idx_print_stat(const mp_idx_t *mi, int32_t max_occ) // index.c:138-152
{
	const uint32_t n = idx_n_bucket(&mi->opt);
	int64_t tot = 0, big = 0;
	uint32_t used = 0, n_big = 0;
	for (uint32_t i = 0; i + 1 < n; ++i) {
		int64_t c = mi->ki[i + 1] - mi->ki[i];
		if (c > 0) ++used;
		if (c > max_occ) ++n_big, big += c; else tot += c;
	}
	fprintf(stderr, "[M::%s] %d distinct k-mers; mean occ of infrequent k-mers: %.2f; %d frequent k-mers accounting for %ld occurrences\n",
	        __func__, used, (double)tot / (used - n_big), n_big, (long)big);
}

} // extern "C"
