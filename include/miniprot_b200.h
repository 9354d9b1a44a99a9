/*
 * miniprot_b200.h -- C ABI of libminiprot_b200.so, the H100-native protein-to-genome mapping
 * hot path.  Two groups of entry points:
 *
 * (1) mp_*  : drop-in replacements for the reference library API (reference miniprot.h:148-286).
 *             A program compiled against the reference's miniprot.h (e.g. its main.c) links
 *             against this library unchanged; struct layouts below are ABI and mirror the
 *             reference field for field (miniprot.h:32-143).
 * (2) mpb_* : the batch interface the reference's per-query worker (map.c:264 worker_for ->
 *             map.c:143 mp_map) is replaced by: one call maps a whole mini-batch of proteins
 *             through GPU stages (seed+lookup, chaining, refinement, nasw DP waves).
 *
 * All compute stages run as hand-written sm_90a CUDA kernels; there is NO CPU fallback.
 * Without a usable CUDA device mpb_ctx_create() returns NULL and mp_map()/mp_map_file() abort.
 */
#ifndef MINIPROT_B200_H
#define MINIPROT_B200_H

#include <stdint.h>
#include <stdio.h>
#include "nasw_b200.h"

#define MPB_VERSION "0.1-b200 (API of miniprot 0.18-r281)"

/* mp_mapopt_t::flag bits (reference miniprot.h:8-17) */
#define MP_F_NO_SPLICE    0x1
#define MP_F_NO_ALIGN     0x2
#define MP_F_SHOW_UNMAP   0x4
#define MP_F_GFF          0x8
#define MP_F_NO_PAF       0x10
#define MP_F_GTF          0x20
#define MP_F_NO_PRE_CHAIN 0x40
#define MP_F_SHOW_RESIDUE 0x80
#define MP_F_SHOW_TRANS   0x100
#define MP_F_NO_CS        0x200

/* mp_dbg_flag bits, set by the CLI's debugging switches (reference mppriv.h:9-14, main.c:162-167); read once per mapping call */
#define MP_DBG_NO_KALLOC   0x1  /* --no-kalloc: allocator choice of the reference; nothing to do here */
#define MP_DBG_QNAME       0x2  /* --dbg-qname: "QR\tname\tlen\ttid" on stderr before each protein (file and batch calls, not mp_map) */
#define MP_DBG_NO_REFINE   0x4  /* --dbg-no-refine: no second-round refinement; needs MP_F_NO_ALIGN (-A), refused (-3) without */
#define MP_DBG_MORE_DP     0x8  /* --dbg-aflt: no seed filter, one global DP over the whole region instead of fills between anchors */
#define MP_DBG_ANCHOR      0x10 /* --dbg-anchor: "X" lines, every seed anchor of the protein, on stderr */
#define MP_DBG_CHAIN       0x20 /* --dbg-chain: "Y1" lines, the anchors of every first-round region, on stderr */

#define MP_FEAT_CDS  0
#define MP_FEAT_STOP 1
#define MP_IDX_MAGIC "MPI\3"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- ABI structs ---------- */

typedef struct { uint64_t x, y; } mp128_t;                     /* miniprot.h:32 */
typedef struct { int32_t n, m; uint64_t *a; } mp64_v;          /* miniprot.h:34 */

typedef struct {                                               /* miniprot.h:36-41 */
	int32_t bbit;       /* log2 of the genome block size (8 => 256 bp blocks) */
	int32_t min_aa_len; /* ORFs shorter than this are not indexed */
	int32_t kmer, mod_bit;
	uint32_t trans_code;
} mp_idxopt_t;

typedef struct {                                               /* miniprot.h:43-77 */
	uint32_t flag;
	int64_t mini_batch_size;
	int32_t max_occ;
	int32_t max_gap;
	int32_t max_intron;
	int32_t min_max_intron, max_max_intron;
	int32_t bw;
	int32_t max_ext;
	int32_t max_ava;
	int32_t min_chn_cnt;
	int32_t max_chn_max_skip;
	int32_t max_chn_iter;
	int32_t min_chn_sc;
	float chn_coef_log;
	float mask_level;
	int32_t mask_len;
	float pri_ratio;
	float out_sim, out_cov;
	int32_t best_n, out_n;
	int32_t kmer2;
	int32_t go, ge, io, fs;
	int32_t io_end;
	float ie_coef;
	int32_t sp_model;
	int32_t sp_null_bonus, sp_max_bonus;
	float sp_scale;
	int32_t xdrop;
	int32_t end_bonus;
	int32_t asize;
	int32_t gff_delim;
	int32_t max_intron_flank;
	const char *gff_prefix;
	int8_t mat[484];
} mp_mapopt_t;

typedef struct { uint32_t n, m; uint64_t *a; } mp_spsc_t;      /* miniprot.h:79-82 */
typedef struct { int64_t off, len; char *name; } mp_ctg_t;     /* miniprot.h:84-87 */

typedef struct {                                               /* miniprot.h:89-98 */
	int32_t n_ctg, m_ctg;
	int32_t l_name;
	int64_t l_seq, m_seq;
	uint8_t *seq;   /* 4 bits per base, low nibble = even offset */
	mp_ctg_t *ctg;
	char *name;
	void *h;
	mp_spsc_t *spsc;
} mp_ntdb_t;

typedef struct {                                               /* miniprot.h:100-106 */
	mp_idxopt_t opt;
	uint32_t n_block;
	mp_ntdb_t *nt;
	int64_t n_kb, *ki;  /* ki[bucket] = start of the bucket in kb[]; no sentinel */
	uint32_t *bo, *kb;  /* bo[ctg*2+strand] = first block id; kb[] = block ids */
} mp_idx_t;

typedef struct {                                               /* miniprot.h:108-118 */
	int32_t dp_score, dp_max, dp_max2;
	int32_t n_cigar, m_cigar;
	int32_t blen;
	int32_t n_fs;
	int32_t n_stop;
	int32_t dist_stop;
	int32_t dist_start;
	int32_t n_iden, n_plus;
	uint32_t cigar[];
} mp_extra_t;

typedef struct {                                               /* miniprot.h:120-127 */
	int64_t vs, ve;
	int32_t qs, qe;
	int16_t type, phase;
	int32_t n_fs, n_stop;
	int32_t score, n_iden, blen;
	char donor[2], acceptor[2];
} mp_feat_t;

typedef struct {                                               /* miniprot.h:129-143 */
	int32_t off, cnt;
	int32_t id, parent;
	int32_t n_sub, subsc;
	int32_t n_feat, m_feat, n_exon;
	int32_t chn_sc;
	int32_t chn_sc_ungap;
	uint32_t hash;
	uint32_t vid;      /* contig<<1 | strand */
	int32_t qs, qe;
	int64_t vs, ve;    /* on the strand given by vid */
	uint64_t *a;       /* NOT valid after mp_map()/mpb_map_batch() return */
	mp_feat_t *feat;   /* malloc'ed; caller frees */
	mp_extra_t *p;     /* malloc'ed; caller frees */
} mp_reg1_t;

struct mp_tbuf_s;
typedef struct mp_tbuf_s mp_tbuf_t;

extern int32_t mp_verbose, mp_dbg_flag;

/* ------------------------------------------- (1) reference-compatible entry points ------ */

void mp_start(void);                                                    /* miniprot.h:158 (misc.c:12)     */
void mp_idxopt_init(mp_idxopt_t *io);                                   /* miniprot.h:165 (options.c:10)  */
void mp_mapopt_init(mp_mapopt_t *mo);                                   /* miniprot.h:172 (options.c:42)  */
void mp_mapopt_set_fs(mp_mapopt_t *mo, int32_t fs);                     /* miniprot.h:182 (options.c:24)  */
void mp_mapopt_set_max_intron(mp_mapopt_t *mo, int64_t gsize);          /* miniprot.h:190 (options.c:31)  */
int32_t mp_mapopt_check(const mp_mapopt_t *mo);                         /* miniprot.h:199 (options.c:92)  */
mp_idx_t *mp_idx_load(const char *fn, const mp_idxopt_t *io, int32_t n_threads); /* miniprot.h:214 (index.c:231) */
void mp_idx_destroy(mp_idx_t *mi);                                      /* miniprot.h:221 (index.c:154)   */
int mp_idx_dump(const char *fn, const mp_idx_t *mi);                    /* miniprot.h:231 (index.c:189)   */
mp_idx_t *mp_idx_restore(const char *fn);                               /* miniprot.h:240 (index.c:204)   */
void mp_idx_print_stat(const mp_idx_t *mi, int32_t max_occ);            /* miniprot.h:285 (index.c:138)   */
mp_tbuf_t *mp_tbuf_init(void);                                          /* miniprot.h:275 (map.c:16)      */
void mp_tbuf_destroy(mp_tbuf_t *b);                                     /* miniprot.h:282 (map.c:25)      */
/* Map one protein: a GPU batch of one.  Return value and r->p / r->feat are malloc'ed (caller frees).  Safe to call from several
 * threads at once, as the reference's worker threads do: without MPB_DEVICES the calls take turns on the default context; with
 * MPB_DEVICES each call takes an idle context of that pool (and waits while all are busy).  ns_global_gs16b does the same. */
mp_reg1_t *mp_map(const mp_idx_t *mi, int qlen, const char *seq, int *n_reg, mp_tbuf_t *b,
                  const mp_mapopt_t *opt, const char *qname);           /* miniprot.h:268 (map.c:143)     */
/* Read FASTA proteins from fn, map them in mini-batches on the GPU, write PAF/GFF to stdout in input order.  n_threads is not
 * used.  MPB_DEVICES=<device>[,<device>...] (read once; repeats allowed, "0,0" = two contexts on device 0) maps the file over one
 * context per entry (mpb_map_file_multi); the output is the same byte for byte. */
int32_t mp_map_file(const mp_idx_t *idx, const char *fn, const mp_mapopt_t *opt, int n_threads); /* miniprot.h:286 (map.c:330) */
double mp_realtime(void);                                               /* mppriv.h:47 (sys.c:93)  */
double mp_cputime(void);                                                /* mppriv.h:48 (sys.c:107) */
long mp_peakrss(void);                                                  /* mppriv.h:49 (sys.c:116) */
/* --spsc splice-score input (SURVEY 8f #4; ntseq.c:234-296, index.c:239-248): the score file is read into mi->nt->spsc
 * (sorted per contig and strand, as the reference keeps them); the mapping context scatters it into a dense per-base table in
 * HBM on first use and the DP prep kernels apply nasw-sse.c:138-152,189-203. */
int32_t mp_ntseq_read_spsc(mp_ntdb_t *nt, const char *fn, int32_t max_sc);  /* miniprot.h:251 */
void mp_set_spsc(const char *fn, mp_idx_t *mi, mp_mapopt_t *mo, int32_t keep_io); /* miniprot.h:253 */

/* ------------------------------------------- (2) GPU batch interface -------------------- */

typedef struct mpb_ctx_s mpb_ctx_t; /* stream, device arenas, resident index; several may share one GPU */

/* Create the context on CUDA device `device` and keep the calling thread on the device's NUMA node (MPB_AFFINITY=0: leave it).
 * NULL (with a message on stderr) if there is no device.  Every mpb_* call that uses a context holds the context's mutex, so
 * calls on one context from several threads take turns; calls on different contexts run concurrently. */
mpb_ctx_t *mpb_ctx_create(int device);
void mpb_ctx_destroy(mpb_ctx_t *ctx);
/* Process-wide default context used by mp_map()/mp_map_file()/ns_global_gs16b(); created on first use, on device LOCAL_RANK (or 0),
 * or on the first device of MPB_DEVICES when that is set (context 0 of the pool). */
mpb_ctx_t *mpb_ctx_default(void);

/* Make the read-only index resident in HBM (ki, kb, bo, 4-bit genome, contig table). */
int mpb_idx_upload(mpb_ctx_t *ctx, const mp_idx_t *mi);
/* Restore a .mpi index straight into HBM: the k-mer tables are streamed from the file through pinned staging buffers and
 * never materialise on the host (the returned index has ki == kb == NULL; the genome section is kept on the host too).
 * Replaces mp_idx_restore (index.c:204) + mpb_idx_upload for a process that only maps.  NULL on failure. */
mp_idx_t *mpb_idx_load_device(mpb_ctx_t *ctx, const char *fn);
/* Host part of a .mpi file only (options, contig table, block offsets, genome): for the ranks whose k-mer tables arrive by
 * broadcast (mpb_idx_attach_device).  mpb_idx_device_ptrs: where a context keeps its resident index (broadcast source). */
mp_idx_t *mpb_idx_load_meta(const char *fn);
int mpb_idx_device_ptrs(mpb_ctx_t *ctx, void **d_ki, void **d_kb, void **d_seq);
/* Multi-GPU: adopt device buffers that were filled by an NCCL broadcast from rank 0 instead of
 * uploading from the host (sizes: ki 8*n_bucket, kb 4*n_kb, seq (l_seq+1)/2 bytes). The host-side
 * mp_idx_t must still carry nt->ctg[], bo[], n_kb and opt (small metadata). */
int mpb_idx_attach_device(mpb_ctx_t *ctx, const mp_idx_t *mi_meta, void *d_ki, void *d_kb, void *d_seq);
/* Make the index resident in `src` resident in `dst` too; 0, or -1 when src holds none.  On one device dst adopts src's k-mer
 * tables and genome (nothing is copied); on another device they are copied device to device.  An index loaded with
 * mpb_idx_load_device reaches other contexts this way (the mapping calls do it themselves when another context holds the index).
 * A context that adopted must not be in use while the owner of the buffers is destroyed or replaces its index; when that
 * happens the adopter forgets the index (and shares or uploads it again on its next call). */
int mpb_idx_share(mpb_ctx_t *dst, mpb_ctx_t *src);

/* Replacement for the reference's kt_for(worker_for) step (map.c:291): map n_seq proteins.
 * reg_out[i] / n_reg_out[i] receive what mp_map() would have returned for protein i.
 * Returns 0; -1 without a context; -3 (with a message on stderr, nothing mapped) for scoring parameters whose reference
 * result cannot be reproduced bit for bit: a gap open penalty below 1 (with -O 0 the reference's lazy-F loop stops at once,
 * nasw-sse.c:411,530, and its scores depend on the SSE stripe layout) or an ie_coef whose length penalty has more steps
 * than the kernels' table (> ~5); or an index built with a minimum ORF length (-L) above 40, which the tile halos of the
 * window kernels do not cover.  mpb_map_file() and mpb_nasw_batch() apply the same checks, and mpb_refine_batch() the
 * index check. */
int mpb_map_batch(mpb_ctx_t *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq,
                  const char *const *seqs, const int32_t *lens, const char *const *names,
                  int32_t *n_reg_out, mp_reg1_t **reg_out);

/* Locus mode: align proteins to genomic loci the caller already knows (lifting gene models over, re-aligning the hits of a
 * translated search, checking annotated loci).  Pair k is protein seqs[loci[k].qid] against [st, en) of contig cid, both strands.
 * reg_out[k] / n_reg_out[k] receive what the reference reports when that locus alone is the genome (its index built with mi->opt,
 * the mapping options as given; -I is not applied, opt->max_intron is used as it is), secondary hits included, moved to the
 * coordinates of the real genome: vid = cid<<1|rev, and vs / ve and every feat[].vs / ve gain st on the + strand, len(cid) - en
 * on the - strand.  mpb_format_paf() with mi then prints the reference's PAF line for the locus, with the contig's name and
 * length in columns 6-7 and start and end moved by st.  Free the regions with mpb_regs_free(n_loci, ...).
 * mi needs its genome only (an index from mpb_idx_load_meta will do): the loci are seeded without a k-mer table.  A context that
 * holds mi resident uploads nothing of it; otherwise only the packed genome and the contig table are uploaded.
 * Returns 0; -1 (nothing mapped) for a null context or a malformed locus: qid or cid out of range, st < 0, en > len(cid) or
 * st >= en; -3 (with a message, nothing mapped) for what mpb_map_batch() refuses, an index with --spsc scores, or any
 * mp_dbg_flag bit other than MP_DBG_NO_KALLOC. */
typedef struct { int32_t qid, cid; int64_t st, en; } mpb_locus_t;
int mpb_map_loci(mpb_ctx_t *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs,
                 const int32_t *lens, const char *const *names, int32_t n_loci, const mpb_locus_t *loci,
                 int32_t *n_reg_out, mp_reg1_t **reg_out);

/* An index for locus mode only, from a FASTA or FASTA.gz file (genome, contig table and block offsets as mp_idx_load() sets them,
 * with the options io, or mp_idxopt_init()'s when io is NULL) or from a .mpi file (its head, as mpb_idx_load_meta(); io is ignored).
 * Nothing of a k-mer table is built, read or uploaded: ki == kb == NULL, n_kb == 0.  Enough for mpb_map_loci() and
 * mpb_map_loci_file*(), not for whole-genome mapping.  Free with mp_idx_destroy().  NULL if the file cannot be read. */
mp_idx_t *mpb_idx_load_genome(const char *fn, const mp_idxopt_t *io);

/* Locus mode over files: proteins from prot_fn (FASTA, gzip allowed, read whole; a repeated name stands for its last record), pairs
 * from loci_fn, a TSV of `protein contig start end` (0-based, end exclusive; blank lines and lines starting with '#' skipped).  For
 * every pair, in file order, writes what the reference CLI prints with the same options when that locus alone is the genome --
 * PAF with or without cs, --gff / --gff-only / --gtf, --aln, --trans, -P, --gff-delim, --max-intron-out, -u, --outn / --outs /
 * --outc applied per pair -- moved to the real contig: its name and length in PAF columns 6-7 (and in the ##PAF lines), start and
 * end moved by st in PAF columns 8-9 and GFF / GTF columns 4-5, the contig's name in GFF / GTF column 1.  The output as a whole is
 * one file: "##gff-version 3" once at the top with --gff, and one counter numbers the ids of all pairs.  Genome bases past a locus
 * end are never read (--aln's codon after a hit is clipped there, as in the reference given the locus alone).
 * Everything is validated before anything is written.  Returns 0; -1 (with "file:line: why" on stderr) for an unreadable file, a
 * malformed line, an unknown protein or contig or a range outside 0 <= start < end <= contig length, and for a null, missing or
 * repeated context; -3 (with a message) for what mpb_map_loci() refuses; -2 when out_path cannot be created.
 * _multi: over n_ctx distinct contexts as mpb_map_file_multi() (units of at most mini_batch_size / n_ctx residues, one mapper thread
 * per context, written in input order); the output is the same byte for byte for any n_ctx and mini_batch_size.  The genome is made
 * resident in every context (the packed genome and the contig table only, unless the context holds the whole index). */
int32_t mpb_map_loci_file(mpb_ctx_t *ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, FILE *out);
int32_t mpb_map_loci_file_path(mpb_ctx_t *ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt, const char *out_path);
int32_t mpb_map_loci_file_multi(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn, const mp_mapopt_t *opt,
                                FILE *out);
int32_t mpb_map_loci_file_multi_path(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *prot_fn, const char *loci_fn,
                                     const mp_mapopt_t *opt, const char *out_path);

/* mp_map_file() with an explicit output stream and context (tests, benchmarks).  The index is made resident in the context before
 * anything is mapped: shared from another context that holds it, else uploaded from its host tables.  Returns 0; -1 for a null
 * context, an unreadable input, or an index that has no host tables (mpb_idx_load_device) and is held by no context (with a
 * message); -3 (with a message) for refused options.  mpb_map_file_multi(&ctx, 1, ...). */
int32_t mpb_map_file(mpb_ctx_t *ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out);
/* mpb_map_file() over n_ctx distinct contexts (on one or several GPUs) at once: the input is cut into units of at most
 * mini_batch_size / n_ctx residues, each context maps the next unit on a thread of its own, and the output is written in input
 * order -- byte for byte what mpb_map_file() writes.  The index is made resident in every context first (shared from one that holds
 * it, else uploaded).  Returns what mpb_map_file() returns; -1 also for a repeated or null context. */
int32_t mpb_map_file_multi(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, FILE *out);
int32_t mpb_map_file_multi_path(mpb_ctx_t *const *ctx, int32_t n_ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, const char *out_path);
/* Format one hit exactly like the reference's PAF writer (format.c:333); appends to a malloc'ed buffer. */
int64_t mpb_format_paf(const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen,
                       const char *qseq, const mp_reg1_t *r, char **buf, int64_t *len, int64_t *cap);

/* ---- stage-level batch entry points (each is one GPU stage; HOST buffers in and out) ---- */

typedef struct {
	const uint8_t *nt; /* nl nucleotide codes 0..4 (or ASCII) */
	const char *aa;    /* al residues, ASCII */
	const uint8_t *ss; /* optional per-base splice bytes, or NULL */
	int32_t nl, al;
	int32_t flag;      /* NS_F_CIGAR | NS_F_EXT_LEFT | NS_F_EXT_RIGHT */
	int32_t io;        /* intron-open penalty for this problem (mp_align retries with io_end) */
} mpb_dp_problem_t;

typedef struct {
	int32_t score, nt_len, aa_len;
	int32_t n_cigar;
	uint32_t *cigar;   /* malloc'ed when n_cigar > 0; caller frees */
} mpb_dp_result_t;

/* nasw DP over a batch (replaces n calls of ns_global_gs16b, nasw-sse.c:340). opt->flag/io are
 * taken per problem; everything else from *opt. */
int mpb_nasw_batch(mpb_ctx_t *ctx, const ns_opt_t *opt, int32_t n, const mpb_dp_problem_t *prob, mpb_dp_result_t *rst);

typedef struct {
	int32_t max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float chn_coef_log;
	int32_t is_spliced, kmer, bbit;
} mpb_chain_par_t;

/* Anchor chaining over a batch (replaces n calls of mp_chain, chain.c:160).  a_off[n+1] delimits the
 * sorted anchors of each problem inside a[].  On return u_off[n+1] / u[] hold the chains (score<<32|cnt)
 * and b_off[n+1] / b[] the compacted anchors; u and b are malloc'ed. */
int mpb_chain_batch(mpb_ctx_t *ctx, const mpb_chain_par_t *par, int32_t n, const int64_t *a_off, const uint64_t *a,
                    int64_t *u_off, uint64_t **u, int64_t *b_off, uint64_t **b);

/* Protein sketch + index lookup + anchor sort for a batch (replaces map.c:155-177 per query).
 * On return a_off[n+1] / *a hold each query's sorted anchors (block<<32|qpos); *a is malloc'ed. */
int mpb_seed_batch(mpb_ctx_t *ctx, const mp_idx_t *mi, int32_t max_occ, int32_t n_seq, const char *const *seqs,
                   const int32_t *lens, int64_t *a_off, uint64_t **a);

/* The seeding of locus mode alone (mpb_map_loci): a_off[n_loci+1] / *a hold each pair's sorted, max_occ-filtered anchors
 * (block<<32|qpos), the blocks numbered as in an index of the locus alone (the - strand's from ceil(len / 2^bbit)); *a is
 * malloc'ed.  Returns 0; -1 as mpb_map_loci(); -3 (with a message) for an index mpb_map_batch() refuses, --spsc scores or
 * debugging bits as mpb_map_loci(). */
int mpb_seed_loci_batch(mpb_ctx_t *ctx, const mp_idx_t *mi, int32_t max_occ, int32_t n_seq, const char *const *seqs,
                        const int32_t *lens, int32_t n_loci, const mpb_locus_t *loci, int64_t *a_off, uint64_t **a);

/* Second-round refinement over a batch of windows (replaces map.c:41-97 per region): window k is [as, ae) on strand
 * vid = contig<<1|rev of query qid.  On return a_off[n_win+1] / *a hold the best chain of each window
 * (window-relative nt end position<<32 | residue end position; empty = no chain) and sc[n_win] its score; *a is malloc'ed.
 * Returns 0; -1 for a bad argument; -3 (with a message on stderr) for an index with a minimum ORF length above 40. */
typedef struct { int32_t qid; uint32_t vid; int64_t as, ae; } mpb_window_t;
int mpb_refine_batch(mpb_ctx_t *ctx, const mp_idx_t *mi, const mp_mapopt_t *opt, int32_t n_seq, const char *const *seqs, const int32_t *lens,
                     int32_t n_win, const mpb_window_t *win, int64_t *a_off, uint64_t **a, int32_t *sc);

/* The segmented sort of the seeding / refinement stages alone: keys[off[s] .. off[s+1]) sorted ascending for every s, in place. */
int mpb_sort_segments(mpb_ctx_t *ctx, int32_t n_seg, const int64_t *off, uint64_t *keys);

void mpb_free(void *p);                                   /* free() for buffers this library malloc'ed */
void mpb_regs_free(int32_t n, const int32_t *n_reg, mp_reg1_t **reg); /* free what mpb_map_batch returned */
int32_t mpb_map_file_path(mpb_ctx_t *ctx, const mp_idx_t *mi, const char *fn, const mp_mapopt_t *opt, const char *out_path);
void mpb_event_begin(mpb_ctx_t *ctx);                     /* CUDA-event bracket on the context's stream */
double mpb_event_end_ms(mpb_ctx_t *ctx);

/* Measured integer-issue peak of the device (SURVEY 8d): variant 0 = 32-bit fused add-max, 1 = 32-bit three-way max, 2 = packed
 * int16x2 add-max, 3 = packed int16x2 three-way max, 4 = packed add-max with the zero floor.  Outputs: thread-level instructions
 * per second and elementary integer operations per second (an add-max or three-way max = 2, packed forms = 4). */
int mpb_int_peak(mpb_ctx_t *ctx, int variant, double *thread_instr_per_s, double *int_ops_per_s);

/* counters since context creation (for bench.py): */
typedef struct {
	int64_t dp_cells_ext, dp_cells_tb; /* sum nl*al over executed DP problems */
	int64_t n_dp_ext, n_dp_tb;
	int64_t n_anchors, n_chain_problems, n_refine_regions;
	int64_t kernel_launches;
	int64_t h2d_bytes, d2h_bytes;
	double ms_seed, ms_chain, ms_refine, ms_dp_ext, ms_dp_tb; /* CUDA-event time per stage (kernels of one stage may overlap) */
	double ms_wall[6]; /* host wall clock per dispatcher phase: S1, H1, S2, H2, S3 (three DP waves incl. their host steps), H3 */
	/* nasw kernels by class: [0] score-only extension, [1] global alignment with traceback; classes 0..3 = block-wide
	 * wavefront kernels with 1 / 2 / 4 / 8 warps per problem, 4..8 = the column-pass family, 9..12 = pair-lane kernels with
	 * 1 / 2 / 4 / 8 warps per problem.  ms = CUDA-event time of the
	 * DP kernel alone on its own stream (classes of one wave overlap in time), cells = sum nl*al, n = launches. */
	double ms_class[2][16];
	int64_t cells_class[2][16], n_class[2][16];
	double ms_bt;      /* CIGAR backtrack kernels */
	double ms_dp_wave; /* device wall time of the DP waves: fork of the class streams -> last join */
	double ms_prep;    /* row preparation kernels */
} mpb_stats_t;
void mpb_get_stats(const mpb_ctx_t *ctx, mpb_stats_t *st);
void mpb_reset_stats(mpb_ctx_t *ctx);

#ifdef __cplusplus
}
#endif
#endif
