// annot.cpp -- the reference's other output formats, byte-compatible: GFF3 (format.c:360), GTF (format.c:414), and the
// residue-level alignment / translation blocks of --aln and --trans (format.c:189).  Host formatting of what the GPU
// stages produced (SURVEY 8f #2): everything is derived from r->p (CIGAR + statistics), r->feat (one record per exon
// and the stop codon, align.cpp fill_statistics) and the packed genome.
#include <ctype.h>
#include <stdio.h>
#include <string>
#include "internal.hpp"

namespace mpb {

static inline uint8_t codon_aa(uint8_t n1, uint8_t n2, uint8_t n3)
{
	return (n1 > 3 || n2 > 3 || n3 > 3) ? ns_tab_aa20[(uint8_t)'X'] : ns_tab_codon[n1 << 4 | n2 << 2 | n3];
}

static void put_ratio4(Str &o, double x) // "%.4f"
{
	char dec[32];
	snprintf(dec, sizeof(dec), "%.4f", x);
	o.puts(dec);
}

// "<prefix><6-digit id>" (format.c:377) or "<query name><delim><hit rank>" with --gff-delim (format.c:373)
static std::string hit_id(const mp_mapopt_t *opt, const char *qname, int64_t id, int32_t hit_idx, const char *infix)
{
	char num[40];
	if (infix[0] == 0 && opt->gff_delim >= 33 && opt->gff_delim <= 126 && hit_idx >= 0) {
		snprintf(num, sizeof(num), "%c%d", (char)opt->gff_delim, hit_idx);
		return std::string(qname) + num;
	}
	snprintf(num, sizeof(num), "%.6ld", (long)id);
	return std::string(opt->gff_prefix ? opt->gff_prefix : "MP") + infix + num;
}

// mRNA line + one line per feature; coordinates 1-based inclusive on the forward strand; in GFF3 the last CDS includes the
// stop codon (format.c:390-392)
void format_gff(Str &o, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const mp_reg1_t *r, int64_t id, int32_t hit_idx)
{
	if (!r || !r->p) return;
	const mp_ctg_t *c = &mi->nt->ctg[r->vid >> 1];
	const bool rev = r->vid & 1, has_stop = r->qe == qlen && r->p->dist_stop == 0;
	const int64_t ve_mrna = has_stop ? r->ve + 3 : r->ve;
	const std::string ids = hit_id(opt, qname, id, hit_idx, "");
	const char strand = "+-"[r->vid & 1];
	auto span = [&](int64_t vs, int64_t ve) { // strand coordinates [vs, ve) -> "start\tend" on the contig
		o.puti((rev ? c->len - ve : vs) + 1), o.putc('\t'), o.puti(rev ? c->len - vs : ve);
	};
	o.puts(c->name), o.puts("\tminiprot\tmRNA\t"), span(r->vs, ve_mrna), o.putc('\t'), o.puti(r->p->dp_max), o.putc('\t'), o.putc(strand);
	o.puts("\t.\tID="), o.puts(ids.c_str()), o.puts(";Rank="), o.puti(hit_idx);
	o.puts(";Identity="), put_ratio4(o, (double)r->p->n_iden * 3 / r->p->blen);
	o.puts(";Positive="), put_ratio4(o, (double)r->p->n_plus * 3 / r->p->blen);
	if (r->p->n_fs > 0) o.puts(";Frameshift="), o.puti(r->p->n_fs);
	if (r->p->n_stop > 0) o.puts(";StopCodon="), o.puti(r->p->n_stop);
	o.puts(";Target="), o.puts(qname), o.putc(' '), o.puti(r->qs + 1), o.putc(' '), o.puti(r->qe), o.putc('\n');
	for (int32_t j = 0; j < r->n_feat; ++j) {
		const mp_feat_t *f = &r->feat[j];
		int64_t ve = f->ve;
		if (has_stop && f->type == MP_FEAT_CDS && j + 1 < r->n_feat && r->feat[j + 1].type == MP_FEAT_STOP) ve += 3;
		o.puts(c->name), o.puts("\tminiprot\t"), o.puts(f->type == MP_FEAT_STOP ? "stop_codon" : "CDS"), o.putc('\t'), span(f->vs, ve);
		o.putc('\t'), o.puti(f->score), o.putc('\t'), o.putc(strand), o.putc('\t'), o.puti(f->phase);
		o.puts("\tParent="), o.puts(ids.c_str()), o.puts(";Rank="), o.puti(hit_idx);
		if (f->type == MP_FEAT_CDS) {
			o.puts(";Identity="), put_ratio4(o, (double)f->n_iden * 3 / f->blen);
			if (f->acceptor[0] && !(f->acceptor[0] == 'A' && f->acceptor[1] == 'G')) o.puts(";Acceptor="), o.putc(f->acceptor[0]), o.putc(f->acceptor[1]);
			if (f->donor[0] && !(f->donor[0] == 'G' && f->donor[1] == 'T')) o.puts(";Donor="), o.putc(f->donor[0]), o.putc(f->donor[1]);
			if (f->n_fs > 0) o.puts(";Frameshift="), o.puti(f->n_fs);
			if (f->n_stop > 0) o.puts(";StopCodon="), o.puti(f->n_stop);
			o.puts(";Target="), o.puts(qname), o.putc(' '), o.puti(f->qs + 1), o.putc(' '), o.puti(f->qe);
		}
		o.putc('\n');
	}
}

// gene + transcript + (exon, CDS) per coding exon; the exon line of the last exon includes the stop codon, the CDS line does not
void format_gtf(Str &o, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const mp_reg1_t *r, int64_t id)
{
	if (!r || !r->p) return;
	const mp_ctg_t *c = &mi->nt->ctg[r->vid >> 1];
	const bool rev = r->vid & 1, has_stop = r->qe == qlen && r->p->dist_stop == 0;
	const int64_t ve_mrna = has_stop ? r->ve + 3 : r->ve;
	const std::string gid = hit_id(opt, qname, id, -1, "G"), tid = hit_id(opt, qname, id, -1, "T");
	const char strand = "+-"[r->vid & 1];
	auto head = [&](const char *what, int64_t vs, int64_t ve, int32_t score) {
		o.puts(c->name), o.puts("\tminiprot\t"), o.puts(what), o.putc('\t'), o.puti((rev ? c->len - ve : vs) + 1), o.putc('\t'), o.puti(rev ? c->len - vs : ve);
		o.putc('\t'), o.puti(score), o.putc('\t'), o.putc(strand), o.putc('\t');
	};
	auto ids = [&]() { o.puts("transcript_id \""), o.puts(tid.c_str()), o.puts("\"; gene_id \""), o.puts(gid.c_str()), o.puts("\";\n"); };
	head("gene", r->vs, ve_mrna, r->p->dp_max), o.puts(".\tgene_id \""), o.puts(gid.c_str()), o.puts("\";\n");
	head("transcript", r->vs, ve_mrna, r->p->dp_max), o.puts(".\t"), ids();
	for (int32_t j = 0; j < r->n_feat; ++j) {
		const mp_feat_t *f = &r->feat[j];
		if (f->type != MP_FEAT_CDS) continue;
		head("exon", f->vs, f->ve == r->ve ? ve_mrna : f->ve, f->score), o.puts(".\t"), ids();
		head("CDS", f->vs, f->ve, f->score), o.puti(f->phase), o.putc('\t'), ids();
	}
}

// --aln / --trans (format.c:189-331): four aligned text rows (genome bases, their translation, match line, protein residues:
// "##ATN", "##ATA", "##AAS", "##AQA") and the translated protein ("##STA"); long introns are abbreviated to their flanks.
// The one read of the genome past the hit: the codon after r->ve (format.c:219), clipped at the contig end or at nt_lim (>= 0).
void format_residue(Str &o, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qseq, const mp_reg1_t *r, int64_t nt_lim)
{
	static const char UC[] = "ACGTN", LC[] = "acgtn";
	const mp_extra_t *e = r->p;
	if (!e) return;
	const int32_t max_flank = opt->max_intron_flank;
	std::vector<uint8_t> nt((size_t)(r->ve - r->vs + 3));
	const int64_t l_nt = nt_fetch_v(mi->nt, r->vid, r->vs, nt_lim >= 0 && nt_lim < r->ve + 3 ? nt_lim : r->ve + 3, nt.data());
	std::string atn = "##ATN\t", ata = "##ATA\t", aas = "##AAS\t", aqa = "##AQA\t", sta = "##STA\t";
	auto col = [&](char a, char b, char c, char d) { atn += a, ata += b, aas += c, aqa += d; };
	auto codon_cols = [&](int32_t i, char match, char res, bool translate) { // three columns of one genome codon
		const uint8_t na = codon_aa(nt[(size_t)i], nt[(size_t)i + 1], nt[(size_t)i + 2]);
		if (translate) sta += ns_tab_aa_i2c[na];
		col(UC[nt[(size_t)i]], ns_tab_aa_i2c[na], match, res), col(UC[nt[(size_t)i + 1]], '.', ' ', ' '), col(UC[nt[(size_t)i + 2]], '.', ' ', ' ');
	};
	int32_t al = r->qs, nl = 0;
	for (int32_t k = 0; k < e->n_cigar; ++k) {
		const int32_t op = (int32_t)(e->cigar[k] & 0xf), len = (int32_t)(e->cigar[k] >> 4);
		if (op == NS_CIGAR_M) {
			for (int32_t l = 0; l < len; ++l) {
				const int32_t i = nl + l * 3;
				const uint8_t na = codon_aa(nt[(size_t)i], nt[(size_t)i + 1], nt[(size_t)i + 2]), qa = ns_tab_aa20[(uint8_t)qseq[al + l]];
				codon_cols(i, na == qa ? '|' : opt->mat[na * opt->asize + qa] > 0 ? '+' : ' ', (char)toupper(qseq[al + l]), true);
			}
			nl += len * 3, al += len;
		} else if (op == NS_CIGAR_I) {
			for (int32_t j = 0; j < len; ++j) col('-', '-', ' ', (char)toupper(qseq[al + j])), col('-', '.', ' ', ' '), col('-', '.', ' ', ' ');
			al += len;
		} else if (op == NS_CIGAR_D) {
			for (int32_t l = 0; l < len; ++l) codon_cols(nl + l * 3, ' ', '-', true);
			nl += len * 3;
		} else if (op == NS_CIGAR_F) {
			for (int32_t l = 0; l < len; ++l) col(UC[nt[(size_t)(nl + l)]], '!', ' ', ' ');
			nl += len;
		} else if (op == NS_CIGAR_G) {
			for (int32_t l = 0; l < len; ++l) col(UC[nt[(size_t)(nl + l)]], '$', ' ', l == 0 ? (char)toupper(qseq[al]) : ' ');
			nl += len, ++al;
		} else if (op == NS_CIGAR_N || op == NS_CIGAR_U || op == NS_CIGAR_V) {
			const int32_t intron_len = op == NS_CIGAR_N ? len : len - 3;
			if (op != NS_CIGAR_N) { // the codon split by a phase-1 / phase-2 intron: its bases before the intron
				const uint8_t n1 = nt[(size_t)nl], n2 = op == NS_CIGAR_U ? nt[(size_t)(nl + len - 2)] : nt[(size_t)nl + 1], n3 = nt[(size_t)(nl + len - 1)];
				const uint8_t na = codon_aa(n1, n2, n3), qa = ns_tab_aa20[(uint8_t)qseq[al]];
				sta += ns_tab_aa_i2c[na];
				col(UC[nt[(size_t)nl]], ns_tab_aa_i2c[na], na == qa ? '|' : opt->mat[na * opt->asize + qa] > 0 ? '+' : ' ', (char)toupper(qseq[al]));
				++nl;
				if (op == NS_CIGAR_V) col(UC[nt[(size_t)nl]], '.', ' ', ' '), ++nl;
				++al;
			}
			if (intron_len <= max_flank * 2) {
				for (int32_t l = 0; l < intron_len; ++l) col(LC[nt[(size_t)(nl + l)]], ' ', ' ', ' ');
			} else {
				for (int32_t l = 0; l < max_flank; ++l) col(LC[nt[(size_t)(nl + l)]], ' ', ' ', ' ');
				col('~', ' ', ' ', ' ');
				char num[24];
				const int il = snprintf(num, sizeof(num), "%d", intron_len);
				for (int l = 0; l < il; ++l) col(num[l], ' ', ' ', ' ');
				col('~', ' ', ' ', ' ');
				for (int32_t l = 0; l < max_flank; ++l) col(LC[nt[(size_t)(nl + intron_len - max_flank + l)]], ' ', ' ', ' ');
			}
			nl += intron_len;
			if (op != NS_CIGAR_N) { // ... and after it
				col(UC[nt[(size_t)nl]], '.', ' ', ' '), ++nl;
				if (op == NS_CIGAR_U) col(UC[nt[(size_t)nl]], '.', ' ', ' '), ++nl;
			}
		}
	}
	if (l_nt == r->ve - r->vs + 3 && sta.back() != '*') { // one more codon when the translation does not end in a stop (format.c:318)
		const uint8_t na = codon_aa(nt[(size_t)nl], nt[(size_t)nl + 1], nt[(size_t)nl + 2]);
		sta += ns_tab_aa_i2c[na];
		col(UC[nt[(size_t)nl]], ns_tab_aa_i2c[na], ' ', ' '), col(UC[nt[(size_t)nl + 1]], '.', ' ', ' '), col(UC[nt[(size_t)nl + 2]], '.', ' ', ' ');
	}
	if (opt->flag & MP_F_SHOW_RESIDUE) {
		for (const std::string *s : { &atn, &ata, &aas, &aqa }) o.put(s->data(), (int64_t)s->size()), o.putc('\n');
	}
	if (opt->flag & MP_F_SHOW_TRANS) o.put(sta.data(), (int64_t)sta.size()), o.putc('\n');
}

// everything the reference prints for one hit, in its order (format.c:453-473); r == 0: the unmapped line of -u
void format_output(Str &o, const mp_idx_t *mi, const mp_mapopt_t *opt, const char *qname, int32_t qlen, const char *qseq, const mp_reg1_t *r, int64_t id,
                   int32_t hit_idx, int64_t nt_lim)
{
	if (!r) {
		if (opt->flag & MP_F_SHOW_UNMAP) format_hit(o, mi, opt, qname, qlen, qseq, 0);
	} else if (opt->flag & MP_F_GTF) {
		if (opt->flag & (MP_F_SHOW_RESIDUE | MP_F_SHOW_TRANS)) format_hit(o, mi, opt, qname, qlen, qseq, r), format_residue(o, mi, opt, qseq, r, nt_lim);
		format_gtf(o, mi, opt, qname, qlen, r, id);
	} else {
		if (!(opt->flag & MP_F_NO_PAF)) format_hit(o, mi, opt, qname, qlen, qseq, r);
		if (opt->flag & (MP_F_SHOW_RESIDUE | MP_F_SHOW_TRANS)) format_residue(o, mi, opt, qseq, r, nt_lim);
		if (opt->flag & MP_F_GFF) format_gff(o, mi, opt, qname, qlen, r, id, hit_idx);
	}
}

} // namespace mpb
