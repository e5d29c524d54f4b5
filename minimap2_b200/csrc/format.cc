// minimap2_b200/csrc/format.cc -- PAF / SAM record formatting and the cs/ds/MD tags (host; defines the parity surface).
// Field order, tag set and number formatting follow reference format.c (write_tags :397-423, mm_write_paf4 :425-461,
// mm_write_sam3 :522-680, cs/ds/MD :150-395) so that records compare byte-for-byte with the reference's output.
#include "hostlogic.h"
#include <cstring>
#include <cstdlib>
#include <cassert>

static inline void put_int(std::string &s, int64_t v) { s += std::to_string(v); }

static char g_rg_id[256]; // ID of the -R read group (format.c:9), set by the header writer, printed as RG:Z: on every SAM record

static void write_tags(std::string &s, const mm_reg1_t *r) // format.c:397-423
{
	int type;
	if (r->id == r->parent) type = r->inv? 'I' : 'P';
	else type = r->inv? 'i' : 'S';
	if (r->p) {
		s += "\tNM:i:"; put_int(s, r->blen - r->mlen + r->p->n_ambi);
		s += "\tms:i:"; put_int(s, r->p->dp_max0);
		s += "\tAS:i:"; put_int(s, r->p->dp_score);
		s += "\tnn:i:"; put_int(s, r->p->n_ambi);
		if (r->p->trans_strand == 1 || r->p->trans_strand == 2) { s += "\tts:A:"; s += "?+-?"[r->p->trans_strand]; }
	}
	s += "\ttp:A:"; s += (char)type;
	s += "\tcm:i:"; put_int(s, r->cnt);
	s += "\ts1:i:"; put_int(s, r->score);
	if (r->parent == r->id) { s += "\ts2:i:"; put_int(s, r->subsc); }
	if (r->p) {
		char buf[16];
		double div = 1.0 - hl_event_identity(r);
		if (div == 0.0) buf[0] = '0', buf[1] = 0;
		else snprintf(buf, 16, "%.4f", 1.0 - hl_event_identity(r));
		s += "\tde:f:"; s += buf;
	} else if (r->div >= 0.0f && r->div <= 1.0f) {
		char buf[16];
		if (r->div == 0.0f) buf[0] = '0', buf[1] = 0;
		else snprintf(buf, 16, "%.4f", r->div);
		s += "\tdv:f:"; s += buf;
	}
	if (r->split) { s += "\tzd:i:"; put_int(s, r->split); }
}

// ---- cs / ds / MD (format.c:150-395) ----
static void write_indel_ds(std::string &s, int64_t len, const uint8_t *seq, int64_t ll, int64_t lr)
{
	if (ll + lr >= len) {
		s += '[';
		for (int64_t i = 0; i < len; ++i) s += "acgtn"[seq[i]];
		s += ']';
	} else {
		int64_t k = 0;
		if (ll > 0) { s += '['; for (int64_t i = 0; i < ll; ++i) s += "acgtn"[seq[k + i]]; s += ']'; k += ll; }
		for (int64_t i = 0; i < len - lr - ll; ++i) s += "acgtn"[seq[k + i]];
		k += len - lr - ll;
		if (lr > 0) { s += '['; for (int64_t i = 0; i < lr; ++i) s += "acgtn"[seq[k + i]]; s += ']'; }
	}
}

static void write_cs_ds_core(std::string &s, const uint8_t *tseq, const uint8_t *qseq, const mm_reg1_t *r, int no_iden, int is_ds, int write_tag)
{
	int q_off = 0, t_off = 0, q_len = 0, t_len = 0;
	if (write_tag) { s += is_ds? "\tds:Z:" : "\tcs:Z:"; }
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		int op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == MM_CIGAR_MATCH || op == MM_CIGAR_EQ_MATCH || op == MM_CIGAR_X_MISMATCH) q_len += len, t_len += len;
		else if (op == MM_CIGAR_INS) q_len += len;
		else if (op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) t_len += len;
	}
	std::string run;
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		int op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == MM_CIGAR_MATCH || op == MM_CIGAR_EQ_MATCH || op == MM_CIGAR_X_MISMATCH) {
			run.clear();
			for (int j = 0; j < len; ++j) {
				if (qseq[q_off + j] != tseq[t_off + j]) {
					if (!run.empty()) {
						if (!no_iden) { s += '='; s += run; } else { s += ':'; put_int(s, (int64_t)run.size()); }
						run.clear();
					}
					s += '*'; s += "acgtn"[tseq[t_off + j]]; s += "acgtn"[qseq[q_off + j]];
				} else run += "ACGTN"[qseq[q_off + j]];
			}
			if (!run.empty()) { if (!no_iden) { s += '='; s += run; } else { s += ':'; put_int(s, (int64_t)run.size()); } }
			q_off += len, t_off += len;
		} else if (op == MM_CIGAR_INS) {
			if (is_ds) {
				int z, ll, lr, y = q_off;
				for (z = 1; z <= len; ++z) if (y - z < 0 || qseq[y + len - z] != qseq[y - z]) break;
				lr = z - 1;
				for (z = 0; z < len; ++z) if (y + len + z >= q_len || qseq[y + len + z] != qseq[y + z]) break;
				ll = z;
				s += '+';
				write_indel_ds(s, len, &qseq[y], ll, lr);
			} else { s += '+'; for (int j = 0; j < len; ++j) s += "acgtn"[qseq[q_off + j]]; }
			q_off += len;
		} else if (op == MM_CIGAR_DEL) {
			if (is_ds) {
				int z, ll, lr, x = t_off;
				for (z = 1; z <= len; ++z) if (x - z < 0 || tseq[x + len - z] != tseq[x - z]) break;
				lr = z - 1;
				for (z = 0; z < len; ++z) if (x + len + z >= t_len || tseq[x + z] != tseq[x + len + z]) break;
				ll = z;
				s += '-';
				write_indel_ds(s, len, &tseq[x], ll, lr);
			} else { s += '-'; for (int j = 0; j < len; ++j) s += "acgtn"[tseq[t_off + j]]; }
			t_off += len;
		} else { // intron
			s += '~'; s += "acgtn"[tseq[t_off]]; s += "acgtn"[tseq[t_off + 1]];
			put_int(s, len);
			s += "acgtn"[tseq[t_off + len - 2]]; s += "acgtn"[tseq[t_off + len - 1]];
			t_off += len;
		}
	}
}

static void write_MD_core(std::string &s, const uint8_t *tseq, const uint8_t *qseq, const mm_reg1_t *r, int write_tag)
{
	int q_off = 0, t_off = 0, l_MD = 0;
	if (write_tag) s += "\tMD:Z:";
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		int op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == MM_CIGAR_MATCH || op == MM_CIGAR_EQ_MATCH || op == MM_CIGAR_X_MISMATCH) {
			for (int j = 0; j < len; ++j) {
				if (qseq[q_off + j] != tseq[t_off + j]) { put_int(s, l_MD); s += "ACGTN"[tseq[t_off + j]]; l_MD = 0; }
				else ++l_MD;
			}
			q_off += len, t_off += len;
		} else if (op == MM_CIGAR_INS) q_off += len;
		else if (op == MM_CIGAR_DEL) {
			put_int(s, l_MD); s += '^';
			for (int j = 0; j < len; ++j) s += "ACGTN"[tseq[t_off + j]];
			l_MD = 0;
			t_off += len;
		} else if (op == MM_CIGAR_N_SKIP) t_off += len;
	}
	if (l_MD > 0) put_int(s, l_MD);
}

static void write_cs_ds_or_MD(std::string &s, const mm_idx_t *mi, const char *seq, const mm_reg1_t *r, int no_iden, int is_MD, int is_ds, int write_tag, int is_qstrand = 0)
{
	if (r->p == 0) return;
	std::vector<uint8_t> qseq(r->qe - r->qs + 1), tseq(r->re - r->rs + 1);
	if (is_qstrand && r->rev) { // mm_idx_getseq2 / mm_idx_getseq_rev (index.c:176-196): the other strand of the target, forward query (format.c:343-346)
		const int len = (int)mi->seq[r->rid].len, n = r->re - r->rs;
		mm_idx_getseq(mi, r->rid, len - r->re, len - r->rs, tseq.data());
		for (int i = 0, j = n - 1; i <= j; ++i, --j) { const uint8_t x = tseq[i], y = tseq[j]; tseq[i] = y < 4? 3 - y : y, tseq[j] = x < 4? 3 - x : x; }
	} else mm_idx_getseq(mi, r->rid, r->rs, r->re, tseq.data());
	if (!r->rev || is_qstrand) for (int i = r->qs; i < r->qe; ++i) qseq[i - r->qs] = mmx_nt4((uint8_t)seq[i]);
	else for (int i = r->qs; i < r->qe; ++i) { uint8_t c = mmx_nt4((uint8_t)seq[i]); qseq[r->qe - i - 1] = c >= 4? 4 : 3 - c; }
	if (is_MD) write_MD_core(s, tseq.data(), qseq.data(), r, write_tag);
	else write_cs_ds_core(s, tseq.data(), qseq.data(), r, no_iden, is_ds, write_tag);
}

static int gen_tag(char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq, int is_MD, int is_ds, int no_iden)
{
	std::string s;
	write_cs_ds_or_MD(s, mi, seq, r, no_iden, is_MD, is_ds, 0);
	if ((int)s.size() + 1 > *max_len) {
		uint32_t m = (uint32_t)s.size() + 1;
		--m; m |= m >> 1; m |= m >> 2; m |= m >> 4; m |= m >> 8; m |= m >> 16; ++m;
		*max_len = (int)m;
		*buf = (char*)realloc(*buf, *max_len);
	}
	memcpy(*buf, s.c_str(), s.size() + 1);
	return (int)s.size();
}
extern "C" int mm_gen_cs(void *, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq, int no_iden) { return gen_tag(buf, max_len, mi, r, seq, 0, 0, no_iden); }
extern "C" int mm_gen_ds(void *, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq, int no_iden) { return gen_tag(buf, max_len, mi, r, seq, 0, 1, no_iden); }
extern "C" int mm_gen_MD(void *, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq) { return gen_tag(buf, max_len, mi, r, seq, 1, 0, 0); }

// mm_write_junc (format.c:256-300): one BED6 line per intron of a spliced hit with a preferred transcript strand (contig, start, end,
// read name, donor + acceptor score, strand), each ended by a newline
void hl_write_junc(std::string &s, const mm_idx_t *mi, const char *qname, const mm_reg1_t *r)
{
	if (!r->is_spliced || r->p == 0) return;
	if (r->p->trans_strand != 1 && r->p->trans_strand != 2) return;
	auto revcomp_splice = [](uint8_t x[2]) { const uint8_t c = x[1] < 4? 3 - x[1] : 4; x[1] = x[0] < 4? 3 - x[0] : 4; x[0] = c; };
	int32_t t_off = r->rs;
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		const int op = r->p->cigar[i] & 0xf, len = (int)(r->p->cigar[i] >> 4);
		if (op == MM_CIGAR_MATCH || op == MM_CIGAR_EQ_MATCH || op == MM_CIGAR_X_MISMATCH || op == MM_CIGAR_DEL) t_off += len;
		else if (op == MM_CIGAR_N_SKIP) {
			uint8_t donor[2], acceptor[2];
			int score1 = 0, score2 = 0;
			const int rev = (r->p->trans_strand == 2) ^ r->rev;
			if (!rev) {
				mm_idx_getseq(mi, r->rid, t_off, t_off + 2, donor);
				mm_idx_getseq(mi, r->rid, t_off + len - 2, t_off + len, acceptor);
			} else {
				mm_idx_getseq(mi, r->rid, t_off, t_off + 2, acceptor);
				mm_idx_getseq(mi, r->rid, t_off + len - 2, t_off + len, donor);
				revcomp_splice(donor), revcomp_splice(acceptor);
			}
			if (donor[0] == 2 && donor[1] == 3) score1 = 3;
			else if (donor[0] == 2 && donor[1] == 1) score1 = 2;
			else if (donor[0] == 0 && donor[1] == 3) score1 = 1;
			if (acceptor[0] == 0 && acceptor[1] == 2) score2 = 3;
			else if (acceptor[0] == 0 && acceptor[1] == 1) score2 = 1;
			s += mi->seq[r->rid].name; s += '\t'; put_int(s, t_off); s += '\t'; put_int(s, t_off + len); s += '\t';
			s += qname; s += '\t'; put_int(s, score1 + score2); s += '\t'; s += "+-"[rev]; s += '\n';
			t_off += len;
		}
	}
}

// NB: cs/MD need the query sequence; the PAF writer receives it through hl_write_paf_seq below
static thread_local const char *tl_seq = nullptr;
void hl_set_seq_for_tags(const char *seq) { tl_seq = seq; }

void hl_write_paf(std::string &s, const mm_idx_t *mi, const char *qname, int qlen, const mm_reg1_t *r, int64_t opt_flag, int rep_len) // format.c:425-461
{
	s += qname;
	if (r == 0) {
		s += '\t'; put_int(s, qlen); s += "\t0\t0\t*\t*\t0\t0\t0\t0\t0\t0";
		if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
		return;
	}
	s += '\t'; put_int(s, qlen); s += '\t'; put_int(s, r->qs); s += '\t'; put_int(s, r->qe); s += '\t'; s += "+-"[r->rev]; s += '\t';
	if (mi->seq[r->rid].name) s += mi->seq[r->rid].name; else put_int(s, r->rid);
	s += '\t'; put_int(s, mi->seq[r->rid].len);
	if ((opt_flag & MM_F_QSTRAND) && r->rev) { s += '\t'; put_int(s, (int64_t)mi->seq[r->rid].len - r->re); s += '\t'; put_int(s, (int64_t)mi->seq[r->rid].len - r->rs); } // format.c:440-443
	else { s += '\t'; put_int(s, r->rs); s += '\t'; put_int(s, r->re); }
	s += '\t'; put_int(s, r->mlen); s += '\t'; put_int(s, r->blen);
	s += '\t'; put_int(s, r->mapq);
	write_tags(s, r);
	if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
	if (r->p && (opt_flag & MM_F_OUT_CG)) {
		s += "\tcg:Z:";
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { put_int(s, r->p->cigar[k] >> 4); s += MM_CIGAR_STR[r->p->cigar[k] & 0xf]; }
	}
	if (r->p && (opt_flag & (MM_F_OUT_CS | MM_F_OUT_DS | MM_F_OUT_MD)) && tl_seq)
		write_cs_ds_or_MD(s, mi, tl_seq, r, !(opt_flag & MM_F_OUT_CS_LONG), !!(opt_flag & MM_F_OUT_MD), !!(opt_flag & MM_F_OUT_DS), 1, !!(opt_flag & MM_F_QSTRAND));
}

static const unsigned char comp_tab[128] = { // bseq.c:11-28 (ASCII range)
	  0,   1,   2,   3,   4,   5,   6,   7,   8,   9,  10,  11,  12,  13,  14,  15,
	 16,  17,  18,  19,  20,  21,  22,  23,  24,  25,  26,  27,  28,  29,  30,  31,
	 32,  33,  34,  35,  36,  37,  38,  39,  40,  41,  42,  43,  44,  45,  46,  47,
	 48,  49,  50,  51,  52,  53,  54,  55,  56,  57,  58,  59,  60,  61,  62,  63,
	 64, 'T', 'V', 'G', 'H', 'E', 'F', 'C', 'D', 'I', 'J', 'M', 'L', 'K', 'N', 'O',
	'P', 'Q', 'Y', 'S', 'A', 'A', 'B', 'W', 'X', 'R', 'Z',  91,  92,  93,  94,  95,
	 96, 't', 'v', 'g', 'h', 'e', 'f', 'c', 'd', 'i', 'j', 'm', 'l', 'k', 'n', 'o',
	'p', 'q', 'y', 's', 'a', 'a', 'b', 'w', 'x', 'r', 'z', 123, 124, 125, 126, 127
};

// the exported form (bseq.h:29; mappy's cmappy.h reverse-complements the mate with it): identity outside the ASCII letters
extern "C" { unsigned char seq_comp_table[256]; }
namespace { struct CompTabInit { CompTabInit() { for (int i = 0; i < 256; ++i) seq_comp_table[i] = i < 128? comp_tab[i] : (unsigned char)i; } } g_comp_tab_init; }

static void sam_write_sq(std::string &s, const char *seq, int l, int rev, int comp) // format.c:463-476
{
	if (rev) {
		for (int i = 0; i < l; ++i) {
			int c = (unsigned char)seq[l - 1 - i];
			s += (char)(c < 128 && comp? comp_tab[c] : c);
		}
	} else s.append(seq, l);
}

static void write_sam_cigar(std::string &s, int sam_flag, int in_tag, int qlen, const mm_reg1_t *r, int64_t opt_flag) // format.c:487-520
{
	if (r->p == 0) { s += '*'; return; }
	uint32_t clip_len[2];
	clip_len[0] = r->rev? qlen - r->qe : r->qs;
	clip_len[1] = r->rev? r->qs : qlen - r->qe;
	const bool hard = ((sam_flag & 0x800) || ((sam_flag & 0x100) && (opt_flag & MM_F_SECONDARY_SEQ))) && !(opt_flag & MM_F_SOFTCLIP);
	if (in_tag) {
		int clip_char = hard? 5 : 4;
		s += "\tCG:B:I";
		if (clip_len[0]) { s += ','; put_int(s, clip_len[0] << 4 | clip_char); }
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { s += ','; put_int(s, r->p->cigar[k]); }
		if (clip_len[1]) { s += ','; put_int(s, clip_len[1] << 4 | clip_char); }
	} else {
		char clip_char = hard? 'H' : 'S';
		if (clip_len[0]) { put_int(s, clip_len[0]); s += clip_char; }
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { put_int(s, r->p->cigar[k] >> 4); s += MM_CIGAR_STR[r->p->cigar[k] & 0xf]; }
		if (clip_len[1]) { put_int(s, clip_len[1]); s += clip_char; }
	}
}

// single-segment subset of mm_write_sam3 (format.c:522-680)
void hl_write_sam(std::string &s, const mm_idx_t *mi, const char *qname, const char *seq, const char *qual, int qlen, int reg_idx,
				  int n_regs, const mm_reg1_t *regs, int64_t opt_flag, int rep_len)
{
	const int max_bam_cigar_op = 65535;
	int flag = 0, cigar_in_tag = 0;
	const mm_reg1_t *r = n_regs > 0 && reg_idx < n_regs && reg_idx >= 0? &regs[reg_idx] : NULL;
	s += qname;
	if (r == 0) flag |= 0x4;
	else {
		if (r->rev) flag |= 0x10;
		if (r->parent != r->id) flag |= 0x100;
		else if (!r->sam_pri) flag |= 0x800;
	}
	s += '\t'; put_int(s, flag);
	if (r == 0) s += "\t*\t0\t0\t*";
	else {
		s += '\t'; s += mi->seq[r->rid].name; s += '\t'; put_int(s, r->rs + 1); s += '\t'; put_int(s, r->mapq); s += '\t';
		if ((opt_flag & MM_F_LONG_CIGAR) && r->p && r->p->n_cigar > (uint32_t)max_bam_cigar_op - 2) {
			int n_cigar = r->p->n_cigar;
			if (r->qs != 0) ++n_cigar;
			if (r->qe != qlen) ++n_cigar;
			if (n_cigar > max_bam_cigar_op) cigar_in_tag = 1;
		}
		if (cigar_in_tag) {
			int slen;
			if ((flag & 0x900) == 0 || (opt_flag & MM_F_SOFTCLIP)) slen = qlen;
			else if ((flag & 0x100) && !(opt_flag & MM_F_SECONDARY_SEQ)) slen = 0;
			else slen = r->qe - r->qs;
			put_int(s, slen); s += 'S'; put_int(s, r->re - r->rs); s += 'N';
		} else write_sam_cigar(s, flag, 0, qlen, r, opt_flag);
	}
	s += "\t*\t0\t0\t";
	if (r == 0) {
		sam_write_sq(s, seq, qlen, 0, 0);
		s += '\t';
		if (qual) sam_write_sq(s, qual, qlen, 0, 0); else s += '*';
	} else {
		if ((flag & 0x900) == 0 || (opt_flag & MM_F_SOFTCLIP)) {
			sam_write_sq(s, seq, qlen, r->rev, r->rev);
			s += '\t';
			if (qual) sam_write_sq(s, qual, qlen, r->rev, 0); else s += '*';
		} else if ((flag & 0x100) && !(opt_flag & MM_F_SECONDARY_SEQ)) s += "*\t*";
		else {
			sam_write_sq(s, seq + r->qs, r->qe - r->qs, r->rev, r->rev);
			s += '\t';
			if (qual) sam_write_sq(s, qual + r->qs, r->qe - r->qs, r->rev, 0); else s += '*';
		}
	}
	if (g_rg_id[0]) { s += "\tRG:Z:"; s += g_rg_id; } // format.c:639
	if (r) {
		write_tags(s, r);
		if (r->parent == r->id && r->p && n_regs > 1 && regs && r >= regs && r - regs < n_regs) { // SA tag
			int n_sa = 0;
			for (int i = 0; i < n_regs; ++i) if (i != r - regs && regs[i].parent == regs[i].id && regs[i].p) ++n_sa;
			if (n_sa > 0) {
				s += "\tSA:Z:";
				for (int i = 0; i < n_regs; ++i) {
					const mm_reg1_t *q = &regs[i];
					int l_M, l_I = 0, l_D = 0, clip5 = 0, clip3 = 0;
					if (r == q || q->parent != q->id || q->p == 0) continue;
					if (q->qe - q->qs < q->re - q->rs) l_M = q->qe - q->qs, l_D = (q->re - q->rs) - l_M;
					else l_M = q->re - q->rs, l_I = (q->qe - q->qs) - l_M;
					clip5 = q->rev? qlen - q->qe : q->qs;
					clip3 = q->rev? q->qs : qlen - q->qe;
					s += mi->seq[q->rid].name; s += ','; put_int(s, q->rs + 1); s += ','; s += "+-"[q->rev]; s += ',';
					if (clip5) { put_int(s, clip5); s += 'S'; }
					if (l_M) { put_int(s, l_M); s += 'M'; }
					if (l_I) { put_int(s, l_I); s += 'I'; }
					if (l_D) { put_int(s, l_D); s += 'D'; }
					if (clip3) { put_int(s, clip3); s += 'S'; }
					s += ','; put_int(s, q->mapq); s += ','; put_int(s, q->blen - q->mlen + q->p->n_ambi); s += ';';
				}
			}
		}
		if (r->p && (opt_flag & (MM_F_OUT_CS | MM_F_OUT_DS | MM_F_OUT_MD)))
			write_cs_ds_or_MD(s, mi, seq, r, !(opt_flag & MM_F_OUT_CS_LONG), !!(opt_flag & MM_F_OUT_MD), !!(opt_flag & MM_F_OUT_DS), 1);
		if (cigar_in_tag) write_sam_cigar(s, flag, 1, qlen, r, opt_flag);
	}
	if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
}

// read group (format.c:9,82-117): the @RG line goes into the header with its escapes resolved and its ID is repeated as RG:Z: on every record
static int sam_rg_line(std::string &s, const char *rg)
{
	memset(g_rg_id, 0, 256);
	if (rg == 0) return 0;
	if (strstr(rg, "@RG") != rg) { if (mm_verbose >= 1) fprintf(stderr, "[ERROR] the read group line is not started with @RG\n"); return -1; }
	if (strstr(rg, "\t") != NULL) { if (mm_verbose >= 1) fprintf(stderr, "[ERROR] the read group line contained literal <tab> characters -- replace with escaped tabs: \\t\n"); return -1; }
	std::string line;
	for (const char *p = rg; *p; ++p) { // mm_escape: \t -> tab, \\ -> backslash, any other escape is dropped
		if (*p == '\\') { ++p; if (*p == 't') line += '\t'; else if (*p == '\\') line += '\\'; if (*p == 0) break; }
		else line += *p;
	}
	const size_t id = line.find("\tID:");
	if (id == std::string::npos) { if (mm_verbose >= 1) fprintf(stderr, "[ERROR] no ID within the read group line\n"); return -1; }
	size_t e = id + 4;
	while (e < line.size() && line[e] != '\t' && line[e] != '\n') ++e;
	if (e - (id + 4) + 1 > 256) { if (mm_verbose >= 1) fprintf(stderr, "[ERROR] @RG:ID is longer than 255 characters\n"); return -1; }
	memcpy(g_rg_id, line.data() + id + 4, e - (id + 4));
	s += line; s += '\n';
	return 0;
}

int hl_write_sam_hdr(std::string &s, const mm_idx_t *mi, const char *rg, const char *ver, int argc, char *argv[]) // format.c:119-148
{
	int ret = 0;
	s += "@HD\tVN:1.6\tSO:unsorted\tGO:query\n";
	if (mi) for (uint32_t i = 0; i < mi->n_seq; ++i) { s += "@SQ\tSN:"; s += mi->seq[i].name; s += "\tLN:"; put_int(s, mi->seq[i].len); s += '\n'; }
	if (rg) ret = sam_rg_line(s, rg);
	s += "@PG\tID:minimap2\tPN:minimap2";
	if (ver) { s += "\tVN:"; s += ver; }
	if (argc > 1) {
		s += "\tCL:minimap2";
		for (int i = 1; i < argc; ++i) { s += ' '; s += argv[i]; }
	}
	return ret;
}

// mmpriv.h:104: what main.c:446-452 calls (the header goes to stdout through mm_err_puts, one line feed appended)
extern "C" int mm_write_sam_hdr(const mm_idx_t *mi, const char *rg, const char *ver, int argc, char *argv[])
{
	std::string s;
	const int ret = hl_write_sam_hdr(s, mi, rg, ver, argc, argv);
	puts(s.c_str());
	return ret;
}
