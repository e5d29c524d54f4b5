// annot.h -- junction annotation of the index (mm_idx_t::I): BED reader and per-window junction flags, host side.
// Restates mm_idx_bed_read_core / mm_idx_bed_read_merge / mm_idx_bed_junc (index.c:672-826). The two structs keep the reference's
// layout, so an mm_idx_t annotated by either implementation can be read by the other.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cctype>
#include <string>
#include <vector>
#include <algorithm>
#include <zlib.h>
#include "mm_algo.cuh"

typedef struct { // index.c:35-38
	int32_t st, en, cnt;
	int32_t score:30, strand:2;
} mm_idx_intv1_t;
struct MmxKeyIntvSt { MM_HD uint64_t operator()(const mm_idx_intv1_t &v) const { return (uint64_t)(uint32_t)v.st; } }; // sort_key_bed, index.c:676
struct MmxKeyIntvEn { MM_HD uint64_t operator()(const mm_idx_intv1_t &v) const { return (uint64_t)(uint32_t)v.en; } }; // sort_key_end, index.c:679

struct mm_idx_intv_s { // index.c:40-43
	int32_t n, m;
	mm_idx_intv1_t *a;
};

// one BED line -> intervals (BED12 with read_junc: the introns between the blocks), appended to I[id] (index.c:693-757)
template<class Name2Id> static inline void mmx_bed_line(char *line, int read_junc, int min_sc, Name2Id name2id, mm_idx_intv_s *I)
{
	mm_idx_intv1_t t = {-1, -1, -1, -1, 0};
	char *p, *q, *bl = 0, *bs = 0;
	int32_t i, id = -1, n_blk = 0;
	for (p = q = line, i = 0;; ++p) {
		if (*p == 0 || *p == '\t') {
			const int32_t c = *p;
			*p = 0;
			if (i == 0) { id = name2id(q); if (id < 0) break; }
			else if (i == 1) { t.st = atol(q); if (t.st < 0) break; }
			else if (i == 2) { t.en = atol(q); if (t.en < 0) break; }
			else if (i == 4) t.score = *q >= '0' && *q <= '9'? atol(q) : -1;
			else if (i == 5) t.strand = *q == '+'? 1 : *q == '-'? -1 : 0;
			else if (i == 9) { if (!isdigit((unsigned char)*q)) break; n_blk = atol(q); }
			else if (i == 10) bl = q;
			else if (i == 11) { bs = q; break; }
			if (c == 0) break;
			++i, q = p + 1;
		}
	}
	if (id < 0 || t.st < 0 || t.st >= t.en) return;
	if (min_sc > 0 && t.score < min_sc) return;
	mm_idx_intv_s *r = &I[id];
	auto push = [&](const mm_idx_intv1_t &s) {
		if (r->n == r->m) {
			r->m = r->m? r->m + (r->m >> 1) : 16;
			r->a = (mm_idx_intv1_t*)realloc(r->a, sizeof(*r->a) * r->m);
		}
		r->a[r->n++] = s;
	};
	if (i >= 11 && read_junc) { // BED12
		int32_t st, sz, en;
		st = strtol(bs, &bs, 10); ++bs;
		sz = strtol(bl, &bl, 10); ++bl;
		en = t.st + st + sz;
		for (i = 1; i < n_blk; ++i) {
			mm_idx_intv1_t s = t;
			st = strtol(bs, &bs, 10); ++bs;
			sz = strtol(bl, &bl, 10); ++bl;
			s.st = en, s.en = t.st + st;
			en = t.st + st + sz;
			if (s.en > s.st) push(s);
		}
	} else push(t);
}

// index.c:682-794: read, sort by (st, en), merge identical intervals (cnt = multiplicity). Returns NULL if the file cannot be opened.
template<class Name2Id> static inline mm_idx_intv_s *mmx_bed_read(const char *fn, uint32_t n_seq, int read_junc, int min_sc, Name2Id name2id, long *n_raw, long *n_merged)
{
	gzFile fp = fn && strcmp(fn, "-")? gzopen(fn, "r") : gzdopen(0, "r");
	if (fp == 0) return 0;
	mm_idx_intv_s *I = (mm_idx_intv_s*)calloc(n_seq, sizeof(mm_idx_intv_s));
	std::string line;
	int c;
	bool any = false;
	auto flush = [&]() { std::vector<char> buf(line.begin(), line.end()); buf.push_back(0); mmx_bed_line(buf.data(), read_junc, min_sc, name2id, I); line.clear(); any = false; };
	while ((c = gzgetc(fp)) >= 0) {
		if (c == '\n') flush();
		else line += (char)c, any = true;
	}
	if (any) flush();
	gzclose(fp);
	long n = 0, n0 = 0;
	for (uint32_t i = 0; i < n_seq; ++i) {
		mm_idx_intv_s *v = &I[i];
		n0 += v->n;
		// (st, en) order exactly as index.c:776-783 establishes it: radix_sort_bed by st, then radix_sort_end inside each group of
		// equal st. Both are the unstable American-flag sort of ksort.h:101-151, so which of several identical (st, en) lines
		// comes first -- and hence whose strand the merged interval keeps -- is defined by that sort's walk; mmx_rs_sort replays it.
		if (v->n > 1) {
			std::vector<int32_t> stk((size_t)mmx_rs_stack_len(v->n));
			mmx_rs_sort(v->a, (int64_t)v->n, stk.data(), MmxKeyIntvSt());
			for (int32_t j = 1, j0 = 0; j <= v->n; ++j)
				if (j == v->n || v->a[j].st != v->a[j0].st) {
					if (j - j0 > 1) mmx_rs_sort(v->a + j0, (int64_t)(j - j0), stk.data(), MmxKeyIntvEn());
					j0 = j;
				}
		}
		int32_t j, j0, k;
		for (j = 1, j0 = 0, k = 0; j <= v->n; ++j)
			if (j == v->n || v->a[j].st != v->a[j0].st || v->a[j].en != v->a[j0].en) {
				v->a[k] = v->a[j0];
				v->a[k++].cnt = j - j0;
				j0 = j;
			}
		v->a = (mm_idx_intv1_t*)realloc(v->a, sizeof(mm_idx_intv1_t) * (k > 0? k : 1));
		v->n = v->m = k;
		n += k;
	}
	if (n_raw) *n_raw = n0;
	if (n_merged) *n_merged = n;
	return I;
}

// index.c:802-826: bit 1/2 = first/last base of a '+' intron, 8/4 = first/last base of a '-' intron; only introns that lie
// entirely inside [st,en) are marked
static inline int mmx_bed_junc(const mm_idx_intv_s *I, int32_t n_seq, int32_t ctg, int32_t st, int32_t en, uint8_t *s)
{
	memset(s, 0, en - st);
	if (I == 0 || ctg < 0 || ctg >= n_seq) return -1;
	const mm_idx_intv_s *r = &I[ctg];
	int32_t left = 0, right = r->n;
	while (right > left) {
		const int32_t mid = left + ((right - left) >> 1);
		if (r->a[mid].st >= st) right = mid;
		else left = mid + 1;
	}
	for (int32_t i = left; i < r->n; ++i) {
		if (r->a[i].st >= en) break; // sorted by st: nothing further can lie inside the window
		if (st <= r->a[i].st && en >= r->a[i].en && r->a[i].strand != 0) {
			if (r->a[i].strand > 0) s[r->a[i].st - st] |= 1, s[r->a[i].en - 1 - st] |= 2;
			else s[r->a[i].st - st] |= 8, s[r->a[i].en - 1 - st] |= 4;
		}
	}
	return left;
}

// ---- junction jumps (mm_idx_t::J; index.c:828-959) ----
#ifndef MM_JUNC_ANNO
#define MM_JUNC_ANNO 0x1 // mmpriv.h:27-28
#define MM_JUNC_MISC 0x2
#endif
typedef struct { // mmpriv.h:59-63; also the entry of the device table (index.h: d_jump)
	int32_t off, off2, cnt;
	int16_t strand;
	uint16_t flag;
} mm_idx_jjump1_t;
struct mm_idx_jjump_s { // one per contig: both ends of every intron, sorted by (off, off2), equal pairs merged
	int32_t n, m;
	mm_idx_jjump1_t *a;
};
struct MmxKeyJjOff  { MM_HD uint64_t operator()(const mm_idx_jjump1_t &v) const { return (uint64_t)(uint32_t)v.off; } };  // sort_key_jj, index.c:832
struct MmxKeyJjOff2 { MM_HD uint64_t operator()(const mm_idx_jjump1_t &v) const { return (uint64_t)(uint32_t)v.off2; } }; // sort_key_jj2, index.c:835

// sort_jjump (index.c:838-863). Both radix sorts have 4-byte keys; mmx_rs_sort starts at the most significant byte in which the
// keys differ, which for keys below 2^32 is the walk a 4-byte sort takes. The merged entry keeps the strand of the first entry of
// its run, so the unstable order of equal keys is replayed, not just the sorted result.
static inline void mmx_jjump_sort(mm_idx_jjump_s *jj)
{
	if (jj->n == 0) return;
	std::vector<int32_t> stk((size_t)mmx_rs_stack_len(jj->n));
	mmx_rs_sort(jj->a, (int64_t)jj->n, stk.data(), MmxKeyJjOff());
	for (int32_t j0 = 0, j = 1; j <= jj->n; ++j)
		if (j == jj->n || jj->a[j0].off != jj->a[j].off) {
			mmx_rs_sort(jj->a + j0, (int64_t)(j - j0), stk.data(), MmxKeyJjOff2());
			j0 = j;
		}
	int32_t k = 0;
	for (int32_t j0 = 0, j = 1; j <= jj->n; ++j)
		if (j == jj->n || jj->a[j0].off != jj->a[j].off || jj->a[j0].off2 != jj->a[j].off2) {
			int32_t cnt = 0;
			uint16_t flag = 0;
			for (int32_t t = j0; t < j; ++t) cnt += jj->a[t].cnt, flag |= jj->a[t].flag;
			jj->a[k] = jj->a[j0];
			jj->a[k].cnt = cnt;
			jj->a[k++].flag = flag;
			j0 = j;
		}
	jj->n = jj->m = k;
}

// mm_idx_bed2jjump (index.c:865-883): each intron as {off=st, off2=en} and {off=en, off2=st}
static inline mm_idx_jjump_s *mmx_bed2jjump(const mm_idx_intv_s *I, uint32_t n_seq, uint16_t flag)
{
	mm_idx_jjump_s *J = (mm_idx_jjump_s*)calloc(n_seq, sizeof(mm_idx_jjump_s));
	for (uint32_t i = 0; i < n_seq; ++i) {
		const mm_idx_intv_s *v = &I[i];
		mm_idx_jjump_s *jj = &J[i];
		jj->n = jj->m = v->n * 2;
		jj->a = (mm_idx_jjump1_t*)calloc(jj->n > 0? jj->n : 1, sizeof(mm_idx_jjump1_t));
		for (int32_t j = 0, k = 0; j < v->n; ++j) {
			const mm_idx_intv1_t &t = v->a[j];
			jj->a[k].off = t.st, jj->a[k].off2 = t.en, jj->a[k].cnt = t.cnt, jj->a[k].strand = (int16_t)t.strand, jj->a[k++].flag = flag;
			jj->a[k].off = t.en, jj->a[k].off2 = t.st, jj->a[k].cnt = t.cnt, jj->a[k].strand = (int16_t)t.strand, jj->a[k++].flag = flag;
		}
		mmx_jjump_sort(jj);
	}
	return J;
}

// mm_idx_jjump_merge (index.c:885-901): J0's entries, then J1's, through the same sort; J0 and J1 are freed
static inline mm_idx_jjump_s *mmx_jjump_merge(mm_idx_jjump_s *J0, mm_idx_jjump_s *J1, uint32_t n_seq)
{
	mm_idx_jjump_s *J2 = (mm_idx_jjump_s*)calloc(n_seq, sizeof(mm_idx_jjump_s));
	for (uint32_t i = 0; i < n_seq; ++i) {
		mm_idx_jjump_s *jj = &J2[i];
		jj->n = jj->m = J0[i].n + J1[i].n;
		jj->a = (mm_idx_jjump1_t*)calloc(jj->n > 0? jj->n : 1, sizeof(mm_idx_jjump1_t));
		if (J0[i].n) memcpy(jj->a, J0[i].a, sizeof(mm_idx_jjump1_t) * J0[i].n);
		if (J1[i].n) memcpy(jj->a + J0[i].n, J1[i].a, sizeof(mm_idx_jjump1_t) * J1[i].n);
		mmx_jjump_sort(jj);
		free(J0[i].a), free(J1[i].a);
	}
	free(J0), free(J1);
	return J2;
}

// mm_idx_jump_get_core (index.c:932-944): the last entry with off <= x, -1 if there is none
MM_HD int32_t mmx_jump_get_core(int32_t n, const mm_idx_jjump1_t *a, int32_t x)
{
	int32_t s = 0, e = n;
	if (n == 0 || x < a[0].off) return -1;
	while (s < e) {
		const int32_t mid = s + (e - s) / 2;
		if (x >= a[mid].off && (mid + 1 >= n || x < a[mid + 1].off)) return mid;
		else if (x < a[mid].off) e = mid;
		else s = mid + 1;
	}
	return n - 1; // not reached: a is sorted by off
}

// mm_idx_jump_get (index.c:946-959): the entries of one contig with off in (st, en], en clamped to the contig length
MM_HD const mm_idx_jjump1_t *mmx_jump_get(int32_t n_a, const mm_idx_jjump1_t *a, int32_t seq_len, int32_t st, int32_t en, int32_t *n)
{
	*n = 0;
	if (en < 0 || en > seq_len) en = seq_len;
	if (n_a == 0) return 0;
	const int32_t l = mmx_jump_get_core(n_a, a, st), r = mmx_jump_get_core(n_a, a, en);
	*n = r - l;
	return &a[l + 1];
}

// ---- splice scores (mm_idx_t::spsc; index.c:963-1075) ----
struct mm_idx_spsc_s { // index.c:963-966; one entry per (contig, strand): a[] = pos<<8 | (score+64)<<1 | acceptor, sorted
	uint32_t n, m;
	uint64_t *a;
};

// index.c:968-1040. Line format: contig, position, strand (+/-), type (D/A), score. Returns NULL if the file cannot be opened.
template<class Name2Id, class SeqLen> static inline mm_idx_spsc_s *mmx_spsc_read(const char *fn, uint32_t n_seq, int32_t max_sc, float scale, Name2Id name2id, SeqLen seq_len, long *n_read_)
{
	gzFile fp = fn && strcmp(fn, "-") != 0? gzopen(fn, "rb") : gzdopen(0, "rb");
	if (fp == 0) return 0;
	if (max_sc > 63) max_sc = 63;
	mm_idx_spsc_s *S = (mm_idx_spsc_s*)calloc((size_t)n_seq * 2, sizeof(mm_idx_spsc_s));
	long n_read = 0;
	std::string line;
	int c;
	bool any = false;
	auto flush = [&]() {
		std::vector<char> buf(line.begin(), line.end()); buf.push_back(0);
		line.clear(), any = false;
		char *p, *q, *name = 0;
		int32_t i, type = -1, strand = 0, cid = -1, score = -1;
		int64_t pos = -1;
		for (i = 0, p = q = buf.data();; ++p) {
			if (*p == '\t' || *p == 0) {
				const int ch = *p;
				*p = 0;
				if (i == 0) name = q;
				else if (i == 1) pos = atol(q);
				else if (i == 2) strand = *q == '+'? 1 : -1; // index.c:1001 as written: anything but '+' counts as the minus strand
				else if (i == 3) type = *q == 'D'? 0 : *q == 'A'? 1 : -1;
				else if (i == 4) { score = atoi(q); break; }
				if (ch == 0) break;
				q = p + 1, ++i;
			}
		}
		if (i < 4) return;
		if (scale > 0.0f && scale < 1.0f) score = score > 0.0f? (int)(score * scale + .499) : (int)(score * scale - .499);
		if (score > max_sc) score = max_sc;
		if (score < -max_sc) score = -max_sc;
		cid = name2id(name);
		if (cid < 0 || type < 0 || strand == 0 || pos < 0) return;
		mm_idx_spsc_s *s = &S[cid << 1 | (strand > 0? 0 : 1)];
		if (s->n == s->m) { s->m = s->m? s->m + (s->m >> 1) + 1 : 16; s->a = (uint64_t*)realloc(s->a, sizeof(uint64_t) * s->m); }
		if (pos > 0 && pos < (int64_t)seq_len(cid)) { // scores at the ends are ignored
			s->a[s->n++] = (uint64_t)pos << 8 | (uint64_t)(score + 64) << 1 | (uint64_t)type;
			++n_read;
		}
	};
	while ((c = gzgetc(fp)) >= 0) {
		if (c == '\n') flush();
		else line += (char)c, any = true;
	}
	if (any) flush();
	gzclose(fp);
	for (uint32_t j = 0; j < n_seq * 2; ++j) if (S[j].n > 0) std::sort(S[j].a, S[j].a + S[j].n); // radix_sort_64: plain ascending order of distinct-or-equal keys
	if (n_read_) *n_read_ = n_read;
	return S;
}

// index.c:1042-1053
static inline int32_t mmx_spsc_find(int32_t n, const uint64_t *a, int64_t x)
{
	int32_t s = 0, e = n;
	if (n == 0) return -1;
	if (x < (int64_t)(a[0] >> 8)) return -1;
	while (s < e) {
		const int32_t mid = s + (e - s) / 2;
		if (x >= (int64_t)(a[mid] >> 8) && (mid + 1 >= n || x < (int64_t)(a[mid + 1] >> 8))) return mid;
		else if (x < (int64_t)(a[mid] >> 8)) e = mid;
		else s = mid + 1;
	}
	return n - 1;
}

// index.c:1055-1075: per-position score bytes of (st, en) on one strand, 0xff where there is none; the largest byte wins
static inline int64_t mmx_spsc_get(const mm_idx_spsc_s *S, int32_t n_seq, int32_t cid, int64_t seq_len, int64_t st, int64_t en, int32_t rev, uint8_t *sc)
{
	if (cid >= n_seq || cid < 0 || S == 0) return -1;
	if (en < 0 || en > seq_len) en = seq_len;
	memset(sc, 0xff, en - st);
	const mm_idx_spsc_s *s = &S[cid << 1 | (!!rev)];
	if (s->n > 0) {
		const int32_t l = mmx_spsc_find((int32_t)s->n, s->a, st), r = mmx_spsc_find((int32_t)s->n, s->a, en);
		for (int32_t j = l + 1; j <= r; ++j) {
			const int64_t x = (int64_t)(s->a[j] >> 8) - st;
			const uint8_t score = s->a[j] & 0xff;
			if (x == en - st) continue;
			if (sc[x] == 0xff || sc[x] < score) sc[x] = score;
		}
	}
	return en - st;
}
