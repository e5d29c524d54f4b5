/* oracle/mm2o_seed.c -- TEST INFRASTRUCTURE ONLY (see mm2o.h).
 * Restates the seeding stage between the sketch and the chaining DP:
 *   the minimizer index as a lookup structure (index.c:226-275 worker_post: occurrences of a key in ascending position
 *   order; index.c:93-110 mm_idx_get), mm_seed_mz_flt (seed.c:5-28), mm_seed_collect_all (seed.c:30-52), mm_seed_select
 *   (seed.c:56-96) with the ksort.h max-heap (ksort.h:44-66), mm_collect_matches (seed.c:98-132), skip_seed (map.c:78-100)
 *   and collect_seed_hits (map.c:168-204) including its final radix_sort_128x.
 * The index here is a sorted array with binary search: only the *content* of a lookup is part of the contract.
 */
#include <stdlib.h>
#include <string.h>
#include "mm2o.h"

#define F_NO_DIAG   0x001LL
#define F_NO_DUAL   0x002LL
#define F_FOR_ONLY  0x100000LL
#define F_REV_ONLY  0x200000LL
#define F_QSTRAND   0x100000000LL
#define SEED_TANDEM (1ULL<<42)
#define SEED_SELF   (1ULL<<43)
#define SEED_SEG_SHIFT 48

struct mm2o_idx_s {
	int w, k, is_hpc, n_seq;
	char **name; int *len;
	int64_t n_keys, n_pos;
	uint64_t *key;     /* distinct minimizer values (x>>8), ascending */
	int64_t *start;    /* n_keys+1 offsets into pos */
	uint64_t *pos;     /* y = rid<<32 | lastPos<<1 | strand, ascending inside a key */
};

typedef struct { uint64_t key, y; } kv_t;
static int kv_cmp(const void *a, const void *b)
{
	const kv_t *x = (const kv_t*)a, *y = (const kv_t*)b;
	if (x->key != y->key) return x->key < y->key? -1 : 1;
	return x->y < y->y? -1 : x->y > y->y? 1 : 0;
}

mm2o_idx_t *mm2o_idx_build(int n_seq, const char **seqs, const int *lens, const char **names, int w, int k, int is_hpc)
{
	mm2o_idx_t *mi = (mm2o_idx_t*)calloc(1, sizeof(*mi));
	int64_t i, cap = 0, n = 0;
	kv_t *kv;
	int s;
	mi->w = w, mi->k = k, mi->is_hpc = is_hpc, mi->n_seq = n_seq;
	mi->name = (char**)calloc(n_seq, sizeof(char*)), mi->len = (int*)calloc(n_seq, sizeof(int));
	for (s = 0; s < n_seq; ++s) cap += lens[s];
	kv = (kv_t*)malloc((cap + 1) * sizeof(kv_t));
	for (s = 0; s < n_seq; ++s) { /* index.c:322-326: every sequence is sketched with rid = its index */
		mm2o_128_t *m = (mm2o_128_t*)malloc(((size_t)lens[s] + 1) * sizeof(mm2o_128_t));
		int nm = mm2o_sketch(seqs[s], lens[s], w, k, (uint32_t)s, is_hpc, m), j;
		for (j = 0; j < nm; ++j) kv[n].key = m[j].x >> 8, kv[n++].y = m[j].y;
		free(m);
		mi->name[s] = strdup(names? names[s] : ""), mi->len[s] = lens[s];
	}
	qsort(kv, n, sizeof(kv_t), kv_cmp);
	mi->key = (uint64_t*)malloc((n + 1) * 8), mi->start = (int64_t*)malloc((n + 2) * 8), mi->pos = (uint64_t*)malloc((n + 1) * 8);
	for (i = 0; i < n; ++i) {
		if (i == 0 || kv[i].key != kv[i-1].key) mi->key[mi->n_keys] = kv[i].key, mi->start[mi->n_keys++] = i;
		mi->pos[i] = kv[i].y;
	}
	mi->start[mi->n_keys] = n, mi->n_pos = n;
	free(kv);
	return mi;
}

void mm2o_idx_destroy(mm2o_idx_t *mi)
{
	int s;
	if (!mi) return;
	for (s = 0; s < mi->n_seq; ++s) free(mi->name[s]);
	free(mi->name); free(mi->len); free(mi->key); free(mi->start); free(mi->pos); free(mi);
}

const uint64_t *mm2o_idx_get(const mm2o_idx_t *mi, uint64_t minier, int *n) /* index.c:93-110 */
{
	int64_t lo = 0, hi = mi->n_keys;
	while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (mi->key[mid] < minier) lo = mid + 1; else hi = mid; }
	if (lo < mi->n_keys && mi->key[lo] == minier) { *n = (int)(mi->start[lo + 1] - mi->start[lo]); return mi->pos + mi->start[lo]; }
	*n = 0;
	return 0;
}

int64_t mm2o_idx_keys(const mm2o_idx_t *mi, const uint64_t **keys, const int64_t **start, const uint64_t **pos)
{
	*keys = mi->key, *start = mi->start, *pos = mi->pos;
	return mi->n_keys;
}

typedef struct { uint32_t n, q_pos; uint32_t q_span:8, flt:1, seg_id:8, is_tandem:1; const uint64_t *cr; } seed_t; /* mmpriv.h:45-51 */

static void heap_down(size_t i, size_t n, uint64_t *l) /* ksort.h:44-56 with '<' */
{
	size_t k = i;
	uint64_t tmp = l[i];
	while ((k = (k << 1) + 1) < n) {
		if (k != n - 1 && l[k] < l[k+1]) ++k;
		if (l[k] < tmp) break;
		l[i] = l[k]; i = k;
	}
	l[i] = tmp;
}
static void heap_make(size_t n, uint64_t *l) /* ksort.h:57-62 */
{
	size_t i;
	for (i = (n >> 1) - 1; i != (size_t)(-1); --i) heap_down(i, n, l);
}

static int mz_flt(mm2o_128_t *mv, int n, int32_t q_occ_max, float q_occ_frac) /* seed.c:5-28; returns the new count */
{
	mm2o_128_t *a;
	int i, j, st;
	if (n <= q_occ_max || q_occ_frac <= 0.0f || q_occ_max <= 0) return n;
	a = (mm2o_128_t*)malloc((size_t)n * sizeof(*a));
	for (i = 0; i < n; ++i) a[i].x = mv[i].x, a[i].y = (uint64_t)i;
	mm2o_radix_sort_128x(a, a + n);
	for (st = 0, i = 1; i <= n; ++i)
		if (i == n || a[i].x != a[st].x) {
			int32_t cnt = i - st;
			if (cnt > q_occ_max && cnt > (size_t)n * q_occ_frac)
				for (j = st; j < i; ++j) mv[a[j].y].x = 0;
			st = i;
		}
	free(a);
	for (i = j = 0; i < n; ++i) if (mv[i].x != 0) mv[j++] = mv[i];
	return j;
}

static void seed_select(int32_t n, seed_t *a, int len, int max_occ, int max_max_occ, int dist) /* seed.c:56-96 */
{
	int32_t i, last0, m;
	uint64_t b[128];
	if (n == 0 || n == 1) return;
	for (i = m = 0; i < n; ++i) if ((int32_t)a[i].n > max_occ) ++m;
	if (m == 0) return;
	for (i = 0, last0 = -1; i <= n; ++i) {
		if (i == n || (int32_t)a[i].n <= max_occ) {
			if (i - last0 > 1) {
				int32_t ps = last0 < 0? 0 : (int32_t)(a[last0].q_pos >> 1);
				int32_t pe = i == n? len : (int32_t)(a[i].q_pos >> 1);
				int32_t j, k, st = last0 + 1, en = i;
				int32_t max_high_occ = (int32_t)((double)(pe - ps) / dist + .499);
				if (max_high_occ > 0) {
					if (max_high_occ > 128) max_high_occ = 128;
					for (j = st, k = 0; j < en && k < max_high_occ; ++j, ++k) b[k] = (uint64_t)a[j].n << 32 | (uint32_t)j;
					heap_make(k, b);
					for (; j < en; ++j)
						if ((int32_t)a[j].n < (int32_t)(b[0] >> 32)) { b[0] = (uint64_t)a[j].n << 32 | (uint32_t)j; heap_down(0, k, b); }
					for (j = 0; j < k; ++j) a[(uint32_t)b[j]].flt = 1;
				}
				for (j = st; j < en; ++j) a[j].flt ^= 1;
				for (j = st; j < en; ++j) if ((int32_t)a[j].n > max_max_occ) a[j].flt = 1;
			}
			last0 = i;
		}
	}
}

static int skip_seed(int64_t flag, uint64_t r, const seed_t *q, const char *qname, int qlen, const mm2o_idx_t *mi, int *is_self) /* map.c:78-100 */
{
	*is_self = 0;
	if (qname && (flag & (F_NO_DIAG | F_NO_DUAL))) {
		const int rid = (int)(r >> 32);
		int cmp = strcmp(qname, mi->name[rid]);
		if ((flag & F_NO_DIAG) && cmp == 0 && mi->len[rid] == qlen) {
			if ((uint32_t)r >> 1 == (q->q_pos >> 1)) return 1;
			if ((r & 1) == (q->q_pos & 1)) *is_self = 1;
		}
		if ((flag & F_NO_DUAL) && cmp > 0) return 1;
	}
	if (flag & (F_FOR_ONLY | F_REV_ONLY)) {
		if ((r & 1) == (q->q_pos & 1)) { if (flag & F_REV_ONLY) return 1; }
		else if (flag & F_FOR_ONLY) return 1;
	}
	return 0;
}

/* collect_minimizers for one segment + mm_seed_mz_flt + collect_seed_hits (map.c:59-76,168-204, map.c:252-254).
 * Outputs are malloc'd: sorted anchors, mini_pos[]; returns the number of anchors. */
int64_t mm2o_collect_seed_hits(const mm2o_idx_t *mi, const char *qname, const char *seq, int qlen, int64_t flag, int mid_occ, float q_occ_frac,
							   int max_max_occ, int occ_dist, mm2o_128_t **a_out, int *rep_len, int *n_mini_pos, uint64_t **mini_pos)
{
	mm2o_128_t *mv = (mm2o_128_t*)malloc(((size_t)qlen + 1) * sizeof(*mv)), *a;
	int n_mv = mm2o_sketch(seq, qlen, mi->w, mi->k, 0, mi->is_hpc, mv), i, n_m0 = 0, n_m = 0, rep_st = 0, rep_en = 0;
	int64_t n_a = 0;
	seed_t *m;
	if (q_occ_frac > 0.0f) n_mv = mz_flt(mv, n_mv, mid_occ, q_occ_frac);
	m = (seed_t*)calloc((size_t)n_mv + 1, sizeof(seed_t));
	*mini_pos = (uint64_t*)malloc(((size_t)n_mv + 1) * 8), *n_mini_pos = 0;
	for (i = 0; i < n_mv; ++i) { /* mm_seed_collect_all */
		int t;
		const uint64_t *cr = mm2o_idx_get(mi, mv[i].x >> 8, &t);
		seed_t *q;
		if (t == 0) continue;
		q = &m[n_m0++];
		q->q_pos = (uint32_t)mv[i].y, q->q_span = mv[i].x & 0xff, q->cr = cr, q->n = t, q->seg_id = mv[i].y >> 32;
		q->is_tandem = q->flt = 0;
		if (i > 0 && mv[i].x >> 8 == mv[i-1].x >> 8) q->is_tandem = 1;
		if (i < n_mv - 1 && mv[i].x >> 8 == mv[i+1].x >> 8) q->is_tandem = 1;
	}
	if (occ_dist > 0 && max_max_occ > mid_occ) seed_select(n_m0, m, qlen, mid_occ, max_max_occ, occ_dist);
	else for (i = 0; i < n_m0; ++i) if ((int32_t)m[i].n > mid_occ) m[i].flt = 1;
	for (i = 0, *rep_len = 0; i < n_m0; ++i) { /* seed.c:113-130 */
		seed_t *q = &m[i];
		if (q->flt) {
			int en = (int)(q->q_pos >> 1) + 1, st = en - (int)q->q_span;
			if (st > rep_en) { *rep_len += rep_en - rep_st; rep_st = st, rep_en = en; }
			else rep_en = en;
		} else {
			n_a += q->n;
			(*mini_pos)[(*n_mini_pos)++] = (uint64_t)q->q_span << 32 | q->q_pos >> 1;
			m[n_m++] = *q;
		}
	}
	*rep_len += rep_en - rep_st;
	a = (mm2o_128_t*)malloc(((size_t)n_a + 1) * sizeof(*a));
	for (i = 0, n_a = 0; i < n_m; ++i) { /* map.c:176-199 */
		const seed_t *q = &m[i];
		uint32_t k;
		for (k = 0; k < q->n; ++k) {
			const uint64_t r = q->cr[k];
			int is_self;
			int32_t rpos = (int32_t)((uint32_t)r >> 1);
			mm2o_128_t *p;
			if (skip_seed(flag, r, q, qname, qlen, mi, &is_self)) continue;
			p = &a[n_a++];
			if ((r & 1) == (q->q_pos & 1)) {
				p->x = (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
				p->y = (uint64_t)q->q_span << 32 | q->q_pos >> 1;
			} else if (!(flag & F_QSTRAND)) {
				p->x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
				p->y = (uint64_t)q->q_span << 32 | (uint32_t)(qlen - ((int32_t)(q->q_pos >> 1) + 1 - (int32_t)q->q_span) - 1);
			} else {
				int32_t len = mi->len[r >> 32];
				p->x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)(len - (rpos + 1 - (int32_t)q->q_span) - 1);
				p->y = (uint64_t)q->q_span << 32 | q->q_pos >> 1;
			}
			p->y |= (uint64_t)q->seg_id << SEED_SEG_SHIFT;
			if (q->is_tandem) p->y |= SEED_TANDEM;
			if (is_self) p->y |= SEED_SELF;
		}
	}
	mm2o_radix_sort_128x(a, a + n_a);
	free(m); free(mv);
	*a_out = a;
	return n_a;
}
