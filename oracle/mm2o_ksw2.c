/* oracle/mm2o_ksw2.c -- TEST INFRASTRUCTURE ONLY (see mm2o.h).
 *
 * Scalar restatement of the reference's SSE ksw2 kernels. The reference has no scalar ksw2, so the SSE
 * code is the specification, including what its 16-byte chunking does at band edges
 * (ksw2_extd2_sse.c:146-184). This file models one byte lane at a time over the same flat arrays
 * (u|v|x|y|x2|y2|s, each tlen_*16 bytes, zero/(-q-e)-initialised exactly as ksw2_extd2_sse.c:107-116).
 */
#include <stdlib.h>
#include <string.h>
#include "mm2o.h"

static void ez_reset(mm2o_ez_t *ez) /* ksw2.h:164-169 */
{
	ez->max_q = ez->max_t = ez->mqe_t = ez->mte_q = -1;
	ez->max = 0, ez->score = ez->mqe = ez->mte = MM2O_KSW_NEG_INF;
	ez->n_cigar = 0, ez->zdropped = 0, ez->reach_end = 0;
}

static void push_cigar(mm2o_ez_t *ez, uint32_t op, int len) /* ksw2.h:114-124 */
{
	if (ez->n_cigar == 0 || op != (ez->cigar[ez->n_cigar - 1] & 0xf)) {
		if (ez->n_cigar == ez->m_cigar) {
			ez->m_cigar = ez->m_cigar? ez->m_cigar << 1 : 4;
			ez->cigar = (uint32_t*)realloc(ez->cigar, (size_t)ez->m_cigar << 2);
		}
		ez->cigar[ez->n_cigar++] = (uint32_t)len << 4 | op;
	} else ez->cigar[ez->n_cigar - 1] += (uint32_t)len << 4;
}

/* ksw2.h:130-162, rotated (anti-diagonal) layout only */
static void backtrack_rot(mm2o_ez_t *ez, int is_rev, int min_intron_len, const uint8_t *p, const int *off, const int *off_end,
						  int n_col, int i0, int j0)
{
	int i = i0, j = j0, state = 0;
	ez->n_cigar = 0;
	while (i >= 0 && j >= 0) {
		int r = i + j, force = -1;
		uint32_t tmp;
		if (i < off[r]) force = 2;
		if (i > off_end[r]) force = 1;
		tmp = force < 0? p[(size_t)r * n_col + i - off[r]] : 0;
		if (state == 0) state = tmp & 7;
		else if (!(tmp >> (state + 2) & 1)) state = 0;
		if (state == 0) state = tmp & 7;
		if (force >= 0) state = force;
		if (state == 0) push_cigar(ez, 0, 1), --i, --j;
		else if (state == 1 || (state == 3 && min_intron_len <= 0)) push_cigar(ez, 2, 1), --i;
		else if (state == 3 && min_intron_len > 0) push_cigar(ez, 3, 1), --i;
		else push_cigar(ez, 1, 1), --j;
	}
	if (i >= 0) push_cigar(ez, min_intron_len > 0 && i >= min_intron_len? 3 : 2, i + 1);
	if (j >= 0) push_cigar(ez, 1, j + 1);
	if (!is_rev) {
		int k;
		for (k = 0; k < ez->n_cigar >> 1; ++k) {
			uint32_t t = ez->cigar[k];
			ez->cigar[k] = ez->cigar[ez->n_cigar - 1 - k], ez->cigar[ez->n_cigar - 1 - k] = t;
		}
	}
}

static int apply_zdrop_rot(mm2o_ez_t *ez, int32_t H, int r, int t, int zdrop, int e) /* ksw2.h:171-187 */
{
	if (H > ez->max) {
		ez->max = H, ez->max_t = t, ez->max_q = r - t;
	} else if (t >= ez->max_t && r - t >= ez->max_q) {
		int tl = t - ez->max_t, ql = (r - t) - ez->max_q, l;
		l = tl > ql? tl - ql : ql - tl;
		if (zdrop >= 0 && ez->max - H > zdrop + l * e) {
			ez->zdropped = 1;
			return 1;
		}
	}
	return 0;
}

#define I8(v) ((int8_t)(v))

void mm2o_extd2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
				int q_, int e_, int q2_, int e2_, int w, int zdrop, int end_bonus, int flag, mm2o_ez_t *ez)
{
	int8_t q = I8(q_), e = I8(e_), q2 = I8(q2_), e2 = I8(e2_);
	const int qe0 = q + e; /* :68: taken before the swap below, so H(0,0) keeps the caller's first gap pair */
	int r, t, n_col, tlen16, qlen16, last_st, last_en, max_sc, min_sc, long_thres, long_diff;
	int with_cigar = !(flag & MM2O_EZ_SCORE_ONLY), approx_max = !!(flag & MM2O_EZ_APPROX_MAX), right = !!(flag & MM2O_EZ_RIGHT);
	int8_t *u, *v, *x, *y, *x2, *y2, *s, *ou, *ov, *ox, *oy, *ox2, *oy2;
	int8_t sc_mch, sc_mis, sc_N, qe, qe2;
	uint8_t *sf, *qr, *p = 0;
	int *off = 0, *off_end = 0;
	int32_t *H = 0, H0 = 0, last_H0_t = 0;

	ez->cigar = 0, ez->m_cigar = 0;
	ez_reset(ez);
	if (m <= 1 || qlen <= 0 || tlen <= 0) return;
	if (q2 + e2 < q + e) { int8_t tt; tt = q, q = q2, q2 = tt, tt = e, e = e2, e2 = tt; } /* :78 */
	qe = I8(q + e), qe2 = I8(q2 + e2);
	sc_mch = mat[0], sc_mis = mat[1];
	sc_N = mat[m*m-1] == 0? I8(-e2) : mat[m*m-1]; /* :87 */
	if (w < 0) w = tlen > qlen? tlen : qlen;
	tlen16 = (tlen + 15) / 16 * 16;
	qlen16 = (qlen + 15) / 16 * 16;
	n_col = qlen < tlen? qlen : tlen;
	n_col = (((n_col < w + 1? n_col : w + 1) + 15) / 16 + 1) * 16; /* :93-94, in bytes */
	for (t = 1, max_sc = mat[0], min_sc = mat[1]; t < m * m; ++t) {
		max_sc = max_sc > mat[t]? max_sc : mat[t];
		min_sc = min_sc < mat[t]? min_sc : mat[t];
	}
	if (-min_sc > 2 * (q + e)) return; /* :100 */
	long_thres = e != e2? (q2 - q) / (e - e2) - 1 : 0; /* :102-105 */
	if (q2 + e2 + long_thres * e2 > q + e + long_thres * e) ++long_thres;
	long_diff = long_thres * (e - e2) - (q2 - q) - e2;

	u = (int8_t*)malloc((size_t)tlen16 * 13);
	v = u + tlen16, x = v + tlen16, y = x + tlen16, x2 = y + tlen16, y2 = x2 + tlen16, s = y2 + tlen16;
	ou = s + tlen16, ov = ou + tlen16, ox = ov + tlen16, oy = ox + tlen16, ox2 = oy + tlen16, oy2 = ox2 + tlen16;
	memset(u, -q - e, tlen16), memset(v, -q - e, tlen16), memset(x, -q - e, tlen16), memset(y, -q - e, tlen16);
	memset(x2, -q2 - e2, tlen16), memset(y2, -q2 - e2, tlen16);
	memset(s, 0, tlen16);
	sf = (uint8_t*)calloc(tlen16 + qlen16 + 32, 1); /* sf then qr contiguous as in :109-110 (+16 zero slack) */
	qr = sf + tlen16;
	memcpy(sf, target, tlen);
	for (t = 0; t < qlen; ++t) qr[t] = query[qlen - 1 - t];
	if (!approx_max) {
		H = (int32_t*)malloc((size_t)tlen16 * 4);
		for (t = 0; t < tlen16; ++t) H[t] = MM2O_KSW_NEG_INF;
	}
	if (with_cigar) {
		p = (uint8_t*)malloc((size_t)(qlen + tlen - 1) * n_col + 16);
		off = (int*)malloc((size_t)(qlen + tlen - 1) * sizeof(int) * 2);
		off_end = off + qlen + tlen - 1;
	}

	for (r = 0, last_st = last_en = -1; r < qlen + tlen - 1; ++r) {
		int st = 0, en = tlen - 1, st0, en0;
		int8_t x1, x21, v1;
		const uint8_t *qrr = qr + (qlen - 1 - r);
		if (st < r - qlen + 1) st = r - qlen + 1;
		if (en > r) en = r;
		if (st < (r - w + 1) >> 1) st = (r - w + 1) >> 1;
		if (en > (r + w) >> 1) en = (r + w) >> 1;
		if (st > en) { ez->zdropped = 1; break; }
		st0 = st, en0 = en;
		st = st / 16 * 16, en = (en + 16) / 16 * 16 - 1;
		if (st > 0) { /* :149-163 */
			if (st - 1 >= last_st && st - 1 <= last_en) x1 = x[st - 1], x21 = x2[st - 1], v1 = v[st - 1];
			else x1 = I8(-q - e), x21 = I8(-q2 - e2), v1 = I8(-q - e);
		} else {
			x1 = I8(-q - e), x21 = I8(-q2 - e2);
			v1 = r == 0? I8(-q - e) : r < long_thres? I8(-e) : r == long_thres? I8(long_diff) : I8(-e2);
		}
		if (en >= r) {
			y[r] = I8(-q - e), y2[r] = I8(-q2 - e2);
			u[r] = r == 0? I8(-q - e) : r < long_thres? I8(-e) : r == long_thres? I8(long_diff) : I8(-e2);
		}
		/* scores: 16-byte chunks from st0 (:165-184) */
		if (!(flag & MM2O_EZ_GENERIC_SC)) {
			int t0;
			for (t0 = st0; t0 <= en0; t0 += 16)
				for (t = t0; t < t0 + 16 && t < tlen16; ++t) { /* lanes >= tlen16 spill into sf[] but are never read */
					uint8_t sq = sf[t], sr = qrr[t];
					int8_t sc = sq == sr? sc_mch : sc_mis;
					if (sq == (uint8_t)(m - 1) || sr == (uint8_t)(m - 1)) sc = sc_N;
					s[t] = sc;
				}
		} else {
			for (t = st0; t <= en0; ++t) s[t] = mat[sf[t] * m + qrr[t]];
		}
		/* core: all lanes st..en read row r-1 values (Jacobi), lane st gets the x1/v1 scalars */
		memcpy(ou, u, tlen16), memcpy(ov, v, tlen16), memcpy(ox, x, tlen16);
		memcpy(oy, y, tlen16), memcpy(ox2, x2, tlen16), memcpy(oy2, y2, tlen16);
		if (with_cigar) off[r] = st, off_end[r] = en;
		for (t = st; t <= en; ++t) {
			int8_t z = s[t], xt1, vt1, x2t1, ut, a, b, a2, b2, tmp, d = 0;
			xt1 = t == st? x1 : ox[t - 1];
			vt1 = t == st? v1 : ov[t - 1];
			x2t1 = t == st? x21 : ox2[t - 1];
			ut = ou[t];
			a = I8(xt1 + vt1), b = I8(oy[t] + ut), a2 = I8(x2t1 + vt1), b2 = I8(oy2[t] + ut);
			if (!with_cigar) {
				z = z > a? z : a; z = z > b? z : b; z = z > a2? z : a2; z = z > b2? z : b2;
				z = z < sc_mch? z : sc_mch;
			} else if (!right) { /* :232-243 */
				d = a > z? 1 : 0;  z = z > a? z : a;
				d = b > z? 2 : d;  z = z > b? z : b;
				d = a2 > z? 3 : d; z = z > a2? z : a2;
				d = b2 > z? 4 : d; z = z > b2? z : b2;
				z = z < sc_mch? z : sc_mch;
			} else { /* :279-290 */
				d = z > a? 0 : 1;  z = z > a? z : a;
				d = z > b? d : 2;  z = z > b? z : b;
				d = z > a2? d : 3; z = z > a2? z : a2;
				d = z > b2? d : 4; z = z > b2? z : b2;
				z = z < sc_mch? z : sc_mch;
			}
			u[t] = I8(z - vt1), v[t] = I8(z - ut); /* :58-66 */
			tmp = I8(z - q);  a = I8(a - tmp),  b = I8(b - tmp);
			tmp = I8(z - q2); a2 = I8(a2 - tmp), b2 = I8(b2 - tmp);
			if (!with_cigar || !right) { /* "a > 0" variant */
				x[t]  = I8((a  > 0? a  : 0) - qe);  if (a  > 0) d |= 0x08;
				y[t]  = I8((b  > 0? b  : 0) - qe);  if (b  > 0) d |= 0x10;
				x2[t] = I8((a2 > 0? a2 : 0) - qe2); if (a2 > 0) d |= 0x20;
				y2[t] = I8((b2 > 0? b2 : 0) - qe2); if (b2 > 0) d |= 0x40;
			} else { /* right-aligned: "!(0 > a)" (:308-320) */
				x[t]  = I8((0 > a?  0 : a)  - qe);  if (!(0 > a))  d |= 0x08;
				y[t]  = I8((0 > b?  0 : b)  - qe);  if (!(0 > b))  d |= 0x10;
				x2[t] = I8((0 > a2? 0 : a2) - qe2); if (!(0 > a2)) d |= 0x20;
				y2[t] = I8((0 > b2? 0 : b2) - qe2); if (!(0 > b2)) d |= 0x40;
			}
			if (with_cigar) p[(size_t)r * n_col + (t - st)] = (uint8_t)d;
		}
		if (!approx_max) { /* :323-366 */
			int32_t max_H, max_t;
			if (r > 0) {
				int32_t HH[4], tt[4], en1 = st0 + (en0 - st0) / 4 * 4, i;
				max_H = H[en0] = en0 > 0? H[en0 - 1] + u[en0] : H[en0] + v[en0];
				max_t = en0;
				for (i = 0; i < 4; ++i) HH[i] = max_H, tt[i] = max_t;
				for (t = st0; t < en1; t += 4)
					for (i = 0; i < 4; ++i) {
						H[t + i] += v[t + i];
						if (H[t + i] > HH[i]) HH[i] = H[t + i], tt[i] = t; /* lane keeps the block start t */
					}
				for (i = 0; i < 4; ++i)
					if (max_H < HH[i]) max_H = HH[i], max_t = tt[i] + i;
				for (; t < en0; ++t) {
					H[t] += (int32_t)v[t];
					if (H[t] > max_H) max_H = H[t], max_t = t;
				}
			} else H[0] = v[0] - qe0, max_H = H[0], max_t = 0; /* :358 */
			if (en0 == tlen - 1 && H[en0] > ez->mte) ez->mte = H[en0], ez->mte_q = r - en0;
			if (r - st0 == qlen - 1 && H[st0] > ez->mqe) ez->mqe = H[st0], ez->mqe_t = st0;
			if (apply_zdrop_rot(ez, max_H, r, max_t, zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez->score = H[tlen - 1];
		} else { /* :367-383 */
			if (r > 0) {
				if (last_H0_t >= st0 && last_H0_t <= en0 && last_H0_t + 1 >= st0 && last_H0_t + 1 <= en0) {
					int32_t d0 = v[last_H0_t], d1 = u[last_H0_t + 1];
					if (d0 > d1) H0 += d0;
					else H0 += d1, ++last_H0_t;
				} else if (last_H0_t >= st0 && last_H0_t <= en0) {
					H0 += v[last_H0_t];
				} else {
					++last_H0_t, H0 += u[last_H0_t];
				}
			} else H0 = v[0] - qe0, last_H0_t = 0; /* :379 */
			if ((flag & MM2O_EZ_APPROX_DROP) && apply_zdrop_rot(ez, H0, r, last_H0_t, zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez->score = H0;
		}
		last_st = st, last_en = en;
	}
	free(u); free(sf); free(H);
	if (with_cigar) { /* :388-400 */
		int rev_cigar = !!(flag & MM2O_EZ_REV_CIGAR);
		if (!ez->zdropped && !(flag & MM2O_EZ_EXTZ_ONLY)) {
			backtrack_rot(ez, rev_cigar, 0, p, off, off_end, n_col, tlen - 1, qlen - 1);
		} else if (!ez->zdropped && (flag & MM2O_EZ_EXTZ_ONLY) && ez->mqe + end_bonus > ez->max) {
			ez->reach_end = 1;
			backtrack_rot(ez, rev_cigar, 0, p, off, off_end, n_col, ez->mqe_t, qlen - 1);
		} else if (ez->max_t >= 0 && ez->max_q >= 0) {
			backtrack_rot(ez, rev_cigar, 0, p, off, off_end, n_col, ez->max_t, ez->max_q);
		}
		free(p); free(off);
	}
}

/* ksw2_ll_sse.c:37-152. The striped layout only matters for (a) int16 saturation and (b) which query end is
 * reported on ties (the LAST striped slot with H==gmax, :148-150), so lanes are modelled as slot = seg + k*slen. */
int mm2o_ll_i16(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
				int gapo, int gape, int *qe, int *te)
{
	int slen = (qlen + 7) / 8, n = slen * 8, i, j, k, gmax = 0;
	/* striped arrays: vector j, lane k <-> query position j + k*slen; stored [j*8+k] */
	int16_t *H0 = (int16_t*)calloc(n, 2), *H1 = (int16_t*)calloc(n, 2), *E = (int16_t*)calloc(n, 2), *Hmax = (int16_t*)calloc(n, 2);
	uint16_t go = (uint16_t)(gapo + gape), ge = (uint16_t)gape;
#define QPOS(j,k) ((j) + (k) * slen)
#define SUBS_U16(a,b) ((uint16_t)(a) > (uint16_t)(b)? (int16_t)((uint16_t)(a) - (uint16_t)(b)) : (int16_t)0)
#define MAX16(a,b) ((int16_t)(a) > (int16_t)(b)? (int16_t)(a) : (int16_t)(b))
	*qe = *te = -1;
	for (i = 0; i < tlen; ++i) {
		int16_t h[8], f[8], mx[8], e8[8], imax;
		const int8_t *ma = mat + target[i] * m;
		int done = 0;
		for (k = 0; k < 8; ++k) f[k] = 0, mx[k] = 0;
		/* h = H0[slen-1] shifted by one lane */
		h[0] = 0;
		for (k = 1; k < 8; ++k) h[k] = H0[(slen - 1) * 8 + k - 1];
		for (j = 0; j < slen; ++j) {
			for (k = 0; k < 8; ++k) {
				int qp = QPOS(j, k);
				int16_t sc = qp >= qlen? -1 : ma[query[qp]];
				int32_t t32 = (int32_t)h[k] + sc; /* _mm_adds_epi16: signed saturation */
				int16_t hh, hs;
				if (t32 > 32767) t32 = 32767;
				if (t32 < -32768) t32 = -32768;
				hh = (int16_t)t32;
				e8[k] = E[j * 8 + k];
				hh = MAX16(hh, e8[k]);
				hh = MAX16(hh, f[k]);
				mx[k] = MAX16(mx[k], hh);
				H1[j * 8 + k] = hh;
				hs = SUBS_U16(hh, go);
				e8[k] = SUBS_U16(e8[k], ge);
				e8[k] = MAX16(e8[k], hs);
				E[j * 8 + k] = e8[k];
				f[k] = SUBS_U16(f[k], ge);
				f[k] = MAX16(f[k], hs);
				h[k] = H0[j * 8 + k];
			}
		}
		for (k = 0; k < 8 && !done; ++k) { /* lazy-F loop (:124-135) */
			int kk;
			for (kk = 7; kk > 0; --kk) f[kk] = f[kk - 1];
			f[0] = 0;
			for (j = 0; j < slen; ++j) {
				int any = 0;
				for (kk = 0; kk < 8; ++kk) {
					int16_t hh = H1[j * 8 + kk], hs;
					hh = MAX16(hh, f[kk]);
					H1[j * 8 + kk] = hh;
					hs = SUBS_U16(hh, go);
					f[kk] = SUBS_U16(f[kk], ge);
					if ((int16_t)f[kk] > (int16_t)hs) any = 1;
				}
				if (!any) { done = 1; break; }
			}
		}
		imax = mx[0];
		for (k = 1; k < 8; ++k) imax = MAX16(imax, mx[k]);
		if ((int)imax >= gmax) {
			gmax = imax, *te = i;
			memcpy(Hmax, H1, (size_t)n * 2);
		}
		{ int16_t *tmp = H1; H1 = H0; H0 = tmp; }
	}
	/* :148-150: H8[i] over the raw striped memory, i = vector*8 + lane; qe = i/8 + i%8*slen; last match wins */
	for (i = 0; i < n; ++i)
		if ((int)(uint16_t)Hmax[i] == gmax) *qe = i / 8 + i % 8 * slen;
	free(H0); free(H1); free(E); free(Hmax);
	return gmax;
}

void mm2o_free(void *p) { free(p); }
