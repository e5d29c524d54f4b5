// minimap2_b200/csrc/jump.cuh -- K5: junction jumps of spliced hits (mm_jump_split, jump.c:5-201). Included once, by map.cu.
// The device decides, for each hit, whether its left end and then its right end move across an entry of the index's jump table
// (mm_idx_jjump_read); the host applies the decisions to the hit and its CIGAR (mmb_jump_apply). The read bases stay on the device.
#pragma once
#include "mmb_internal.h"
#include "index.h"
#include "annot.h"
#include "mm_algo.cuh"

#define MMX_MIN_EXON_LEN 20 // jump.c:5

// the hit fields a decision reads; the left decision's effect on them is what the right decision sees
struct JumpState { int32_t rs, re, qs, qe, n_cigar; uint32_t first, last; };

// mm_jump_check (jump.c:7-22) as written: the clip it tests is the one of the opposite end for forward hits
MM_HD bool jump_check(const JumpState &s, int32_t rev, int32_t qlen, int32_t seq_len, int32_t ext, int is_left)
{
	if (s.n_cigar <= 0) return false;
	const int e = !rev ^ !is_left;
	const int32_t clip = e == 0? s.qs : qlen - s.qe;
	const uint32_t c = is_left? s.first : s.last;
	const int32_t clen = (c & 0xf) == MM_CIGAR_MATCH? (int32_t)(c >> 4) : 0;
	if (clen <= ext) return false;
	return is_left? clip < s.rs : clip < seq_len - s.re;
}

struct JumpArgs {
	const mmb_jump_hit_t *hits; int n_hits;
	const uint8_t *seq;                          // the batch's reads, nt4
	const uint32_t *S; const uint64_t *seq_off; const uint32_t *seq_len;
	const int64_t *jump_off; const mm_idx_jjump1_t *jump; // per-contig entry offsets (n_seq+1), entries
	int32_t ext, jump_min_match;
	mmb_jump_dec_t *out;
};

// One end of one hit (mm_jump_split_left / _right, jump.c:50-194), by a whole warp: candidates in table order, the bases of each
// compared 32 at a time (warp sums). A candidate is abandoned as soon as it cannot match (mm1 > 0 or mm2 > 1): the decision does not change.
__device__ mmb_jump_side_t jump_side(const JumpArgs &A, const mmb_jump_hit_t &h, const JumpState &s, int is_left, int lane)
{
	mmb_jump_side_t d = {0, 0, 0, 0, 0};
	const int32_t ext = A.ext, seq_len = (int32_t)A.seq_len[h.rid];
	if (!jump_check(s, h.rev, h.qlen, seq_len, ext + MMX_MIN_EXON_LEN, is_left)) return d;
	const int32_t clip = is_left? (!h.rev? s.qs : h.qlen - s.qe) : (!h.rev? h.qlen - s.qe : s.qs);
	const int32_t extt = clip < ext? clip : ext, L = clip + ext;
	int32_t n;
	const int64_t j0 = A.jump_off[h.rid];
	const mm_idx_jjump1_t *a = mmx_jump_get((int32_t)(A.jump_off[h.rid + 1] - j0), A.jump + j0, seq_len,
											is_left? s.rs - extt : s.re - ext, is_left? s.rs + ext : s.re + extt, &n);
	const uint8_t *q = A.seq + h.q_off;
	const uint64_t t0 = A.seq_off[h.rid];
	int32_t i0_anno = -1, n_anno = 0, mm0_anno = 0, i0_misc = -1, n_misc = 0, mm0_misc = 0;
	for (int32_t i = 0; i < n; ++i) {
		const int32_t off = a[i].off, off2 = a[i].off2;
		int32_t tl1;
		if (is_left) {
			if (off2 >= off || off - off2 < 6 || off2 < L) continue; // wrong direction / intron too small / not long enough
			tl1 = clip + (off - s.rs);
		} else {
			if (off2 <= off || off2 - off < 6 || off2 + L > seq_len) continue;
			tl1 = clip + (s.re - off);
		}
		// left: query [0,tl1) against the target before off2 (mm1), the rest against [off, rs+ext) (mm2);
		// right: query [0,L-tl1) against [re-ext, off) (mm2), the rest against [off2, off2+tl1) (mm1)
		const int32_t cut = is_left? tl1 : L - tl1;
		int32_t mm1 = 0, mm2 = 0;
		for (int32_t j00 = 0; j00 < L; j00 += 32) {
			const int32_t j = j00 + lane;
			bool mis1 = false, mis2 = false;
			if (j < L) {
				uint8_t c;
				if (!h.rev) c = q[is_left? j : h.qlen - L + j];
				else { c = q[is_left? h.qlen - 1 - j : L - 1 - j]; c = c >= 4? c : 3 - c; }
				int64_t tp;
				if (is_left) tp = j < tl1? (int64_t)off2 - tl1 + j : (int64_t)off + (j - tl1);
				else tp = j < cut? (int64_t)s.re - ext + j : (int64_t)off2 + (j - cut);
				const uint32_t t = mmx_seq4_get(A.S, t0 + (uint64_t)tp);
				const bool mis = c != t || c > 3 || t > 3;
				if (j < cut) (is_left? mis1 : mis2) = mis;
				else (is_left? mis2 : mis1) = mis;
			}
			mm1 += __reduce_add_sync(0xffffffffu, (int)mis1);
			mm2 += __reduce_add_sync(0xffffffffu, (int)mis2);
			if (mm1 > 0 || mm2 > 1) break;
		}
		if (mm1 == 0 && mm2 <= 1) { // left keeps the last match, right the first (jump.c:89-92, 161-167)
			if (a[i].flag & MM_JUNC_ANNO) {
				if (is_left || i0_anno < 0) i0_anno = i, mm0_anno = mm2;
				++n_anno;
			} else {
				if (is_left || i0_misc < 0) i0_misc = i, mm0_misc = mm2;
				++n_misc;
			}
		}
	}
	const int32_t m = n_anno > 0? n_anno : n_misc, i0 = n_anno > 0? i0_anno : i0_misc;
	if (m == 0) return d;
	d.off = a[i0].off, d.off2 = a[i0].off2, d.mm0 = n_anno > 0? mm0_anno : mm0_misc;
	d.l = is_left? d.off - s.rs : s.re - d.off;
	if (m == 1 && clip + d.l >= A.jump_min_match) d.act = 2;
	else if (is_left? d.off > s.rs : s.re > d.off) d.act = 1;
	return d;
}

// the left decision's effect on what the right decision reads (the same edits mmb_jump_apply makes)
MM_HD void jump_left_effect(JumpState &s, const mmb_jump_side_t &d, int32_t rev, int32_t qlen)
{
	const int32_t clip = !rev? s.qs : qlen - s.qe;
	if (d.act == 2) {
		const uint32_t third = (uint32_t)((int32_t)(s.first >> 4) - d.l) << 4 | MM_CIGAR_MATCH; // the old first op after the new exon
		if (s.n_cigar == 1) s.last = third;
		s.first = (uint32_t)(clip + d.l) << 4 | MM_CIGAR_MATCH;
		s.n_cigar += 2;
		s.rs = d.off2 - (clip + d.l);
		if (!rev) s.qs = 0; else s.qe = qlen;
	} else if (d.act == 1) {
		s.first -= (uint32_t)d.l << 4;
		if (s.n_cigar == 1) s.last = s.first;
		s.rs += d.l;
		if (!rev) s.qs += d.l; else s.qe -= d.l;
	}
}

__global__ void __launch_bounds__(256) jump_kernel(JumpArgs A)
{
	const int w = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
	if (w >= A.n_hits) return;
	const mmb_jump_hit_t h = A.hits[w];
	JumpState s = {h.rs, h.re, h.qs, h.qe, h.n_cigar, h.cig_first, h.cig_last};
	mmb_jump_dec_t d;
	d.side[0] = jump_side(A, h, s, 1, lane);
	jump_left_effect(s, d.side[0], h.rev, h.qlen);
	d.side[1] = jump_side(A, h, s, 0, lane);
	if (lane == 0) A.out[w] = d;
}

// whether K5 has anything to decide for this hit: mm_jump_check of either end (the right end's check on the hit as it is; when the
// left end changes the hit, the hit is in the batch anyway)
bool mmb_jump_wanted(const mm_idx_t *mi, const mm_mapopt_t *opt, int qlen, const mm_reg1_t *r)
{
	if (r->p == 0 || r->p->n_cigar == 0) return false;
	const int32_t ext = 1 + (opt->b + opt->a - 1) / opt->a + 1 + MMX_MIN_EXON_LEN;
	const JumpState s = {r->rs, r->re, r->qs, r->qe, (int32_t)r->p->n_cigar, r->p->cigar[0], r->p->cigar[r->p->n_cigar - 1]};
	const int32_t len = (int32_t)mi->seq[r->rid].len;
	return jump_check(s, r->rev, qlen, len, ext, 1) || jump_check(s, r->rev, qlen, len, ext, 0);
}

// mm_enlarge_cigar (align.c:305-318) for an r->p that exists
static void jump_enlarge_cigar(mm_reg1_t *r, uint32_t n_cigar)
{
	if (r->p->n_cigar + n_cigar + sizeof(mm_extra_t) / 4 > r->p->capacity) {
		uint32_t c = r->p->n_cigar + n_cigar + sizeof(mm_extra_t) / 4;
		--c, c |= c >> 1, c |= c >> 2, c |= c >> 4, c |= c >> 8, c |= c >> 16, ++c; // kroundup32
		r->p->capacity = c;
		r->p = (mm_extra_t*)realloc(r->p, (size_t)c * 4);
	}
}

// the edits of jump.c:100-119 (left) and 175-193 (right). A trim leaves blen, mlen and the scores as they were, as the reference does.
extern "C" void mmb_jump_apply(const mm_mapopt_t *opt, int qlen, mm_reg1_t *r, const mmb_jump_dec_t *dec)
{
	for (int side = 0; side < 2; ++side) {
		const mmb_jump_side_t &d = dec->side[side];
		if (d.act == 0) continue;
		const int32_t l = d.l, clip = side == 0? (!r->rev? r->qs : qlen - r->qe) : (!r->rev? qlen - r->qe : r->qs);
		if (d.act == 1) { // trim by l (l > 0)
			if (side == 0) {
				r->p->cigar[0] -= (uint32_t)l << 4 | MM_CIGAR_MATCH;
				r->rs += l;
				if (!r->rev) r->qs += l; else r->qe -= l;
			} else {
				r->p->cigar[r->p->n_cigar - 1] -= (uint32_t)l << 4 | MM_CIGAR_MATCH;
				r->re -= l;
				if (!r->rev) r->qe -= l; else r->qs += l;
			}
			continue;
		}
		jump_enlarge_cigar(r, 2); // add one more exon
		uint32_t *c = r->p->cigar;
		if (side == 0) {
			memmove(c + 2, c, r->p->n_cigar * 4);
			c[0] = (uint32_t)(clip + l) << 4 | MM_CIGAR_MATCH;
			c[1] = (uint32_t)(d.off - d.off2) << 4 | MM_CIGAR_N_SKIP;
			c[2] = (uint32_t)((int32_t)(c[2] >> 4) - l) << 4 | MM_CIGAR_MATCH;
			r->rs = d.off2 - (clip + l);
			if (!r->rev) r->qs = 0; else r->qe = qlen;
		} else {
			const uint32_t nc = r->p->n_cigar;
			c[nc - 1] = (uint32_t)((int32_t)(c[nc - 1] >> 4) - l) << 4 | MM_CIGAR_MATCH;
			c[nc] = (uint32_t)(d.off2 - d.off) << 4 | MM_CIGAR_N_SKIP;
			c[nc + 1] = (uint32_t)(clip + l) << 4 | MM_CIGAR_MATCH;
			r->re = d.off2 + (clip + l);
			if (!r->rev) r->qe = qlen; else r->qs = 0;
		}
		r->p->n_cigar += 2;
		r->blen += clip, r->mlen += clip - d.mm0;
		r->p->dp_max0 += (clip - d.mm0) * opt->a - d.mm0 * opt->b;
		r->p->dp_max += (clip - d.mm0) * opt->a - d.mm0 * opt->b;
		if (!r->is_spliced) r->is_spliced = 1, r->p->dp_max += (opt->a + opt->b) + ((opt->a + opt->b) >> 1);
	}
}
