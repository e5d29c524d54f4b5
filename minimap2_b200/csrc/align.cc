// minimap2_b200/csrc/align.cc -- host side of base-level alignment: chooses DP windows from chains, issues ksw2 jobs to
// the GPU (K3) and stitches CIGARs. Semantics follow the reference's align.c: mm_align_skeleton :1048-1120, mm_align1
// :645-914, mm_align1_inv :916-975, mm_test_zdrop :61-103, mm_update_extra/mm_fix_cigar/eqx :105-303, end/seed filters
// :418-616. The control flow is written as a REPLAYABLE routine: every ksw2 call is looked up in the read's result cache;
// a miss is recorded as a GPU job request and the routine keeps walking (without consuming results) so that all jobs that
// do not depend on the missing one -- the remaining gap fills and the right extension of the region, other regions -- are
// requested in the same wave. The batch scheduler (map.cc) replays a read after each wave until nothing is missing;
// the last replay then executes exactly the reference's sequence of decisions.
#include "hostlogic.h"
#include <emmintrin.h>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <cassert>

#define KSW_NEG_INF_H (-0x40000000)

void hl_gen_mat(int8_t *mat, const mm_mapopt_t *opt) // align.c:11-38 (m = 5)
{
	const int m = 5;
	int8_t aa = (int8_t)(opt->a < 0? -opt->a : opt->a), bb = (int8_t)(opt->b > 0? -opt->b : opt->b);
	int8_t sa = (int8_t)(opt->sc_ambi > 0? -opt->sc_ambi : opt->sc_ambi);
	for (int i = 0; i < m - 1; ++i) {
		for (int j = 0; j < m - 1; ++j) mat[i * m + j] = i == j? aa : bb;
		mat[i * m + m - 1] = sa;
	}
	for (int j = 0; j < m; ++j) mat[(m - 1) * m + j] = sa;
	if (opt->transition == 0 || opt->transition == opt->b) return;
	int8_t t = (int8_t)(opt->transition > 0? -opt->transition : opt->transition);
	mat[0 * m + 2] = t, mat[1 * m + 3] = t, mat[2 * m + 0] = t, mat[3 * m + 1] = t;
}

namespace {

struct Ez {
	int max, zdropped, max_q, max_t, mqe, mqe_t, mte, mte_q, score, n_cigar, reach_end;
	const uint32_t *cigar;
	const uint32_t *dcigar;   // device copy of the CIGAR (K4 input)
	int zd_max, zd_pos[2][2]; // mm_test_zdrop's scan evaluated by the kernel (MMB_JOB_ZDROP); zd_max < 0: not available
};

inline void ez_reset(Ez *ez) // ksw2.h:164-169
{
	ez->max_q = ez->max_t = ez->mqe_t = ez->mte_q = -1;
	ez->max = 0, ez->score = ez->mqe = ez->mte = KSW_NEG_INF_H;
	ez->n_cigar = 0, ez->zdropped = 0, ez->reach_end = 0, ez->cigar = 0, ez->dcigar = 0;
	ez->zd_max = -1;
}

struct Seg { // a piece of the query (on strand `rev`, strand coordinates) and of the target
	int rev, qs, qlen, q_reversed;
	uint32_t rid; int rs, tlen, t_reversed;
	int t_rc = 0; // query-strand mode, reverse hit: rs counts on the reverse-complement strand of the target (mm_idx_getseq_rev, index.c:176-190)
};

inline uint32_t roundup32(uint32_t x) { --x; x |= x >> 1; x |= x >> 2; x |= x >> 4; x |= x >> 8; x |= x >> 16; return ++x; }

struct Driver {
	const mm_mapopt_t *opt;
	const mm_idx_t *mi;
	ReadAlign &ra;
	int qlen;
	int8_t mat[25];
	bool pending; // set while walking a region whose results are not all available

	Driver(const mm_mapopt_t *o, const mm_idx_t *m, ReadAlign &r) : opt(o), mi(m), ra(r), qlen(r.qlen), pending(false) {
		hl_gen_mat(mat, o);
	}

	KswKey make_key(const Seg &s, int w, int zdrop, int end_bonus, int flag) const {
		KswKey k;
		if (s.rev == 0) {
			if (!s.q_reversed) k.q_start = ra.q_dev_off + s.qs, k.q_step = 1;
			else k.q_start = ra.q_dev_off + s.qs + s.qlen - 1, k.q_step = -1;
		} else {
			flag |= MMB_JOB_Q_COMP;
			if (!s.q_reversed) k.q_start = ra.q_dev_off + qlen - 1 - s.qs, k.q_step = -1;
			else k.q_start = ra.q_dev_off + qlen - s.qs - s.qlen, k.q_step = 1;
		}
		if (!s.t_rc) {
			const int64_t toff = (int64_t)mi->seq[s.rid].offset + s.rs;
			if (!s.t_reversed) k.t_start = toff, k.t_step = 1;
			else k.t_start = toff + s.tlen - 1, k.t_step = -1;
		} else { // element i of the piece is reverse-strand position rs+i = forward position len-1-rs-i, complemented
			const int64_t off = (int64_t)mi->seq[s.rid].offset, len = (int64_t)mi->seq[s.rid].len;
			flag |= MMB_JOB_T_COMP;
			if (!s.t_reversed) k.t_start = off + len - 1 - s.rs, k.t_step = -1;
			else k.t_start = off + len - s.rs - s.tlen, k.t_step = 1;
		}
		k.qlen = s.qlen, k.tlen = s.tlen, k.w = w, k.zdrop = zdrop, k.end_bonus = end_bonus, k.flag = flag;
		return k;
	}

	// cache lookup; on a miss the job is queued for the GPU and false is returned. slot_out (optional) receives the job's cache slot.
	bool fetch(const KswKey &k, Ez *ez, int *slot_out = nullptr) {
		HpScope hp_(HP_FETCH);
		int slot = ra.find(k);
		if (slot_out) *slot_out = slot >= 0? slot : (int)ra.keys.size();
		return fetch_slot(slot, &k, ez);
	}
	// the same for a job whose slot is known (k may be null then)
	bool fetch_slot(int slot, const KswKey *kp, Ez *ez) {
		if (slot >= 0 && ra.done_idx[slot] >= 0) {
			ra.hint = (size_t)slot + 1;
			const KswDone &d = ra.done[ra.done_idx[slot]];
			ez->max = d.r.max, ez->zdropped = d.r.zdropped, ez->max_q = d.r.max_q, ez->max_t = d.r.max_t;
			ez->mqe = d.r.mqe, ez->mqe_t = d.r.mqe_t, ez->mte = d.r.mte, ez->mte_q = d.r.mte_q;
			ez->score = d.r.score, ez->n_cigar = d.r.n_cigar, ez->reach_end = d.r.reach_end;
			ez->cigar = d.cig, ez->dcigar = d.dcig;
			ez->zd_max = d.r.zd_max, ez->zd_pos[0][0] = d.r.zd_t0, ez->zd_pos[0][1] = d.r.zd_t1, ez->zd_pos[1][0] = d.r.zd_q0, ez->zd_pos[1][1] = d.r.zd_q1;
			return true;
		}
		if (slot < 0) {
			const KswKey &k = *kp;
			ra.keys.push_back(k); ra.done_idx.push_back(-1);
			mmb_ksw_job_t j;
			j.q_start = k.q_start, j.t_start = k.t_start, j.q_step = k.q_step, j.t_step = k.t_step;
			j.qlen = k.qlen, j.tlen = k.tlen, j.w = k.w, j.zdrop = k.zdrop, j.end_bonus = k.end_bonus, j.flag = k.flag;
			ra.want.push_back(j);
			ra.want_slot.push_back((int)ra.keys.size() - 1);
		}
		ra.incomplete = true;
		pending = true;
		return false;
	}

	// mm_align_pair (align.c:336-368). Single-affine scoring (q == q2, e == e2: ksw_extz2_sse, align.c:360-361) runs the same
	// dual-affine kernels with both gap terms equal: on every flag combination align.c uses, ksw_extz2_sse(q,e) and
	// ksw_extd2_sse(q,e,q,e) return identical ksw_extz_t and CIGARs (tests/test_oracle_vs_ref.py::test_extz2_is_extd2_with_equal_gaps).
	bool align_pair(const Seg &s, int w, int end_bonus, int zdrop, int ksw_flag, Ez *ez, int *slot = nullptr) {
		if (slot && *slot >= 0) { HpScope hp_(HP_FETCH); return fetch_slot(*slot, nullptr, ez); } // planned job, requested by an earlier replay
		if (opt->transition != 0 && opt->b != opt->transition) ksw_flag |= MMB_KSW_GENERIC_SC;
		if (opt->flag & MM_F_SPLICE) { // ksw_exts2 (align.c:352-355): the splice-model bits travel in the job flag
			ksw_flag |= MMB_JOB_SPLICE;
			if (!(opt->flag & MM_F_SPLICE_OLD)) ksw_flag |= MMB_KSW_SPLICE_CMPLX;
		}
		if (opt->max_sw_mat > 0 && (int64_t)s.tlen * s.qlen > opt->max_sw_mat) {
			ez_reset(ez);
			ez->zdropped = 1;
			return true;
		}
		return fetch(make_key(s, w, zdrop, end_bonus, ksw_flag), ez, slot);
	}

	bool ll_i16(const Seg &s, int *score, int *q_off, int *t_off) { // ksw_ll_qinit + ksw_ll_i16
		Ez ez;
		if (!fetch(make_key(s, opt->q, opt->e, 0, MMB_JOB_LL), &ez)) return false;
		*score = ez.score, *q_off = ez.max_q, *t_off = ez.max_t;
		return true;
	}

	const uint8_t *qptr(int rev, int qs) const { ra.ensure_qseq(); return ra.qseq[rev] + qs; }
	void get_tseq(uint32_t rid, int st, int en, std::vector<uint8_t> &buf, int t_rc = 0) const { // mm_idx_getseq2 (index.c:192-196)
		HpScope hp_(HP_TSEQ);
		buf.resize((en > st? en - st : 0) + 16); // 16 bytes of slack: update_extra compares 16-byte blocks
		if (en <= st) return;
		if (!t_rc) { mm_idx_getseq(mi, rid, st, en, buf.data()); return; }
		const int len = (int)mi->seq[rid].len; // mm_idx_getseq_rev: reverse complement of [len-en, len-st)
		if (en > len) en = len;
		mm_idx_getseq(mi, rid, len - en, len - st, buf.data());
		for (int i = 0, j = en - st - 1; i <= j; ++i, --j) {
			const uint8_t x = buf[i], y = buf[j];
			buf[i] = y < 4? 3 - y : y, buf[j] = x < 4? 3 - x : x;
		}
	}

	static void update_max_zdrop(int32_t score, int i, int j, int32_t *max, int *max_i, int *max_j, int e, int *max_zdrop, int pos[2][2]) { // align.c:46-59
		if (score < *max) {
			int li = i - *max_i, lj = j - *max_j, diff = li > lj? li - lj : lj - li, z = *max - score - diff * e;
			if (z > *max_zdrop) {
				*max_zdrop = z;
				pos[0][0] = *max_i, pos[0][1] = i;
				pos[1][0] = *max_j, pos[1][1] = j;
			}
		} else *max = score, *max_i = i, *max_j = j;
	}

	// align.c:61-103. Returns 0/1/2, or -1 if the inversion probe (ksw_ll_i16) is still pending on the GPU.
	// zd: the scan's result when the kernel already evaluated it (max_zdrop, pos), else null and the CIGAR is scanned here
	int test_zdrop(const Seg &s, const uint8_t *qseq, const uint8_t *tseq, uint32_t n_cigar, const uint32_t *cigar, const Ez *zd) {
		HpScope hp_(HP_ZDROP);
		int32_t score = 0, max = INT32_MIN, max_i = -1, max_j = -1, i = 0, j = 0, max_zdrop = 0;
		int pos[2][2] = {{-1, -1}, {-1, -1}}, q_len, t_len;
		if (zd) {
			max_zdrop = zd->zd_max;
			pos[0][0] = zd->zd_pos[0][0], pos[0][1] = zd->zd_pos[0][1], pos[1][0] = zd->zd_pos[1][0], pos[1][1] = zd->zd_pos[1][1];
		} else for (uint32_t k = 0; k < n_cigar; ++k) {
			uint32_t op = cigar[k] & 0xf, len = cigar[k] >> 4;
			if (op == MM_CIGAR_MATCH) {
				for (uint32_t l = 0; l < len; ++l) {
					score += mat[tseq[i + l] * 5 + qseq[j + l]];
					update_max_zdrop(score, i + l, j + l, &max, &max_i, &max_j, opt->e, &max_zdrop, pos);
				}
				i += len, j += len;
			} else if (op == MM_CIGAR_INS || op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) {
				score -= opt->q + opt->e * len;
				if (op == MM_CIGAR_INS) j += len; else i += len;
				update_max_zdrop(score, i, j, &max, &max_i, &max_j, opt->e, &max_zdrop, pos);
			}
		}
		q_len = pos[1][1] - pos[1][0], t_len = pos[0][1] - pos[0][0];
		if (!(opt->flag & (MM_F_SPLICE|MM_F_SR|MM_F_FOR_ONLY|MM_F_REV_ONLY)) && max_zdrop > opt->zdrop_inv && q_len < opt->max_gap && t_len < opt->max_gap) {
			// reverse complement of query[pos10, pos11) == forward piece of the opposite strand (see make_key)
			Seg v;
			v.rev = 1 - s.rev, v.q_reversed = 0, v.qlen = q_len;
			// strand position of piece element 0: qlen - (s.qs' + pos11) where s.qs' is the forward-orientation start on strand s.rev
			v.qs = qlen - s.qs - pos[1][1]; // test_zdrop is only applied to (non-reversed) gap fills
			v.rid = s.rid, v.rs = s.rs + pos[0][0], v.tlen = t_len, v.t_reversed = 0, v.t_rc = s.t_rc;
			int sc, qo, to;
			if (q_len <= 0 || t_len <= 0) sc = 0; // ksw_ll_i16 on an empty query/target yields 0
			else if (!ll_i16(v, &sc, &qo, &to)) return -1;
			if (sc >= opt->min_chain_score * opt->a && sc >= opt->min_dp_max) return 2;
		}
		return max_zdrop > opt->zdrop? 1 : 0;
	}

	// ---- CIGAR bookkeeping on mm_reg1_t::p (align.c:305-334) ----
	static void enlarge_cigar(mm_reg1_t *r, uint32_t n_cigar) {
		if (n_cigar == 0) return;
		if (r->p == 0) {
			uint32_t capacity = roundup32(n_cigar + sizeof(mm_extra_t) / 4);
			r->p = (mm_extra_t*)calloc(capacity, 4);
			r->p->capacity = capacity;
		} else if (r->p->n_cigar + n_cigar + sizeof(mm_extra_t) / 4 > r->p->capacity) {
			r->p->capacity = roundup32(r->p->n_cigar + n_cigar + sizeof(mm_extra_t) / 4);
			r->p = (mm_extra_t*)realloc(r->p, r->p->capacity * 4);
		}
	}
	static void append_cigar(mm_reg1_t *r, uint32_t n_cigar, const uint32_t *cigar) {
		HpScope hp_(HP_APPEND);
		if (n_cigar == 0) return;
		enlarge_cigar(r, n_cigar);
		mm_extra_t *p = r->p;
		if (p->n_cigar > 0 && (p->cigar[p->n_cigar - 1] & 0xf) == (cigar[0] & 0xf)) {
			p->cigar[p->n_cigar - 1] += cigar[0] >> 4 << 4;
			if (n_cigar > 1) memcpy(p->cigar + p->n_cigar, cigar + 1, (n_cigar - 1) * 4);
			p->n_cigar += n_cigar - 1;
		} else {
			memcpy(p->cigar + p->n_cigar, cigar, n_cigar * 4);
			p->n_cigar += n_cigar;
		}
	}

	// one piece of a hit's CIGAR: appended here, or (device tail) only recorded -- the hit keeps a header-only mm_extra_t for dp_score
	int fin_first = 0; // first piece of the hit being walked
	void add_cigar(mm_reg1_t *r, const Ez &ez) {
		if (!ra.defer) { append_cigar(r, ez.n_cigar, ez.cigar); return; }
		if (ez.n_cigar == 0) return;
		if (r->p == 0) {
			uint32_t capacity = roundup32(sizeof(mm_extra_t) / 4);
			r->p = (mm_extra_t*)calloc(capacity, 4);
			r->p->capacity = capacity;
		}
		HlFinJob j; j.dcig = ez.dcigar, j.n = (uint32_t)ez.n_cigar;
		ra.fin_jobs.push_back(j);
	}

	static void fix_cigar(mm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq, int *qshift, int *tshift) { // align.c:105-181
		mm_extra_t *p = r->p;
		int32_t toff = 0, qoff = 0, to_shrink = 0;
		*qshift = *tshift = 0;
		if (p->n_cigar <= 1) return;
		for (uint32_t k = 0; k < p->n_cigar; ++k) { // left-align indels
			uint32_t op = p->cigar[k] & 0xf, len = p->cigar[k] >> 4;
			if (len == 0) to_shrink = 1;
			if (op == MM_CIGAR_MATCH) toff += len, qoff += len;
			else if (op == MM_CIGAR_INS || op == MM_CIGAR_DEL) {
				if (k > 0 && k < p->n_cigar - 1 && (p->cigar[k-1] & 0xf) == 0 && (p->cigar[k+1] & 0xf) == 0) {
					int l, prev_len = p->cigar[k-1] >> 4;
					if (op == MM_CIGAR_INS) { for (l = 0; l < prev_len; ++l) if (qseq[qoff - 1 - l] != qseq[qoff + len - 1 - l]) break; }
					else { for (l = 0; l < prev_len; ++l) if (tseq[toff - 1 - l] != tseq[toff + len - 1 - l]) break; }
					if (l > 0) p->cigar[k-1] -= l << 4, p->cigar[k+1] += l << 4, qoff -= l, toff -= l;
					if (l == prev_len) to_shrink = 1;
				}
				if (op == MM_CIGAR_INS) qoff += len; else toff += len;
			} else if (op == MM_CIGAR_N_SKIP) toff += len;
		}
		assert(qoff == r->qe - r->qs && toff == r->re - r->rs);
		for (uint32_t k = 0; k + 2 < p->n_cigar; ++k) { // merge runs like 5I6D7I (n_cigar >= 2 here; k < n_cigar-2)
			if ((p->cigar[k] & 0xf) > 0 && (p->cigar[k] & 0xf) + (p->cigar[k+1] & 0xf) == 3) {
				uint32_t l, s[3] = {0, 0, 0};
				for (l = k; l < p->n_cigar; ++l) {
					uint32_t op = p->cigar[l] & 0xf;
					if (op == MM_CIGAR_INS || op == MM_CIGAR_DEL || p->cigar[l] >> 4 == 0) s[op] += p->cigar[l] >> 4;
					else break;
				}
				if (s[1] > 0 && s[2] > 0 && l - k > 2) {
					p->cigar[k] = s[1] << 4 | MM_CIGAR_INS;
					p->cigar[k+1] = s[2] << 4 | MM_CIGAR_DEL;
					for (k += 2; k < l; ++k) p->cigar[k] &= 0xf;
					to_shrink = 1;
				}
				k = l;
			}
		}
		if (to_shrink) {
			int32_t l = 0;
			for (uint32_t k = 0; k < p->n_cigar; ++k) if (p->cigar[k] >> 4 != 0) p->cigar[l++] = p->cigar[k];
			p->n_cigar = l;
			l = 0;
			for (uint32_t k = 0; k < p->n_cigar; ++k)
				if (k == p->n_cigar - 1 || (p->cigar[k] & 0xf) != (p->cigar[k+1] & 0xf)) p->cigar[l++] = p->cigar[k];
				else p->cigar[k+1] += p->cigar[k] >> 4 << 4;
			p->n_cigar = l;
		}
		if ((p->cigar[0] & 0xf) == MM_CIGAR_INS || (p->cigar[0] & 0xf) == MM_CIGAR_DEL) { // drop a leading I/D
			int32_t l = p->cigar[0] >> 4;
			if ((p->cigar[0] & 0xf) == MM_CIGAR_INS) {
				if (r->rev) r->qe -= l; else r->qs += l;
				*qshift = l;
			} else r->rs += l, *tshift = l;
			--p->n_cigar;
			memmove(p->cigar, p->cigar + 1, p->n_cigar * 4);
		}
	}

	static void update_cigar_eqx(mm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq) { // align.c:183-252
		uint32_t n_EQX = 0, k, l, m, cap, toff = 0, qoff = 0, n_M = 0;
		if (r->p == 0) return;
		for (k = 0; k < r->p->n_cigar; ++k) {
			uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
			if (op == MM_CIGAR_MATCH) {
				while (len > 0) {
					for (l = 0; l < len && qseq[qoff + l] == tseq[toff + l]; ++l) {}
					if (l > 0) { ++n_EQX; len -= l; toff += l; qoff += l; }
					for (l = 0; l < len && qseq[qoff + l] != tseq[toff + l]; ++l) {}
					if (l > 0) { ++n_EQX; len -= l; toff += l; qoff += l; }
				}
				++n_M;
			} else if (op == MM_CIGAR_INS) qoff += len;
			else if (op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) toff += len;
		}
		if (n_EQX == n_M) {
			for (k = 0; k < r->p->n_cigar; ++k) {
				uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
				if (op == MM_CIGAR_MATCH) r->p->cigar[k] = len << 4 | MM_CIGAR_EQ_MATCH;
			}
			return;
		}
		cap = roundup32(r->p->n_cigar + (n_EQX - n_M) + sizeof(mm_extra_t));
		mm_extra_t *p = (mm_extra_t*)calloc(cap, 4);
		memcpy(p, r->p, sizeof(mm_extra_t));
		p->capacity = cap;
		toff = qoff = m = 0;
		for (k = 0; k < r->p->n_cigar; ++k) {
			uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
			if (op == MM_CIGAR_MATCH) {
				while (len > 0) {
					for (l = 0; l < len && qseq[qoff + l] == tseq[toff + l]; ++l) {}
					if (l > 0) p->cigar[m++] = l << 4 | MM_CIGAR_EQ_MATCH;
					len -= l; toff += l, qoff += l;
					for (l = 0; l < len && qseq[qoff + l] != tseq[toff + l]; ++l) {}
					if (l > 0) p->cigar[m++] = l << 4 | MM_CIGAR_X_MISMATCH;
					len -= l; toff += l, qoff += l;
				}
				continue;
			} else if (op == MM_CIGAR_INS) qoff += len;
			else if (op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) toff += len;
			p->cigar[m++] = r->p->cigar[k];
		}
		p->n_cigar = m;
		free(r->p);
		r->p = p;
	}

	void update_extra(mm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq, int8_t q, int8_t e, int is_eqx, int log_gap) { // align.c:254-303
		HpScope hp_(HP_EXTRA);
		int32_t qshift, tshift, toff = 0, qoff = 0;
		mm_extra_t *p = r->p;
		if (p == 0) return;
		fix_cigar(r, qseq, tseq, &qshift, &tshift);
		qseq += qshift, tseq += tshift;
		// The reference's running score (align.c:266-297) is a double; here it is an integer in units of 2^-32, which is exact. With
		// int8_t q and e, mmx_log2(1+len) is a float in [1,33) and so a multiple of 2^-23; q + e * mmx_log2(1+len) is then an exact
		// double, a multiple of 2^-23 below 2^13 in magnitude, and times 2^32 an integer below 2^45 (tests/test_tail_penalty_exact.py).
		int64_t matfx[25];
		for (int i = 0; i < 25; ++i) matfx[i] = (int64_t)mat[i] << 32;
		int64_t sfx = 0, maxfx = 0;
		const int64_t afx = matfx[0];
		const bool diag_ok = mat[0] > 0 && mat[6] == mat[0] && mat[12] == mat[0] && mat[18] == mat[0]; // one positive match score
		int32_t blen = 0, mlen = 0, n_ambi_tot = 0, is_spliced = 0;
		for (uint32_t k = 0; k < p->n_cigar; ++k) {
			uint32_t op = p->cigar[k] & 0xf, len = p->cigar[k] >> 4;
			if (op == MM_CIGAR_MATCH) {
				int n_ambi = 0, n_diff = 0;
				const uint8_t *pq = qseq + qoff, *pt = tseq + toff;
				if (diag_ok) {
					// runs of identical unambiguous bases add run * a at once (the running score only rises there, so
					// testing the maximum at the end of the run is the same as testing it at every base); 16 bases
					// per comparison, both buffers carry 16 bytes of slack
					for (uint32_t l0 = 0; l0 < len; l0 += 16) {
						const uint32_t nb = len - l0 < 16? len - l0 : 16;
						const __m128i vq = _mm_loadu_si128((const __m128i*)(pq + l0)), vt = _mm_loadu_si128((const __m128i*)(pt + l0));
						const __m128i same = _mm_cmpeq_epi8(vq, vt), amb = _mm_cmpgt_epi8(_mm_or_si128(vq, vt), _mm_set1_epi8(3));
						uint32_t ev = (uint32_t)_mm_movemask_epi8(_mm_or_si128(amb, _mm_xor_si128(same, _mm_set1_epi8(-1)))) & ((1u << nb) - 1);
						uint32_t pos = 0;
						while (ev) {
							const uint32_t b = (uint32_t)__builtin_ctz(ev);
							if (b > pos) { sfx += (int64_t)(b - pos) * afx; maxfx = maxfx > sfx? maxfx : sfx; }
							const int cq = pq[l0 + b], ct = pt[l0 + b];
							if ((ct | cq) > 3) ++n_ambi; else ++n_diff;
							sfx += matfx[ct * 5 + cq];
							if (sfx < 0) sfx = 0;
							else maxfx = maxfx > sfx? maxfx : sfx;
							pos = b + 1, ev &= ev - 1;
						}
						if (nb > pos) { sfx += (int64_t)(nb - pos) * afx; maxfx = maxfx > sfx? maxfx : sfx; }
					}
				} else
				for (uint32_t l = 0; l < len; ++l) {
					const int cq = pq[l], ct = pt[l];
					const int amb = (ct | cq) > 3;
					n_ambi += amb, n_diff += (ct != cq) & !amb;
					sfx += matfx[ct * 5 + cq];
					if (sfx < 0) sfx = 0;
					else maxfx = maxfx > sfx? maxfx : sfx;
				}
				blen += len - n_ambi, mlen += len - (n_ambi + n_diff), n_ambi_tot += n_ambi;
				toff += len, qoff += len;
			} else if (op == MM_CIGAR_INS || op == MM_CIGAR_DEL) {
				int n_ambi = 0;
				const uint8_t *sq = op == MM_CIGAR_INS? qseq + qoff : tseq + toff;
				for (uint32_t l = 0; l < len; ++l) if (sq[l] > 3) ++n_ambi;
				blen += len - n_ambi, n_ambi_tot += n_ambi;
				const double pen = log_gap? q + (double)e * mmx_log2(1.0 + len) : (double)(q + e);
				sfx -= (int64_t)(pen * 4294967296.0);
				if (sfx < 0) sfx = 0;
				if (op == MM_CIGAR_INS) qoff += len; else toff += len;
			} else if (op == MM_CIGAR_N_SKIP) is_spliced = 1, toff += len;
		}
		r->blen = blen, r->mlen = mlen, r->is_spliced = is_spliced, p->n_ambi += n_ambi_tot;
		p->dp_max = p->dp_max0 = (int32_t)((double)maxfx / 4294967296.0 + .499);
		assert(qoff == r->qe - r->qs && toff == r->re - r->rs);
		if (is_eqx) update_cigar_eqx(r, qseq, tseq);
	}

	// ---- seed/end filters (align.c:418-566) ----
	int hplen_back(uint32_t rid, uint32_t x) const { // align.c:409-416
		int64_t i, off0 = mi->seq[rid].offset, off = off0 + x;
		int c = mmx_seq4_get(mi->S, off);
		for (i = off - 1; i >= off0; --i) if ((int)mmx_seq4_get(mi->S, i) != c) break;
		return (int)(off - i);
	}
	void adjust_minier(const m128 *a, int32_t *r, int32_t *q) const { // align.c:418-433
		if (mi->flag & MM_I_HPC) {
			ra.ensure_qseq();
			const uint8_t *qs = ra.qseq[a->x >> 63];
			int i, c;
			*q = (int32_t)a->y;
			for (i = *q - 1, c = qs[*q]; i > 0; --i) if (qs[i] != c) break;
			*q = i + 1;
			c = hplen_back((uint32_t)(a->x << 1 >> 33), (uint32_t)(int32_t)a->x);
			*r = (int32_t)a->x + 1 - c;
		} else {
			*r = (int32_t)a->x - (mi->k >> 1);
			*q = (int32_t)a->y - (mi->k >> 1);
		}
	}
	static inline int gap_of(const m128 *a, int i) { return ((int32_t)a[i].y - (int32_t)a[i-1].y) - ((int32_t)a[i].x - (int32_t)a[i-1].x); }
	static void long_gaps(int as1, int cnt1, const m128 *a, int min_gap, std::vector<int> &K) { // align.c:435-452
		K.clear();
		int n = 0;
		for (int i = 1; i < cnt1; ++i) { int g = gap_of(a + as1, i); if (g < -min_gap || g > min_gap) ++n; }
		if (n <= 1) return;
		for (int i = 1; i < cnt1; ++i) { int g = gap_of(a + as1, i); if (g < -min_gap || g > min_gap) K.push_back(i); }
	}
	static void filter_bad_seeds(int as1, int cnt1, m128 *a, int min_gap, int diff_thres, int max_ext_len, int max_ext_cnt) { // align.c:454-489
		std::vector<int> K;
		long_gaps(as1, cnt1, a, min_gap, K);
		const int n = (int)K.size();
		if (n == 0) return;
		int max = 0, max_st = -1, max_en = -1;
		for (int k = 0;; ++k) {
			int gap, l, n_ins = 0, n_del = 0, qs, rs, max_diff = 0, max_diff_l = -1;
			if (k == n || k >= max_en) {
				if (max_en > 0) for (int i = K[max_st]; i < K[max_en]; ++i) a[as1 + i].y |= MMX_SEED_IGNORE;
				max = 0, max_st = max_en = -1;
				if (k == n) break;
			}
			int i = K[k];
			gap = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - (int32_t)(a[as1 + i].x - a[as1 + i - 1].x);
			if (gap > 0) n_ins += gap; else n_del += -gap;
			qs = (int32_t)a[as1 + i - 1].y, rs = (int32_t)a[as1 + i - 1].x;
			for (l = k + 1; l < n && l <= k + max_ext_cnt; ++l) {
				int j = K[l], diff;
				if ((int32_t)a[as1 + j].y - qs > max_ext_len || (int32_t)a[as1 + j].x - rs > max_ext_len) break;
				gap = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
				if (gap > 0) n_ins += gap; else n_del += -gap;
				diff = n_ins + n_del - abs(n_ins - n_del);
				if (max_diff < diff) max_diff = diff, max_diff_l = l;
			}
			if (max_diff > diff_thres && max_diff > max) max = max_diff, max_st = k, max_en = max_diff_l;
		}
	}
	static void filter_bad_seeds_alt(int as1, int cnt1, m128 *a, int min_gap, int max_ext) { // align.c:491-525
		std::vector<int> K;
		long_gaps(as1, cnt1, a, min_gap, K);
		const int n = (int)K.size();
		if (n == 0) return;
		for (int k = 0; k < n;) {
			int i = K[k], l;
			int gap1 = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - ((int32_t)a[as1 + i].x - (int32_t)a[as1 + i - 1].x);
			int re1 = (int32_t)a[as1 + i].x, qe1 = (int32_t)a[as1 + i].y;
			gap1 = gap1 > 0? gap1 : -gap1;
			for (l = k + 1; l < n; ++l) {
				int j = K[l], gap2, q_span_pre, rs2, qs2, m;
				if ((int32_t)a[as1 + j].y - qe1 > max_ext || (int32_t)a[as1 + j].x - re1 > max_ext) break;
				gap2 = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
				q_span_pre = (int)(a[as1 + j - 1].y >> 32 & 0xff);
				rs2 = (int32_t)a[as1 + j - 1].x + q_span_pre;
				qs2 = (int32_t)a[as1 + j - 1].y + q_span_pre;
				m = rs2 - re1 < qs2 - qe1? rs2 - re1 : qs2 - qe1;
				gap2 = gap2 > 0? gap2 : -gap2;
				if (m > gap1 + gap2) break;
				re1 = (int32_t)a[as1 + j].x, qe1 = (int32_t)a[as1 + j].y;
				gap1 = gap2;
			}
			if (l > k + 1) {
				int end = K[l - 1];
				for (int j = K[k]; j < end; ++j) a[as1 + j].y |= MMX_SEED_IGNORE;
				a[as1 + end].y |= MMX_SEED_LONG_JOIN;
			}
			k = l;
		}
	}
	static void fix_bad_ends(const mm_reg1_t *r, const m128 *a, int bw, int min_match, int32_t *as, int32_t *cnt) { // align.c:527-564
		int32_t i, l, m;
		*as = r->as, *cnt = r->cnt;
		if (r->cnt < 3) return;
		m = l = (int32_t)(a[r->as].y >> 32 & 0xff);
		for (i = r->as + 1; i < r->as + r->cnt - 1; ++i) {
			int32_t lq, lr, min, max, q_span = (int32_t)(a[i].y >> 32 & 0xff);
			if (a[i].y & MMX_SEED_LONG_JOIN) break;
			lr = (int32_t)a[i].x - (int32_t)a[i-1].x, lq = (int32_t)a[i].y - (int32_t)a[i-1].y;
			min = lr < lq? lr : lq, max = lr > lq? lr : lq;
			if (max - min > l >> 1) *as = i;
			l += min;
			m += min < q_span? min : q_span;
			if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= r->mlen >> 1) break;
		}
		*cnt = r->as + r->cnt - *as;
		m = l = (int32_t)(a[r->as + r->cnt - 1].y >> 32 & 0xff);
		for (i = r->as + r->cnt - 2; i > *as; --i) {
			int32_t lq, lr, min, max, q_span = (int32_t)(a[i+1].y >> 32 & 0xff);
			if (a[i+1].y & MMX_SEED_LONG_JOIN) break;
			lr = (int32_t)a[i+1].x - (int32_t)a[i].x, lq = (int32_t)a[i+1].y - (int32_t)a[i].y;
			min = lr < lq? lr : lq, max = lr > lq? lr : lq;
			if (max - min > l >> 1) *cnt = i + 1 - *as;
			l += min;
			m += min < q_span? min : q_span;
			if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= r->mlen >> 1) break;
		}
	}

	// mm_seed_ext_score (align.c:592-616): local score of the anchor extended by anchor_ext_len on both sides. False while pending.
	bool seed_ext_score(const m128 *a, int *score) {
		const int q_span = (int)(a->y >> 32 & 0xff), ext_len = opt->anchor_ext_len, rid = (int)(a->x << 1 >> 33);
		int re = (int)(uint32_t)a->x + 1, rs = re - q_span, qe = (int)(uint32_t)a->y + 1, qs = qe - q_span, q_off, t_off;
		rs = rs - ext_len > 0? rs - ext_len : 0;
		qs = qs - ext_len > 0? qs - ext_len : 0;
		re = re + ext_len < (int32_t)mi->seq[rid].len? re + ext_len : (int)mi->seq[rid].len;
		qe = qe + ext_len < qlen? qe + ext_len : qlen;
		Seg s; s.rev = (int)(a->x >> 63), s.qs = qs, s.qlen = qe - qs, s.q_reversed = 0, s.rid = rid, s.rs = rs, s.tlen = re - rs, s.t_reversed = 0;
		return ll_i16(s, score, &q_off, &t_off);
	}
	// mm_fix_bad_ends_splice (align.c:618-637): drop a boundary anchor that sits far from its neighbour and extends poorly
	bool fix_bad_ends_splice(const mm_reg1_t *r, const m128 *a, int32_t *as1, int32_t *cnt1) {
		int score;
		double log_gap;
		*as1 = r->as, *cnt1 = r->cnt;
		if (r->cnt < 3) return true;
		log_gap = log((int32_t)a[r->as + 1].x - (int32_t)a[r->as].x);
		if ((double)(a[r->as].y >> 32 & 0xff) < log_gap + opt->anchor_ext_shift) {
			if (!seed_ext_score(&a[r->as], &score)) return false;
			if ((double)score / mat[0] < log_gap + opt->anchor_ext_shift) ++(*as1), --(*cnt1);
		}
		log_gap = log((int32_t)a[r->as + r->cnt - 1].x - (int32_t)a[r->as + r->cnt - 2].x);
		if ((double)(a[r->as + r->cnt - 1].y >> 32 & 0xff) < log_gap + opt->anchor_ext_shift) {
			if (!seed_ext_score(&a[r->as + r->cnt - 1], &score)) return false;
			if ((double)score / mat[0] < log_gap + opt->anchor_ext_shift) --(*cnt1);
		}
		return true;
	}

	// ---- mm_align1 (align.c:645-914), long-read path (genomic or spliced). Returns false if some ksw result is still pending. ----
	// splice_flag: which transcript strand(s) to assume (MM_F_SPLICE_FOR / MM_F_SPLICE_REV), as in align.c:684-689.
	bool align1(mm_reg1_t *r, mm_reg1_t *r2, int n_a, m128 *a, int64_t splice_flag) {
		const int32_t rid = (int32_t)(a[r->as].x << 1 >> 33), rev = (int32_t)(a[r->as].x >> 63);
		// query-strand mode (align.c:780-783,815-818,875-878,899-901): the query stays forward, a reverse hit reads the target's other strand
		const bool qst = (opt->flag & MM_F_QSTRAND) != 0;
		const int qrev = qst? 0 : rev, trc = qst && rev? 1 : 0;
		int32_t as1, cnt1, i, l, bw, bw_long, dropped = 0, rs0, re0, qs0, qe0, rs, re, qs, qe, rs1, qs1, re1, qe1;
		const int32_t ref_len = (int32_t)mi->seq[rid].len;
		std::vector<uint8_t> tseq;
		Ez ez;
		pending = false;
		r2->cnt = 0;
		if (r->cnt == 0) return true;
		fin_first = (int)ra.fin_jobs.size();
		bw = (int)(opt->bw * 1.5 + 1.);
		bw_long = (int)(opt->bw_long * 1.5 + 1.);
		if (bw_long < bw) bw_long = bw;
		const bool is_splice = (opt->flag & MM_F_SPLICE) != 0;
		int sflag = 0; // KSW_EZ_SPLICE_* for every ksw call of this region
		if (is_splice) {
			if (splice_flag & MM_F_SPLICE_FOR) sflag |= rev? MMB_KSW_SPLICE_REV : MMB_KSW_SPLICE_FOR;
			if (splice_flag & MM_F_SPLICE_REV) sflag |= rev? MMB_KSW_SPLICE_FOR : MMB_KSW_SPLICE_REV;
			if (opt->flag & MM_F_SPLICE_FLANK) sflag |= MMB_KSW_SPLICE_FLANK;
			if (mi->spsc) sflag |= MMB_KSW_SPLICE_SCORE; // align.c:688: junc[] carries splice scores (mm_idx_spsc_get)
		}
		// What follows up to the gap-fill list depends on the anchors only (spliced reads: and on the end probes, which are awaited first):
		// it is computed by the first replay that gets this far and kept in the read's plan list; later replays start at the extensions.
		const int32_t key_as = r->as, key_cnt = r->cnt;
		HlHitPlan *P = nullptr;
		for (HlHitPlan &hp : ra.plans) if (hp.as == key_as && hp.cnt == key_cnt && hp.splice_flag == (splice_flag << 1 | (r->split_inv? 1 : 0))) { P = &hp; break; }
		HlHitPlan fresh; // used when the hit has no stored plan yet
		if (P) {
			as1 = P->as1, cnt1 = P->cnt1, rs = P->rs, qs = P->qs, re = P->re, qe = P->qe, rs0 = P->rs0, qs0 = P->qs0, re0 = P->re0, qe0 = P->qe0;
			for (const auto &m : P->marks) a[m.first].y |= m.second;
		} else {
		if (!(opt->flag & MM_F_NO_END_FLT)) {
			if (is_splice) { if (!fix_bad_ends_splice(r, a, &as1, &cnt1)) return false; } // the probe is pending: nothing below can be planned yet
			else fix_bad_ends(r, a, opt->bw, opt->min_chain_score * 2, &as1, &cnt1);
		} else as1 = r->as, cnt1 = r->cnt;
		filter_bad_seeds(as1, cnt1, a, 10, 40, opt->max_gap >> 1, 10);
		filter_bad_seeds_alt(as1, cnt1, a, 30, opt->max_gap >> 1);
		for (i = 0; i < cnt1; ++i) if (a[as1 + i].y & (MMX_SEED_IGNORE | MMX_SEED_LONG_JOIN)) fresh.marks.emplace_back(as1 + i, a[as1 + i].y & (MMX_SEED_IGNORE | MMX_SEED_LONG_JOIN));
		adjust_minier(&a[as1], &rs, &qs);
		adjust_minier(&a[as1 + cnt1 - 1], &re, &qe);
		assert(cnt1 > 0);

		// DP window (align.c:704-767)
		rs0 = (int32_t)a[r->as].x + 1 - (int32_t)(a[r->as].y >> 32 & 0xff);
		qs0 = (int32_t)a[r->as].y + 1 - (int32_t)(a[r->as].y >> 32 & 0xff);
		if (rs0 < 0) rs0 = 0;
		assert(qs0 >= 0);
		rs1 = qs1 = 0;
		for (i = r->as - 1, l = 0; i >= 0 && a[i].x >> 32 == a[r->as].x >> 32; --i) {
			int32_t x = (int32_t)a[i].x + 1 - (int32_t)(a[i].y >> 32 & 0xff);
			int32_t y = (int32_t)a[i].y + 1 - (int32_t)(a[i].y >> 32 & 0xff);
			if (x < rs0 && y < qs0) {
				if (++l > opt->min_cnt) {
					l = rs0 - x > qs0 - y? rs0 - x : qs0 - y;
					rs1 = rs0 - l, qs1 = qs0 - l;
					if (rs1 < 0) rs1 = 0;
					break;
				}
			}
		}
		if (qs > 0 && rs > 0) {
			l = qs < opt->max_gap? qs : opt->max_gap;
			qs1 = qs1 > qs - l? qs1 : qs - l;
			qs0 = qs0 < qs1? qs0 : qs1;
			l += l * opt->a > opt->q? (l * opt->a - opt->q) / opt->e : 0;
			l = l < opt->max_gap? l : opt->max_gap;
			l = l < rs? l : rs;
			rs1 = rs1 > rs - l? rs1 : rs - l;
			rs0 = rs0 < rs1? rs0 : rs1;
			rs0 = rs0 < rs? rs0 : rs;
		} else rs0 = rs, qs0 = qs;
		re0 = (int32_t)a[r->as + r->cnt - 1].x + 1;
		qe0 = (int32_t)a[r->as + r->cnt - 1].y + 1;
		re1 = ref_len, qe1 = qlen;
		for (i = r->as + r->cnt, l = 0; i < n_a && a[i].x >> 32 == a[r->as].x >> 32; ++i) {
			int32_t x = (int32_t)a[i].x + 1, y = (int32_t)a[i].y + 1;
			if (x > re0 && y > qe0) {
				if (++l > opt->min_cnt) {
					l = x - re0 > y - qe0? x - re0 : y - qe0;
					re1 = re0 + l, qe1 = qe0 + l;
					break;
				}
			}
		}
		if (qe < qlen && re < ref_len) {
			l = qlen - qe < opt->max_gap? qlen - qe : opt->max_gap;
			qe1 = qe1 < qe + l? qe1 : qe + l;
			qe0 = qe0 > qe1? qe0 : qe1;
			l += l * opt->a > opt->q? (l * opt->a - opt->q) / opt->e : 0;
			l = l < opt->max_gap? l : opt->max_gap;
			l = l < ref_len - re? l : ref_len - re;
			re1 = re1 < re + l? re1 : re + l;
			re0 = re0 > re1? re0 : re1;
		} else re0 = re, qe0 = qe;
		if (a[r->as].y & MMX_SEED_SELF) {
			int max_ext = r->qs > r->rs? r->qs - r->rs : r->rs - r->qs;
			if (r->rs - rs0 > max_ext) rs0 = r->rs - max_ext;
			if (r->qs - qs0 > max_ext) qs0 = r->qs - max_ext;
			max_ext = r->qe > r->re? r->qe - r->re : r->re - r->qe;
			if (re0 - r->re > max_ext) re0 = r->re + max_ext;
			if (qe0 - r->qe > max_ext) qe0 = r->qe + max_ext;
		}
		assert(re0 > rs0);
			// the gap fills (align.c:803-813): anchor pairs far enough apart, long joins, the last anchor
			fresh.as = key_as, fresh.cnt = key_cnt, fresh.splice_flag = splice_flag << 1 | (r->split_inv? 1 : 0);
			fresh.as1 = as1, fresh.cnt1 = cnt1, fresh.rs = rs, fresh.qs = qs, fresh.re = re, fresh.qe = qe, fresh.rs0 = rs0, fresh.qs0 = qs0, fresh.re0 = re0, fresh.qe0 = qe0;
			{
				int32_t prs = rs, pqs = qs, pre = re, pqe = qe;
				for (i = 1; i < cnt1; ++i) {
					if ((a[as1 + i].y & (MMX_SEED_IGNORE | MMX_SEED_TANDEM)) && i != cnt1 - 1) continue;
					adjust_minier(&a[as1 + i], &pre, &pqe);
					if (i == cnt1 - 1 || (a[as1 + i].y & MMX_SEED_LONG_JOIN) || (pqe - pqs >= opt->min_ksw_len && pre - prs >= opt->min_ksw_len)) {
						HlFill f;
						f.i = i, f.qs = pqs, f.qe = pqe, f.rs = prs, f.re = pre, f.slot = -1;
						f.bw1 = (a[as1 + i].y & MMX_SEED_LONG_JOIN)? (pqe - pqs > pre - prs? pqe - pqs : pre - prs) : bw_long;
						fresh.fills.push_back(f);
						prs = pre, pqs = pqe;
					}
				}
			}
			ra.plans.push_back(std::move(fresh));
			P = &ra.plans.back();
		} // planning

		// left extension (align.c:779-799)
		if (qs > 0 && rs > 0) {
			Seg s; s.rev = qrev, s.qs = qs0, s.qlen = qs - qs0, s.q_reversed = 1, s.rid = rid, s.rs = rs0, s.tlen = rs - rs0, s.t_reversed = 1, s.t_rc = trc;
			bool ok = align_pair(s, bw, opt->end_bonus, r->split_inv? opt->zdrop_inv : opt->zdrop, sflag | MMB_KSW_EXTZ_ONLY | MMB_KSW_RIGHT | MMB_KSW_REV_CIGAR, &ez, &P->slot_left);
			if (ok) {
				if (ez.n_cigar > 0) { add_cigar(r, ez); r->p->dp_score += ez.max; }
				rs1 = rs - (ez.reach_end? ez.mqe_t + 1 : ez.max_t + 1);
				qs1 = qs - (ez.reach_end? qs - qs0 : ez.max_q + 1);
			} else rs1 = rs, qs1 = qs; // placeholder while the result is pending; the region is replayed later
		} else rs1 = rs, qs1 = qs;
		re1 = rs, qe1 = qs;
		if (!pending) assert(qs1 >= 0 && rs1 >= 0);

		// gap filling (align.c:803-872)
		for (size_t fk = 0; fk < P->fills.size(); ++fk) {
			HlFill &F = P->fills[fk];
			i = F.i, qs = F.qs, qe = F.qe, rs = F.rs, re = F.re;
			re1 = re, qe1 = qe;
			{
				int j, zdrop_code;
				const int bw1 = F.bw1;
				Seg s; s.rev = qrev, s.qs = qs, s.qlen = qe - qs, s.q_reversed = 0, s.rid = rid, s.rs = rs, s.tlen = re - rs, s.t_reversed = 0, s.t_rc = trc;
				bool ok = align_pair(s, bw1, -1, opt->zdrop, sflag | MMB_KSW_APPROX_MAX | MMB_JOB_ZDROP, &ez, &F.slot); // first pass
				if (ok) { // results that are available are consumed even if an earlier call is pending: this surfaces second-pass jobs one wave earlier
					const bool have_zd = ez.zd_max >= 0 && !ez.zdropped;
					const uint8_t *qseq = have_zd? nullptr : qptr(qrev, qs); // the host only scans the bases itself when the kernel did not
					if (!have_zd) get_tseq(rid, rs, re, tseq, trc);
					zdrop_code = test_zdrop(s, qseq, tseq.data(), ez.n_cigar, ez.cigar, have_zd? &ez : nullptr);
					if (zdrop_code > 0) ok = align_pair(s, bw1, -1, zdrop_code == 2? opt->zdrop_inv : opt->zdrop, sflag, &ez); // second pass
					else if (zdrop_code < 0) ok = false;
					if (ok) {
						if (ez.n_cigar > 0) add_cigar(r, ez);
						if (ez.zdropped) { // truncated by Z-drop
							if (!r->p) {
								uint32_t capacity = roundup32(sizeof(mm_extra_t) / 4);
								r->p = (mm_extra_t*)calloc(capacity, 4);
								r->p->capacity = capacity;
							}
							for (j = i - 1; j >= 0; --j) if ((int32_t)a[as1 + j].x <= rs + ez.max_t) break;
							dropped = 1;
							if (j < 0) j = 0;
							r->p->dp_score += ez.max;
							re1 = rs + (ez.max_t + 1);
							qe1 = qs + (ez.max_q + 1);
							if (cnt1 - (j + 1) >= opt->min_cnt) {
								hl_split_reg(r, r2, as1 + j + 1 - r->as, qlen, a, !!(opt->flag & MM_F_QSTRAND));
								if (zdrop_code == 2) r2->split_inv = 1;
							}
							break;
						} else if (r->p) r->p->dp_score += ez.score;
					}
				}
				rs = re, qs = qe;
			}
		}

		// right extension (align.c:874-890)
		if (!dropped && qe < qe0 && re < re0) {
			Seg s; s.rev = qrev, s.qs = qe, s.qlen = qe0 - qe, s.q_reversed = 0, s.rid = rid, s.rs = re, s.tlen = re0 - re, s.t_reversed = 0, s.t_rc = trc;
			bool ok = align_pair(s, bw, opt->end_bonus, opt->zdrop, sflag | MMB_KSW_EXTZ_ONLY, &ez, &P->slot_right);
			if (ok) {
				if (ez.n_cigar > 0) { add_cigar(r, ez); r->p->dp_score += ez.max; }
				re1 = re + (ez.reach_end? ez.mqe_t + 1 : ez.max_t + 1);
				qe1 = qe + (ez.reach_end? qe0 - qe : ez.max_q + 1);
			}
		}
		if (pending) { ra.fin_jobs.resize(fin_first); return false; }
		assert(qe1 <= qlen);
		r->rs = rs1, r->re = re1;
		if (!rev || (opt->flag & MM_F_QSTRAND)) r->qs = qs1, r->qe = qe1;
		else r->qs = qlen - qe1, r->qe = qlen - qs1;
		assert(re1 - rs1 <= re0 - rs0);
		if (r->p && ra.defer) { // the device tail assembles, fixes and rescans this hit (K4)
			HlFinHit h;
			h.p = r->p, h.rev = r->rev, h.qs = qs1, h.rid = rid, h.rs = rs1, h.qspan = qe1 - qs1, h.tspan = re1 - rs1;
			h.job_first = fin_first, h.n_jobs = (int)ra.fin_jobs.size() - fin_first, h.n_cig_max = 0;
			for (int k = fin_first; k < (int)ra.fin_jobs.size(); ++k) h.n_cig_max += ra.fin_jobs[k].n;
			ra.fin_hits.push_back(h);
		} else if (r->p) {
			get_tseq(rid, rs1, re1, tseq, trc);
			update_extra(r, qptr(qst? 0 : r->rev, qs1), tseq.data(), opt->q, opt->e, opt->flag & MM_F_EQX, 1);
			if (rev && r->p->trans_strand) r->p->trans_strand ^= 3;
		}
		return true;
	}

	// mm_align1_inv (align.c:916-975). Returns 1 if an inversion hit was produced, 0 if not, -1 if pending.
	int align1_inv(const mm_reg1_t *r1, const mm_reg1_t *r2, mm_reg1_t *r_inv) {
		int tl, ql, score, q_off, t_off;
		Ez ez;
		memset(r_inv, 0, sizeof(mm_reg1_t));
		if (!(r1->split & 1) || !(r2->split & 2)) return 0;
		if (r1->id != r1->parent && r1->parent != HL_PARENT_TMP_PRI) return 0;
		if (r2->id != r2->parent && r2->parent != HL_PARENT_TMP_PRI) return 0;
		if (r1->rid != r2->rid || r1->rev != r2->rev) return 0;
		ql = r1->rev? r1->qs - r2->qe : r2->qs - r1->qe;
		tl = r2->rs - r1->re;
		if (ql < opt->min_chain_score || ql > opt->max_gap) return 0;
		if (tl < opt->min_chain_score || tl > opt->max_gap) return 0;
		// qseq = r1->rev? &qseq0[0][r2->qe] : &qseq0[1][qlen - r2->qs]
		Seg s; s.rev = r1->rev? 0 : 1, s.qs = r1->rev? r2->qe : qlen - r2->qs, s.qlen = ql, s.q_reversed = 1;
		s.rid = r1->rid, s.rs = r1->re, s.tlen = tl, s.t_reversed = 1;
		pending = false;
		if (!ll_i16(s, &score, &q_off, &t_off)) return -1;
		if (score < opt->min_dp_max) return 0;
		q_off = ql - (q_off + 1), t_off = tl - (t_off + 1);
		Seg e = s; e.q_reversed = 0, e.t_reversed = 0, e.qs = s.qs + q_off, e.qlen = ql - q_off, e.rs = s.rs + t_off, e.tlen = tl - t_off;
		if (!align_pair(e, (int)(opt->bw * 1.5), -1, opt->zdrop, MMB_KSW_EXTZ_ONLY, &ez)) return -1;
		if (ez.n_cigar == 0) return 0;
		append_cigar(r_inv, ez.n_cigar, ez.cigar);
		r_inv->p->dp_score = ez.max;
		r_inv->id = -1;
		r_inv->parent = HL_PARENT_UNSET;
		r_inv->inv = 1;
		r_inv->rev = !r1->rev;
		r_inv->rid = r1->rid;
		r_inv->div = -1.0f;
		if (r_inv->rev == 0) {
			r_inv->qs = r2->qe + q_off;
			r_inv->qe = r_inv->qs + ez.max_q + 1;
		} else {
			r_inv->qe = r2->qs - q_off;
			r_inv->qs = r_inv->qe - (ez.max_q + 1);
		}
		r_inv->rs = r1->re + t_off;
		r_inv->re = r_inv->rs + ez.max_t + 1;
		std::vector<uint8_t> tseq;
		get_tseq(r1->rid, r1->re + t_off, r2->rs, tseq);
		update_extra(r_inv, qptr(s.rev, s.qs + q_off), tseq.data(), opt->q, opt->e, opt->flag & MM_F_EQX, !(opt->flag & (MM_F_SR | MM_F_SR_RNA)));
		return 1;
	}
};

inline mm_reg1_t *insert_reg(const mm_reg1_t *r, int i, int *n_regs, mm_reg1_t *regs) // align.c:977-986
{
	regs = (mm_reg1_t*)realloc(regs, (*n_regs + 1) * sizeof(mm_reg1_t));
	if (i + 1 != *n_regs) memmove(&regs[i + 2], &regs[i + 1], sizeof(mm_reg1_t) * (*n_regs - i - 1));
	regs[i + 1] = *r;
	++*n_regs;
	return regs;
}

} // namespace

uint64_t g_hp[HP_N] = {0};
thread_local uint64_t tl_hp[HP_N] = {0};
void hl_hp_flush()
{
	if (!g_hp_on) return;
	for (int i = 0; i < HP_N; ++i) if (tl_hp[i]) { __atomic_fetch_add(&g_hp[i], tl_hp[i], __ATOMIC_RELAXED); tl_hp[i] = 0; }
}
bool g_hp_on = getenv("MM_B200_TIMING") != nullptr;
void hl_hp_dump(const char *tag)
{
	if (!g_hp_on) return;
	static const char *nm[HP_N] = { "skeleton", "tseq", "zdrop", "extra", "fetch", "append", "pre", "post", "hits" };
	fprintf(stderr, "[hostprof %s]", tag);
	for (int i = 0; i < HP_N; ++i) fprintf(stderr, " %s=%.1fms", nm[i], (double)__atomic_exchange_n(&g_hp[i], 0, __ATOMIC_RELAXED) / 2.0e6); // ~2 GHz TSC
	fprintf(stderr, "\n");
}

mm_reg1_t *hl_align_skeleton(const mm_mapopt_t *opt, const mm_idx_t *mi, ReadAlign &ra, int *n_regs_, mm_reg1_t *regs, int n_a_in, m128 *a)
{
	HpScope hp_(HP_SKEL);
	int32_t n_regs = *n_regs_, n_a;
	Driver D(opt, mi, ra);
	ra.incomplete = false, ra.defer_abort = false;
	ra.fin_hits.clear(), ra.fin_jobs.clear();
	if (ra.defer && !hl_defer_supported(opt)) ra.defer = false;
	(void)n_a_in;
	n_a = hl_squeeze_a(n_regs, regs, a); // idempotent across replays: after the first call regions are already packed in order
	for (int i = 0; i < n_regs; ++i) {
		mm_reg1_t r2;
		if ((opt->flag & MM_F_SPLICE) && (opt->flag & MM_F_SPLICE_FOR) && (opt->flag & MM_F_SPLICE_REV)) { // both transcript strands (align.c:1068-1098)
			mm_reg1_t s[2], s2[2];
			s[0] = s[1] = regs[i];
			const bool ok0 = D.align1(&s[0], &s2[0], n_a, a, MM_F_SPLICE_FOR);
			const bool ok1 = D.align1(&s[1], &s2[1], n_a, a, MM_F_SPLICE_REV); // walked even if the first is pending: its jobs join the same wave
			if (!ok0 || !ok1) { free(s[0].p); free(s[1].p); continue; }
			int which, trans_strand;
			if (s[0].p->dp_score > s[1].p->dp_score) which = 0, trans_strand = 1;
			else if (s[0].p->dp_score < s[1].p->dp_score) which = 1, trans_strand = 2;
			else trans_strand = 3, which = (ra.qlen + s[0].p->dp_score) & 1;
			regs[i] = s[which], r2 = s2[which];
			free(s[1 - which].p);
			mm_reg1_t *r = &regs[i];
			r->p->trans_strand = trans_strand;
			if (r->is_spliced) {
				if (trans_strand == 1 || trans_strand == 2) r->p->dp_max += (opt->a + opt->b) + ((opt->a + opt->b) >> 1);
				else if (trans_strand == 3) r->p->dp_max -= opt->a + opt->b;
			}
		} else {
			if (!D.align1(&regs[i], &r2, n_a, a, opt->flag)) continue; // results pending: other regions are still walked to collect their jobs
			if (opt->flag & MM_F_SPLICE) regs[i].p->trans_strand = opt->flag & MM_F_SPLICE_FOR? 1 : 2;
		}
		if (r2.cnt > 0) regs = insert_reg(&r2, i, &n_regs, regs);
		if (i > 0 && regs[i].split_inv && !(opt->flag & MM_F_NO_INV)) {
			if (ra.defer) { ra.defer_abort = true; *n_regs_ = n_regs; return regs; } // the probe reads the two hits' final coordinates
			int ret = D.align1_inv(&regs[i-1], &regs[i], &r2);
			if (ret > 0) {
				regs = insert_reg(&r2, i, &n_regs, regs);
				++i;
			}
		}
	}
	*n_regs_ = n_regs;
	if (ra.incomplete) return regs;
	if (ra.defer && !ra.fin_hits.empty()) return regs; // hl_align_apply_fin() + hl_align_finish() complete the read
	hl_align_finish(opt, ra, n_regs_, regs);
	return regs;
}

bool hl_align_apply_fin(ReadAlign &ra, int n_regs, mm_reg1_t *regs, const HlFinOut *fin, const uint32_t *const *cig)
{
	for (size_t k = 0; k < ra.fin_hits.size(); ++k) if (fin[k].status != 0) return false;
	for (size_t k = 0; k < ra.fin_hits.size(); ++k) {
		const HlFinHit &h = ra.fin_hits[k];
		const HlFinOut &o = fin[k];
		mm_reg1_t *r = nullptr;
		for (int i = 0; i < n_regs; ++i) if (regs[i].p == h.p) { r = &regs[i]; break; }
		assert(r);
		const uint32_t capacity = roundup32((uint32_t)o.n_cigar + sizeof(mm_extra_t) / 4);
		mm_extra_t *p = (mm_extra_t*)realloc(r->p, (size_t)capacity * 4);
		p->capacity = capacity, p->n_cigar = (uint32_t)o.n_cigar;
		if (o.n_cigar > 0) memcpy(p->cigar, cig[k], (size_t)o.n_cigar * 4);
		r->p = p;
		if (o.qshift) { if (r->rev) r->qe -= o.qshift; else r->qs += o.qshift; } // mm_fix_cigar's leading I/D (align.c:172-180)
		r->rs += o.tshift;
		r->blen = o.blen, r->mlen = o.mlen, r->is_spliced = o.is_spliced;
		p->n_ambi += (uint32_t)o.n_ambi;
		p->dp_max = p->dp_max0 = o.dp_max;
	}
	return true;
}

void hl_align_finish(const mm_mapopt_t *opt, ReadAlign &ra, int *n_regs_, mm_reg1_t *regs)
{
	hl_filter_regs(opt, ra.qlen, n_regs_, regs);
	if (!(opt->flag & (MM_F_SR | MM_F_SR_RNA | MM_F_ALL_CHAINS)) && !opt->split_prefix && ra.qlen >= opt->rank_min_len) {
		hl_update_dp_max(ra.qlen, *n_regs_, regs, opt->rank_frac, opt->a, opt->b);
		hl_filter_regs(opt, ra.qlen, n_regs_, regs);
	}
	hl_hit_sort(n_regs_, regs, opt->alt_drop);
}
