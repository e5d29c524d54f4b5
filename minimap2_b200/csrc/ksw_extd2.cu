// minimap2_b200/csrc/ksw_extd2.cu
//
// K3: banded dual-affine-gap extension / global alignment with traceback on sm_90a.
// Replaces ksw_extd2_sse (reference ksw2_extd2_sse.c:27-401), ksw_backtrack / ksw_apply_zdrop (ksw2.h:130-187).
//
// "Universal" kernel: one worker (a warp, or a whole CTA for long jobs) per alignment, anti-diagonal order, the
// same difference recurrence on int8 with wrap-around arithmetic, the same flat per-target-position state arrays
// and the same 16-lane chunk rounding of every anti-diagonal, so results (score, z-drop, max/mqe/mte end points,
// CIGAR) are bit-identical to the reference even when the band clips the matrix and stale lanes are consumed
// (SURVEY 7.2 items 4-6). Four DP cells are packed per 32-bit word (SIMD-in-register byte ops), 128 cells per
// warp step; state lives in shared memory, the 1 B/cell traceback matrix in HBM (L2-resident while hot).
//
// Design notes
//  * v/x/x2 are double-buffered by row parity so every lane reads row r-1 values without ordering constraints
//    (the SSE code gets the same effect by carrying lane 15 in a register). u/y/y2/s are read and written at the
//    same target position only. Because st/en are non-decreasing in r, a lane is active for one contiguous run of
//    rows, which makes the parity double-buffer exact (both buffers start with the same fill).
//  * off[]/off_end[] of the reference (ksw2_extd2_sse.c:230) are pure functions of r and are recomputed in the
//    traceback instead of being stored.
//  * Jobs are pulled from a queue (atomic counter) by persistent workers: grid = SMs x resident CTAs.
#include "mmb_internal.h"
#include "ksw_plan.h"
#include <algorithm>
#include <numeric>
#include <mutex>

#define KSW_NEG_INF (-0x40000000)

namespace {

struct KswArgs {
	const mmb_ksw_job_t *jobs;
	const int *order;      // job indices of this tier, largest first
	int n;                 // jobs in this tier
	const uint8_t *query;
	const void *target;
	int t_packed;
	mmb_ksw_res_t *res;
	uint32_t *cigar;
	long long cigar_cap;
	unsigned long long *cigar_used;
	uint8_t *pws;          // traceback workspace, pws_stride bytes per worker
	size_t pws_stride;
	uint32_t *cigws;       // cigar scratch, cigws_stride uint32 per worker
	size_t cigws_stride;
	int *counter;          // job queue head
	int L, LQ;             // state array length (multiple of 16) / reversed-query length (multiple of 16)
	int8_t mat[25];
	int8_t q, e, q2, e2;   // already ordered so that q+e <= q2+e2
	int qe0;               // q+e as the caller gave them, before that reordering: H(0,0) = v - qe0 (ksw2_extd2_sse.c:68,358,379)
	int8_t skip;           // -min(mat) > 2(q+e): the reference returns immediately (:100)
	int long_thres, long_diff;
	int8_t sp[4];          // spliced variant: penalties of the four signal classes (ksw2_exts2_sse.c:113-121)
	const long long *jst, *jen; // annotated introns sorted by jst, [jst,jen) in target coordinates (mm_idx_bed_junc, index.c:802-826); spliced variant
	const int8_t *jstrand;
	int n_junc;            // 0: no annotation
	const long long *sps_pos[2]; const uint8_t *sps_val[2]; int n_sps[2]; // splice scores per strand (mm_idx_spsc_get, index.c:1055-1075)
	int8_t junc_pen;
	int8_t junc_bonus;
	uint8_t *gws;          // per-worker DP state in HBM for targets that do not fit shared memory (null: shared memory)
	size_t gws_stride;
};

__device__ __forceinline__ uint32_t blend4(uint32_t a, uint32_t b, uint32_t m) { return (a & ~m) | (b & m); } // m ? b : a
__device__ __forceinline__ uint32_t rep4(int8_t v) { return 0x01010101u * (uint8_t)v; }

template<int G> __device__ __forceinline__ void gsync()
{
	if (G == 32) __syncwarp(); else __syncthreads();
}

// group-wide argmax of (h, lower rank wins). scratch: 2*(G/32) ints of shared memory (G>32 only)
template<int G> __device__ __forceinline__ void greduce_max(int &h, int &rank, int *scratch, int g)
{
	const unsigned full = 0xffffffffu;
	int m = __reduce_max_sync(full, h);
	int rk = h == m? rank : 0x7fffffff;
	rk = __reduce_min_sync(full, rk);
	h = m, rank = rk;
	if (G > 32) {
		const int nw = G / 32;
		__syncthreads();
		if ((g & 31) == 0) scratch[(g >> 5) * 2] = h, scratch[(g >> 5) * 2 + 1] = rank;
		__syncthreads();
		int bh = scratch[0], br = scratch[1];
		for (int i = 1; i < nw; ++i) {
			int hh = scratch[i * 2], rr = scratch[i * 2 + 1];
			if (hh > bh || (hh == bh && rr < br)) bh = hh, br = rr;
		}
		h = bh, rank = br;
		__syncthreads();
	}
}

__device__ __forceinline__ uint8_t fetch_target(const void *target, int packed, long long idx)
{
	if (packed) {
		const uint32_t *S = (const uint32_t*)target;
		return (uint8_t)(S[idx >> 3] >> ((idx & 7) << 2) & 0xf);
	}
	return ((const uint8_t*)target)[idx];
}

// bounds of anti-diagonal r (ksw2_extd2_sse.c:132-147)
__device__ __forceinline__ bool diag_bounds(int r, int qlen, int tlen, int w, int &st0, int &en0)
{
	int st = 0, en = tlen - 1;
	if (st < r - qlen + 1) st = r - qlen + 1;
	if (en > r) en = r;
	if (st < (r - w + 1) >> 1) st = (r - w + 1) >> 1;
	if (en > (r + w) >> 1) en = (r + w) >> 1;
	st0 = st, en0 = en;
	return st <= en;
}

struct EzState {
	int max, zdropped, max_q, max_t, mqe, mqe_t, mte, mte_q, score, n_cigar, reach_end;
};

__device__ __forceinline__ void push_cigar(uint32_t *cig, int &n, uint32_t op, int len) // ksw2.h:114-124
{
	if (n == 0 || op != (cig[n - 1] & 0xf)) cig[n++] = (uint32_t)len << 4 | op;
	else cig[n - 1] += (uint32_t)len << 4;
}

// ksw2.h:130-162 (rotated layout), off/off_end recomputed. The walk is inherently serial (one state machine), but each
// step only needs one traceback byte that lies inside a 32-row x 32-column window below-left of the current cell (a step
// lowers r by 1 or 2 and i by 0 or 1). The warp therefore stages that window from HBM/L2 into shared memory with 32
// independent loads per lane (one memory latency per ~16-32 steps instead of one per step), then lane 0 walks inside it.
__device__ int backtrack_tiled(const uint8_t *p, int n_col, int qlen, int tlen, int w, int i0, int j0, uint32_t *cig, uint8_t *tile, int lane, int min_intron_len)
{
	int n = 0, i = i0, j = j0, state = 0;
	for (;;) {
		int go = i >= 0 && j >= 0;
		go = __shfl_sync(0xffffffffu, go, 0);
		if (!go) break;
		const int rt = __shfl_sync(0xffffffffu, i + j, 0), it = __shfl_sync(0xffffffffu, i, 0); // tile anchor: row rt, right column it
		{ // lane k stages row rt-k, columns it-31..it
			const int rr = rt - lane;
			uint8_t *trow = tile + lane * 32;
			if (rr >= 0) {
				int st0, en0;
				diag_bounds(rr, qlen, tlen, w, st0, en0);
				const int off = st0 / 16 * 16, off_end = (en0 + 16) / 16 * 16 - 1;
				const uint8_t *prow = p + (size_t)rr * n_col - off;
				#pragma unroll 8
				for (int c = 0; c < 32; ++c) {
					const int col = it - 31 + c;
					trow[c] = (col >= off && col <= off_end)? prow[col] : 0;
				}
			}
		}
		__syncwarp();
		if (lane == 0) {
			while (i >= 0 && j >= 0) {
				const int r = i + j;
				if (rt - r > 31) break; // left the staged window
				int st0, en0, force = -1;
				diag_bounds(r, qlen, tlen, w, st0, en0);
				const int off = st0 / 16 * 16, off_end = (en0 + 16) / 16 * 16 - 1;
				if (i < off) force = 2;
				if (i > off_end) force = 1;
				const uint32_t tmp = force < 0? tile[(rt - r) * 32 + (i - (it - 31))] : 0;
				if (state == 0) state = tmp & 7;
				else if (!(tmp >> (state + 2) & 1)) state = 0;
				if (state == 0) state = tmp & 7;
				if (force >= 0) state = force;
				if (state == 0) push_cigar(cig, n, 0, 1), --i, --j;
				else if (state == 1 || (state == 3 && min_intron_len <= 0)) push_cigar(cig, n, 2, 1), --i;
				else if (state == 3) push_cigar(cig, n, 3, 1), --i; // an intron (ksw2.h:152)
				else push_cigar(cig, n, 1, 1), --j;
			}
		}
		__syncwarp();
	}
	if (lane == 0) {
		if (i >= 0) push_cigar(cig, n, min_intron_len > 0 && i >= min_intron_len? 3 : 2, i + 1);
		if (j >= 0) push_cigar(cig, n, 1, j + 1);
	}
	return n;
}

// SP = true is ksw_exts2_sse (ksw2_exts2_sse.c:26-465): the second gap state is an intron (open q2, free extension, A.e2 == 0 here)
// whose closing / opening is scored with the acceptor / donor signal of the target position; no band; y2[] holds the donor array.
template<int G, bool SP>
#ifndef KE_MINB
#define KE_MINB 3 // CTAs per SM the register allocation leaves room for: the small-job tiers are latency-bound, residency is their throughput
#endif
__global__ void __launch_bounds__(256, KE_MINB) ksw_extd2_kernel(KswArgs A)
{
	extern __shared__ __align__(16) uint8_t smem_raw[];
	__shared__ int s_job[8];
	__shared__ int s_red[16];
	const int NW = blockDim.x / G;               // workers per CTA
	const int wk = threadIdx.x / G, g = threadIdx.x % G;
	const int worker = blockIdx.x * NW + wk;
	const int L = A.L, LQ = A.LQ;
	const size_t wbytes = (size_t)16 * L + LQ + 64 + 1024;
	uint8_t *base = A.gws? A.gws + A.gws_stride * worker : smem_raw + wbytes * wk;
	uint8_t *bt_tile = A.gws? smem_raw + (size_t)1024 * wk : base + wbytes - 1024;
	// state arrays (all offsets multiples of 16)
	uint8_t *u = base, *y = u + L, *y2 = y + L, *s = y2 + L, *sf = s + L;
	uint8_t *vb[2] = { sf + L, sf + 2 * L }, *xb[2] = { sf + 3 * L, sf + 4 * L }, *x2b[2] = { sf + 5 * L, sf + 6 * L };
	uint8_t *qr = sf + 7 * L + 16;               // 16 zero bytes in front, >=32 behind
	int32_t *H = (int32_t*)(sf + 7 * L + LQ + 64);
	uint8_t *acc = (uint8_t*)(H + L);             // acceptor signals (SP only)
	uint8_t *p = A.pws + A.pws_stride * worker;
	uint32_t *cig = A.cigws + A.cigws_stride * worker;
	const int8_t q = A.q, e = A.e, q2 = A.q2, e2 = A.e2;
	const int8_t qe = (int8_t)(q + e), qe2 = (int8_t)(q2 + e2);
	const uint32_t Q4 = rep4(q), Q24 = rep4(q2), QE4 = rep4(qe), QE24 = rep4(qe2);
	const uint32_t NQE4 = rep4((int8_t)(-q - e)), NQE24 = rep4((int8_t)(-q2 - e2));
	const uint32_t MCH4 = rep4(A.mat[0]), MIS4 = rep4(A.mat[1]);
	const uint32_t SCN4 = rep4(A.mat[24] == 0? (int8_t)(SP? -e : -e2) : A.mat[24]); // ksw2_extd2_sse.c:87 / ksw2_exts2_sse.c:80

	for (;;) {
		if (g == 0) s_job[wk] = atomicAdd(A.counter, 1);
		gsync<G>();
		const int slot = s_job[wk];
		gsync<G>();
		if (slot >= A.n) break;
		const int jid = A.order[slot];
		const mmb_ksw_job_t jb = A.jobs[jid];
		const int qlen = jb.qlen, tlen = jb.tlen, flag = jb.flag;
		int w = jb.w;
		EzState ez;
		ez.max_q = ez.max_t = ez.mqe_t = ez.mte_q = -1;
		ez.max = 0, ez.score = ez.mqe = ez.mte = KSW_NEG_INF;
		ez.n_cigar = 0, ez.zdropped = 0, ez.reach_end = 0;
		if (qlen <= 0 || tlen <= 0 || A.skip) {
			if (g == 0) {
				mmb_ksw_res_t o;
				o.zd_max = -1, o.zd_t0 = o.zd_t1 = o.zd_q0 = o.zd_q1 = -1;
				o.max = ez.max, o.zdropped = 0, o.max_q = o.max_t = o.mqe_t = o.mte_q = -1;
				o.mqe = o.mte = o.score = KSW_NEG_INF, o.n_cigar = 0, o.reach_end = 0, o.cigar_off = 0;
				A.res[jid] = o;
			}
			continue;
		}
		const bool with_cigar = !(flag & MMB_KSW_SCORE_ONLY), approx_max = (flag & MMB_KSW_APPROX_MAX) != 0;
		const bool right = (flag & MMB_KSW_RIGHT) != 0, generic = (flag & MMB_KSW_GENERIC_SC) != 0;
		if (SP || w < 0) w = tlen > qlen? tlen : qlen; // ksw_exts2_sse takes no band (ksw2_exts2_sse.c:26-31): the driver's bandwidth is not part of a spliced call
		const int tlen16 = (tlen + 15) / 16 * 16;
		int n_col = qlen < tlen? qlen : tlen;
		n_col = (((n_col < w + 1? n_col : w + 1) + 15) / 16 + 1) * 16;

		// ---- stage sequences and initialise state (ksw2_extd2_sse.c:107-129) ----
		for (int i = g * 4; i < tlen16; i += G * 4) {
			*(uint32_t*)(u + i) = NQE4, *(uint32_t*)(y + i) = NQE4, *(uint32_t*)(y2 + i) = NQE24, *(uint32_t*)(s + i) = 0;
			*(uint32_t*)(vb[0] + i) = NQE4, *(uint32_t*)(vb[1] + i) = NQE4;
			*(uint32_t*)(xb[0] + i) = NQE4, *(uint32_t*)(xb[1] + i) = NQE4;
			*(uint32_t*)(x2b[0] + i) = NQE24, *(uint32_t*)(x2b[1] + i) = NQE24;
			if (!approx_max) { H[i] = H[i + 1] = H[i + 2] = H[i + 3] = KSW_NEG_INF; }
		}
		{
			const bool tc = (flag & MMB_JOB_T_COMP) != 0;
			for (int i = g; i < tlen16; i += G) {
				uint8_t c = i < tlen? fetch_target(A.target, A.t_packed, jb.t_start + (long long)i * jb.t_step) : 0;
				if (tc && c < 4 && i < tlen) c = 3 - c;
				sf[i] = c;
			}
		}
		for (int i = g; i < LQ + 48; i += G) { // qr[-16 .. LQ+32)
			int k = i - 16; // position in qr
			uint8_t c = 0;
			if (k >= 0 && k < qlen) {
				c = A.query[jb.q_start + (long long)(qlen - 1 - k) * jb.q_step];
				if ((flag & MMB_JOB_Q_COMP) && c < 4) c = 3 - c;
			}
			qr[k] = c;
		}
		gsync<G>();
		if (SP) { // donor / acceptor arrays (ksw2_exts2_sse.c:111-190) + annotated junctions (:220-241)
			const bool fo = (flag & MMB_KSW_SPLICE_FOR) != 0, re = (flag & MMB_KSW_SPLICE_REV) != 0, rc = (flag & MMB_KSW_REV_CIGAR) != 0;
			const bool with_score = (flag & MMB_KSW_SPLICE_SCORE) != 0; // junc[] carries per-site scores (ksw2_exts2_sse.c:213-219)
			const bool with_junc = !with_score && A.n_junc > 0 && (fo || re);
			if (with_score) {
				// junc[] = mm_idx_spsc_get over the job's window on the strand SPLICE_REV selects (align.c:638-640): 0xff, or the
				// score byte of the positions strictly inside the window; staged in s[] and cleared again below
				for (int i = g * 4; i < tlen16; i += G * 4) *(uint32_t*)(s + i) = 0xffffffffu;
				gsync<G>();
				const int sd = re? 1 : 0;
				const long long wlo = jb.t_step > 0? jb.t_start : jb.t_start - (tlen - 1), whi = wlo + tlen;
				int lo = 0, hi = A.n_sps[sd];
				while (hi > lo) { const int mid = lo + ((hi - lo) >> 1); if (A.sps_pos[sd][mid] > wlo) hi = mid; else lo = mid + 1; }
				for (int k = lo + g; k < A.n_sps[sd]; k += G) {
					const long long pos = A.sps_pos[sd][k];
					if (pos >= whi) break;
					s[jb.t_step > 0? pos - jb.t_start : jb.t_start - pos] = A.sps_val[sd][k];
				}
				gsync<G>();
			}
			if (with_junc) {
				// junc[] of this call = mm_idx_bed_junc over the job's target window, reversed with the target for a reversed job
				// (align.c:787-790): flags of the introns lying entirely inside the window, OR-ed into s[] (all zero here) and
				// cleared again below
				const long long wlo = jb.t_step > 0? jb.t_start : jb.t_start - (tlen - 1), whi = wlo + tlen;
				int lo = 0, hi = A.n_junc;
				while (hi > lo) { const int mid = lo + ((hi - lo) >> 1); if (A.jst[mid] >= wlo) hi = mid; else lo = mid + 1; }
				for (int k = lo + g; k < A.n_junc; k += G) {
					const long long st = A.jst[k];
					if (st >= whi) break;
					const long long en = A.jen[k];
					const int sd = A.jstrand[k];
					if (en <= whi && sd != 0) {
						const int i1 = (int)(jb.t_step > 0? st - jb.t_start : jb.t_start - st);
						const int i2 = (int)(jb.t_step > 0? en - 1 - jb.t_start : jb.t_start - (en - 1));
						atomicOr((unsigned*)(s + (i1 & ~3)), (unsigned)(sd > 0? 1 : 8) << ((i1 & 3) * 8));
						atomicOr((unsigned*)(s + (i2 & ~3)), (unsigned)(sd > 0? 2 : 4) << ((i2 & 3) * 8));
					}
				}
				gsync<G>();
			}
			for (int i = g; i < tlen16; i += G) {
				int8_t d = 0, a = 0;
				if (fo || re) {
					d = a = (int8_t)-A.sp[3];
					if (i < tlen - 4) {
						const int c1 = sf[i + 1], c2 = sf[i + 2], c3 = sf[i + 3];
						int z = 3;
						if (!rc) {
							if (fo) { if (c1 == 2 && c2 == 3) z = c3 == 0 || c3 == 2? -1 : 0; else if (c1 == 2 && c2 == 1) z = 1; else if (c1 == 0 && c2 == 3) z = 2; }
							else { if (c1 == 1 && c2 == 3) z = c3 == 0 || c3 == 2? -1 : 0; else if (c1 == 2 && c2 == 3) z = 2; }
						} else {
							if (fo) { if (c1 == 2 && c2 == 0) z = c3 == 1 || c3 == 3? -1 : 0; else if (c1 == 1 && c2 == 0) z = 2; }
							else { if (c1 == 1 && c2 == 0) z = c3 == 1 || c3 == 3? -1 : 0; else if (c1 == 1 && c2 == 2) z = 1; else if (c1 == 3 && c2 == 0) z = 2; }
						}
						d = z < 0? 0 : (int8_t)-A.sp[z];
					}
					if (i >= 2 && i < tlen) {
						const int c0 = sf[i - 2], c1 = sf[i - 1], c2 = sf[i];
						int z = 3;
						if (!rc) {
							if (fo) { if (c1 == 0 && c2 == 2) z = c0 == 1 || c0 == 3? -1 : 0; else if (c1 == 0 && c2 == 1) z = 2; }
							else { if (c1 == 0 && c2 == 1) z = c0 == 1 || c0 == 3? -1 : 0; else if (c1 == 2 && c2 == 1) z = 1; else if (c1 == 0 && c2 == 3) z = 2; }
						} else {
							if (fo) { if (c1 == 3 && c2 == 2) z = c0 == 0 || c0 == 2? -1 : 0; else if (c1 == 1 && c2 == 2) z = 1; else if (c1 == 3 && c2 == 0) z = 2; }
							else { if (c1 == 3 && c2 == 1) z = c0 == 0 || c0 == 2? -1 : 0; else if (c1 == 3 && c2 == 2) z = 2; }
						}
						a = z < 0? 0 : (int8_t)-A.sp[z];
					}
					if (with_junc) { // ksw2_exts2_sse.c:220-241 (int8 wrap-around like the reference's array arithmetic)
						const int jd = i < tlen - 1? s[i + 1] : 0, ja = i < tlen? s[i] : 0;
						const int dm = rc? (fo? 2 : 0) | (re? 4 : 0) : (fo? 1 : 0) | (re? 8 : 0);
						const int am = rc? (fo? 1 : 0) | (re? 8 : 0) : (fo? 2 : 0) | (re? 4 : 0);
						if (jd & dm) d = (int8_t)(d + A.junc_bonus);
						if (ja & am) a = (int8_t)(a + A.junc_bonus);
					}
				}
				if (with_score && i < tlen - 1) { // :213-219
					const int donor_val = fo == !rc? 0 : 1, jv = s[i + 1];
					d = (int8_t)(d + (jv == 0xff || (jv & 1) != donor_val? -A.junc_pen : (int8_t)(jv >> 1) - (int8_t)64));
					a = (int8_t)(a + (jv == 0xff || (jv & 1) != !donor_val? -A.junc_pen : (int8_t)(jv >> 1) - (int8_t)64));
				}
				y2[i] = (uint8_t)d, acc[i] = (uint8_t)a;
			}
			gsync<G>();
			if (with_junc || with_score) {
				for (int i = g * 4; i < tlen16; i += G * 4) *(uint32_t*)(s + i) = 0;
				gsync<G>();
			}
		}

		int last_st = -1, last_en = -1;
		int H0 = 0, last_H0_t = 0;      // approximate-max tracker (thread 0)
		const int n_rows = qlen + tlen - 1;
		int r;
		for (r = 0; r < n_rows; ++r) {
			int st0, en0;
			if (!diag_bounds(r, qlen, tlen, w, st0, en0)) { ez.zdropped = 1; break; }
			const int st = st0 / 16 * 16, en = (en0 + 16) / 16 * 16 - 1;
			const int nb = r & 1, ob = nb ^ 1;
			uint8_t *vn = vb[nb], *xn = xb[nb], *x2n = x2b[nb];
			const uint8_t *vo = vb[ob], *xo = xb[ob], *x2o = x2b[ob];
			int8_t x1, x21, v1;
			const int8_t vbound = r == 0? (int8_t)(-q - e) : r < A.long_thres? (int8_t)(-e) : r == A.long_thres? (int8_t)A.long_diff : (int8_t)(-e2);
			if (st > 0) { // :149-158
				if (st - 1 >= last_st && st - 1 <= last_en) x1 = (int8_t)xo[st - 1], x21 = (int8_t)x2o[st - 1], v1 = (int8_t)vo[st - 1];
				else x1 = (int8_t)(-q - e), x21 = (int8_t)(-q2 - e2), v1 = (int8_t)(-q - e);
			} else x1 = (int8_t)(-q - e), x21 = (int8_t)(-q2 - e2), v1 = vbound;
			const bool set_top = en >= r; // :159-162 (applied in registers: only lane r reads y[r], y2[r], u[r] this row)
			// fresh score range [st0, s_end) in 16-byte chunks from st0 (:165-180); generic: [st0, en0]
			const int s_end = generic? en0 + 1 : min(st0 + ((en0 - st0) / 16 + 1) * 16, tlen16);
			const int t_hi = max(en, s_end - 1);
			const int qoff = qlen - 1 - r;
			uint8_t *prow = p + (size_t)r * n_col;

			for (int t0 = st + 4 * g; t0 <= t_hi; t0 += 4 * G) {
				uint32_t S = *(const uint32_t*)(s + t0);
				if (t0 + 3 >= st0 && t0 < s_end) { // some byte of this word gets a fresh score
					uint32_t fresh;
					if (!generic) {
						uint32_t sq = *(const uint32_t*)(sf + t0);
						int qi = qoff + t0; // >= -16 thanks to the front pad
						const uint32_t *qw = (const uint32_t*)(qr + (qi & ~3));
						uint32_t sr = __funnelshift_r(qw[0], qw[1], (qi & 3) * 8);
						uint32_t nmask = __vcmpeq4(sq, 0x04040404u) | __vcmpeq4(sr, 0x04040404u);
						fresh = blend4(MIS4, MCH4, __vcmpeq4(sq, sr));
						fresh = blend4(fresh, SCN4, nmask);
					} else {
						fresh = 0;
						for (int b = 0; b < 4; ++b) {
							int t = t0 + b;
							if (t >= st0 && t < s_end) fresh |= (uint32_t)(uint8_t)A.mat[sf[t] * 5 + qr[qoff + t]] << (8 * b);
						}
					}
					uint32_t m = 0;
					#pragma unroll
					for (int b = 0; b < 4; ++b) if (t0 + b >= st0 && t0 + b < s_end) m |= 0xffu << (8 * b);
					S = blend4(S, fresh, m);
					*(uint32_t*)(s + t0) = S;
				}
				if (t0 > en) continue; // score-only overshoot lanes
				uint32_t U = *(const uint32_t*)(u + t0), Y = *(const uint32_t*)(y + t0), Y2 = *(const uint32_t*)(y2 + t0);
				uint32_t Vo = *(const uint32_t*)(vo + t0), Xo = *(const uint32_t*)(xo + t0), X2o = *(const uint32_t*)(x2o + t0);
				uint32_t vp, xp, x2p;
				if (t0 == st) vp = (uint8_t)v1, xp = (uint8_t)x1, x2p = (uint8_t)x21;
				else vp = vo[t0 - 1], xp = xo[t0 - 1], x2p = x2o[t0 - 1];
				if (set_top && r >= t0 && r < t0 + 4) {
					uint32_t sh = (r - t0) * 8, m = 0xffu << sh;
					Y = (Y & ~m) | ((NQE4 & 0xff) << sh);
					Y2 = (Y2 & ~m) | ((NQE24 & 0xff) << sh);
					U = (U & ~m) | ((uint32_t)(uint8_t)vbound << sh);
				}
				const uint32_t VT1 = Vo << 8 | vp, XT1 = Xo << 8 | xp, X2T1 = X2o << 8 | x2p;
				uint32_t Aa = __vadd4(XT1, VT1), Bb = __vadd4(Y, U), A2 = __vadd4(X2T1, VT1), B2 = __vadd4(Y2, U);
				uint32_t Z = S, D = 0, m;
				if (SP) { // ksw2_exts2_sse.c:36-66,283-380: three candidates, no clip, the intron state is floored by the donor signal
					const uint32_t DON = *(const uint32_t*)(y2 + t0), A2A = __vadd4(A2, *(const uint32_t*)(acc + t0));
					if (!right) {
						m = __vcmpgts4(Aa, Z);  D = m & 0x01010101u;            Z = blend4(Z, Aa, m);
						m = __vcmpgts4(Bb, Z);  D = blend4(D, 0x02020202u, m);  Z = blend4(Z, Bb, m);
						m = __vcmpgts4(A2A, Z); D = blend4(D, 0x03030303u, m);  Z = blend4(Z, A2A, m);
					} else {
						m = __vcmpgts4(Z, Aa);  D = ~m & 0x01010101u;           Z = blend4(Aa, Z, m);
						m = __vcmpgts4(Z, Bb);  D = blend4(0x02020202u, D, m);  Z = blend4(Bb, Z, m);
						m = __vcmpgts4(Z, A2A); D = blend4(0x03030303u, D, m);  Z = blend4(A2A, Z, m);
					}
					*(uint32_t*)(u + t0) = __vsub4(Z, VT1);
					*(uint32_t*)(vn + t0) = __vsub4(Z, U);
					uint32_t T = __vsub4(Z, Q4);
					Aa = __vsub4(Aa, T), Bb = __vsub4(Bb, T);
					A2 = __vsub4(A2, __vsub4(Z, Q24));
					if (!right) {
						m = __vcmpgts4(Aa, 0);   *(uint32_t*)(xn + t0)  = __vsub4(Aa & m, QE4);             D |= m & 0x08080808u;
						m = __vcmpgts4(Bb, 0);   *(uint32_t*)(y + t0)   = __vsub4(Bb & m, QE4);             D |= m & 0x10101010u;
						m = __vcmpgts4(A2, DON); *(uint32_t*)(x2n + t0) = __vsub4(blend4(DON, A2, m), Q24); D |= m & 0x20202020u;
					} else {
						m = ~__vcmpgts4(0, Aa);   *(uint32_t*)(xn + t0)  = __vsub4(Aa & m, QE4);             D |= m & 0x08080808u;
						m = ~__vcmpgts4(0, Bb);   *(uint32_t*)(y + t0)   = __vsub4(Bb & m, QE4);             D |= m & 0x10101010u;
						m = ~__vcmpgts4(DON, A2); *(uint32_t*)(x2n + t0) = __vsub4(blend4(DON, A2, m), Q24); D |= m & 0x20202020u;
					}
				} else {
				if (!right) { // :232-243
					m = __vcmpgts4(Aa, Z); D = m & 0x01010101u;            Z = blend4(Z, Aa, m);
					m = __vcmpgts4(Bb, Z); D = blend4(D, 0x02020202u, m);  Z = blend4(Z, Bb, m);
					m = __vcmpgts4(A2, Z); D = blend4(D, 0x03030303u, m);  Z = blend4(Z, A2, m);
					m = __vcmpgts4(B2, Z); D = blend4(D, 0x04040404u, m);  Z = blend4(Z, B2, m);
				} else {      // :279-290
					m = __vcmpgts4(Z, Aa); D = ~m & 0x01010101u;           Z = blend4(Aa, Z, m);
					m = __vcmpgts4(Z, Bb); D = blend4(0x02020202u, D, m);  Z = blend4(Bb, Z, m);
					m = __vcmpgts4(Z, A2); D = blend4(0x03030303u, D, m);  Z = blend4(A2, Z, m);
					m = __vcmpgts4(Z, B2); D = blend4(0x04040404u, D, m);  Z = blend4(B2, Z, m);
				}
				Z = __vmins4(Z, MCH4);
				*(uint32_t*)(u + t0) = __vsub4(Z, VT1);
				*(uint32_t*)(vn + t0) = __vsub4(Z, U);
				uint32_t T = __vsub4(Z, Q4);
				Aa = __vsub4(Aa, T), Bb = __vsub4(Bb, T);
				T = __vsub4(Z, Q24);
				A2 = __vsub4(A2, T), B2 = __vsub4(B2, T);
				if (!right) { // keep if > 0 (:261-273)
					m = __vcmpgts4(Aa, 0); *(uint32_t*)(xn + t0)  = __vsub4(Aa & m, QE4);  D |= m & 0x08080808u;
					m = __vcmpgts4(Bb, 0); *(uint32_t*)(y + t0)   = __vsub4(Bb & m, QE4);  D |= m & 0x10101010u;
					m = __vcmpgts4(A2, 0); *(uint32_t*)(x2n + t0) = __vsub4(A2 & m, QE24); D |= m & 0x20202020u;
					m = __vcmpgts4(B2, 0); *(uint32_t*)(y2 + t0)  = __vsub4(B2 & m, QE24); D |= m & 0x40404040u;
				} else {      // keep if >= 0 (:308-320)
					m = ~__vcmpgts4(0, Aa); *(uint32_t*)(xn + t0)  = __vsub4(Aa & m, QE4);  D |= m & 0x08080808u;
					m = ~__vcmpgts4(0, Bb); *(uint32_t*)(y + t0)   = __vsub4(Bb & m, QE4);  D |= m & 0x10101010u;
					m = ~__vcmpgts4(0, A2); *(uint32_t*)(x2n + t0) = __vsub4(A2 & m, QE24); D |= m & 0x20202020u;
					m = ~__vcmpgts4(0, B2); *(uint32_t*)(y2 + t0)  = __vsub4(B2 & m, QE24); D |= m & 0x40404040u;
				}
				}
				if (with_cigar) *(uint32_t*)(prow + (t0 - st)) = D;
			}
			gsync<G>();

			int stop = 0;
			if (!approx_max) { // exact max with the reference's tie rules (:323-366)
				int max_H, max_t;
				if (r > 0) {
					int Hen0 = 0;
					if (g == 0) Hen0 = en0 > 0? H[en0 - 1] + (int8_t)u[en0] : H[en0] + (int8_t)vn[en0];
					gsync<G>();
					const int nblk = (en0 - st0) / 4, en1 = st0 + nblk * 4;
					int bh = KSW_NEG_INF, brank = 0x7fffffff;
					for (int t = st0 + g; t < en0; t += G) {
						int hv = H[t] + (int8_t)vn[t];
						H[t] = hv;
						int idx = t - st0;
						int rank = t < en1? 1 + (idx & 3) * nblk + (idx >> 2) : 1 + 4 * nblk + (t - en1);
						if (hv > bh || (hv == bh && rank < brank)) bh = hv, brank = rank;
					}
					if (g == 0) {
						H[en0] = Hen0;
						if (Hen0 > bh || Hen0 == bh) bh = Hen0, brank = 0; // the seed candidate wins ties (strict > to displace it)
					}
					greduce_max<G>(bh, brank, s_red, g);
					max_H = bh;
					if (brank == 0) max_t = en0;
					else if (brank <= 4 * nblk) { int k = brank - 1; max_t = st0 + (k % nblk) * 4 + k / nblk; }
					else max_t = en1 + (brank - 1 - 4 * nblk);
				} else {
					if (g == 0) H[0] = (int8_t)vn[0] - A.qe0;
					gsync<G>();
					max_H = H[0], max_t = 0;
				}
				gsync<G>();
				// every thread keeps ez in registers and applies the same updates (values are group-uniform)
				if (en0 == tlen - 1 && H[en0] > ez.mte) ez.mte = H[en0], ez.mte_q = r - en0;
				if (r - st0 == qlen - 1 && H[st0] > ez.mqe) ez.mqe = H[st0], ez.mqe_t = st0;
				// ksw_apply_zdrop (ksw2.h:171-187)
				if (max_H > ez.max) ez.max = max_H, ez.max_t = max_t, ez.max_q = r - max_t;
				else if (max_t >= ez.max_t && r - max_t >= ez.max_q) {
					int tl = max_t - ez.max_t, ql = (r - max_t) - ez.max_q, l = tl > ql? tl - ql : ql - tl;
					if (jb.zdrop >= 0 && ez.max - max_H > jb.zdrop + l * e2) ez.zdropped = 1, stop = 1;
				}
				if (!stop && r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H[tlen - 1];
				gsync<G>(); // H is rewritten next row
			} else { // approximate max: follow one path (:367-383); thread 0 tracks it, result broadcast at the end
				if (g == 0) {
					if (r > 0) {
						if (last_H0_t >= st0 && last_H0_t <= en0 && last_H0_t + 1 >= st0 && last_H0_t + 1 <= en0) {
							int d0 = (int8_t)vn[last_H0_t], d1 = (int8_t)u[last_H0_t + 1];
							if (d0 > d1) H0 += d0; else H0 += d1, ++last_H0_t;
						} else if (last_H0_t >= st0 && last_H0_t <= en0) H0 += (int8_t)vn[last_H0_t];
						else ++last_H0_t, H0 += (int8_t)u[last_H0_t];
					} else H0 = (int8_t)vn[0] - A.qe0, last_H0_t = 0;
				}
				if (flag & MMB_KSW_APPROX_DROP) { // not used by align.c; supported for API completeness
					int hh = __shfl_sync(0xffffffffu, H0, 0), tt = __shfl_sync(0xffffffffu, last_H0_t, 0);
					if (G > 32) { if (g == 0) s_red[0] = H0, s_red[1] = last_H0_t; __syncthreads(); hh = s_red[0], tt = s_red[1]; __syncthreads(); }
					if (hh > ez.max) ez.max = hh, ez.max_t = tt, ez.max_q = r - tt;
					else if (tt >= ez.max_t && r - tt >= ez.max_q) {
						int tl = tt - ez.max_t, ql = (r - tt) - ez.max_q, l = tl > ql? tl - ql : ql - tl;
						if (jb.zdrop >= 0 && ez.max - hh > jb.zdrop + l * e2) ez.zdropped = 1, stop = 1;
					}
				}
				if (!stop && r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H0; // only thread 0's copy is meaningful
				gsync<G>(); // thread 0 read u[]/v[] of this row: the other lanes must not start overwriting them for the next row before that
			}
			if (stop) break;
			last_st = st, last_en = en;
		}

		// ---- traceback (ksw2_extd2_sse.c:388-400) and result write-out ----
		int n_cig = 0;
		bool rev_cigar = (flag & MMB_KSW_REV_CIGAR) != 0;
		if (with_cigar) {
			int bi = -1, bj = -1;
			if (!ez.zdropped && !(flag & MMB_KSW_EXTZ_ONLY)) bi = tlen - 1, bj = qlen - 1;
			else if (!ez.zdropped && (flag & MMB_KSW_EXTZ_ONLY) && ez.mqe + jb.end_bonus > ez.max) ez.reach_end = 1, bi = ez.mqe_t, bj = qlen - 1;
			else if (ez.max_t >= 0 && ez.max_q >= 0) bi = ez.max_t, bj = ez.max_q;
			__threadfence_block();
			gsync<G>();
			if (g < 32 && bi >= 0) n_cig = backtrack_tiled(p, n_col, qlen, tlen, w, bi, bj, cig, bt_tile, g, SP? A.long_thres : 0);
			if (G == 32) n_cig = __shfl_sync(0xffffffffu, n_cig, 0);
			else { if (g == 0) s_red[0] = n_cig; __syncthreads(); n_cig = s_red[0]; __syncthreads(); }
		}
		unsigned long long coff = 0;
		if (n_cig > 0) {
			if (g == 0) coff = atomicAdd(A.cigar_used, (unsigned long long)n_cig);
			if (G == 32) coff = __shfl_sync(0xffffffffu, coff, 0);
			else { if (g == 0) *(unsigned long long*)s_red = coff; __syncthreads(); coff = *(unsigned long long*)s_red; __syncthreads(); }
			if ((long long)(coff + n_cig) <= A.cigar_cap)
				for (int i = g; i < n_cig; i += G)
					A.cigar[coff + i] = rev_cigar? cig[i] : cig[n_cig - 1 - i];
		}
		if (g == 0) {
			mmb_ksw_res_t o;
			o.zd_max = -1, o.zd_t0 = o.zd_t1 = o.zd_q0 = o.zd_q1 = -1;
			o.max = ez.max, o.zdropped = ez.zdropped, o.max_q = ez.max_q, o.max_t = ez.max_t;
			o.mqe = ez.mqe, o.mqe_t = ez.mqe_t, o.mte = ez.mte, o.mte_q = ez.mte_q;
			o.score = ez.score, o.n_cigar = n_cig, o.reach_end = ez.reach_end, o.cigar_off = (uint32_t)coff;
			A.res[jid] = o;
		}
		gsync<G>();
	}
}

// ---------------------------------------------------------------------------------------------------------
// ksw_ll_i16 (reference ksw2_ll_sse.c:37-152): Farrar-striped local alignment score with int16 saturation, used only for
// inversion probes (align.c:95-96, :940-941). The 8 int16 lanes of an SSE register map to 8 threads; a warp runs 4 jobs.
// The striped order is part of the contract: the lazy-F loop leaves E uncorrected and the reported query end is the LAST
// striped slot holding the maximum (:148-150).
// ---------------------------------------------------------------------------------------------------------
struct LLArgs {
	const mmb_ksw_job_t *jobs;
	const int *order;
	int n;
	const uint8_t *query;
	const void *target;
	int t_packed;
	mmb_ksw_res_t *res;
	int16_t *ws;          // per group: 4 arrays of slen_max*8 int16 + query bytes
	size_t ws_stride;     // bytes per group
	int slen_max;
	int *counter;
	int8_t mat[25];
};

__device__ __forceinline__ int16_t subs_u16(int16_t a, uint16_t b) { uint16_t ua = (uint16_t)a; return ua > b? (int16_t)(ua - b) : (int16_t)0; }
__device__ __forceinline__ int16_t max16(int16_t a, int16_t b) { return a > b? a : b; }

__global__ void __launch_bounds__(128) ksw_ll_kernel(LLArgs A)
{
	const int lane = threadIdx.x & 31, k = lane & 7, grp = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
	const unsigned gmask = 0xffu << (lane & 24);
	uint8_t *wsb = (uint8_t*)A.ws + A.ws_stride * grp;
	const int SM = A.slen_max * 8;
	int16_t *H0 = (int16_t*)wsb, *H1 = H0 + SM, *E = H1 + SM, *Hmax = E + SM;
	uint8_t *qs = (uint8_t*)(Hmax + SM);
	for (;;) {
		int slot = 0;
		if (k == 0) slot = atomicAdd(A.counter, 1);
		slot = __shfl_sync(gmask, slot, lane & 24);
		if (slot >= A.n) break;
		const int jid = A.order[slot];
		const mmb_ksw_job_t jb = A.jobs[jid];
		const int qlen = jb.qlen, tlen = jb.tlen, slen = (qlen + 7) / 8;
		const uint16_t go = (uint16_t)(jb.w + jb.zdrop), ge = (uint16_t)jb.zdrop; // w = gap open, zdrop = gap extension for LL jobs
		for (int i = k; i < slen * 8; i += 8) {
			H0[i] = 0, E[i] = 0, Hmax[i] = 0, H1[i] = 0;
			uint8_t c = 0;
			if (i < qlen) {
				c = A.query[jb.q_start + (long long)i * jb.q_step];
				if ((jb.flag & MMB_JOB_Q_COMP) && c < 4) c = 3 - c;
			}
			qs[i] = c;
		}
		__syncwarp(gmask);
		int gmax = 0, qe = -1, te = -1;
		for (int i = 0; i < tlen; ++i) {
			int t = fetch_target(A.target, A.t_packed, jb.t_start + (long long)i * jb.t_step);
			if ((jb.flag & MMB_JOB_T_COMP) && t < 4) t = 3 - t;
			const int8_t *ma = A.mat + t * 5;
			int16_t f = 0, mx = 0, h, e;
			h = slen > 0? H0[(slen - 1) * 8 + k] : 0;
			h = __shfl_up_sync(gmask, h, 1, 8);
			if (k == 0) h = 0;
			for (int j = 0; j < slen; ++j) {
				const int qp = j + k * slen;
				const int sc = qp >= qlen? -1 : ma[qs[qp]];
				int t32 = (int)h + sc;
				t32 = t32 > 32767? 32767 : t32 < -32768? -32768 : t32;
				h = (int16_t)t32;
				e = E[j * 8 + k];
				h = max16(h, e); h = max16(h, f); mx = max16(mx, h);
				H1[j * 8 + k] = h;
				const int16_t hs = subs_u16(h, go);
				e = subs_u16(e, ge); e = max16(e, hs);
				E[j * 8 + k] = e;
				f = subs_u16(f, ge); f = max16(f, hs);
				h = H0[j * 8 + k];
			}
			bool done = false;
			for (int kk = 0; kk < 8 && !done; ++kk) { // lazy F (:124-135)
				f = __shfl_up_sync(gmask, f, 1, 8);
				if (k == 0) f = 0;
				for (int j = 0; j < slen; ++j) {
					int16_t hh = H1[j * 8 + k];
					hh = max16(hh, f);
					H1[j * 8 + k] = hh;
					const int16_t hs = subs_u16(hh, go);
					f = subs_u16(f, ge);
					if (!(__ballot_sync(gmask, f > hs) & gmask)) { done = true; break; }
				}
			}
			int imax = mx;
			for (int o = 4; o > 0; o >>= 1) imax = max(imax, __shfl_xor_sync(gmask, imax, o, 8));
			if (imax >= gmax) {
				gmax = imax, te = i;
				for (int j = 0; j < slen; ++j) Hmax[j * 8 + k] = H1[j * 8 + k];
			}
			int16_t *tmp = H1; H1 = H0; H0 = tmp;
		}
		int best = -1;
		for (int j = 0; j < slen; ++j) if ((int)(uint16_t)Hmax[j * 8 + k] == gmax) best = j * 8 + k;
		for (int o = 4; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(gmask, best, o, 8));
		if (best >= 0) qe = best / 8 + best % 8 * slen;
		if (k == 0) {
			mmb_ksw_res_t o;
			o.zd_max = -1, o.zd_t0 = o.zd_t1 = o.zd_q0 = o.zd_q1 = -1;
			o.max = 0, o.zdropped = 0, o.max_q = qe, o.max_t = te, o.mqe = o.mte = KSW_NEG_INF, o.mqe_t = o.mte_q = -1;
			o.score = gmax, o.n_cigar = 0, o.reach_end = 0, o.cigar_off = 0;
			A.res[jid] = o;
		}
		__syncwarp(gmask);
	}
}

} // namespace

bool mmb_ksw_fast_eligible(const mmb_ksw_job_t &j);
void mmb_ksw_fast_plan(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, const std::vector<int> &idx, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
					   const uint8_t *d_query, const void *d_target, int t_packed, mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap,
					   unsigned long long *d_cigar_used, int *d_order_all, std::vector<KswPlan> &plans);

// Host-side tiering. Tiers by max(qlen,tlen): warp-per-job for <=1024, CTA-per-job above. Nothing goes on the stream.
void mmb_ksw_plan(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
				  const uint8_t *d_query, const void *d_target, int t_packed,
				  mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap, unsigned long long *d_cigar_used, KswLaunch &K)
{
	if (n_jobs <= 0) return;
	KswArgs A;
	A.jobs = d_jobs, A.query = d_query, A.target = d_target, A.t_packed = t_packed, A.res = d_res;
	A.cigar = d_cigar, A.cigar_cap = cigar_cap, A.cigar_used = d_cigar_used;
	for (int i = 0; i < 25; ++i) A.mat[i] = sc->mat[i];
	int8_t q = sc->q, e = sc->e, q2 = sc->q2, e2 = sc->e2;
	A.qe0 = q + e; // the same in both passes: ksw_exts2_sse does not reorder (ksw2_exts2_sse.c:65)
	if (q2 + e2 < q + e) std::swap(q, q2), std::swap(e, e2); // ksw2_extd2_sse.c:78
	A.q = q, A.e = e, A.q2 = q2, A.e2 = e2;
	int min_sc = sc->mat[1];
	for (int i = 1; i < 25; ++i) min_sc = std::min<int>(min_sc, sc->mat[i]);
	A.skip = -min_sc > 2 * (q + e);
	int lt = e != e2? (q2 - q) / (e - e2) - 1 : 0; // :102-105
	if (q2 + e2 + lt * e2 > q + e + lt * e) ++lt;
	A.long_thres = lt, A.long_diff = lt * (e - e2) - (q2 - q) - e2;
	A.gws = nullptr, A.gws_stride = 0;
	{ // signal-class penalties of the spliced kernel (ksw2_exts2_sse.c:113-121); the model bits are the same for every job of a batch
		bool cmplx = false, flank = false;
		for (int i = 0; i < n_jobs; ++i) if (h_jobs[i].flag & MMB_JOB_SPLICE) { cmplx = (h_jobs[i].flag & MMB_KSW_SPLICE_CMPLX) != 0, flank = (h_jobs[i].flag & MMB_KSW_SPLICE_FLANK) != 0; break; }
		static const int sp0[4] = { 8, 15, 21, 30 };
		for (int t = 0; t < 4; ++t) A.sp[t] = cmplx? (int8_t)((double)sp0[t] / 3. + .499) : (int8_t)(t == 0? (flank? sc->noncan / 2 : 0) : sc->noncan);
		A.jst = (const long long*)ctx->junc_st, A.jen = (const long long*)ctx->junc_en, A.jstrand = ctx->junc_strand;
		A.n_junc = (int)ctx->n_junc, A.junc_bonus = sc->junc_bonus, A.junc_pen = sc->junc_pen;
		for (int t = 0; t < 2; ++t) A.sps_pos[t] = (const long long*)ctx->spsc_pos[t], A.sps_val[t] = ctx->spsc_val[t], A.n_sps[t] = (int)ctx->n_spsc[t];
	}

	// tiers: {max len16, group size, workers per CTA}; the last tier keeps the DP state in HBM instead of shared memory
	struct Tier { int maxlen, G, nw; };
	Tier tiers[] = { {256, 32, 8}, {512, 32, 8}, {1024, 32, 4}, {13000, 256, 1}, {1 << 20, 256, 1} };
	const int n_tiers = 5;
	static const int smem_maxlen = getenv("MM_B200_KSW_SMEM_MAXLEN")? atoi(getenv("MM_B200_KSW_SMEM_MAXLEN")) : 13000; // test hook: push shorter jobs into the HBM-state tier
	for (int k = 0; k < n_tiers - 1; ++k) tiers[k].maxlen = std::min(tiers[k].maxlen, std::max(16, smem_maxlen));
	std::vector<std::vector<int>> tj(2 * (n_tiers + 1)); // [0, n_tiers]: ksw_extd2 jobs, [n_tiers+1, ..]: spliced (ksw_exts2) jobs
	uint64_t cells = 0, io_bytes = 0;
	std::vector<int> llj, fastj;
	for (int i = 0; i < n_jobs; ++i) {
		if (h_jobs[i].flag & MMB_JOB_LL) { llj.push_back(i); continue; }
		const bool spl = (h_jobs[i].flag & MMB_JOB_SPLICE) != 0;
		if (!spl && mmb_ksw_fast_eligible(h_jobs[i])) {
			fastj.push_back(i);
			cells += (uint64_t)h_jobs[i].qlen * h_jobs[i].tlen, io_bytes += (uint64_t)h_jobs[i].qlen + h_jobs[i].tlen + 40;
			continue;
		}
		int m = std::max(h_jobs[i].qlen, h_jobs[i].tlen), k = 0;
		cells += (uint64_t)std::max(h_jobs[i].qlen, 0) * std::max(h_jobs[i].tlen, 0);
		io_bytes += (uint64_t)std::max(h_jobs[i].qlen, 0) + std::max(h_jobs[i].tlen, 0) + 40;
		while (k < n_tiers && m > tiers[k].maxlen) ++k;
		tj[(spl? n_tiers + 1 : 0) + k].push_back(i);
	}
	static const bool ksw_stats = getenv("MM_B200_KSW_STATS") != nullptr; // development aid: shapes of the jobs the universal tiers get
	if (ksw_stats) {
		for (int k = 0; k < n_tiers; ++k) {
			uint64_t c = 0, sq = 0, st = 0; int ext = 0, right = 0;
			for (int i : tj[k]) c += (uint64_t)h_jobs[i].qlen * h_jobs[i].tlen, sq += h_jobs[i].qlen, st += h_jobs[i].tlen, ext += !!(h_jobs[i].flag & MMB_KSW_EXTZ_ONLY), right += !!(h_jobs[i].flag & MMB_KSW_RIGHT);
			if (!tj[k].empty()) fprintf(stderr, "[ksw] tier %d: %zu jobs (ext-only %d, right-aligned %d), mean qlen %.1f tlen %.1f, cells %.3g\n", k, tj[k].size(), ext, right, (double)sq / tj[k].size(), (double)st / tj[k].size(), (double)c);
		}
		uint64_t c = 0; for (int i : fastj) c += (uint64_t)h_jobs[i].qlen * h_jobs[i].tlen;
		fprintf(stderr, "[ksw] packed path: %zu jobs, cells %.3g; ll %zu\n", fastj.size(), (double)c, llj.size());
	}
	if (!tj[n_tiers].empty() || !tj[2 * n_tiers + 1].empty()) {
		fprintf(stderr, "[ERROR] ksw job longer than %d not supported by this build\n", tiers[n_tiers - 1].maxlen);
		abort();
	}
	if (!llj.empty()) {
		LLArgs L;
		int maxq = 1;
		for (int i : llj) maxq = std::max(maxq, h_jobs[i].qlen);
		L.jobs = d_jobs, L.query = d_query, L.target = d_target, L.t_packed = t_packed, L.res = d_res, L.n = (int)llj.size();
		for (int i = 0; i < 25; ++i) L.mat[i] = sc->mat[i];
		L.slen_max = (maxq + 7) / 8;
		L.ws_stride = ((size_t)L.slen_max * 8 * 2 * 4 + (size_t)L.slen_max * 8 + 255) & ~(size_t)255;
		int groups = std::min((int)llj.size(), ctx->n_sm * 16 * 4);
		int grid = (groups * 8 + 127) / 128;
		groups = grid * 16;
		int *d_order = (int*)ctx->d_g.reserve(((size_t)n_jobs * 3 + 256) * sizeof(int)) + (size_t)n_jobs * 2 + 128;
		L.counter = d_order, L.order = d_order + 1;
		K.ll.pws_bytes = L.ws_stride * (size_t)groups; // the probes' workspace is the traceback workspace of the kernels after them
		K.ll.order = std::move(llj), K.ll.d_order = d_order;
		K.ll.go = [=](uint8_t *ws, uint32_t *) {
			LLArgs B = L;
			B.ws = (int16_t*)ws;
			ksw_ll_kernel<<<grid, 128, 0, ctx->stream>>>(B);
			MMB_CUDA_CHECK(cudaGetLastError());
			++ctx->n_launch;
		};
	}
	if (ctx->profiling) ctx->prof_bytes[MMB_PROF_KSW] += io_bytes + cells; // reference-layout algorithmic bytes: sequences + 1 B/cell traceback (+4 B per CIGAR op, added by the caller)
	int *d_queues = (int*)ctx->d_g.reserve(((size_t)n_jobs * 3 + 256) * sizeof(int)); // queues: [0,n+64) fast path | [n+64,2n+128) universal tiers | [2n+128,..) ll
	size_t g_off = (size_t)n_jobs + 64;
	std::vector<KswPlan> &plans = K.plans;
	K.cells = cells;
	mmb_ksw_fast_plan(ctx, sc, fastj, h_jobs, d_jobs, d_query, d_target, t_packed, d_res, d_cigar, cigar_cap, d_cigar_used, d_queues, plans);
	for (int pass = 0; pass < 2; ++pass) { // 0: dual-affine (ksw_extd2), 1: spliced (ksw_exts2)
		if (pass == 1) { // ksw2_exts2_sse.c:71-95: no (q,e)/(q2,e2) reordering; the intron state has no extension cost
			A.q = sc->q, A.e = sc->e, A.q2 = sc->q2, A.e2 = 0;
			A.skip = (-min_sc > 2 * (sc->q + sc->e)) || sc->q2 <= sc->q + sc->e;
			int lt2 = sc->e > 0? (sc->q2 - sc->q) / sc->e - 1 : 0;
			if (sc->q2 > sc->q + sc->e + lt2 * sc->e) ++lt2;
			A.long_thres = lt2, A.long_diff = lt2 * sc->e - (sc->q2 - sc->q);
		}
	for (int k = 0; k < n_tiers; ++k) {
		std::vector<int> &v = tj[pass * (n_tiers + 1) + k];
		if (v.empty()) continue;
		mmb_order_by_cells(v, h_jobs);
		int maxq = 0, maxt = 0; size_t maxp = 0; int maxsum = 0;
		for (int i : v) {
			const mmb_ksw_job_t &j = h_jobs[i];
			maxq = std::max(maxq, j.qlen), maxt = std::max(maxt, j.tlen), maxsum = std::max(maxsum, j.qlen + j.tlen);
			int w = j.w < 0 || pass == 1? std::max(j.qlen, j.tlen) : j.w;
			int n_col = std::min(j.qlen, j.tlen);
			n_col = ((std::min(n_col, w + 1) + 15) / 16 + 1) * 16;
			maxp = std::max(maxp, (size_t)(j.qlen + j.tlen - 1) * n_col + 16);
		}
		A.L = (maxt + 15) / 16 * 16, A.LQ = (maxq + 15) / 16 * 16;
		const int G = tiers[k].G, nw = tiers[k].nw, threads = G * nw;
		const bool gstate = k == n_tiers - 1;
		const size_t state_bytes = (size_t)16 * A.L + A.LQ + 64 + 1024;
		size_t smem = gstate? (size_t)1024 * nw : state_bytes * nw;
		int cta_per_sm = 1;
		{ // opt in to the full shared-memory carve-out once (never lowered: several scheduler groups launch concurrently)
			static std::once_flag once;
			std::call_once(once, [&]() {
				MMB_CUDA_CHECK(cudaFuncSetAttribute(ksw_extd2_kernel<32, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024));
				MMB_CUDA_CHECK(cudaFuncSetAttribute(ksw_extd2_kernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024));
				MMB_CUDA_CHECK(cudaFuncSetAttribute(ksw_extd2_kernel<32, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024));
				MMB_CUDA_CHECK(cudaFuncSetAttribute(ksw_extd2_kernel<256, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024));
			});
		}
		void (*kern)(KswArgs) = G == 32? (pass? ksw_extd2_kernel<32, true> : ksw_extd2_kernel<32, false>) : (pass? ksw_extd2_kernel<256, true> : ksw_extd2_kernel<256, false>);
		MMB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cta_per_sm, kern, threads, smem));
		if (smem > ctx->smem_optin - 1024 || cta_per_sm < 1) {
			fprintf(stderr, "[ERROR] ksw tier %d needs %zu B shared memory per CTA\n", k, smem);
			abort();
		}
		int grid = ctx->n_sm * cta_per_sm;
		int need = ((int)v.size() + nw - 1) / nw;
		grid = std::max(1, std::min(grid, need));
		maxp = (maxp + 255) & ~(size_t)255;
		const size_t gws_stride = gstate? (state_bytes + 255) & ~(size_t)255 : 0;
		// bound the workspace (2 GB per launch; every scheduler group keeps its own): fewer resident workers for very large matrices
		while ((size_t)grid * nw * (maxp + gws_stride) > ((size_t)2 << 30) && grid > 1) grid = (grid + 1) / 2;
		A.pws_stride = maxp, A.cigws_stride = (size_t)maxsum + 8;
		int *d_order = d_queues + g_off; g_off += v.size() + 1;
		A.counter = d_order, A.order = d_order + 1, A.n = (int)v.size();
		KswPlan pl;
		pl.order = std::move(v), pl.d_order = d_order;
		const size_t pws_area = A.pws_stride * (size_t)grid * nw;
		pl.pws_bytes = pws_area + gws_stride * (size_t)grid * nw, pl.cigws_bytes = A.cigws_stride * 4 * (size_t)grid * nw;
		const KswArgs A0 = A;
		pl.go = [=](uint8_t *pws, uint32_t *cigws) {
			KswArgs B = A0;
			B.pws = pws, B.cigws = cigws;
			B.gws = gstate? pws + pws_area : nullptr, B.gws_stride = gws_stride;
			kern<<<grid, threads, smem, ctx->stream>>>(B);
			MMB_CUDA_CHECK(cudaGetLastError());
			++ctx->n_launch;
		};
		plans.push_back(pl);
	}
	}
}

// The launch set on ctx->stream: the queue uploads, the probes, then the other kernels back to back in one workspace sized for the
// largest launch (they run one after another on the stream).
void mmb_ksw_enqueue(mmb_ctx_t *ctx, const KswLaunch &K)
{
	size_t pws_bytes = K.ll.pws_bytes, cigws_bytes = 0;
	for (const KswPlan &pl : K.plans) pws_bytes = std::max(pws_bytes, pl.pws_bytes), cigws_bytes = std::max(cigws_bytes, pl.cigws_bytes);
	uint8_t *pws = (uint8_t*)ctx->d_e.reserve(pws_bytes);
	uint32_t *cigws = (uint32_t*)ctx->d_f.reserve(cigws_bytes);
	auto upload = [&](const KswPlan &pl) {
		MMB_CUDA_CHECK(cudaMemcpyAsync(pl.d_order + 1, pl.order.data(), pl.order.size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
		MMB_CUDA_CHECK(cudaMemsetAsync(pl.d_order, 0, sizeof(int), ctx->stream));
	};
	if (K.ll.go) {
		upload(K.ll);
		ProfScope prof(ctx, MMB_PROF_OTHER, 0);
		K.ll.go(pws, nullptr);
	}
	for (const KswPlan &pl : K.plans) upload(pl);
	ProfScope prof(ctx, MMB_PROF_KSW, K.cells);
	for (const KswPlan &pl : K.plans) pl.go(pws, cigws);
}

void mmb_ksw_launch(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
					const uint8_t *d_query, const void *d_target, int t_packed,
					mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap, unsigned long long *d_cigar_used)
{
	if (n_jobs <= 0) return;
	KswLaunch K;
	mmb_ksw_plan(ctx, sc, n_jobs, h_jobs, d_jobs, d_query, d_target, t_packed, d_res, d_cigar, cigar_cap, d_cigar_used, K);
	mmb_ksw_enqueue(ctx, K);
}
