// minimap2_b200/csrc/ksw_fast.cu
//
// K3 fast path: global dual-affine alignment with traceback for the gap-fill shape that dominates map-ont
// (align.c:803-872 first pass: KSW_EZ_APPROX_MAX, w >= max(qlen,tlen) so the band never clips, ~230 x 230 cells,
// ~41 such calls per 10 kb read = 95% of all DP cells).
//
// Same recurrence and tie rules as ksw_extd2_sse (ksw2_extd2_sse.c:39-66, 232-273), but the per-cell difference values
// are pure functions of the cell's two predecessors, so any evaluation order gives the reference's bytes as long as the
// band is not clipping (then no stale SSE lane is ever consumed). That freedom is used for a register-resident
// wavefront: lane l of a warp owns C consecutive target columns, all lanes walk the query rows with a skew of one row
// per lane (lane l is at row s-l in step s), the vertical state (u,y,y2 per column) never leaves registers, the
// horizontal state (v,x,x2) is handed to the next lane with one packed shuffle per step, and the only memory traffic is
// the 1 B/cell traceback row (one coalesced 8/16-byte store per lane per step). 88% of lane-steps do useful cells
// (qlen/(qlen+31)) versus ~60% for an anti-diagonal sweep, and there is no shared-memory round trip per cell.
// Valid cells never leave the int8 range (guaranteed by mm_check_opt: (q+e)+(q2+e2) <= 127), so int32 arithmetic
// reproduces the reference's wrapping int8 arithmetic bit for bit.
//
// Jobs that do not qualify (exact max / extension / right-aligned / clipped band / long) go to the universal kernel
// in ksw_extd2.cu, which emulates the SSE lane semantics exactly.
#include "mmb_internal.h"
#include "ksw_plan.h"
#include <algorithm>

#define KSW_NEG_INF (-0x40000000)

namespace {

struct FastArgs {
	const mmb_ksw_job_t *jobs;
	const int *order;
	int n;
	const uint8_t *query;
	const void *target;
	int t_packed;
	mmb_ksw_res_t *res;
	uint32_t *cigar;
	long long cigar_cap;
	unsigned long long *cigar_used;
	uint8_t *pws; size_t pws_stride;      // traceback rows: qlen x (32*C) bytes per worker
	uint32_t *cigws; size_t cigws_stride;
	int *counter;
	int qmax;                             // shared-memory query staging capacity per warp
	int8_t mch, mis, scn;
	int8_t q, e, q2, e2;
	int qe0;                              // q+e before the (q,e)/(q2,e2) reordering: H(0,0) = v - qe0 (ksw2_extd2_sse.c:68,358)
	int8_t zd_q, zd_e;                    // gap open/extension as mm_test_zdrop uses them (opt->q, opt->e: not reordered)
	int8_t zd_scn;                        // that scan's score for an ambiguous base: the matrix entry, also when it is 0 and the DP scores -e2
	int zd_skip;                          // > 0: skip that scan when the path's total penalty cannot exceed it (mmb_ksw_score_t::zd_skip)
	int long_thres, long_diff;
	int8_t mat[25];
	uint32_t one, neg1;                   // 1 and 0xffffffff, passed at run time so that ptxas keeps the IMAD form of PK_FADD/PK_FSUB
};

__device__ __forceinline__ uint8_t fetch_t(const void *target, int packed, long long idx)
{
	if (packed) {
		const uint32_t *S = (const uint32_t*)target;
		return (uint8_t)(S[idx >> 3] >> ((idx & 7) << 2) & 0xf);
	}
	return ((const uint8_t*)target)[idx];
}

__device__ __forceinline__ void push_cig(uint32_t *cig, int &n, uint32_t op, int len)
{
	if (n == 0 || op != (cig[n - 1] & 0xf)) cig[n++] = (uint32_t)len << 4 | op;
	else cig[n - 1] += (uint32_t)len << 4;
}

template<int C>
__global__ void __launch_bounds__(128) ksw_fast_kernel(FastArgs A)
{
	extern __shared__ __align__(16) uint8_t smem[];
	const int lane = threadIdx.x & 31, wk = threadIdx.x >> 5, nwk = blockDim.x >> 5;
	const int worker = blockIdx.x * nwk + wk;
	uint8_t *qs = smem + (size_t)wk * (A.qmax + 1024);   // staged query bytes
	uint8_t *tile = qs + A.qmax;                          // 32x32 traceback window
	uint8_t *p = A.pws + A.pws_stride * worker;
	uint32_t *cig = A.cigws + A.cigws_stride * worker;
	constexpr int CP = C <= 4? 4 : C <= 8? 8 : 16;        // bytes reserved per lane per row (one aligned vector store)
	const int W = 32 * CP;                                // traceback row stride
	const int q = A.q, e = A.e, q2 = A.q2, e2 = A.e2, qe = q + e, qe2 = q2 + e2;
	const int mch = A.mch, mis = A.mis, scn = A.scn;
	const unsigned full = 0xffffffffu;

	#pragma unroll 1
	for (;;) {
		int slot = 0;
		if (lane == 0) slot = atomicAdd(A.counter, 1);
		slot = __shfl_sync(full, slot, 0);
		if (slot >= A.n) break;
		const int jid = A.order[slot];
		const mmb_ksw_job_t jb = A.jobs[jid];
		const int qlen = jb.qlen, tlen = jb.tlen;
		const bool generic = (jb.flag & MMB_KSW_GENERIC_SC) != 0;
		// stage the query (row j -> base) and this lane's target columns
		for (int i = lane; i < qlen; i += 32) {
			uint8_t c = A.query[jb.q_start + (long long)i * jb.q_step];
			if ((jb.flag & MMB_JOB_Q_COMP) && c < 4) c = 3 - c;
			qs[i] = c;
		}
		const int t0 = lane * C;
		int tb[C], u[C], y[C], y2[C], msc[C];
		#pragma unroll
		for (int c = 0; c < C; ++c) {
			const int t = t0 + c;
			tb[c] = t < tlen? fetch_t(A.target, A.t_packed, jb.t_start + (long long)t * jb.t_step) : 4;
			// top boundary (ksw2_extd2_sse.c:159-162): the cell above row 0 in column t carries the gap-open ramp of diagonal r=t
			u[c] = t == 0? -q - e : t < A.long_thres? -e : t == A.long_thres? A.long_diff : -e2;
			y[c] = -q - e, y2[c] = -q2 - e2;
			msc[c] = tb[c] == 4? scn : mis; // mismatch score of this column (ambiguous target base scores sc_N)
		}
		__syncwarp();
		int hcol0 = 0, hrow = 0;           // score pieces: lane 0 sums v down column 0, every lane sums u along the last row
		int pk_prev = 0;                   // (v,x,x2) of this lane's last column, packed, from the previous step
		const int n_steps = qlen + 31;
		#pragma unroll 1
		for (int s = 0; s < n_steps; ++s) {
			const int j = s - lane;
			// hand the right edge of lane l-1 (same query row) to lane l
			int pk_in = __shfl_up_sync(full, pk_prev, 1);
			if (j >= 0 && j < qlen && t0 < tlen) {
				int vl, xl, x2l;
				if (lane == 0) { // left boundary (ksw2_extd2_sse.c:149-158 with st == 0): diagonal r = j
					xl = -q - e, x2l = -q2 - e2;
					vl = j == 0? -q - e : j < A.long_thres? -e : j == A.long_thres? A.long_diff : -e2;
				} else {
					vl = (int)(int8_t)(pk_in & 0xff), xl = (int)(int8_t)(pk_in >> 8 & 0xff), x2l = (int)(int8_t)(pk_in >> 16 & 0xff);
				}
				const int qb = qs[j];
				int hc0 = 0;
				uint32_t dw[(C + 3) / 4];
				#pragma unroll
				for (int k = 0; k < (C + 3) / 4; ++k) dw[k] = 0;
				// Lean cell update (~40 integer ops): the 4 "open/extend" maxima are folded with the -(q+e) shift
				// (x' = max(a - (z-q) - qe, -qe)), rows with an ambiguous query base take the generic-score path.
				const int nqe = -qe, nqe2 = -qe2;
				if (!generic && qb < 4) {
					#pragma unroll
					for (int c = 0; c < C; ++c) {
						const int sc = tb[c] == qb? mch : msc[c];
						const int uc = u[c];
						int a = xl + vl, b = y[c] + uc, a2 = x2l + vl, b2 = y2[c] + uc;
						int z = sc, d = 0;
						if (a > z) d = 1;  z = max(z, a);      // ksw2_extd2_sse.c:235-243: strict '>' keeps the earlier state
						if (b > z) d = 2;  z = max(z, b);
						if (a2 > z) d = 3; z = max(z, a2);
						if (b2 > z) d = 4; z = max(z, b2);
						z = min(z, mch);
						const int un = z - vl, vn = z - uc;
						const int t1 = z - q + qe, t2 = z - q2 + qe2;
						a -= t1, b -= t1, a2 -= t2, b2 -= t2;           // = (a - (z-q)) - qe : value before the max(.,0) shifted by -qe
						if (a > nqe) d |= 0x08;
						if (b > nqe) d |= 0x10;
						if (a2 > nqe2) d |= 0x20;
						if (b2 > nqe2) d |= 0x40;
						xl = max(a, nqe), y[c] = max(b, nqe), x2l = max(a2, nqe2), y2[c] = max(b2, nqe2);
						u[c] = un, vl = vn;
						dw[c >> 2] |= (uint32_t)d << ((c & 3) * 8);
						if (c == 0) hc0 = vn;
					}
				} else {
					#pragma unroll
					for (int c = 0; c < C; ++c) {
						int sc;
						if (!generic) sc = (tb[c] == 4 || qb == 4)? scn : tb[c] == qb? mch : mis;
						else sc = A.mat[tb[c] * 5 + qb];
						const int uc = u[c];
						int a = xl + vl, b = y[c] + uc, a2 = x2l + vl, b2 = y2[c] + uc;
						int z = sc, d = 0;
						if (a > z) d = 1;  z = max(z, a);
						if (b > z) d = 2;  z = max(z, b);
						if (a2 > z) d = 3; z = max(z, a2);
						if (b2 > z) d = 4; z = max(z, b2);
						z = min(z, mch);
						const int un = z - vl, vn = z - uc;
						const int t1 = z - q + qe, t2 = z - q2 + qe2;
						a -= t1, b -= t1, a2 -= t2, b2 -= t2;
						if (a > nqe) d |= 0x08;
						if (b > nqe) d |= 0x10;
						if (a2 > nqe2) d |= 0x20;
						if (b2 > nqe2) d |= 0x40;
						xl = max(a, nqe), y[c] = max(b, nqe), x2l = max(a2, nqe2), y2[c] = max(b2, nqe2);
						u[c] = un, vl = vn;
						dw[c >> 2] |= (uint32_t)d << ((c & 3) * 8);
						if (c == 0) hc0 = vn;
					}
				}
				if (j == qlen - 1) { // H(t,qlen-1) = H(t-1,qlen-1) + u(t,qlen-1): sum u along the last row
					#pragma unroll
					for (int c = 0; c < C; ++c) if (t0 + c >= 1 && t0 + c < tlen) hrow += u[c];
				}
				if (lane == 0) hcol0 += j == 0? hc0 - A.qe0 : hc0; // H(0,0) = v - (q+e) (:358, q+e as given); then H(0,j) = H(0,j-1) + v(0,j)
				pk_prev = (vl & 0xff) | (xl & 0xff) << 8 | (x2l & 0xff) << 16;
				uint8_t *prow = p + (size_t)j * W + lane * CP;
				if (CP == 4) *(uint32_t*)prow = dw[0];
				else if (CP == 8) *(uint2*)prow = make_uint2(dw[0], dw[1 % ((C + 3) / 4)]);
				else *(uint4*)prow = make_uint4(dw[0], dw[1 % ((C + 3) / 4)], dw[2 % ((C + 3) / 4)], dw[3 % ((C + 3) / 4)]);
			}
		}
		// score = H(tlen-1, qlen-1): down column 0, then along the last row
		int score = hrow;
		for (int o = 16; o > 0; o >>= 1) score += __shfl_xor_sync(full, score, o);
		score += __shfl_sync(full, hcol0, 0);
		__syncwarp();
		// ---- traceback from (tlen-1, qlen-1) (ksw2.h:130-162; no forced states: the band is never clipped) ----
		int n = 0, i = tlen - 1, jj = qlen - 1, state = 0;
		for (;;) {
			int go = i >= 0 && jj >= 0;
			go = __shfl_sync(full, go, 0);
			if (!go) break;
			const int jt = __shfl_sync(full, jj, 0), it = __shfl_sync(full, i, 0);
			{ // lane k stages row jt-k, columns it-31..it
				const int rr = jt - lane;
				if (rr >= 0) {
					const uint8_t *prow = p + (size_t)rr * W;
					#pragma unroll 8
					for (int c = 0; c < 32; ++c) {
						const int col = it - 31 + c;
						tile[lane * 32 + c] = col >= 0? prow[(col / C) * CP + col % C] : 0;
					}
				}
			}
			__syncwarp();
			if (lane == 0) {
				while (i >= 0 && jj >= 0 && jt - jj < 32 && it - i < 32) {
					const uint32_t tmp = tile[(jt - jj) * 32 + (i - (it - 31))];
					if (state == 0) state = tmp & 7;
					else if (!(tmp >> (state + 2) & 1)) state = 0;
					if (state == 0) state = tmp & 7;
					if (state == 0) push_cig(cig, n, 0, 1), --i, --jj;
					else if (state == 1 || state == 3) push_cig(cig, n, 2, 1), --i;
					else push_cig(cig, n, 1, 1), --jj;
				}
			}
			__syncwarp();
		}
		if (lane == 0) {
			if (i >= 0) push_cig(cig, n, 2, i + 1);
			if (jj >= 0) push_cig(cig, n, 1, jj + 1);
		}
		n = __shfl_sync(full, n, 0);
		unsigned long long coff = 0;
		if (n > 0) {
			if (lane == 0) coff = atomicAdd(A.cigar_used, (unsigned long long)n);
			coff = __shfl_sync(full, coff, 0);
			const bool rev_cigar = (jb.flag & MMB_KSW_REV_CIGAR) != 0;
			if ((long long)(coff + n) <= A.cigar_cap)
				for (int k = lane; k < n; k += 32) A.cigar[coff + k] = rev_cigar? cig[k] : cig[n - 1 - k];
		}
		if (lane == 0) {
			mmb_ksw_res_t o;
			o.zd_max = -1, o.zd_t0 = o.zd_t1 = o.zd_q0 = o.zd_q1 = -1;
			o.max = 0, o.zdropped = 0, o.max_q = o.max_t = o.mqe_t = o.mte_q = -1, o.mqe = o.mte = KSW_NEG_INF;
			o.score = score, o.n_cigar = n, o.reach_end = 0, o.cigar_off = (uint32_t)coff;
			A.res[jid] = o;
		}
		__syncwarp();
	}
}


// ---------------------------------------------------------------------------------------------------------------------
// Packed variant: two DP cells per 32-bit operation.
//
// The kernel above is issue-bound (~40 integer instructions per cell). Every quantity of the difference recurrence fits
// in 8 bits, so two cells are packed as 16-bit halves of one register and updated with VIMNMX(3).S16x2 and plain 32-bit
// adds. Layout of a half: ((value + 128) << 8) | low byte (unsigned 16-bit compares). Biasing keeps both halves non-negative, hence a 32-bit
// add/subtract of packed words never carries between halves; the low byte is scratch: a candidate carries the tag
// 7-k of the state k it stands for, so one 3-input maximum returns both max(z) and the reference's tie rule (the earlier
// state wins, ksw2_extd2_sse.c:235-243), and the gap-open floor carries one "not extended" bit per gap state, so the
// four continuation flags (:244-273) drop out of the maxima as well. ~28 instructions per PAIR of cells.
// The two cells of a pair must be independent: lane l owns columns [l*C, l*C+C), split in a left block A and a right
// block B of H = C/2 columns; B runs one query row behind A (its left input is A's right edge of the previous step), and
// lane l+1 runs two rows behind lane l. Traceback bytes are stored as (tag | flags), i.e. the reference byte XOR 0x7f.
// Jobs with tlen <= 256 use LN = 16 lanes (two jobs per warp, up to 16 columns per lane): more columns per lane amortise
// the per-step overhead (shuffles, stores, row bookkeeping) and halve the pipeline fill/drain of the lane skew.
// Pipe balancing. IADD3/LOP3/VIMNMX/PRMT issue on the ALU pipe and IMAD on the FMA pipe, so the recurrence written with plain
// adds would queue on the ALU pipe while the FMA pipe idles. (The per-pipe issue rates and the balance this buys have not been
// profiled on H100: no Nsight Compute capture exists for the sm_90a build.) The linear steps are therefore written as two-input multiply-adds
// x * 1 + y / y * (-1) + x whose multiplier is a kernel argument: ptxas cannot fold it back into an IADD3, and packed words add
// exactly like before (the halves never carry into each other in the final values; intermediate borrows cancel modulo 2^32).
#if defined(MMB_EMU) || defined(MMB_PK_NO_FMA)
#define PK_FADD(x, y) ((x) + (y))
#define PK_FSUB(x, y) ((x) - (y))
#else
#define PK_FADD(x, y) pk_mad((x), ONE, (y))
#define PK_FSUB(x, y) pk_mad((y), NEG1, (x))
__device__ __forceinline__ uint32_t pk_mad(uint32_t a, uint32_t b, uint32_t c)
{
	uint32_t d;
	asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
	return d;
}
#endif

template<int H, int LN>
#ifndef PK_MINB
#define PK_MINB (H <= 8? 4 : 3) // CTAs per SM the register allocation must leave room for (128 / 168 registers)
#endif
__global__ void __launch_bounds__(128, PK_MINB) ksw_pk_kernel(FastArgs A)
{
	extern __shared__ __align__(16) uint8_t smem[];
	constexpr int C = 2 * H;
	constexpr int CPH = H <= 1? 1 : H <= 2? 2 : H <= 4? 4 : H <= 8? 8 : 16; // traceback bytes per block per row (one aligned store)
	constexpr int CP = 2 * CPH;
	constexpr int NW = (H + 3) / 4;
	constexpr int NJ = 32 / LN;                                // jobs per warp
	constexpr int W = LN * CP;                                 // traceback row stride
	const int lane = threadIdx.x & 31, wk = threadIdx.x >> 5, nwk = blockDim.x >> 5;
	const int sub = lane & (LN - 1), grp = lane / LN, lead = lane & ~(LN - 1);
	const int worker0 = (blockIdx.x * nwk + wk) * NJ;
	uint8_t *qs = smem + (size_t)(wk * NJ + grp) * A.qmax;   // staged query, one-hot (0x80 = ambiguous), one sentinel past the end
	constexpr int TSM = LN * C;                              // staged target (nt4 codes) per job, for the z-drop scan
	constexpr int TW = 80, TILE = 32 * TW;                   // traceback tile: 32 rows x 80 physical bytes per warp
	uint8_t *ts = smem + (size_t)nwk * NJ * A.qmax + (size_t)(wk * NJ + grp) * TSM;
	uint8_t *tile = smem + (size_t)nwk * NJ * (A.qmax + TSM) + (size_t)wk * TILE;
	uint8_t *p = A.pws + A.pws_stride * (size_t)(worker0 + grp);
	const int q = A.q, e = A.e, q2 = A.q2, e2 = A.e2, qe = q + e, qe2 = q2 + e2;
	const unsigned full = 0xffffffffu;
	#define PK_ENC(v) ((uint32_t)((v) + 128) << 8)
	#define PK2(v) (PK_ENC(v) * 0x10001u)
	const uint32_t BB2 = 0x80008000u, CLEAN = 0xff00ff00u;
	// state words carry the tag of the candidate they feed (x: 6, y: 5, x2: 4, y2: 3; sc: 7) in the low byte of each half
	const uint32_t TAGS = 0x03040506u, NBB2 = 0u - BB2;
	const uint32_t ONE = A.one, NEG1 = A.neg1;
	(void)ONE; (void)NEG1;
	const uint32_t KX = BB2 - ((uint32_t)e << 8) * 0x10001u - 0x00060006u, KY = BB2 - ((uint32_t)e << 8) * 0x10001u - 0x00050005u;
	const uint32_t KX2 = BB2 - ((uint32_t)e2 << 8) * 0x10001u - 0x00040004u, KY2 = BB2 - ((uint32_t)e2 << 8) * 0x10001u - 0x00030003u;
	const uint32_t NQX = PK2(-qe) | 0x00080008u, NQY = PK2(-qe) | 0x00100010u, NQX2 = PK2(-qe2) | 0x00200020u, NQY2 = PK2(-qe2) | 0x00400040u;
	const uint32_t SCN_T = PK2((int)A.scn) + 0x00070007u;
	const uint32_t KMM = (uint32_t)((int)A.mch - (int)A.mis) << 8;
	const uint32_t E_QE = PK_ENC(-q - e), E_E = PK_ENC(-e), E_E2 = PK_ENC(-e2), E_LD = PK_ENC(A.long_diff), E_QE2 = PK_ENC(-q2 - e2);
	const uint32_t XT0 = E_QE | 6u, YT0 = E_QE | 5u, X2T0 = E_QE2 | 4u, Y2T0 = E_QE2 | 3u; // gap states at a boundary, tagged
	const int lt = A.long_thres;

	#pragma unroll 1
	for (;;) {
		int slot = 0;
		if (sub == 0) slot = atomicAdd(A.counter, 1);
		slot = __shfl_sync(full, slot, lead);
		const bool act = slot < A.n;
		if (!__any_sync(full, act)) break;
		int jid = -1, qlen = 0, tlen = 0, jflag = 0;
		mmb_ksw_job_t jb;
		if (act) { jid = A.order[slot]; jb = A.jobs[jid]; qlen = jb.qlen, tlen = jb.tlen, jflag = jb.flag; }
		for (int i = sub; i <= qlen; i += LN) {
			uint8_t c = 4;
			if (i < qlen) {
				c = A.query[jb.q_start + (long long)i * jb.q_step];
				if ((jflag & MMB_JOB_Q_COMP) && c < 4) c = 3 - c;
			}
			qs[i] = c < 4? (uint8_t)(1u << c) : (uint8_t)0x80;
		}
		const int t0 = sub * C;
		uint32_t TBM[H], MSC[H], U[H], Y[H], Y2[H];
		#pragma unroll
		for (int c = 0; c < H; ++c) {
			uint32_t tbm = 0, msc = 0, u = 0;
			#pragma unroll
			for (int h = 0; h < 2; ++h) {
				const int t = t0 + h * H + c;
				const int b = t < tlen? fetch_t(A.target, A.t_packed, jb.t_start + (long long)t * jb.t_step) : 4;
				ts[t] = (uint8_t)b;
				// top boundary (ksw2_extd2_sse.c:159-162)
				const uint32_t u0 = t == 0? E_QE : t < lt? E_E : t == lt? E_LD : E_E2;
				tbm |= (b < 4? 1u << b : 0u) << (16 * h);
				msc |= (PK_ENC(b == 4? (int)A.scn : (int)A.mis) + 7u) << (16 * h);
				u |= u0 << (16 * h);
			}
			TBM[c] = tbm, MSC[c] = msc, U[c] = u, Y[c] = YT0 * 0x10001u, Y2[c] = Y2T0 * 0x10001u;
		}
		__syncwarp();
		int hrow = 0;
		uint32_t hcol_acc = 0;             // sum over rows of enc(v) in column 0 (only meaningful in the group's first lane)
		uint32_t vl_end = PK2(0), xl_end = XT0 * 0x10001u, x2l_end = X2T0 * 0x10001u; // right edges of the previous step (lo: block A, hi: block B); x words tagged
		uint32_t oh_prev = 0x80;           // one-hot query base of row jA-1
		const int n_lanes = (tlen + C - 1) / C;
		int n_steps = act? qlen + 2 * (n_lanes - 1) + 1 : 0;
		if (NJ == 2) n_steps = max(n_steps, __shfl_xor_sync(full, n_steps, 16));
		uint8_t *pa = p + sub * CP; // traceback bytes of step s: the rows are indexed by STEP (row j of lane l's block A lives in step-row j + 2l, of its block B in j + 2l + 1), so the lanes of a step store one contiguous line
		const bool lane_on = t0 < tlen;
		uint32_t oh_nx = sub == 0? qs[0] : 0x80u; // the query base of the coming step, fetched one step ahead (keeps the shared-memory latency off the step's critical path)
		#pragma unroll 1
		for (int s = 0; s < n_steps; ++s, pa += W) {
			const int jA = s - 2 * sub; // block A row; block B is at jA - 1
			const uint32_t oh = oh_nx;
			{ const int jn = jA + 1; oh_nx = jn >= 0 && jn <= qlen? qs[jn] : 0x80u; }
			const uint32_t sv = __shfl_up_sync(full, vl_end, 1, LN), sx = __shfl_up_sync(full, xl_end, 1, LN), sx2 = __shfl_up_sync(full, x2l_end, 1, LN);
			if (jA >= 0 && jA <= qlen && lane_on) {
				// left inputs: lo <- right edge of the previous lane's block B (same row), hi <- this lane's block A, previous row;
				// the group's first lane takes the left boundary instead (ksw2_extd2_sse.c:149-158 with st == 0)
				uint32_t bv = jA < lt? E_E : E_E2;
				bv = jA == lt? E_LD : bv;
				bv = jA == 0? E_QE : bv;
				const bool first = sub == 0;
				const uint32_t vlE = __byte_perm(first? bv : sv >> 16, vl_end, 0x5410);
				uint32_t xl = __byte_perm(first? XT0 : sx >> 16, xl_end, 0x5410);
				uint32_t x2l = __byte_perm(first? X2T0 : sx2 >> 16, x2l_end, 0x5410);
				// v travels through the column loop without its bias (vl = enc(v) - BB2, a 32-bit difference whose half-borrows cancel in
				// every sum it enters): x + v and z - v are then two-input operations
				uint32_t vl = PK_FADD(vlE, NBB2);
				const uint32_t ohx = oh | oh_prev << 16;
				const uint32_t qbm = ohx & 0x000f000fu;
				const uint32_t mN = (ohx >> 7 & 0x00010001u) * 0xffffu;
				oh_prev = oh;
				uint32_t wd[NW * 4], v_first = 0;
				#pragma unroll
				for (int c = 0; c < NW * 4; ++c) wd[c] = 0;
				#pragma unroll
				for (int c = 0; c < H; ++c) {
					const uint32_t f = __vminu2(TBM[c] & qbm, 0x00010001u);
					uint32_t sc = f * KMM + MSC[c];
					sc = (sc & ~mN) | (SCN_T & mN);
					const uint32_t uc = U[c], ucr = PK_FADD(uc, NBB2);
					const uint32_t a = PK_FADD(xl, vl), a2 = PK_FADD(x2l, vl), b = PK_FADD(Y[c], ucr), b2 = PK_FADD(Y2[c], ucr);
					uint32_t zt = __vimax3_u16x2(sc, a, b);
					zt = __vimax3_u16x2(zt, a2, b2);
					const uint32_t z8 = zt & CLEAN; // no clip to the match score (:243) needed: H(i,j) - H(i-1,j-1) <= match holds in every cell when the band does not clip
					const uint32_t un = PK_FSUB(z8, vl), vn = PK_FSUB(z8, uc); // un = enc(u'), vn = enc(v') - BB2
					const uint32_t xt = __vmaxu2(PK_FADD(a, PK_FSUB(KX, z8)), NQX), yt = __vmaxu2(PK_FADD(b, PK_FSUB(KY, z8)), NQY);
					const uint32_t x2t = __vmaxu2(PK_FADD(a2, PK_FSUB(KX2, z8)), NQX2), y2t = __vmaxu2(PK_FADD(b2, PK_FSUB(KY2, z8)), NQY2);
					wd[c] = (xt | yt | x2t) | y2t | zt; // low byte of each half = tag | flags (the value sits in the high byte)
					// next cell's gap states: value bytes kept, low bytes replaced by the candidate tags (one PRMT each)
					xl = __byte_perm(xt, TAGS, 0x3414), Y[c] = __byte_perm(yt, TAGS, 0x3515), x2l = __byte_perm(x2t, TAGS, 0x3616), Y2[c] = __byte_perm(y2t, TAGS, 0x3717);
					U[c] = un, vl = vn;
					if (c == 0) v_first = vn ^ 0x8000u; // low half back to enc(v)
				}
				vl_end = PK_FADD(vl, BB2), xl_end = xl, x2l_end = x2l;
				if (jA < qlen) hcol_acc += v_first & 0xffffu;
				if (jA == 0) { // block B has not started: put its column state (hi halves) back to the top boundary
					#pragma unroll
					for (int c = 0; c < H; ++c) {
						const int t = t0 + H + c;
						const uint32_t u0 = t < lt? E_E : t == lt? E_LD : E_E2; // t >= 1 here
						U[c] = (U[c] & 0xffffu) | u0 << 16, Y[c] = (Y[c] & 0xffffu) | YT0 << 16, Y2[c] = (Y2[c] & 0xffffu) | Y2T0 << 16;
					}
				}
				// score pieces: H(t, qlen-1) = H(t-1, qlen-1) + u(t, qlen-1) along the last row
				if (jA == qlen - 1) {
					#pragma unroll
					for (int c = 0; c < H; ++c) if (t0 + c >= 1 && t0 + c < tlen) hrow += (int)((U[c] & 0xffffu) >> 8) - 128;
				}
				if (jA == qlen) {
					#pragma unroll
					for (int c = 0; c < H; ++c) if (t0 + H + c < tlen) hrow += (int)(U[c] >> 24) - 128;
				}
				// traceback bytes: lo bytes of the words -> row jA (block A), byte 2 of the words -> row jA-1 (block B)
				uint32_t lo[NW], hi[NW];
				#pragma unroll
				for (int k = 0; k < NW; ++k) {
					const uint32_t r01 = __byte_perm(wd[4 * k], wd[4 * k + 1], 0x6240), r23 = __byte_perm(wd[4 * k + 2], wd[4 * k + 3], 0x6240);
					lo[k] = __byte_perm(r01, r23, 0x5410), hi[k] = __byte_perm(r01, r23, 0x7632);
				}
				if (jA >= 1 && jA < qlen && CPH <= 8) { // both blocks are inside the matrix (all but the first and last row of a lane): one store for the pair
					if constexpr (CPH == 1) *(uint16_t*)pa = (uint16_t)((lo[0] & 0xffu) | hi[0] << 8);
					else if constexpr (CPH == 2) *(uint32_t*)pa = (lo[0] & 0xffffu) | hi[0] << 16;
					else if constexpr (CPH == 4) *(uint2*)pa = make_uint2(lo[0], hi[0]);
					else if constexpr (CPH == 8) *(uint4*)pa = make_uint4(lo[0], lo[NW - 1], hi[0], hi[NW - 1]);
				} else {
					if (jA < qlen) {
						if constexpr (CPH == 1) *pa = (uint8_t)lo[0];
						else if constexpr (CPH == 2) *(uint16_t*)pa = (uint16_t)lo[0];
						else if constexpr (CPH == 4) *(uint32_t*)pa = lo[0];
						else if constexpr (CPH == 8) *(uint2*)pa = make_uint2(lo[0], lo[NW - 1]);
						else *(uint4*)pa = make_uint4(lo[0], lo[1], lo[2], lo[NW - 1]);
					}
					if (jA >= 1) {
						uint8_t *pb = pa + CPH;
						if constexpr (CPH == 1) *pb = (uint8_t)hi[0];
						else if constexpr (CPH == 2) *(uint16_t*)pb = (uint16_t)hi[0];
						else if constexpr (CPH == 4) *(uint32_t*)pb = hi[0];
						else if constexpr (CPH == 8) *(uint2*)pb = make_uint2(hi[0], hi[NW - 1]);
						else *(uint4*)pb = make_uint4(hi[0], hi[1], hi[2], hi[NW - 1]);
					}
				}
			}
		}
		// score = H(tlen-1, qlen-1): down column 0 (H(0,0) = v - (q+e), :366), then along the last row
		int score = hrow;
		#pragma unroll
		for (int o = LN / 2; o > 0; o >>= 1) score += __shfl_xor_sync(full, score, o);
		score += (int)(hcol_acc >> 8) - 128 * qlen - A.qe0;
		score = __shfl_sync(full, score, lead);
		__syncwarp();
		// ---- traceback from (tlen-1, qlen-1) (ksw2.h:130-162; no forced states: the band is never clipped) ----
		// The path is walked run by run instead of cell by cell: in the H state the 32 lanes look down the diagonal, in a gap
		// state along the row/column, and a ballot finds where the run ends -- the per-cell rule of ksw_backtrack is unchanged.
		#pragma unroll 1
		for (int g = 0; g < NJ; ++g) {
			const int src = g * LN;
			if (!__shfl_sync(full, (int)act, src)) continue;
			const int g_tlen = __shfl_sync(full, tlen, src), g_qlen = __shfl_sync(full, qlen, src), g_jid = __shfl_sync(full, jid, src);
			const int g_flag = __shfl_sync(full, jflag, src), g_score = __shfl_sync(full, score, src);
			const uint8_t *gp = A.pws + A.pws_stride * (size_t)(worker0 + g);
			uint32_t *cig = A.cigws + A.cigws_stride * (size_t)(worker0 + g);
			int n = 0, i = g_tlen - 1, jj = g_qlen - 1, state = 0;
			uint32_t run_op = 0, run_len = 0; // pending CIGAR run (lane 0 writes it when the operator changes)
			int n_m = 0, gap_dp = 0, gap_zd = 0; // aligned bases; gap costs as the DP charges them and as mm_test_zdrop does (for the scan-skip bound)
			#define PK_CLOSE() do { if (run_len) { if (run_op == 0) n_m += (int)run_len; else { const int l__c = (int)run_len; \
				gap_dp += min(q + e * l__c, q2 + e2 * l__c), gap_zd += A.zd_q + A.zd_e * l__c; } } } while (0)
			#define PK_EMIT(op_, len_) do { const uint32_t o__ = (op_), l__ = (len_); if (l__) { if (run_len && o__ == run_op) run_len += l__; \
				else { PK_CLOSE(); if (run_len && lane == 0) cig[n] = run_len << 4 | run_op; n += run_len? 1 : 0; run_op = o__, run_len = l__; } } } while (0)
			// The traceback bytes live in HBM/L2; reading them cell by cell along the path is a chain of dependent global loads (the
			// long-scoreboard stall that kept half of the warps waiting in round 1). The warp stages a tile instead -- the 32 rows up from
			// the current cell x the 80 physical bytes that cover the 32 columns left of it, five independent 16-byte loads per lane --
			// and walks inside it at shared-memory latency; a new tile is staged when the path leaves the current one (~every 32 steps).
			bool have = false;
			int tj = 0, tpb = 0;
			while (i >= 0 && jj >= 0) {
				const int di = (state == 0 || state == 1 || state == 3)? 1 : 0, dj = (state == 0 || state == 2 || state == 4)? 1 : 0;
				const int ci = i - lane * di, cj = jj - lane * dj;
				const bool inr = ci >= 0 && cj >= 0;
				int ph = 0, sr = 0; // physical byte and step-row of the cell
				if (inr) { const int wi = ci % C, sb = ci / C; ph = sb * CP + (wi < H? wi : CPH + wi - H); sr = cj + 2 * sb + (wi < H? 0 : 1); }
				const bool intile = have && inr && sr <= tj && sr > tj - 32 && ph >= tpb && ph < tpb + TW;
				if (!__shfl_sync(full, (int)intile, 0)) { // the current cell is not staged: stage the tile that has it in its bottom right corner
					const int c0 = i > 31? i - 31 : 0, w0 = c0 % C;
					tj = __shfl_sync(full, sr, 0), tpb = ((c0 / C) * CP + (w0 < H? w0 : CPH + w0 - H)) & ~15; // every step of the walk lowers the step-row
					__syncwarp();
					const int rr = tj - lane;
					if (rr >= 0) {
						const uint4 *src = (const uint4*)(gp + (size_t)rr * W + tpb);
						uint4 *dst = (uint4*)(tile + lane * TW);
						#pragma unroll
						for (int k = 0; k < TW / 16; ++k) dst[k] = src[k];
					}
					__syncwarp();
					have = true;
					continue;
				}
				uint32_t tmp = 0;
				if (intile) tmp = tile[(tj - sr) * TW + (ph - tpb)] ^ 0x7fu;
				const bool cont = intile && (state == 0? (tmp & 7) == 0 : (tmp >> (state + 2) & 1) != 0);
				const unsigned stop = __ballot_sync(full, !cont);
				const int r = stop? __ffs(stop) - 1 : 32;
				PK_EMIT(state == 0? 0u : di? 2u : 1u, (uint32_t)r);
				i -= r * di, jj -= r * dj;
				if (r < 32) {
					const uint32_t tr = __shfl_sync(full, tmp, r);
					const bool in_r = __shfl_sync(full, (int)inr, r) != 0, in_t = __shfl_sync(full, (int)intile, r) != 0;
					if (!in_r) break;              // ran off the matrix: the leftover is a leading gap (below)
					if (!in_t) continue;           // ran off the tile: the next round stages the tile around the cell the run stopped at
					if (state == 0) {              // first cell that leaves the diagonal: its own step, in its new state
						state = tr & 7;
						if (state == 1 || state == 3) { PK_EMIT(2u, 1u); --i; } else { PK_EMIT(1u, 1u); --jj; }
					} else state = 0;              // the gap closes here: re-read this cell in the H state
				}
			}
			if (i >= 0) PK_EMIT(2u, (uint32_t)(i + 1));
			if (jj >= 0) PK_EMIT(1u, (uint32_t)(jj + 1));
			PK_CLOSE();
			if (run_len) { if (lane == 0) cig[n] = run_len << 4 | run_op; ++n; }
			#undef PK_EMIT
			#undef PK_CLOSE
			__syncwarp();
			// ---- mm_test_zdrop's scan (align.c:61-89) over the path just traced, 32 bases per step: prefix sums give the score at
			// every base, an exclusive prefix maximum the running maximum it is compared with, a max-scan of the updating
			// lanes the position of that maximum, and the first lane holding the largest drop wins (strict '>' in the reference).
			int zd_max = -1, zd_t0 = -1, zd_t1 = -1, zd_q0 = -1, zd_q1 = -1;
			// Every drop the scan could find is at most the total of the path's negative steps under mm_test_zdrop's scoring (align.c:61-89):
			// its gap costs, plus what the non-matching aligned bases cost -- bounded by mch * aligned bases - DP gap costs - DP score, which
			// charges each of them mch more than the scan does. Below the caller's thresholds the answer is "no drop" whatever the exact value.
			const bool zd_skip = A.zd_skip > 0 && A.mch * n_m - gap_dp - g_score + gap_zd <= A.zd_skip;
			if ((g_flag & MMB_JOB_ZDROP) && zd_skip) zd_max = 0;
			else if (g_flag & MMB_JOB_ZDROP) {
				const uint8_t *gq = smem + (size_t)(wk * NJ + g) * A.qmax;
				const uint8_t *gt = smem + (size_t)nwk * NJ * A.qmax + (size_t)(wk * NJ + g) * TSM;
				const int zq = A.zd_q, ze = A.zd_e, mch = A.mch, mis = A.mis, scn = A.zd_scn;
				int sco = 0, mx = INT32_MIN, mi = -1, mj = -1, ti0 = 0, qj0 = 0;
				zd_max = 0;
				for (int k = n - 1; k >= 0; --k) {
					const uint32_t op = cig[k] & 0xf; const int len = (int)(cig[k] >> 4);
					if (op == 0) {
						for (int base = 0; base < len; base += 32) {
							const bool valid = base + lane < len;
							const int ti = ti0 + base + lane, qj = qj0 + base + lane;
							int sc = 0;
							if (valid) {
								const uint32_t oh = gq[qj];
								const int tb = gt[ti];
								sc = (oh == 0x80 || tb == 4)? scn : (oh >> tb & 1)? mch : mis;
							}
							int S = sc;
							#pragma unroll
							for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(full, S, o); if (lane >= o) S += y; }
							S += sco;
							int pm = valid? S : INT32_MIN;
							#pragma unroll
							for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(full, pm, o); if (lane >= o) pm = max(pm, y); }
							int ex = __shfl_up_sync(full, pm, 1);
							if (lane == 0) ex = INT32_MIN;
							const int M = max(mx, ex);               // running maximum this base is compared with
							const bool upd = valid && S >= M;        // '!(score < max)': ties move the maximum forward
							int lu = upd? lane : -1;
							#pragma unroll
							for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(full, lu, o); if (lane >= o) lu = max(lu, y); }
							int exl = __shfl_up_sync(full, lu, 1);
							if (lane == 0) exl = -1;
							const int cmi = exl >= 0? ti0 + base + exl : mi, cmj = exl >= 0? qj0 + base + exl : mj;
							int z = INT32_MIN;
							if (valid && !upd) { const int li = ti - cmi, lj = qj - cmj, diff = li > lj? li - lj : lj - li; z = M - S - diff * ze; }
							int zm = z;
							#pragma unroll
							for (int o = 16; o > 0; o >>= 1) zm = max(zm, __shfl_xor_sync(full, zm, o));
							if (zm > zd_max) {
								const int wl = __ffs(__ballot_sync(full, z == zm)) - 1;
								zd_max = zm, zd_t0 = __shfl_sync(full, cmi, wl), zd_t1 = __shfl_sync(full, ti, wl), zd_q0 = __shfl_sync(full, cmj, wl), zd_q1 = __shfl_sync(full, qj, wl);
							}
							const int L = __shfl_sync(full, lu, 31);
							if (L >= 0) mx = __shfl_sync(full, S, L), mi = ti0 + base + L, mj = qj0 + base + L;
							sco = __shfl_sync(full, S, min(32, len - base) - 1);
						}
						ti0 += len, qj0 += len;
					} else if (op == 1 || op == 2) {
						sco -= zq + ze * len;
						if (op == 1) qj0 += len; else ti0 += len;
						if (sco < mx) {
							const int li = ti0 - mi, lj = qj0 - mj, diff = li > lj? li - lj : lj - li, z = mx - sco - diff * ze;
							if (z > zd_max) zd_max = z, zd_t0 = mi, zd_t1 = ti0, zd_q0 = mj, zd_q1 = qj0;
						} else mx = sco, mi = ti0, mj = qj0;
					}
				}
			}
			unsigned long long coff = 0;
			if (n > 0) {
				if (lane == 0) coff = atomicAdd(A.cigar_used, (unsigned long long)n);
				coff = __shfl_sync(full, coff, 0);
				const bool rev_cigar = (g_flag & MMB_KSW_REV_CIGAR) != 0;
				if ((long long)(coff + n) <= A.cigar_cap)
					for (int k = lane; k < n; k += 32) A.cigar[coff + k] = rev_cigar? cig[k] : cig[n - 1 - k];
			}
			if (lane == 0) {
				mmb_ksw_res_t o;
				o.zd_max = -1, o.zd_t0 = o.zd_t1 = o.zd_q0 = o.zd_q1 = -1;
				o.max = 0, o.zdropped = 0, o.max_q = o.max_t = o.mqe_t = o.mte_q = -1, o.mqe = o.mte = KSW_NEG_INF;
				o.zd_max = zd_max, o.zd_t0 = zd_t0, o.zd_t1 = zd_t1, o.zd_q0 = zd_q0, o.zd_q1 = zd_q1;
				o.score = g_score, o.n_cigar = n, o.reach_end = 0, o.cigar_off = (uint32_t)coff;
				A.res[g_jid] = o;
			}
			__syncwarp();
		}
	}
	#undef PK_ENC
	#undef PK2
}

} // namespace

// Longest-first queue order for the persistent kernels (dynamic scheduling then has a short tail). A counting sort on a
// 4-bit-mantissa logarithmic key is enough: O(n), deterministic, stable within a bucket.
void mmb_order_by_cells(std::vector<int> &v, const mmb_ksw_job_t *h_jobs)
{
	const int NB = 40 * 16;
	auto key = [&](int i) {
		uint64_t c = (uint64_t)std::max(h_jobs[i].qlen, 1) * (uint64_t)std::max(h_jobs[i].tlen, 1);
		int lg = 63 - __builtin_clzll(c);
		int mant = lg >= 4? (int)(c >> (lg - 4)) & 15 : (int)(c << (4 - lg)) & 15;
		return NB - 1 - std::min(NB - 1, lg * 16 + mant);
	};
	std::vector<int> cnt(NB + 1, 0), out(v.size());
	for (int i : v) ++cnt[key(i) + 1];
	for (int b = 0; b < NB; ++b) cnt[b + 1] += cnt[b];
	for (int i : v) out[cnt[key(i)]++] = i;
	v.swap(out);
}

bool mmb_ksw_fast_eligible(const mmb_ksw_job_t &j)
{
	const int f = j.flag;
	if (f & (MMB_JOB_LL | MMB_JOB_SPLICE | MMB_JOB_T_COMP | MMB_KSW_SCORE_ONLY | MMB_KSW_RIGHT | MMB_KSW_APPROX_DROP | MMB_KSW_EXTZ_ONLY)) return false;
	if (!(f & MMB_KSW_APPROX_MAX)) return false;
	if (j.qlen <= 0 || j.tlen <= 0 || j.tlen > 512 || j.qlen > 2048) return false;
	const int w = j.w < 0? std::max(j.qlen, j.tlen) : j.w;
	return w >= std::max(j.qlen, j.tlen);
}

// Launches the fast kernel over the eligible jobs listed in `idx` (indices into the batch). Asynchronous on ctx->stream
// except for the queue-order upload, which is synchronised before returning.
void mmb_ksw_fast_plan(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, const std::vector<int> &idx, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
					   const uint8_t *d_query, const void *d_target, int t_packed, mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap,
					   unsigned long long *d_cigar_used, int *d_order_all, std::vector<KswPlan> &plans)
{
	if (idx.empty()) return;
	FastArgs A;
	A.jobs = d_jobs, A.query = d_query, A.target = d_target, A.t_packed = t_packed, A.res = d_res;
	A.cigar = d_cigar, A.cigar_cap = cigar_cap, A.cigar_used = d_cigar_used;
	int8_t q = sc->q, e = sc->e, q2 = sc->q2, e2 = sc->e2;
	A.qe0 = q + e;
	if (q2 + e2 < q + e) std::swap(q, q2), std::swap(e, e2);
	A.q = q, A.e = e, A.q2 = q2, A.e2 = e2;
	A.zd_q = sc->q, A.zd_e = sc->e, A.zd_scn = sc->mat[24], A.zd_skip = sc->zd_skip;
	A.one = 1u, A.neg1 = 0xffffffffu;
	A.mch = sc->mat[0], A.mis = sc->mat[1], A.scn = sc->mat[24] == 0? (int8_t)(-e2) : sc->mat[24];
	for (int i = 0; i < 25; ++i) A.mat[i] = sc->mat[i];
	int lt = e != e2? (q2 - q) / (e - e2) - 1 : 0;
	if (q2 + e2 + lt * e2 > q + e + lt * e) ++lt;
	A.long_thres = lt, A.long_diff = lt * (e - e2) - (q2 - q) - e2;
	// The packed kernel needs every intermediate of the recurrence inside [-128, 127] with room to spare, and the simple
	// match/mismatch scoring; anything else runs the scalar kernel.
	const int amax = std::max(std::abs((int)A.mch), std::max(std::abs((int)A.mis), std::abs((int)A.scn)));
	const bool pk_ok = 2 * std::max(q + e, q2 + e2) + amax + 8 <= 127 && A.mch > 0 && A.mis <= 0 && A.scn <= 0;
	// column strips: the smallest C with 32*C >= tlen keeps the idle-lane fraction low (C is a template parameter)
	static const int CW[] = { 2, 4, 6, 7, 8, 9, 10, 12, 14, 16,   4, 8, 12, 16, 20, 24,   14, 16 };
	static const int CPW[] = { 4, 4, 8, 8, 8, 16, 16, 16, 16, 16,   4, 8, 16, 16, 32, 32,   16, 16 };
	static const int LNW[] = { 32, 32, 32, 32, 32, 32, 32, 32, 32, 32,   16, 16, 16, 16, 16, 16,   32, 32 };
	const int NS = 10, NC = 18; // [0,NS): scalar kernel widths, [NS,NC): packed kernel widths (16-lane classes up to tlen 384, then 32-lane)
	std::vector<int> v[NC];
	for (int i : idx) {
		const bool pk = pk_ok && !(h_jobs[i].flag & MMB_KSW_GENERIC_SC);
		int k = pk? NS : 0;
		const int last = pk? NC - 1 : NS - 1;
		while (k < last && LNW[k] * CW[k] < h_jobs[i].tlen) ++k;
		v[k].push_back(i);
	}
	size_t order_off = 0;
	for (int k = 0; k < NC; ++k) {
		if (v[k].empty()) continue;
		mmb_order_by_cells(v[k], h_jobs);
		int maxq = 1, maxsum = 2;
		for (int i : v[k]) maxq = std::max(maxq, h_jobs[i].qlen), maxsum = std::max(maxsum, h_jobs[i].qlen + h_jobs[i].tlen);
		const int C = CW[k], W = LNW[k] * CPW[k], NJ = 32 / LNW[k];
		A.qmax = (maxq + 1 + 15) / 16 * 16;
		const int threads = 128, nwk = threads / 32;
		const size_t smem = k >= NS? ((size_t)A.qmax + (size_t)LNW[k] * C) * nwk * NJ + (size_t)32 * 80 * nwk : (size_t)(A.qmax + 1024) * nwk;
		void (*kern)(FastArgs) = nullptr;
		if (k >= NS && NJ == 2) switch (C) {
		case 4: kern = ksw_pk_kernel<2, 16>; break;   case 8: kern = ksw_pk_kernel<4, 16>; break;
		case 12: kern = ksw_pk_kernel<6, 16>; break;  case 16: kern = ksw_pk_kernel<8, 16>; break;
		case 20: kern = ksw_pk_kernel<10, 16>; break; default: kern = ksw_pk_kernel<12, 16>; break;
		}
		else if (k >= NS) switch (C) {
		case 14: kern = ksw_pk_kernel<7, 32>; break;  default: kern = ksw_pk_kernel<8, 32>; break;
		}
		else switch (C) {
		case 2: kern = ksw_fast_kernel<2>; break;   case 4: kern = ksw_fast_kernel<4>; break;
		case 6: kern = ksw_fast_kernel<6>; break;   case 7: kern = ksw_fast_kernel<7>; break;
		case 8: kern = ksw_fast_kernel<8>; break;   case 9: kern = ksw_fast_kernel<9>; break;
		case 10: kern = ksw_fast_kernel<10>; break; case 12: kern = ksw_fast_kernel<12>; break;
		case 14: kern = ksw_fast_kernel<14>; break; default: kern = ksw_fast_kernel<16>; break;
		}
		int cta_per_sm = 1;
		MMB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cta_per_sm, kern, threads, smem));
		if (cta_per_sm < 1) { fprintf(stderr, "[ERROR] ksw_fast: no occupancy\n"); abort(); }
		int grid = ctx->n_sm * cta_per_sm;
		grid = std::max(1, std::min(grid, ((int)v[k].size() + nwk * NJ - 1) / (nwk * NJ)));
		A.pws_stride = ((size_t)(maxq + 2 * LNW[k] + 2) * W + 255) & ~(size_t)255; // one row per step of the lane-skewed sweep
		A.cigws_stride = (size_t)maxsum + 8;
		int *d_order = d_order_all + order_off; order_off += v[k].size() + 1;
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_order + 1, v[k].data(), v[k].size() * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
		MMB_CUDA_CHECK(cudaMemsetAsync(d_order, 0, sizeof(int), ctx->stream));
		A.counter = d_order, A.order = d_order + 1, A.n = (int)v[k].size();
		KswPlan pl;
		pl.pws_bytes = A.pws_stride * (size_t)grid * nwk * NJ + 256 /* the tile loads may read past the last row */, pl.cigws_bytes = A.cigws_stride * 4 * (size_t)grid * nwk * NJ;
		const FastArgs A0 = A;
		pl.go = [=](uint8_t *pws, uint32_t *cigws) {
			FastArgs B = A0;
			B.pws = pws, B.cigws = cigws;
			kern<<<grid, threads, smem, ctx->stream>>>(B);
			MMB_CUDA_CHECK(cudaGetLastError());
			++ctx->n_launch;
		};
		plans.push_back(pl);
	}
}
