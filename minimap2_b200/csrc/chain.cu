// minimap2_b200/csrc/chain.cu
//
// K2c: anchor chaining on sm_90a. Replaces mg_lchain_dp (reference lchain.c:148-217), mg_chain_backtrack /
// mg_chain_bk_end (lchain.c:9-76) and compact_a (lchain.c:78-111).
//
// Reads are the parallel axis: a batch holds 10^4..10^5 reads whose anchor arrays are independent, while inside a
// read the DP is a chain of data-dependent decisions (strict '>' tie rule scanning j downward, the max_skip early
// exit fed by the t[] marks written inside the same scan, the max_ii shortcut, float32 penalties) and the backtrack
// is pointer chasing over an UNSTABLE radix sort whose tie order decides which chain end is peeled first. Each read
// is therefore replayed exactly by one thread over its own slice of the batch-wide SoA arrays in HBM; a launch covers
// the whole batch (grid = ceil(n_reads/128)), scratch comes from one arena sized by the anchor count.
#include "mmb_internal.h"
#include <cstring>
#include "mm_algo.cuh"
#include "mm_rmq.cuh"
#include "pipeline.h"

namespace {

struct ChainArgs {
	mmb_chain_par_t par;
	int n_reads;
	const int64_t *a_off;   // n_reads+1 anchor offsets
	const m128 *a;          // anchors sorted by x (input; not modified)
	// scratch, all indexed by the read's anchor offset
	int32_t *f, *p, *v, *t;
	m128 *z, *b;
	int32_t *stk;           // radix-sort range stack: stk_off[i] per read
	const int64_t *stk_off;
	// outputs
	int32_t *n_u, *n_v;
	uint64_t *u;            // at a_off[i]
	m128 *a_out;            // at a_off[i]
};

__device__ int32_t bk_end(int32_t max_drop, const m128 *z, const int32_t *f, const int32_t *p, int32_t *t, int32_t k) // lchain.c:9-25
{
	int32_t i = (int32_t)z[k].y, end_i = -1, max_i = i, max_s = 0;
	if (i < 0 || t[i] != 0) return i;
	do {
		int32_t s;
		t[i] = 2;
		end_i = i = p[i];
		s = i < 0? (int32_t)z[k].x : (int32_t)z[k].x - f[i];
		if (s > max_s) max_s = s, max_i = i;
		else if (max_s - s > max_drop) break;
	} while (i >= 0 && t[i] == 0);
	for (i = (int32_t)z[k].y; i >= 0 && i != end_i; i = p[i]) t[i] = 0;
	return max_i;
}


// mg_chain_backtrack + compact_a (lchain.c:27-111) for one read; `ao` may alias `a`
__device__ void backtrack_compact(const m128 *a, int32_t n, const int32_t *f, const int32_t *p, int32_t *v, int32_t *t, m128 *z, m128 *b,
								  int32_t *stk, int32_t min_sc, int32_t min_cnt, int32_t max_drop, uint64_t *u, m128 *ao, int32_t *n_u_, int32_t *n_v_)
{
	int32_t n_z = 0;
	*n_u_ = *n_v_ = 0;
	for (int32_t i = 0; i < n; ++i) if (f[i] >= min_sc) z[n_z].x = (uint64_t)(int64_t)f[i], z[n_z++].y = (uint64_t)i;
	if (n_z == 0) return;
	mmx_rs_sort(z, (int64_t)n_z, stk, KeyX128());
	int32_t n_u = 0, n_v = 0;
	// the reference makes a counting pass and a filling pass with identical traversals; one filling pass suffices here
	// because v[] (reused as the index list, as in the reference) and u[] have capacity n
	for (int32_t i = 0; i < n; ++i) t[i] = 0;
	for (int32_t k = n_z - 1; k >= 0; --k) {
		if (t[z[k].y] == 0) {
			const int32_t n_v0 = n_v, end_i = bk_end(max_drop, z, f, p, t, k);
			int32_t i, sc;
			for (i = (int32_t)z[k].y; i != end_i; i = p[i]) v[n_v++] = i, t[i] = 1;
			sc = i < 0? (int32_t)z[k].x : (int32_t)z[k].x - f[i];
			if (sc >= min_sc && n_v > n_v0 && n_v - n_v0 >= min_cnt) u[n_u++] = (uint64_t)sc << 32 | (uint64_t)(n_v - n_v0);
			else n_v = n_v0;
		}
	}
	*n_u_ = n_u, *n_v_ = n_v;
	if (n_u == 0) return;
	m128 *w = z; // z is free now; n_u <= n_z
	int32_t k = 0;
	for (int32_t i = 0; i < n_u; ++i) {
		const int32_t k0 = k, ni = (int32_t)u[i];
		for (int32_t j = 0; j < ni; ++j) b[k++] = a[v[k0 + (ni - j - 1)]];
	}
	k = 0;
	for (int32_t i = 0; i < n_u; ++i) {
		w[i].x = b[k].x, w[i].y = (uint64_t)k << 32 | (uint64_t)i;
		k += (int32_t)u[i];
	}
	mmx_rs_sort(w, (int64_t)n_u, stk, KeyX128());
	k = 0;
	for (int32_t i = 0; i < n_u; ++i) {
		const int32_t j = (int32_t)w[i].y, nn = (int32_t)u[j];
		const int32_t src = (int32_t)(w[i].y >> 32);
		w[i].x = u[j]; // keep the chain's u value next to its order (w[i].x is no longer needed)
		for (int32_t q = 0; q < nn; ++q) ao[k + q] = b[src + q];
		k += nn;
	}
	for (int32_t i = 0; i < n_u; ++i) u[i] = w[i].x;
}

// DP fill (lchain.c:168-207), one WARP per read. Predecessors j = i-1 .. st are scanned 32 at a time: every lane scores
// one predecessor (coalesced loads of a/f/p/t), and the reference's sequential semantics over the 32 candidates -- strict
// '>' running maximum, the t[] marks written by earlier-scanned predecessors, the clamped n_skip counter and its early
// exit -- are reproduced with warp scans: an exclusive prefix-max, a prefix composition of x -> max(x+a, b) maps for the
// counter, a reduce-or for the marks that fall inside the chunk, and ballots for the break position.
__global__ void __launch_bounds__(128) chain_fill_kernel(ChainArgs A)
{
	const int lane = threadIdx.x & 31;
	const int rd = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (rd >= A.n_reads) return;
	const int64_t off = A.a_off[rd];
	const int32_t n = (int32_t)(A.a_off[rd + 1] - off);
	if (n <= 0) return;
	const unsigned full = 0xffffffffu;
	const m128 *a = A.a + off;
	int32_t *f = A.f + off, *p = A.p + off, *v = A.v + off, *t = A.t + off;
	const mmb_chain_par_t &P = A.par;
	int32_t max_dist_x = P.max_dist_x, max_dist_y = P.max_dist_y;
	const int32_t bw = P.bw, max_skip = P.max_skip, max_iter = P.max_iter, is_cdna = P.is_cdna, n_seg = P.n_seg;
	const float pen_gap = P.chn_pen_gap, pen_skip = P.chn_pen_skip;
	if (max_dist_x < bw) max_dist_x = bw;
	if (max_dist_y < bw && !is_cdna) max_dist_y = bw;
	// Pass 1 (all lanes, one anchor each): the start of anchor i's predecessor window has a closed form -- st is monotone
	// in i in the reference (lchain.c:170-172), so st_i = max(lower_bound(x_i - max_dist_x within the same strand/contig),
	// i - max_iter) -- found by binary search. An anchor with x_i - x_{i-1} > max_dist_x (the bulk of the seed hits, which
	// are isolated) has no predecessor in range and is also too far from every earlier max_ii to keep it: it gets f = span,
	// p = -1 and leaves max_ii = i behind, whatever came before (stv = -1 marks it). Every other anchor needs the sequential
	// DP below, including those whose window only the max_iter cut emptied (st_i >= i: they still take the max_ii shortcut)
	// and those whose window is empty because the previous anchor lies on another contig yet within max_dist_x in x.
	// Their indices are compacted in order into `lst`.
	int32_t *stv = (int32_t*)(A.z + off), *lst = (int32_t*)(A.b + off);
	int32_t n_lst = 0;
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		bool nontriv = false;
		if (i < n) {
			const m128 ai = a[i];
			t[i] = 0;
			nontriv = i > 0 && ai.x - a[i - 1].x <= (uint64_t)(int64_t)max_dist_x;
			if (nontriv) {
				const uint64_t base = ai.x >> 32 << 32;
				const uint64_t lo = ai.x - base > (uint64_t)(int64_t)max_dist_x? ai.x - (uint64_t)(int64_t)max_dist_x : base;
				int32_t l = 0, h = i; // first j in [0, i] with a[j].x >= lo
				while (l < h) { const int32_t m = (l + h) >> 1; if (a[m].x < lo) l = m + 1; else h = m; }
				if (i - l > max_iter) l = i - max_iter; // lchain.c:173; st > i when max_iter < 0
				stv[i] = l;
			} else { const int32_t sp = (int32_t)(ai.y >> 32 & 0xff); f[i] = sp, p[i] = -1, v[i] = sp, stv[i] = -1; }
		}
		const unsigned m = __ballot_sync(full, nontriv);
		if (nontriv) lst[n_lst + __popc(m & ((1u << lane) - 1))] = i;
		n_lst += __popc(m);
	}
	__syncwarp();
	int32_t best_prev = -1;
	for (int32_t li = 0; li < n_lst; ++li) {
		const int32_t i = lst[li];
		const m128 ai = a[i];
		const int32_t st = stv[i];
		if (stv[i - 1] < 0) best_prev = i - 1; // the previous anchor was skipped: it reset max_ii to itself
		// end_j: where the scan stopped; i - 1 when it never started (st > i after a negative max_iter's cut)
		int32_t max_f = (int32_t)(ai.y >> 32 & 0xff), max_j = -1, n_skip = 0, end_j = min(st, i) - 1;
		bool brk = false;
		for (int32_t j_hi = i - 1; j_hi >= st && !brk; j_hi -= 32) {
			const int32_t j = j_hi - lane;
			bool valid = false, marked = false;
			int32_t cand = INT32_MIN, pj = -1;
			if (j >= st) {
				const int32_t sc = mmx_comput_sc(ai, a[j], max_dist_x, max_dist_y, bw, pen_gap, pen_skip, is_cdna, n_seg);
				if (sc != INT32_MIN) valid = true, cand = sc + f[j], pj = p[j];
				marked = t[j] == i;
			}
			// marks by predecessors of this chunk that land inside the chunk (p[j'] < j', so the marker is always scanned earlier)
			unsigned bit = 0;
			if (valid && pj >= 0) {
				if (pj >= j_hi - 31) bit = 1u << (j_hi - pj);
				else t[pj] = i; // lands in a later chunk
			}
			const unsigned mask = __reduce_or_sync(full, bit);
			marked = marked || (mask >> lane & 1);
			// exclusive prefix max of the valid candidates
			int32_t pm = valid? cand : INT32_MIN;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { int32_t y = __shfl_up_sync(full, pm, o); if (lane >= o) pm = max(pm, y); }
			int32_t ex = __shfl_up_sync(full, pm, 1);
			if (lane == 0) ex = INT32_MIN;
			const int32_t run = max(max_f, ex);          // running maximum seen by this lane
			const bool improve = valid && cand > run;
			// n_skip as a composition of maps x -> max(x + ca, cb): improve: (-1, 0); counted skip: (+1, -inf); else identity
			int32_t ca = 0, cb = INT32_MIN / 2;
			const bool inc = valid && !improve && marked;
			if (improve) ca = -1, cb = 0;
			else if (inc) ca = 1;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { // inclusive scan: result = (later map) o (earlier map)
				const int32_t pa = __shfl_up_sync(full, ca, o), pb = __shfl_up_sync(full, cb, o);
				if (lane >= o) { const int32_t na = pa + ca, nb = max(pb + ca, cb); ca = na, cb = nb; }
			}
			const int32_t ns_after = max(n_skip + ca, cb);
			const unsigned brk_mask = __ballot_sync(full, inc && ns_after > max_skip);
			int lim = 32; // lanes < lim are processed
			if (brk_mask) { const int b = __ffs(brk_mask) - 1; lim = b; brk = true; end_j = j_hi - b; }
			const unsigned imp_mask = __ballot_sync(full, improve) & (lim >= 32? full : ((1u << lim) - 1));
			if (imp_mask) {
				const int last = 31 - __clz(imp_mask);   // the last improving lane holds the running maximum
				max_f = __shfl_sync(full, cand, last), max_j = j_hi - last;
			}
			if (!brk) n_skip = __shfl_sync(full, ns_after, 31);
			__syncwarp(); // order the t[] marks before the next chunk reads them
		}
		// max_ii shortcut (lchain.c:188-201)
		if (best_prev < 0 || ai.x - a[best_prev].x > (uint64_t)(int64_t)max_dist_x) {
			int32_t mx = INT32_MIN, mxj = -1;
			for (int32_t j = i - 1 - lane; j >= st; j -= 32) { const int32_t fj = f[j]; if (mx < fj) mx = fj, mxj = j; } // per lane: descending j, strict '<'
			#pragma unroll
			for (int o = 16; o > 0; o >>= 1) { // ties go to the larger j (scanned first by the reference)
				const int32_t om = __shfl_xor_sync(full, mx, o), oj = __shfl_xor_sync(full, mxj, o);
				if (om > mx || (om == mx && oj > mxj)) mx = om, mxj = oj;
			}
			best_prev = mxj;
		}
		if (best_prev >= 0 && best_prev < end_j) {
			const int32_t tmp = mmx_comput_sc(ai, a[best_prev], max_dist_x, max_dist_y, bw, pen_gap, pen_skip, is_cdna, n_seg);
			if (tmp != INT32_MIN && max_f < tmp + f[best_prev]) max_f = tmp + f[best_prev], max_j = best_prev;
		}
		if (lane == 0) {
			f[i] = max_f, p[i] = max_j;
			v[i] = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
		}
		__syncwarp();
		if (best_prev < 0 || (ai.x - a[best_prev].x <= (uint64_t)(int64_t)max_dist_x && f[best_prev] < max_f)) best_prev = i;
	}
}

// Backtrack + compaction (mg_chain_backtrack lchain.c:27-76, compact_a :78-111) in three launches, each shaped after its part:
//   chain_bt_collect_kernel  warp per read   candidate chain ends (f >= min_sc) gathered in anchor order with ballots, t[] cleared:
//                                            coalesced streaming over the read's anchors
//   chain_bt_peel_kernel     thread per read the unstable sort of the candidates (exact tie order) and the best-first peeling are
//                                            chains of dependent loads; one thread per read keeps every read of the batch in flight
//                                            at once, which is what hides that latency
//   chain_bt_compact_kernel  warp per read   chains copied into b[] and, ordered by first target position, into a_out by all lanes
__global__ void __launch_bounds__(128) chain_bt_collect_kernel(ChainArgs A)
{
	const int lane = threadIdx.x & 31;
	const int rd = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (rd >= A.n_reads) return;
	const unsigned full = 0xffffffffu;
	const int64_t off = A.a_off[rd];
	const int32_t n = (int32_t)(A.a_off[rd + 1] - off);
	const int32_t min_sc = A.par.min_sc;
	const int32_t *f = A.f + off;
	int32_t *t = A.t + off;
	m128 *z = A.z + off;
	int32_t n_z = 0; // candidate chain ends in anchor order (lchain.c:35-37), t[] cleared on the way
	for (int32_t i0 = 0; i0 < n; i0 += 32) {
		const int32_t i = i0 + lane;
		const int32_t fi = i < n? f[i] : INT32_MIN;
		const bool keep = i < n && fi >= min_sc;
		const unsigned m = __ballot_sync(full, keep);
		if (keep) { const int32_t k = n_z + __popc(m & ((1u << lane) - 1)); z[k].x = (uint64_t)(int64_t)fi, z[k].y = (uint64_t)i; }
		n_z += __popc(m);
		if (i < n) t[i] = 0;
	}
	if (lane == 0) A.n_u[rd] = n_z, A.n_v[rd] = 0; // n_u carries the candidate count to the next launch
}

__global__ void __launch_bounds__(128) chain_bt_peel_kernel(ChainArgs A)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= A.n_reads) return;
	const int32_t n_z = A.n_u[rd];
	if (n_z == 0) return; // n_u = n_v = 0 already
	const int64_t off = A.a_off[rd];
	const mmb_chain_par_t &P = A.par;
	const int32_t max_drop = P.is_cdna? INT32_MAX : P.bw, min_sc = P.min_sc, min_cnt = P.min_cnt;
	const int32_t *f = A.f + off, *p = A.p + off;
	int32_t *v = A.v + off, *t = A.t + off, *stk = A.stk + A.stk_off[rd];
	m128 *z = A.z + off;
	uint64_t *u = A.u + off;
	int32_t n_u = 0, n_v = 0;
	// lchain.c:38-66: best end first; one filling pass suffices (v[] and u[] have capacity n)
	mmx_rs_sort(z, (int64_t)n_z, stk, KeyX128());
	for (int32_t k = n_z - 1; k >= 0; --k) {
		if (t[z[k].y] == 0) {
			const int32_t n_v0 = n_v, end_i = bk_end(max_drop, z, f, p, t, k);
			int32_t i, sc;
			for (i = (int32_t)z[k].y; i != end_i; i = p[i]) v[n_v++] = i, t[i] = 1;
			sc = i < 0? (int32_t)z[k].x : (int32_t)z[k].x - f[i];
			if (sc >= min_sc && n_v > n_v0 && n_v - n_v0 >= min_cnt) u[n_u++] = (uint64_t)sc << 32 | (uint64_t)(n_v - n_v0);
			else n_v = n_v0;
		}
	}
	A.n_u[rd] = n_u, A.n_v[rd] = n_v;
}

__global__ void __launch_bounds__(128) chain_bt_compact_kernel(ChainArgs A)
{
	const int lane = threadIdx.x & 31;
	const int rd = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (rd >= A.n_reads) return;
	const int32_t n_u = A.n_u[rd];
	if (n_u == 0) return;
	const int64_t off = A.a_off[rd];
	const m128 *a = A.a + off;
	const int32_t *v = A.v + off;
	int32_t *stk = A.stk + A.stk_off[rd];
	m128 *z = A.z + off, *b = A.b + off, *ao = A.a_out + off;
	uint64_t *u = A.u + off;
	// compact_a (lchain.c:78-111): chains laid out in b[] with their anchors in ascending order, then ordered by first target position
	m128 *w = z; // z is free now; n_u <= n_z
	int32_t k = 0;
	for (int32_t i = 0; i < n_u; ++i) {
		const int32_t k0 = k, ni = (int32_t)u[i];
		for (int32_t j = lane; j < ni; j += 32) b[k0 + j] = a[v[k0 + (ni - j - 1)]];
		k += ni;
	}
	__syncwarp();
	if (lane == 0) {
		k = 0;
		for (int32_t i = 0; i < n_u; ++i) { w[i].x = b[k].x, w[i].y = (uint64_t)k << 32 | (uint64_t)i; k += (int32_t)u[i]; }
		mmx_rs_sort(w, (int64_t)n_u, stk, KeyX128());
	}
	__syncwarp();
	k = 0;
	for (int32_t i = 0; i < n_u; ++i) {
		const int32_t j = (int32_t)w[i].y, nn = (int32_t)u[j], src = (int32_t)(w[i].y >> 32);
		for (int32_t q = lane; q < nn; q += 32) ao[k + q] = b[src + q];
		k += nn;
	}
	__syncwarp();
	for (int32_t i = lane; i < n_u; i += 32) w[i].x = u[(int32_t)w[i].y]; // the chain's u value travels with its rank
	__syncwarp();
	for (int32_t i = lane; i < n_u; i += 32) u[i] = w[i].x;
}

// ---------------------------------------------------------------------------------------------------------
// Long-join rescue (map.c:283-292): reads whose first-round chaining left more than one chain and whose best chain
// leaves a long unchained part are re-sorted (radix_sort_128x, exact tie order) and re-chained with mg_lchain_rmq
// (lchain.c:250-368) at bw_long. One thread per read; the two balanced trees of the reference live in per-read slices of
// an HBM arena (mm_rmq.cuh).
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ RmqTree tree_at(uint8_t *base, int32_t n)
{
	RmqTree T;
	const size_t m = (size_t)n + 1;
	T.pri = (double*)base;
	T.c[0] = (int32_t*)(base + 8 * m), T.c[1] = T.c[0] + m, T.s = T.c[1] + m;
	T.size = (uint32_t*)(T.s + m), T.y = (int32_t*)(T.size + m);
	T.bal = (int8_t*)(T.y + m);
	T.root = RMQ_NIL, T.n = n;
	return T;
}

__global__ void __launch_bounds__(64) chain_rescue_kernel(ChainArgs A, RescuePar R)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= A.n_reads) return;
	const int64_t off = A.a_off[rd];
	m128 *a = A.a_out + off;
	uint64_t *u = A.u + off;
	int32_t *stk = A.stk + A.stk_off[rd];
	int32_t n;
	if (R.primary) { // first chainer: all anchors of the read, in the order the seed sort left them (already copied into a_out)
		n = (int32_t)(A.a_off[rd + 1] - off);
		if (n == 0) { A.n_u[rd] = 0, A.n_v[rd] = 0; return; } // lchain.c:261-264
	} else {         // map.c:283-291
		if (A.n_u[rd] <= 1) return;
		n = A.n_v[rd];
		const int32_t qlen = R.qlen[rd];
		const int32_t st = (int32_t)a[0].y, en = (int32_t)a[(int32_t)u[0] - 1].y;
		if (!(qlen - (en - st) > R.rescue_size || (float)(en - st) > (float)qlen * R.rescue_ratio)) return;
		mmx_rs_sort(a, (int64_t)n, stk, KeyX128());
	}
	int32_t *f = A.f + off, *p = A.p + off, *v = A.v + off, *t = A.t + off;
	int32_t max_dist = R.max_dist, max_dist_inner = R.max_dist_inner;
	const int32_t bw = R.bw, max_chn_skip = R.max_skip, cap = R.rmq_size_cap;
	const float pen_gap = R.pen_gap, pen_skip = R.pen_skip;
	if (max_dist < bw) max_dist = bw;
	if (max_dist_inner < 0) max_dist_inner = 0;
	if (max_dist_inner > max_dist) max_dist_inner = max_dist;
	uint8_t *tb = R.tree + ((size_t)R.tree_off[rd] + (size_t)rd) * 64;
	RmqTree T0 = tree_at(tb, n), T1 = tree_at(tb + (size_t)32 * (n + 1), n);
	for (int32_t i = 0; i < n; ++i) t[i] = 0;
	int32_t i0 = 0, st = 0, st_inner = 0;
	for (int32_t i = 0; i < n; ++i) {
		int32_t max_j = -1, q_span = (int32_t)(a[i].y >> 32 & 0xff), max_f = q_span;
		if (i0 < i && a[i0].x != a[i].x) { // add in-range anchors (lchain.c:281-294)
			for (int32_t j = i0; j < i; ++j) {
				const double pri = -((double)f[j] + 0.5 * (double)pen_gap * (double)(int32_t)((uint32_t)a[j].x + (uint32_t)a[j].y));
				T0.y[j] = (int32_t)a[j].y, T0.pri[j] = pri;
				rmq_insert(T0, j);
				if (max_dist_inner > 0) { T1.y[j] = (int32_t)a[j].y, T1.pri[j] = pri; rmq_insert(T1, j); }
			}
			i0 = i;
		}
		// drop anchors that fell out of range (lchain.c:296-313)
		while (st < i && (a[i].x >> 32 != a[st].x >> 32 || a[i].x > a[st].x + (uint64_t)(int64_t)max_dist || (T0.root >= 0? (int32_t)T0.size[T0.root] : 0) > cap)) {
			if (rmq_find(T0, (int32_t)a[st].y, st) >= 0) rmq_erase(T0, (int32_t)a[st].y, st);
			++st;
		}
		if (max_dist_inner > 0) {
			while (st_inner < i && (a[i].x >> 32 != a[st_inner].x >> 32 || a[i].x > a[st_inner].x + (uint64_t)(int64_t)max_dist_inner || (T1.root >= 0? (int32_t)T1.size[T1.root] : 0) > cap)) {
				if (rmq_find(T1, (int32_t)a[st_inner].y, st_inner) >= 0) rmq_erase(T1, (int32_t)a[st_inner].y, st_inner);
				++st_inner;
			}
		}
		// RMQ (lchain.c:315-350)
		const int32_t yi = (int32_t)a[i].y;
		int32_t q = rmq_query(T0, yi - max_dist, (int64_t)INT32_MAX, yi, 0);
		if (q >= 0) {
			int32_t sc, exact, width, n_skip = 0, j = q;
			sc = f[j] + mmx_comput_sc_simple(a[i], a[j], pen_gap, pen_skip, &exact, &width);
			if (width <= bw && sc > max_f) max_f = sc, max_j = j;
			if (!exact && T1.root >= 0 && yi > 0) {
				int32_t lo, hi;
				rmq_interval(T1, yi - 1, (int64_t)n, &lo, &hi);
				if (lo >= 0) {
					RmqItr itr;
					rmq_itr_find(T1, T1.y[lo], (int64_t)lo, &itr);
					int32_t qq;
					while ((qq = rmq_itr_at(&itr)) >= 0) {
						if (T1.y[qq] < yi - max_dist_inner) break;
						j = qq;
						sc = f[j] + mmx_comput_sc_simple(a[i], a[j], pen_gap, pen_skip, 0, &width);
						if (width <= bw) {
							if (sc > max_f) {
								max_f = sc, max_j = j;
								if (n_skip > 0) --n_skip;
							} else if (t[j] == i) {
								if (++n_skip > max_chn_skip) break;
							}
							if (p[j] >= 0) t[p[j]] = i;
						}
						if (!rmq_itr_next_bidir(T1, &itr, 0)) break;
					}
				}
			}
		}
		f[i] = max_f, p[i] = max_j;
		v[i] = max_j >= 0 && v[max_j] > max_f? v[max_j] : max_f;
	}
	int32_t n_u, n_v;
	backtrack_compact(a, n, f, p, v, t, A.z + off, A.b + off, stk, R.min_sc, R.min_cnt, bw, u, a, &n_u, &n_v);
	A.n_u[rd] = n_u, A.n_v[rd] = n_v;
}

} // namespace

#include "scan.cuh"

// Scratch of the DP, backtrack and RMQ kernels: f, p, v, t (4 x int32) | z (m128) | b (m128), n_tot+4 entries each, in scratch
// (reserved here when `reserve`), and the per-read sort stacks that mmb_sort_stacks_async laid out in scratch2. The chainers reserve
// the scratch; the rescue that follows them reuses it as it is.
static void chain_scratch_layout(ChainArgs &A, int n_reads, int64_t n_tot, DevBuf &scratch, DevBuf &scratch2, bool reserve)
{
	const size_t n = (size_t)n_tot + 4;
	uint8_t *s = (uint8_t*)(reserve? scratch.reserve(n * (16 + 16 + 16) + 256) : scratch.p);
	A.f = (int32_t*)s, A.p = A.f + n, A.v = A.p + n, A.t = A.v + n;
	A.z = (m128*)(s + n * 16), A.b = A.z + n;
	A.stk_off = (int64_t*)scratch2.p, A.stk = mmb_sort_stacks((int64_t*)scratch2.p, n_reads);
}

static void chain_scratch_setup(mmb_ctx_t *ctx, ChainArgs &A, int n_reads, const m128 *d_a, const int64_t *d_a_off, int64_t n_tot,
								int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2)
{
	A.n_reads = n_reads, A.a_off = d_a_off, A.a = d_a;
	mmb_sort_stacks_async(ctx, d_a_off, n_reads, n_tot, scratch2, 0);
	chain_scratch_layout(A, n_reads, n_tot, scratch, scratch2, true);
	A.n_u = d_n_u, A.n_v = d_n_v, A.u = d_u, A.a_out = d_a_out;
}

// Device-level launcher (asynchronous). d_a: anchors (sorted by x per read), d_a_off: n_reads+1 offsets, total anchors n_tot.
// Outputs (device): d_n_u, d_n_v (n_reads), d_u (n_tot, at the read's anchor offset), d_a_out (n_tot).
void mmb_chain_device(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const m128 *d_a, const int64_t *d_a_off, int64_t n_tot,
					  int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2)
{
	if (n_reads <= 0) return;
	ChainArgs A;
	A.par = *par;
	chain_scratch_setup(ctx, A, n_reads, d_a, d_a_off, n_tot, d_n_u, d_n_v, d_u, d_a_out, scratch, scratch2);
	ProfScope prof(ctx, MMB_PROF_CHAIN, (uint64_t)n_tot);
	chain_fill_kernel<<<(unsigned)(((int64_t)n_reads * 32 + 127) / 128), 128, 0, ctx->stream>>>(A);
	chain_bt_collect_kernel<<<(unsigned)(((int64_t)n_reads * 32 + 127) / 128), 128, 0, ctx->stream>>>(A);
	chain_bt_peel_kernel<<<(n_reads + 127) / 128, 128, 0, ctx->stream>>>(A);
	chain_bt_compact_kernel<<<(unsigned)(((int64_t)n_reads * 32 + 127) / 128), 128, 0, ctx->stream>>>(A);
	MMB_CUDA_CHECK(cudaGetLastError());
	ctx->n_launch += 4;
}

extern "C" int mmb_chain_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const uint64_t *anchors_xy, const int64_t *a_off,
									int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy)
{
	if (n_reads <= 0) return 0;
	if (par->use_rmq) { fprintf(stderr, "[ERROR] mmb_chain_batch_host: rmq chaining goes through mmb_chain_rmq_batch_host\n"); abort(); }
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	const int64_t n_tot = a_off[n_reads];
	m128 *d_a = ctx->d_a.as<m128>((size_t)n_tot + 1);
	int64_t *d_off = ctx->d_b.as<int64_t>((size_t)n_reads + 1);
	int32_t *d_nu = ctx->d_c.as<int32_t>((size_t)n_reads * 2 + 2), *d_nv = d_nu + n_reads;
	uint64_t *d_u = ctx->d_d.as<uint64_t>((size_t)n_tot + 1);
	m128 *d_ao = ctx->d_e.as<m128>((size_t)n_tot + 1);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_a, anchors_xy, sizeof(m128) * n_tot, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, a_off, sizeof(int64_t) * (n_reads + 1), cudaMemcpyHostToDevice, ctx->stream));
	mmb_chain_device(ctx, par, n_reads, d_a, d_off, n_tot, d_nu, d_nv, d_u, d_ao, ctx->d_f, ctx->d_g);
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_u, d_nu, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_v, d_nv, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(u_out, d_u, sizeof(uint64_t) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(a_out_xy, d_ao, sizeof(m128) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return 0;
}

// Re-chain (on the device) the reads that qualify for the long-join rescue. Must follow mmb_chain_device on the same
// buffers (it reuses the scratch set up there). d_tree_off: per-read exclusive offsets of n_v (n_reads+1), total tot_v.
void mmb_chain_rescue_device(mmb_ctx_t *ctx, const RescuePar *rp, int n_reads, const int64_t *d_a_off, int64_t n_tot,
							 int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf, int64_t tot_v)
{
	if (n_reads <= 0) return;
	ChainArgs A;
	memset(&A, 0, sizeof(A));
	A.n_reads = n_reads, A.a_off = d_a_off, A.a = nullptr;
	chain_scratch_layout(A, n_reads, n_tot, scratch, scratch2, false);
	A.n_u = d_n_u, A.n_v = d_n_v, A.u = d_u, A.a_out = d_a_out;
	RescuePar R = *rp;
	R.tree = (uint8_t*)treebuf.reserve(((size_t)tot_v + (size_t)n_reads + 8) * 64);
	ProfScope prof(ctx, MMB_PROF_CHAIN, 0);
	chain_rescue_kernel<<<(n_reads + 63) / 64, 64, 0, ctx->stream>>>(A, R);
	MMB_CUDA_CHECK(cudaGetLastError());
	++ctx->n_launch;
}

void mmb_chain_rmq_primary_device(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const m128 *d_a, const int64_t *d_a_off, int64_t n_tot,
								  int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf)
{
	if (n_reads <= 0) return;
	ChainArgs A;
	memset(&A, 0, sizeof(A));
	chain_scratch_setup(ctx, A, n_reads, d_a, d_a_off, n_tot, d_n_u, d_n_v, d_u, d_a_out, scratch, scratch2);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_a_out, d_a, sizeof(m128) * (size_t)n_tot, cudaMemcpyDeviceToDevice, ctx->stream)); // the kernel chains in place
	RescuePar R;
	memset(&R, 0, sizeof(R));
	R.primary = 1, R.qlen = nullptr;
	R.max_dist = par->max_dist_x, R.max_dist_inner = par->max_dist_inner, R.bw = par->bw, R.max_skip = par->max_skip;
	R.rmq_size_cap = par->rmq_size_cap, R.min_cnt = par->min_cnt, R.min_sc = par->min_sc;
	R.pen_gap = par->chn_pen_gap, R.pen_skip = par->chn_pen_skip;
	R.tree = (uint8_t*)treebuf.reserve(((size_t)n_tot + (size_t)n_reads + 8) * 64), R.tree_off = d_a_off; // 64 B of tree node per anchor
	ProfScope prof(ctx, MMB_PROF_CHAIN, (uint64_t)n_tot);
	chain_rescue_kernel<<<(n_reads + 63) / 64, 64, 0, ctx->stream>>>(A, R);
	MMB_CUDA_CHECK(cudaGetLastError());
	++ctx->n_launch;
}

void mmb_chain_stage(mmb_ctx_t *ctx, const mmb_chain_par_t *par, const RescuePar *rp, int n_reads, const m128 *d_a, const int64_t *d_a_off,
					 int64_t n_tot, int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, int64_t *d_vo,
					 DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf)
{
	if (par->use_rmq) mmb_chain_rmq_primary_device(ctx, par, n_reads, d_a, d_a_off, n_tot, d_n_u, d_n_v, d_u, d_a_out, scratch, scratch2, treebuf);
	else mmb_chain_device(ctx, par, n_reads, d_a, d_a_off, n_tot, d_n_u, d_n_v, d_u, d_a_out, scratch, scratch2);
	if (!rp || n_reads <= 0) return;
	// the rescue's trees take 64 B per compacted anchor plus one node per read: read rd's start at tree_off[rd] + rd
	mmb_widen_i32_async(ctx, d_n_v, n_reads, d_vo);
	const int64_t tot_v = mmb_exclusive_scan_i64(ctx, d_vo, n_reads, true);
	RescuePar R = *rp;
	R.primary = 0, R.tree_off = d_vo;
	mmb_chain_rescue_device(ctx, &R, n_reads, d_a_off, n_tot, d_n_u, d_n_v, d_u, d_a_out, scratch, scratch2, treebuf, tot_v);
}

extern "C" int mmb_chain_rescue_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, const mmb_rescue_par_t *rp, int n_reads, const uint64_t *anchors_xy,
										   const int64_t *a_off, const int32_t *qlen, int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy)
{
	if (n_reads <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	const int64_t n_tot = a_off[n_reads];
	m128 *d_a = ctx->d_a.as<m128>((size_t)n_tot + 1);
	int64_t *d_off = ctx->d_b.as<int64_t>((size_t)(n_reads + 1) * 2), *d_vo = d_off + (n_reads + 1);
	int32_t *d_nu = ctx->d_c.as<int32_t>((size_t)n_reads * 3 + 3), *d_nv = d_nu + n_reads, *d_qlen = d_nv + n_reads;
	uint64_t *d_u = ctx->d_d.as<uint64_t>((size_t)n_tot + 1);
	m128 *d_ao = ctx->d_e.as<m128>((size_t)n_tot + 1);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_a, anchors_xy, sizeof(m128) * n_tot, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, a_off, sizeof(int64_t) * (n_reads + 1), cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_qlen, qlen, sizeof(int32_t) * n_reads, cudaMemcpyHostToDevice, ctx->stream));
	RescuePar R;
	memset(&R, 0, sizeof(R));
	R.qlen = d_qlen, R.rescue_size = rp->rescue_size, R.rescue_ratio = rp->rescue_ratio;
	R.max_dist = rp->max_dist, R.max_dist_inner = rp->max_dist_inner, R.bw = rp->bw_long, R.max_skip = par->max_skip;
	R.rmq_size_cap = rp->rmq_size_cap, R.min_cnt = par->min_cnt, R.min_sc = par->min_sc;
	R.pen_gap = par->chn_pen_gap, R.pen_skip = par->chn_pen_skip;
	mmb_chain_stage(ctx, par, &R, n_reads, d_a, d_off, n_tot, d_nu, d_nv, d_u, d_ao, d_vo, ctx->d_f, ctx->d_g, ctx->d_h);
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_u, d_nu, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_v, d_nv, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(u_out, d_u, sizeof(uint64_t) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(a_out_xy, d_ao, sizeof(m128) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return 0;
}

// Kernel-level entry for mg_lchain_rmq alone (lchain.c:251-357), HOST buffers. Used by the parity tests against the reference function.
// par: max_dist_x = max_dist, max_dist_inner, bw, max_skip, rmq_size_cap, min_cnt, min_sc, chn_pen_gap, chn_pen_skip.
extern "C" int mmb_chain_rmq_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const uint64_t *anchors_xy, const int64_t *a_off,
										int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy)
{
	if (n_reads <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	const int64_t n_tot = a_off[n_reads];
	m128 *d_a = ctx->d_a.as<m128>((size_t)n_tot + 1);
	int64_t *d_off = ctx->d_b.as<int64_t>((size_t)n_reads + 1);
	int32_t *d_nu = ctx->d_c.as<int32_t>((size_t)n_reads * 2 + 2), *d_nv = d_nu + n_reads;
	uint64_t *d_u = ctx->d_d.as<uint64_t>((size_t)n_tot + 1);
	m128 *d_ao = ctx->d_e.as<m128>((size_t)n_tot + 1);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_a, anchors_xy, sizeof(m128) * n_tot, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, a_off, sizeof(int64_t) * (n_reads + 1), cudaMemcpyHostToDevice, ctx->stream));
	mmb_chain_rmq_primary_device(ctx, par, n_reads, d_a, d_off, n_tot, d_nu, d_nv, d_u, d_ao, ctx->d_f, ctx->d_g, ctx->d_h);
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_u, d_nu, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_v, d_nv, sizeof(int32_t) * n_reads, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(u_out, d_u, sizeof(uint64_t) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(a_out_xy, d_ao, sizeof(m128) * n_tot, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return 0;
}
