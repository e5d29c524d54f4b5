// minimap2_b200/csrc/finalize.cu -- K4: the per-hit tail of the alignment driver on the device (SURVEY section 8 row f4).
//
// After the ksw2 jobs of a hit (left extension, gap fills, right extension) have run, the reference assembles the hit's CIGAR with
// mm_append_cigar (align.c:305-334), left-aligns its gaps and drops a leading I/D with mm_fix_cigar (align.c:105-181), and rescans
// every aligned base in mm_update_extra (align.c:254-303) for blen / mlen / n_ambi / dp_max. On the host that was the largest single
// cost of the replay driver (a third of its CPU time: one pass over every aligned base of every read). Here one warp per hit does
// the three steps straight from the job CIGARs that are still in the device arena, so only the final CIGAR and eight integers per
// hit cross PCIe. The running score of mm_update_extra is a sum of integers and of q + e * mg_log2(1+len) gap penalties that are
// exact multiples of 2^-23 for int8_t q and e (see update_extra in align.cc), so it is carried in 2^-32 fixed point -- exactly the
// reference's double arithmetic. A hit whose CIGAR does not consume its query and target spans, which the reference asserts, is
// flagged (status 2) and redone by the host driver.
#include "pipeline.h"

namespace {

struct Acc { // the hit's two sequences as mm_update_extra sees them: query piece on its strand, target piece forward
	const uint8_t *query; const uint32_t *S;
	int64_t q0, t0; int32_t qlen, qs, rev;
	__device__ __forceinline__ int q(int x) const { // base x of the aligned query piece (align.c:1056-1061 for the reverse strand)
		const int p = qs + x;
		if (!rev) return query[q0 + p];
		const int c = query[q0 + (qlen - 1 - p)];
		return c < 4? 3 - c : 4;
	}
	__device__ __forceinline__ int t(int y) const { return (int)mmx_seq4_get(S, (uint64_t)(t0 + y)); }
};

// ---- warp-cooperative pieces ----
#define FIN_INF (1 << 29)
__device__ __forceinline__ int fin_sat(int v) { return v < FIN_INF? v : FIN_INF; }
__device__ __forceinline__ long long shfl_down_ll(long long v, int off) { return __shfl_down_sync(0xffffffffu, v, off); }

// The clamped running score of mm_update_extra, s <- max(s + d, 0) with the running maximum m <- max(m, s), over a stretch of steps is
// the pair of functions s -> max(s + T, C), m -> max(m, s + Mx, Cm); stretches compose associatively, so lanes summarise their own
// operations and an ordered warp reduction joins them (all values in 2^-32 fixed point).
struct Walk { long long T, C, Mx, Cm; };
__device__ __forceinline__ void walk_step(Walk &w, long long d) { w.T += d; w.C = w.C + d > 0? w.C + d : 0; w.Mx = w.Mx > w.T? w.Mx : w.T; w.Cm = w.Cm > w.C? w.Cm : w.C; }
__device__ __forceinline__ Walk walk_join(const Walk &a, const Walk &b) // a, then b
{
	Walk r;
	r.T = a.T + b.T;
	r.C = a.C + b.T > b.C? a.C + b.T : b.C;
	r.Mx = a.Mx > a.T + b.Mx? a.Mx : a.T + b.Mx;
	long long cm = a.Cm > b.Cm? a.Cm : b.Cm;
	r.Cm = cm > a.C + b.Mx? cm : a.C + b.Mx;
	return r;
}

// One WARP per hit. Stage 1 stitches the pieces (lanes fetch 32 piece descriptors at a time, all lanes copy each piece); stage 2 is
// mm_fix_cigar with one operation per lane: the left shift of a gap between two matches is l = min(len(M before) + shift of the gap two
// operations earlier, run of equal bases), a (min,+) recurrence at distance two that a stride-2 warp scan solves, the rare I/D-run
// merge and the squeeze of emptied operations stay sequential on lane 0; stage 3 is mm_update_extra with one operation per lane.
__global__ void __launch_bounds__(128) finalize_kernel(const FinReg *regs, const FinJobRef *jobs, int n, const uint8_t *query, const uint32_t *S,
													   uint32_t *out, FinOut *res, FinPar par)
{
	const unsigned full = 0xffffffffu;
	const int lane = threadIdx.x & 31;
	const int r = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
	if (r >= n) return;
	const FinReg R = regs[r];
	uint32_t *c = out + R.out_off;
	Acc A; A.query = query, A.S = S, A.q0 = R.q0, A.t0 = R.t0, A.qlen = R.qlen, A.qs = R.qs, A.rev = R.rev;
	int status = 0, qshift = 0, tshift = 0;
	// ---- stage 1: mm_append_cigar over the pieces in driver order ----
	uint32_t nc = 0;
	{
		int last_type = -1;
		for (int base = 0; base < R.n_jobs; base += 32) {
			const int j = base + lane;
			FinJobRef J; J.cig = nullptr, J.n = 0, J.pad = 0;
			if (j < R.n_jobs) J = jobs[R.job_first + j];
			uint32_t f = 0; int lt = -1;
			if (J.n) f = J.cig[0], lt = (int)(J.cig[J.n - 1] & 0xf);
			const unsigned ne = __ballot_sync(full, J.n != 0);
			const unsigned below = ne & ((1u << lane) - 1);
			const int pt = __shfl_sync(full, lt, below? 31 - __clz((int)below) : 0);
			const int prev_type = below? pt : last_type;
			const bool merge = J.n != 0 && prev_type == (int)(f & 0xf); // the piece's first operation joins the last one so far
			const uint32_t cnt = J.n - (merge? 1u : 0u);
			uint32_t inc = cnt;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(full, inc, o); if (lane >= o) inc += y; }
			const uint32_t pos = nc + inc - cnt;
			const unsigned long long pbits = (unsigned long long)(uintptr_t)J.cig;
			for (int p = 0; p < 32; ++p) {
				const uint32_t pn = __shfl_sync(full, J.n, p);
				if (!pn) continue;
				const uint32_t *src = (const uint32_t*)(uintptr_t)__shfl_sync(full, pbits, p);
				const uint32_t ppos = __shfl_sync(full, pos, p), pm = __shfl_sync(full, merge? 1u : 0u, p);
				for (uint32_t i = pm + lane; i < pn; i += 32) c[ppos + i - pm] = src[i];
			}
			__syncwarp();
			if (merge) atomicAdd(&c[pos - 1], f >> 4 << 4);
			nc += __shfl_sync(full, inc, 31);
			if (ne) last_type = __shfl_sync(full, lt, 31 - __clz((int)ne));
			__syncwarp();
		}
	}
	// ---- stage 2: mm_fix_cigar (align.c:105-181) ----
	if (nc > 1) {
		int carry_q = 0, carry_t = 0, carry_l0 = 0, carry_l1 = 0; // offsets at the chunk start; shifts of the last even / odd operation of the previous chunk
		uint32_t carry_w = 0;                                       // the previous chunk's last operation as it was before any shift
		bool shrink = false, run_trigger = false;
		for (uint32_t base = 0; base < nc; base += 32) {
			const uint32_t k = base + lane;
			const bool valid = k < nc;
			const uint32_t w = valid? c[k] : 0u;
			const int op = (int)(w & 0xf), len = (int)(w >> 4);
			uint32_t pw = __shfl_up_sync(full, w, 1), nw = __shfl_down_sync(full, w, 1);
			if (lane == 0) pw = carry_w;
			if (lane == 31) nw = k + 1 < nc? c[k + 1] : 0u;
			const bool has_prev = k > 0, has_next = k + 1 < nc;
			int dq = 0, dt = 0;
			if (valid) { if (op == MM_CIGAR_MATCH) dq = dt = len; else if (op == MM_CIGAR_INS) dq = len; else if (op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) dt = len; }
			int iq = dq, it = dt;
			#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { const int yq = __shfl_up_sync(full, iq, o), yt = __shfl_up_sync(full, it, o); if (lane >= o) iq += yq, it += yt; }
			const int qoff = carry_q + iq - dq, toff = carry_t + it - dt;
			if (valid && has_next && op > 0 && op + (int)(nw & 0xf) == 3) run_trigger = true;
			const bool qual = valid && (op == MM_CIGAR_INS || op == MM_CIGAR_DEL) && has_prev && has_next && (pw & 0xf) == 0 && (nw & 0xf) == 0;
			const int lprev = (int)(pw >> 4), xin = (lane & 1)? carry_l1 : carry_l0;
			// upper bound of the shift: the (min,+) scan with no run limit
			int sa = qual? lprev : FIN_INF, sb = qual? FIN_INF : 0;
			#pragma unroll
			for (int o = 2; o < 32; o <<= 1) { const int pa = __shfl_up_sync(full, sa, o), pb = __shfl_up_sync(full, sb, o); if (lane >= o) { const int nb = fin_sat(pb + sa); sb = nb < sb? nb : sb; sa = fin_sat(pa + sa); } }
			const int bound = min(fin_sat(xin + sa), sb);
			int run = 0;
			if (qual) { // equal bases the gap may move over (align.c:119-123)
				if (op == MM_CIGAR_INS) { for (; run < bound; ++run) if (A.q(qoff - 1 - run) != A.q(qoff + len - 1 - run)) break; }
				else { for (; run < bound; ++run) if (A.t(toff - 1 - run) != A.t(toff + len - 1 - run)) break; }
			}
			sa = qual? lprev : FIN_INF, sb = qual? run : 0;
			#pragma unroll
			for (int o = 2; o < 32; o <<= 1) { const int pa = __shfl_up_sync(full, sa, o), pb = __shfl_up_sync(full, sb, o); if (lane >= o) { const int nb = fin_sat(pb + sa); sb = nb < sb? nb : sb; sa = fin_sat(pa + sa); } }
			const int l = qual? min(fin_sat(xin + sa), sb) : 0;
			int l2 = __shfl_up_sync(full, l, 2), l1 = __shfl_up_sync(full, l, 1), ln1 = __shfl_down_sync(full, l, 1);
			if (lane < 2) l2 = xin;
			if (lane == 0) l1 = carry_l1;
			if (lane == 31) ln1 = 0; // the next chunk takes its first shift out of this chunk's last match itself
			if (valid && len + (op == MM_CIGAR_MATCH? l1 : 0) == 0) shrink = true; // empty when the reference's loop reaches it (align.c:115: a match the gap before it has just grown is not)
			if (qual && l == lprev + l2) shrink = true; // the match before the gap is used up (align.c:125)
			if (valid && op == MM_CIGAR_MATCH && (l1 | ln1)) c[k] = (uint32_t)(len + l1 - ln1) << 4;
			__syncwarp();
			if (lane == 0 && base > 0 && l > 0) c[base - 1] -= (uint32_t)l << 4;
			carry_q += __shfl_sync(full, iq, 31), carry_t += __shfl_sync(full, it, 31);
			carry_l0 = __shfl_sync(full, l, 30), carry_l1 = __shfl_sync(full, l, 31);
			carry_w = __shfl_sync(full, w, 31);
			__syncwarp();
		}
		if (carry_q != R.qspan || carry_t != R.tspan) status = 2; // the reference asserts this
		shrink = __any_sync(full, shrink), run_trigger = __any_sync(full, run_trigger);
		if (shrink || run_trigger) { // rare: the reference's own loops, sequentially
			if (lane == 0) {
				int to_shrink = shrink;
				if (run_trigger)
					for (uint32_t k = 0; k + 2 < nc; ++k) { // runs like 5I6D7I become one I and one D (align.c:134-155)
						if ((c[k] & 0xf) > 0 && (c[k] & 0xf) + (c[k + 1] & 0xf) == 3) {
							uint32_t l, s[3] = {0, 0, 0};
							for (l = k; l < nc; ++l) {
								const uint32_t op = c[l] & 0xf;
								if (op == MM_CIGAR_INS || op == MM_CIGAR_DEL || c[l] >> 4 == 0) s[op < 3? op : 0] += c[l] >> 4;
								else break;
							}
							if (s[1] > 0 && s[2] > 0 && l - k > 2) {
								c[k] = s[1] << 4 | MM_CIGAR_INS;
								c[k + 1] = s[2] << 4 | MM_CIGAR_DEL;
								for (k += 2; k < l; ++k) c[k] &= 0xf;
								to_shrink = 1;
							}
							k = l;
						}
					}
				if (to_shrink) { // drop empty operations, then merge equal neighbours (align.c:156-169)
					uint32_t l = 0;
					for (uint32_t k = 0; k < nc; ++k) if (c[k] >> 4 != 0) c[l++] = c[k];
					nc = l, l = 0;
					for (uint32_t k = 0; k < nc; ++k)
						if (k == nc - 1 || (c[k] & 0xf) != (c[k + 1] & 0xf)) c[l++] = c[k];
						else c[k + 1] += c[k] >> 4 << 4;
					nc = l;
				}
			}
			nc = __shfl_sync(full, nc, 0);
			__syncwarp();
		}
		const uint32_t w0 = c[0];
		if ((w0 & 0xf) == MM_CIGAR_INS || (w0 & 0xf) == MM_CIGAR_DEL) { // a leading I/D goes (align.c:170-180); the caller moves qs/qe or rs
			if ((w0 & 0xf) == MM_CIGAR_INS) qshift = (int)(w0 >> 4); else tshift = (int)(w0 >> 4);
			--nc;
			for (uint32_t base = 0; base < nc; base += 32) {
				const uint32_t k = base + lane;
				const uint32_t v = k < nc? c[k + 1] : 0u;
				__syncwarp();
				if (k < nc) c[k] = v;
			}
			__syncwarp();
		}
	}
	// ---- stage 3: mm_update_extra (align.c:266-297) in 2^-32 fixed point, one operation per lane ----
	long long s_run = 0, m_run = 0;
	int blen = 0, mlen = 0, n_ambi = 0, spliced = 0, carry_q = 0, carry_t = 0;
	for (uint32_t base = 0; base < nc; base += 32) {
		const uint32_t k = base + lane;
		const bool valid = k < nc;
		const uint32_t w = valid? c[k] : 0u;
		const int op = (int)(w & 0xf), len = (int)(w >> 4);
		int dq = 0, dt = 0;
		if (valid) { if (op == MM_CIGAR_MATCH) dq = dt = len; else if (op == MM_CIGAR_INS) dq = len; else if (op == MM_CIGAR_DEL || op == MM_CIGAR_N_SKIP) dt = len; }
		int iq = dq, it = dt;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const int yq = __shfl_up_sync(full, iq, o), yt = __shfl_up_sync(full, it, o); if (lane >= o) iq += yq, it += yt; }
		const int qoff = qshift + carry_q + iq - dq, toff = tshift + carry_t + it - dt;
		Walk wk; wk.T = wk.C = wk.Mx = wk.Cm = 0;
		if (valid && op == MM_CIGAR_MATCH) {
			int amb = 0, diff = 0;
			for (int i = 0; i < len; ++i) {
				const int cq = A.q(qoff + i), ct = A.t(toff + i);
				if (ct > 3 || cq > 3) ++amb;
				else if (ct != cq) ++diff;
				walk_step(wk, (long long)par.mat[ct * 5 + cq] << 32);
			}
			blen += len - amb, mlen += len - (amb + diff), n_ambi += amb;
		} else if (valid && (op == MM_CIGAR_INS || op == MM_CIGAR_DEL)) {
			int amb = 0;
			if (op == MM_CIGAR_INS) { for (int i = 0; i < len; ++i) if (A.q(qoff + i) > 3) ++amb; }
			else { for (int i = 0; i < len; ++i) if (A.t(toff + i) > 3) ++amb; }
			blen += len - amb, n_ambi += amb;
			const double pen = par.log_gap? par.q + (double)par.e * mmx_log2((float)(1.0 + len)) : (double)(par.q + par.e);
			walk_step(wk, -(long long)(pen * 4294967296.0));
		} else if (valid && op == MM_CIGAR_N_SKIP) spliced = 1;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { // ordered reduction: lane 0 ends with the chunk's stretch
			Walk ot; ot.T = shfl_down_ll(wk.T, o), ot.C = shfl_down_ll(wk.C, o), ot.Mx = shfl_down_ll(wk.Mx, o), ot.Cm = shfl_down_ll(wk.Cm, o);
			if ((lane & (2 * o - 1)) == 0) wk = walk_join(wk, ot);
		}
		if (lane == 0) {
			long long mm = s_run + wk.Mx > wk.Cm? s_run + wk.Mx : wk.Cm;
			m_run = m_run > mm? m_run : mm;
			s_run = s_run + wk.T > wk.C? s_run + wk.T : wk.C;
		}
		carry_q += __shfl_sync(full, iq, 31), carry_t += __shfl_sync(full, it, 31);
	}
	#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		blen += __shfl_xor_sync(full, blen, o), mlen += __shfl_xor_sync(full, mlen, o), n_ambi += __shfl_xor_sync(full, n_ambi, o);
		spliced |= __shfl_xor_sync(full, spliced, o);
	}
	if (nc > 0 && (carry_q + qshift != R.qspan || carry_t + tshift != R.tspan)) status = 2;
	if (lane == 0) {
		FinOut o;
		o.n_cigar = (int32_t)nc, o.blen = blen, o.mlen = mlen, o.n_ambi = n_ambi, o.qshift = qshift, o.tshift = tshift, o.status = status, o.is_spliced = spliced;
		o.dp_max = (int32_t)((double)m_run / 4294967296.0 + .499);
		o.pad[0] = o.pad[1] = o.pad[2] = 0;
		res[r] = o;
	}
}

} // namespace

void mmb_finalize_device(mmb_ctx_t *ctx, const FinReg *d_regs, const FinJobRef *d_jobs, int n_regs, const uint8_t *d_query, const uint32_t *d_S,
						 uint32_t *d_out, FinOut *d_res, const FinPar &par)
{
	if (n_regs <= 0) return;
	ProfScope ps(ctx, MMB_PROF_OTHER, (uint64_t)n_regs);
	finalize_kernel<<<(n_regs + 3) / 4, 128, 0, ctx->stream>>>(d_regs, d_jobs, n_regs, d_query, d_S, d_out, d_res, par);
	MMB_CUDA_CHECK(cudaGetLastError());
	++ctx->n_launch;
}

// Kernel-level entry with host buffers (parity tests): see include/mm_b200.h
extern "C" int mmb_tail_batch_host(mmb_ctx_t *ctx, int n_hits, const mmb_tail_hit_t *hits, int64_t n_pieces_total, const uint32_t *piece_len, const uint32_t *ops,
								   const uint8_t *query, int64_t query_len, const uint8_t *target, int64_t target_len, const int8_t *mat, int q, int e,
								   const int64_t *cig_off, mmb_tail_out_t *out, uint32_t *cigar_out)
{
	static_assert(sizeof(mmb_tail_out_t) == sizeof(FinOut), "mmb_tail_out_t mirrors FinOut");
	if (n_hits <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	std::vector<int64_t> poff((size_t)n_pieces_total + 1, 0);
	for (int64_t i = 0; i < n_pieces_total; ++i) poff[i + 1] = poff[i] + piece_len[i];
	const int64_t n_ops = poff[n_pieces_total], tot_out = cig_off[n_hits];
	std::vector<uint32_t> S((size_t)(target_len + 7) / 8 + 1, 0);
	for (int64_t i = 0; i < target_len; ++i) S[i >> 3] |= (uint32_t)(target[i] & 0xf) << ((i & 7) << 2);
	uint8_t *d_q = ctx->d_a.as<uint8_t>((size_t)query_len + 16);
	uint32_t *d_S = ctx->d_b.as<uint32_t>(S.size());
	uint32_t *d_ops = ctx->d_c.as<uint32_t>((size_t)n_ops + 1);
	FinReg *d_regs = ctx->d_d.as<FinReg>((size_t)n_hits);
	FinJobRef *d_jobs = ctx->d_e.as<FinJobRef>((size_t)n_pieces_total + 1);
	uint32_t *d_out = ctx->d_f.as<uint32_t>((size_t)tot_out + 1);
	FinOut *d_res = ctx->d_g.as<FinOut>((size_t)n_hits);
	std::vector<FinReg> hr((size_t)n_hits);
	std::vector<FinJobRef> hj((size_t)n_pieces_total + 1);
	for (int64_t i = 0; i < n_pieces_total; ++i) hj[i].cig = d_ops + poff[i], hj[i].n = piece_len[i], hj[i].pad = 0;
	for (int i = 0; i < n_hits; ++i) {
		FinReg &f = hr[i];
		f.q0 = hits[i].q0, f.t0 = hits[i].t0, f.out_off = cig_off[i], f.qlen = hits[i].qlen, f.qs = hits[i].qs, f.rev = hits[i].rev;
		f.qspan = hits[i].qspan, f.tspan = hits[i].tspan, f.job_first = hits[i].piece_first, f.n_jobs = hits[i].n_pieces, f.pad = 0;
	}
	FinPar par;
	for (int i = 0; i < 25; ++i) par.mat[i] = mat[i];
	par.q = (int8_t)q, par.e = (int8_t)e, par.log_gap = 1;
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_q, query, query_len, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_S, S.data(), S.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
	if (n_ops) MMB_CUDA_CHECK(cudaMemcpyAsync(d_ops, ops, (size_t)n_ops * 4, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_regs, hr.data(), sizeof(FinReg) * (size_t)n_hits, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_jobs, hj.data(), sizeof(FinJobRef) * (size_t)n_pieces_total, cudaMemcpyHostToDevice, ctx->stream));
	mmb_finalize_device(ctx, d_regs, d_jobs, n_hits, d_q, d_S, d_out, d_res, par);
	MMB_CUDA_CHECK(cudaMemcpyAsync(out, d_res, sizeof(FinOut) * (size_t)n_hits, cudaMemcpyDeviceToHost, ctx->stream));
	if (tot_out) MMB_CUDA_CHECK(cudaMemcpyAsync(cigar_out, d_out, (size_t)tot_out * 4, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return 0;
}
