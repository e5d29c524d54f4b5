// minimap2_b200/csrc/seed.cu
//
// K2a/K2b: seeds -> anchors on sm_90a. Replaces mm_seed_mz_flt (reference seed.c:5-28), mm_collect_matches /
// mm_seed_collect_all / mm_seed_select (seed.c:30-132), mm_idx_get on the device index (index.c:93-110),
// collect_seed_hits (map.c:168-204) and its radix_sort_128x (ksort.h:98-151, exact tie order).
//
// Stage kernels over a whole read batch (SoA arrays in HBM, per-read slices given by offset arrays):
//   mzflt_smem_kernel  1 CTA / read         query-side high-multiplicity minimizer filter (shared-memory hash; mzflt_kernel for >2048)
//   lookup_kernel      1 thread / minimizer hash-table probe: one 16 B slot load per probe (random HBM sector access)
//   select_kernel      1 warp / read        tandem flags, high-occurrence streak selection (<=128-entry heap, lane 0), rep_len,
//                                           mini_pos, per-seed anchor offsets
//   skip_count/offsets 1 thread / seed,read skip_seed (map.c:78-100) survivors per seed; only for ava / strand-restricted modes
//   expand_kernel      1 thread / seed      occurrence list -> anchors (strand-normalised coordinates)
//   sort_radix_kernel  1 CTA / read         stable LSD radix sort in shared memory, tie detection (one launch per size class)
//   sort_block_kernel  1 CTA / read         bitonic sort of (x, index): the radix kernels' fallback for keys varying in > 33 bits
//   sort_exact_smem    1 warp / read        exact emulation of the reference's unstable in-place MSD radix sort for tie reads
//   sort_exact_kernel  1 thread / read      the same in global memory (mmx_rs_sort) for reads too large for sort_exact_smem
//   heap_merge_kernel  1 thread / read      heap mode (MM_F_HEAP_SORT) instead of the two above: replay of the reference's heap merge
//                                           (collect_seed_hits_heap) for the reads with equal keys and the oversize reads
#include "index.h"
#include "mm_algo.cuh"
#include "scan.cuh"
#include "pipeline.h"
#include <mutex>

namespace {

__device__ __forceinline__ int find_read(const int64_t *off, int n, int64_t t)
{
	int lo = 0, hi = n;
	while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (off[mid] <= t) lo = mid; else hi = mid; }
	return lo;
}

// heap-sort a uint64 array ascending (per-thread, in global scratch)
__device__ void heapsort_u64(uint64_t *a, int n)
{
	for (int start = (n >> 1) - 1; start >= 0; --start) {
		int i = start; uint64_t tmp = a[i];
		for (int k; (k = 2 * i + 1) < n; i = k) { if (k + 1 < n && a[k] < a[k + 1]) ++k; if (a[k] <= tmp) break; a[i] = a[k]; }
		a[i] = tmp;
	}
	for (int end = n - 1; end > 0; --end) {
		uint64_t tmp = a[end]; a[end] = a[0];
		int i = 0;
		for (int k; (k = 2 * i + 1) < end; i = k) { if (k + 1 < end && a[k] < a[k + 1]) ++k; if (a[k] <= tmp) break; a[i] = a[k]; }
		a[i] = tmp;
	}
}

#define MZFLT_SMEM_MAX 2048
#define MZFLT_SLOTS 4096

// mm_seed_mz_flt (seed.c:5-28) for reads with <= 2048 minimizers: one CTA per read counts the multiplicity of every
// minimizer value in a shared-memory hash table (the reference sorts a copy; only the counts matter), then drops the values
// occurring more than max(q_occ_max, n*q_occ_frac) times with an order-preserving compaction. Nearly always nothing is dropped.
__global__ void __launch_bounds__(128) mzflt_smem_kernel(SeedArgs A)
{
	extern __shared__ __align__(16) uint8_t mz_sm[];
	unsigned long long *hkey = (unsigned long long*)mz_sm;
	int *hcnt = (int*)(hkey + MZFLT_SLOTS);
	int *s_part = hcnt + MZFLT_SLOTS;
	int &s_drop = s_part[128];
	for (int rd = blockIdx.x; rd < A.n_reads; rd += gridDim.x) {
		const int64_t base = A.mz_off[rd];
		const int n = A.n_mz[rd];
		if (n <= A.q_occ_max || A.q_occ_frac <= 0.0f || A.q_occ_max <= 0 || n > MZFLT_SMEM_MAX) continue;
		m128 *mz = A.mz + base;
		for (int i = threadIdx.x; i < MZFLT_SLOTS; i += blockDim.x) hkey[i] = ~0ULL, hcnt[i] = 0;
		if (threadIdx.x == 0) s_drop = 0;
		__syncthreads();
		for (int i = threadIdx.x; i < n; i += blockDim.x) {
			const unsigned long long x = mz[i].x;
			unsigned h = (unsigned)((x * 0x9E3779B97F4A7C15ULL) >> 52) & (MZFLT_SLOTS - 1);
			for (;;) {
				const unsigned long long old = atomicCAS(&hkey[h], ~0ULL, x);
				if (old == ~0ULL || old == x) { atomicAdd(&hcnt[h], 1); break; }
				h = (h + 1) & (MZFLT_SLOTS - 1);
			}
		}
		__syncthreads();
		const float thres = (float)(uint64_t)n * A.q_occ_frac;
		// per-thread contiguous slices so that the compaction keeps the original order
		const int per = (n + blockDim.x - 1) / blockDim.x, b0 = threadIdx.x * per, b1 = min(n, b0 + per);
		int keep = 0;
		for (int i = b0; i < b1; ++i) {
			const unsigned long long x = mz[i].x;
			unsigned h = (unsigned)((x * 0x9E3779B97F4A7C15ULL) >> 52) & (MZFLT_SLOTS - 1);
			while (hkey[h] != x) h = (h + 1) & (MZFLT_SLOTS - 1);
			const int cnt = hcnt[h];
			const bool drop = (cnt > A.q_occ_max && (float)cnt > thres) || x == 0;
			if (drop) s_drop = 1; else ++keep;
		}
		s_part[threadIdx.x] = keep;
		__syncthreads();
		if (s_drop) { // rare: order-preserving squeeze (seed.c:24-27)
			int start = 0;
			for (int k = 0; k < (int)threadIdx.x; ++k) start += s_part[k];
			m128 loc[16]; // per <= 2048/128
			int m = 0;
			for (int i = b0; i < b1; ++i) {
				const unsigned long long x = mz[i].x;
				unsigned h = (unsigned)((x * 0x9E3779B97F4A7C15ULL) >> 52) & (MZFLT_SLOTS - 1);
				while (hkey[h] != x) h = (h + 1) & (MZFLT_SLOTS - 1);
				const int cnt = hcnt[h];
				if (!((cnt > A.q_occ_max && (float)cnt > thres) || x == 0)) loc[m++] = mz[i];
			}
			__syncthreads();
			for (int k = 0; k < m; ++k) mz[start + k] = loc[k];
			if (threadIdx.x == blockDim.x - 1) A.n_mz[rd] = start + m;
		}
		__syncthreads();
	}
}

__global__ void __launch_bounds__(128) mzflt_kernel(SeedArgs A) // seed.c:5-28 (reads with more than 2048 minimizers)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= A.n_reads) return;
	const int64_t base = A.mz_off[rd];
	const int n = A.n_mz[rd];
	if (n <= A.q_occ_max || A.q_occ_frac <= 0.0f || A.q_occ_max <= 0) return;
	if (n <= MZFLT_SMEM_MAX) return; // handled by mzflt_smem_kernel
	m128 *mz = A.mz + base;
	uint64_t *tmp = A.mini_pos + base; // free at this point
	for (int i = 0; i < n; ++i) tmp[i] = mz[i].x;
	heapsort_u64(tmp, n);
	const float thres = (float)(uint64_t)n * A.q_occ_frac;
	int k = 0;
	for (int i = 0; i < n; ++i) {
		const uint64_t x = mz[i].x;
		int lo = 0, hi = n; // lower bound
		while (lo < hi) { int mid = (lo + hi) >> 1; if (tmp[mid] < x) lo = mid + 1; else hi = mid; }
		int lo2 = lo, hi2 = n; // upper bound
		while (lo2 < hi2) { int mid = (lo2 + hi2) >> 1; if (tmp[mid] <= x) lo2 = mid + 1; else hi2 = mid; }
		const int cnt = lo2 - lo;
		const bool drop = cnt > A.q_occ_max && (float)cnt > thres;
		// the reference zeroes x of dropped minimizers and then squeezes out x==0 entries (which also drops a genuine x==0)
		if (!drop && x != 0) { if (k != i) mz[k] = mz[i]; ++k; }
	}
	A.n_mz[rd] = k;
}

__global__ void __launch_bounds__(256) lookup_kernel(SeedArgs A, int64_t total)
{
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total) return;
	const int rd = find_read(A.mz_off, A.n_reads, t);
	if (t - A.mz_off[rd] >= A.n_mz[rd]) return;
	uint64_t off;
	const uint32_t n = idx_get_dev(A.ix, A.mz[t].x >> 8, &off);
	A.s_n[t] = n, A.s_off[t] = off;
}

__device__ __forceinline__ void heap_down(uint64_t *b, int i, int n) // max-heap sift-down (ksort.h:44-56 semantics)
{
	uint64_t tmp = b[i];
	int k = i;
	while ((k = (k << 1) + 1) < n) {
		if (k != n - 1 && b[k] < b[k + 1]) ++k;
		if (b[k] < tmp) break;
		b[i] = b[k]; i = k;
	}
	b[i] = tmp;
}

#define SEL_CAP 2048
// Where select_read finds a read's seeds (its minimizers with hits, in query order) and keeps their flags. A read with at most SEL_CAP
// minimizers gets compact copies in shared memory (occurrence count, query position, span, flag: 10 B per seed); a longer one reads
// through the seed list k_idx into s_n and mz, with the flags in A.flt.
struct SelSmem {
	uint32_t *sn_, *qp_; uint8_t *sp_, *fl_;
	__device__ void put(int k, uint32_t cnt, uint64_t x, uint64_t y) const { sn_[k] = cnt, qp_[k] = (uint32_t)y, sp_[k] = (uint8_t)(x & 0xff), fl_[k] = 0; }
	__device__ uint32_t sn(int j) const { return sn_[j]; }
	__device__ uint32_t qpos(int j) const { return qp_[j]; }
	__device__ uint32_t span(int j) const { return sp_[j]; }
	__device__ uint8_t &fl(int j) const { return fl_[j]; }
};
struct SelGlobal {
	const m128 *mz; const uint32_t *s_n, *kidx; uint8_t *flt;
	__device__ void put(int k, uint32_t, uint64_t, uint64_t) const { flt[k] = 0; }
	__device__ uint32_t sn(int j) const { return s_n[kidx[j] & 0x7fffffffu]; }
	__device__ uint32_t qpos(int j) const { return (uint32_t)mz[kidx[j] & 0x7fffffffu].y; }
	__device__ uint32_t span(int j) const { return (uint32_t)(mz[kidx[j] & 0x7fffffffu].x & 0xff); }
	__device__ uint8_t &fl(int j) const { return flt[j]; }
};

// mm_collect_matches (seed.c:98-132) for read rd, one warp: the lookups that hit are compacted by ballots into the seed list k_idx
// (minimizer index | tandem << 31) and the working set W, the high-occurrence streak selection (seed.c:56-96, a sequential scan with a
// 128-entry heap) runs on lane 0, and the final pass (rep_len, anchor offsets by a warp scan, mini_pos, compaction of the kept seeds)
// is lane-parallel again.
template<class Work>
__device__ __forceinline__ void select_read(const SeedArgs &A, int rd, const Work &W)
{
	const int lane = threadIdx.x & 31;
	const unsigned full = 0xffffffffu, lt = (1u << lane) - 1;
	const int64_t base = A.mz_off[rd];
	const int n = A.n_mz[rd], qlen = A.qlen[rd];
	const m128 *mz = A.mz + base;
	const uint32_t *s_n = A.s_n + base;
	uint32_t *kidx = A.k_idx + base;
	// mm_seed_collect_all (seed.c:30-52)
	int n_m0 = 0;
	for (int i0 = 0; i0 < n; i0 += 32) {
		const int i = i0 + lane;
		uint32_t cnt = 0, tandem = 0; uint64_t x = 0, y = 0;
		if (i < n) {
			cnt = s_n[i], x = mz[i].x, y = mz[i].y;
			if (i > 0 && x >> 8 == mz[i - 1].x >> 8) tandem = 1;
			if (i < n - 1 && x >> 8 == mz[i + 1].x >> 8) tandem = 1;
		}
		const bool keep = cnt > 0;
		const unsigned m = __ballot_sync(full, keep);
		if (keep) {
			const int k = n_m0 + __popc(m & lt);
			kidx[k] = (uint32_t)i | tandem << 31;
			W.put(k, cnt, x, y);
		}
		n_m0 += __popc(m);
	}
	__syncwarp();
	const int max_occ = A.max_occ, max_max_occ = A.max_max_occ, dist = A.occ_dist;
	if (dist > 0 && max_max_occ > max_occ) { // mm_seed_select (seed.c:56-96)
		bool any = false;
		for (int j = lane; j < n_m0; j += 32) any = any || (int)W.sn(j) > max_occ;
		if (n_m0 > 1 && __any_sync(full, any)) {
			if (lane == 0) {
				uint64_t b[128];
				for (int i = 0, last0 = -1; i <= n_m0; ++i) {
					if (i == n_m0 || (int)W.sn(i) <= max_occ) {
						if (i - last0 > 1) {
							const int ps = last0 < 0? 0 : (int)(W.qpos(last0) >> 1);
							const int pe = i == n_m0? qlen : (int)(W.qpos(i) >> 1);
							const int st = last0 + 1, en = i;
							int max_high_occ = (int)((double)(pe - ps) / dist + .499);
							if (max_high_occ > 0) {
								if (max_high_occ > 128) max_high_occ = 128;
								int j, k;
								for (j = st, k = 0; j < en && k < max_high_occ; ++j, ++k) b[k] = (uint64_t)W.sn(j) << 32 | (uint32_t)j;
								for (int h = (k >> 1) - 1; h >= 0; --h) heap_down(b, h, k);
								for (; j < en; ++j) {
									const uint32_t c = W.sn(j);
									if ((int32_t)c < (int32_t)(b[0] >> 32)) { b[0] = (uint64_t)c << 32 | (uint32_t)j; heap_down(b, 0, k); }
								}
								for (j = 0; j < k; ++j) W.fl((uint32_t)b[j]) = 1;
							}
							for (int j = st; j < en; ++j) W.fl(j) ^= 1;
							for (int j = st; j < en; ++j) if ((int)W.sn(j) > max_max_occ) W.fl(j) = 1;
						}
						last0 = i;
					}
				}
			}
			__syncwarp();
		}
	} else {
		for (int j = lane; j < n_m0; j += 32) if ((int)W.sn(j) > max_occ) W.fl(j) = 1;
		__syncwarp();
	}
	// seed.c:113-130
	int rep_st = 0, rep_en = 0, rep_len = 0, n_keep = 0; // rep_*: lane 0 only
	int64_t n_a = 0;
	uint64_t *mini_pos = A.mini_pos + base;
	uint32_t *k_aoff = A.k_aoff + base;
	for (int j0 = 0; j0 < n_m0; j0 += 32) {
		const int j = j0 + lane;
		const bool valid = j < n_m0, f = valid && W.fl(j), kept = valid && !f;
		const unsigned mf = __ballot_sync(full, f), mk = __ballot_sync(full, kept);
		if (lane == 0) // masked stretches merge in query order
			for (unsigned mm = mf; mm; mm &= mm - 1) {
				const int jj = j0 + __ffs(mm) - 1;
				const int en = (int)(W.qpos(jj) >> 1) + 1, st = en - (int)W.span(jj);
				if (st > rep_en) { rep_len += rep_en - rep_st; rep_st = st, rep_en = en; }
				else rep_en = en;
			}
		uint32_t e = 0, inc = 0; uint64_t mp = 0;
		if (kept) e = kidx[j], inc = W.sn(j), mp = (uint64_t)W.span(j) << 32 | W.qpos(j) >> 1;
		const uint32_t mine = inc;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t yv = __shfl_up_sync(full, inc, o); if (lane >= o) inc += yv; }
		__syncwarp(); // every lane has read its seed (k_idx[j] and what it indexes) and lane 0 its masked stretches before the compaction overwrites slots <= j
		if (kept) {
			const int dst = n_keep + __popc(mk & lt);
			k_aoff[dst] = (uint32_t)(n_a + (inc - mine));
			mini_pos[dst] = mp;
			kidx[dst] = e;
		}
		n_keep += __popc(mk);
		n_a += __shfl_sync(full, inc, 31);
	}
	if (lane == 0) {
		rep_len += rep_en - rep_st;
		A.n_keep[rd] = n_keep, A.rep_len[rd] = rep_len, A.n_a[rd] = n_a;
	}
}

__global__ void __launch_bounds__(128, 2) select_kernel(SeedArgs A) // one warp per read; 80 KB of shared memory per CTA: two CTAs per SM
{
	extern __shared__ __align__(16) uint8_t sel_sm[];
	const int rd = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	if (rd >= A.n_reads) return;
	const int64_t base = A.mz_off[rd];
	if (A.n_mz[rd] <= SEL_CAP) {
		uint32_t *sn = (uint32_t*)(sel_sm + (size_t)(threadIdx.x >> 5) * SEL_CAP * 10), *qp = sn + SEL_CAP;
		uint8_t *sp = (uint8_t*)(qp + SEL_CAP);
		select_read(A, rd, SelSmem{sn, qp, sp, sp + SEL_CAP});
	} else select_read(A, rd, SelGlobal{A.mz + base, A.s_n + base, A.k_idx + base, A.flt + base});
}

#define MMB_SKIP_FLAGS (MM_F_NO_DIAG | MM_F_NO_DUAL | MM_F_FOR_ONLY | MM_F_REV_ONLY)

// skip_seed (map.c:78-100). strcmp(qname, name[rid]) is evaluated on name ranks: >0 below q_name_lo, 0 inside [lo,hi), <0 above.
__device__ __forceinline__ bool skip_seed_dev(const SeedArgs &A, int rd, uint64_t r, uint32_t q_pos, int qlen, bool *is_self)
{
	*is_self = false;
	if (A.name_rank && (A.flag & (MM_F_NO_DIAG | MM_F_NO_DUAL))) {
		const uint32_t rid = (uint32_t)(r >> 32), rk = A.name_rank[rid];
		const int cmp = rk < A.q_name_lo[rd]? 1 : rk < A.q_name_hi[rd]? 0 : -1;
		if ((A.flag & MM_F_NO_DIAG) && cmp == 0 && (int)A.ix.seq_len[rid] == qlen) {
			if ((uint32_t)r >> 1 == (q_pos >> 1)) return true;      // the diagonal itself
			if ((r & 1) == (q_pos & 1)) *is_self = true;
		}
		if ((A.flag & MM_F_NO_DUAL) && cmp > 0) return true;        // all-vs-all: map each pair once
	}
	if (A.flag & (MM_F_FOR_ONLY | MM_F_REV_ONLY)) {
		if ((r & 1) == (q_pos & 1)) { if (A.flag & MM_F_REV_ONLY) return true; }
		else if (A.flag & MM_F_FOR_ONLY) return true;
	}
	return false;
}

// With skip_seed active the anchor count of a seed is no longer its occurrence count: count the survivors per kept seed,
// then rebuild the per-read offsets (the reference simply appends the survivors, map.c:181-199).
__global__ void __launch_bounds__(256) skip_count_kernel(SeedArgs A, int64_t total)
{
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total) return;
	const int rd = find_read(A.mz_off, A.n_reads, t);
	const int64_t base = A.mz_off[rd];
	if ((int)(t - base) >= A.n_keep[rd]) return;
	const uint32_t mi = A.k_idx[t] & 0x7fffffffu;
	const uint32_t q_pos = (uint32_t)A.mz[base + mi].y, n = A.s_n[base + mi];
	const uint64_t *cr = A.ix.pos + A.s_off[base + mi];
	const int qlen = A.qlen[rd];
	uint32_t c = 0;
	for (uint32_t j = 0; j < n; ++j) { bool self; if (!skip_seed_dev(A, rd, cr[j], q_pos, qlen, &self)) ++c; }
	A.k_cnt[t] = c;
}

__global__ void __launch_bounds__(128) skip_offsets_kernel(SeedArgs A)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= A.n_reads) return;
	const int64_t base = A.mz_off[rd];
	const int n_keep = A.n_keep[rd];
	int64_t run = 0;
	for (int k = 0; k < n_keep; ++k) { A.k_aoff[base + k] = (uint32_t)run; run += A.k_cnt[base + k]; }
	A.n_a[rd] = run;
}

// One anchor of occurrence r of seed q (query minimizer q, seed-list word e: tandem flag in bit 31), as collect_seed_hits writes it
// (map.c:182-197). qstrand selects the query-strand formula for reverse hits; the heap merge never uses it (map.c:134-136).
__device__ __forceinline__ m128 make_anchor(const SeedArgs &A, uint64_t r, m128 q, uint32_t e, bool is_self, int qlen, bool qstrand)
{
	const uint32_t q_pos = (uint32_t)q.y, q_span = (uint32_t)(q.x & 0xff), seg_id = (uint32_t)(q.y >> 32);
	const int32_t rpos = (int32_t)((uint32_t)r >> 1);
	m128 p;
	if ((r & 1) == (q_pos & 1)) {
		p.x = (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
		p.y = (uint64_t)q_span << 32 | q_pos >> 1;
	} else if (!qstrand) {
		p.x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
		p.y = (uint64_t)q_span << 32 | (uint32_t)(qlen - ((int32_t)(q_pos >> 1) + 1 - (int32_t)q_span) - 1);
	} else {
		const int32_t len = (int32_t)A.ix.seq_len[r >> 32];
		p.x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)(len - (rpos + 1 - (int32_t)q_span) - 1);
		p.y = (uint64_t)q_span << 32 | q_pos >> 1;
	}
	p.y |= (uint64_t)seg_id << MMX_SEED_SEG_SHIFT;
	if (e >> 31) p.y |= MMX_SEED_TANDEM;
	if (is_self) p.y |= MMX_SEED_SELF;
	return p;
}

__global__ void __launch_bounds__(256) expand_kernel(SeedArgs A, int64_t total) // map.c:176-199
{
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= total) return;
	const int rd = find_read(A.mz_off, A.n_reads, t);
	const int64_t base = A.mz_off[rd];
	const int k = (int)(t - base);
	if (k >= A.n_keep[rd]) return;
	const uint32_t e = A.k_idx[t], mi = e & 0x7fffffffu;
	const m128 q = A.mz[base + mi];
	const uint32_t q_pos = (uint32_t)q.y;
	const uint32_t n = A.s_n[base + mi];
	const uint64_t *cr = A.ix.pos + A.s_off[base + mi];
	m128 *a = A.a + A.a_off[rd] + A.k_aoff[t];
	const int qlen = A.qlen[rd];
	// heap mode writes reverse hits with the plain formula even in query-strand mode, so the sort below sees the heap merge's keys
	const bool qstrand = (A.flag & MM_F_QSTRAND) && !(A.flag & MM_F_HEAP_SORT), filtered = (A.flag & MMB_SKIP_FLAGS) != 0;
	uint32_t w = 0;
	for (uint32_t j = 0; j < n; ++j) {
		const uint64_t r = cr[j];
		bool is_self = false;
		if (filtered && skip_seed_dev(A, rd, r, q_pos, qlen, &is_self)) continue;
		a[w++] = make_anchor(A, r, q, e, is_self, qlen, qstrand);
	}
}

// ---------------------------------------------------------------------------------------------------------
// Anchor sort (radix_sort_128x of map.c:202). The reference's sort is unstable, but its output is fully determined
// when all keys are distinct, and for n <= 64 it is a stable insertion sort (ksort.h:147-151). So:
//   * sort_block_kernel: one CTA per read, bitonic sort of (x, original index) in shared memory -- the stable order;
//     equal neighbouring keys are detected on the fly;
//   * reads with n > 64 that do contain equal keys (two query minimizers on the same reference position: repeats), or
//     that do not fit the largest shared-memory class, are re-sorted by sort_exact_kernel, the step-by-step emulation of
//     the reference's in-place MSD radix sort (one thread per read).
// ---------------------------------------------------------------------------------------------------------
__global__ void sort_classify_kernel(const int64_t *a_off, int n_reads, int *cls_cnt, int *cls_list, int n_cls, int cap0)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= n_reads) return;
	const int64_t n = a_off[rd + 1] - a_off[rd];
	if (n <= 0) return;
	int c = 0, cap = cap0;
	while (c < n_cls - 1 && n > cap) ++c, cap <<= 1;
	if (n > cap) c = n_cls; // too large for shared memory: exact kernel
	const int pos = atomicAdd(&cls_cnt[c], 1);
	cls_list[(size_t)c * n_reads + pos] = rd;
}

__global__ void sort_block_kernel(const m128 *a_in, m128 *a_out, const int64_t *a_off, const int *list, const int *cnt_ptr, int cap,
								  int *exact_cnt, int *exact_list, int tie_min_n)
{
	extern __shared__ __align__(16) uint8_t sm_raw[];
	uint64_t *key = (uint64_t*)sm_raw;
	uint16_t *idx = (uint16_t*)(key + cap);
	__shared__ int s_tie;
	const int n_list = *cnt_ptr;
	for (int li = blockIdx.x; li < n_list; li += gridDim.x) {
		const int rd = list[li];
		const int64_t off = a_off[rd];
		const int n = (int)(a_off[rd + 1] - off);
		int P = 1;
		while (P < n) P <<= 1;
		if (threadIdx.x == 0) s_tie = 0;
		for (int i = threadIdx.x; i < P; i += blockDim.x) {
			key[i] = i < n? a_in[off + i].x : ~0ULL;
			idx[i] = (uint16_t)i;
		}
		__syncthreads();
		for (int k = 2; k <= P; k <<= 1) {
			for (int j = k >> 1; j > 0; j >>= 1) {
				for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
					const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)); // index with bit j cleared
					const int l = i | j;
					const uint64_t ki = key[i], kl = key[l];
					const uint16_t ii = idx[i], il = idx[l];
					const bool gt = ki > kl || (ki == kl && ii > il);
					const bool up = (i & k) == 0;
					if (gt == up) { key[i] = kl, key[l] = ki; idx[i] = il, idx[l] = ii; }
				}
				__syncthreads();
			}
		}
		int tie = 0;
		for (int i = threadIdx.x; i < n; i += blockDim.x) {
			a_out[off + i] = a_in[off + idx[i]];
			if (i + 1 < n && key[i] == key[i + 1]) tie = 1;
		}
		if (tie) s_tie = 1;
		__syncthreads();
		if (threadIdx.x == 0 && s_tie && n > tie_min_n) exact_list[atomicAdd(exact_cnt, 1)] = rd;
		__syncthreads();
	}
}

// Stable LSD radix sort of one read's anchors by x in shared memory (replaces the O(n log^2 n) bitonic network above for every read
// whose keys differ in at most 33 bit positions -- all of them in practice: strand bit + contig bits + position bits).
//   * the bits in which the read's keys differ are found with one OR-reduction; the keys are squeezed to those bits (order-preserving:
//     all other bits agree), 32 of them in a 32-bit word plus, if there is a 33rd (the strand bit), one flag bit next to the index;
//   * 8-bit digits, least significant first: every warp owns a contiguous segment; __match_any_sync groups equal digits of 32
//     consecutive elements, the group's first lane bumps the warp's counter, so an element's rank inside its segment is known without
//     atomics and in input order (stability); one CTA-wide scan of the (digit, warp) counters turns them into scatter offsets;
//   * the flag bit is a last 1-bit pass.
// Equal keys end up adjacent in input order; reads that have any (and more than 64 anchors) are re-sorted by the exact emulation of the
// reference's unstable radix sort, as before.
template<int CAP, int NT>
__global__ void __launch_bounds__(NT, NT >= 1024? 1 : 1024 / NT) sort_radix_kernel(const m128 *a_in, m128 *a_out, const int64_t *a_off, const int *list, const int *cnt_ptr,
														int *exact_cnt, int *exact_list, int *fallback_cnt, int *fallback_list, int tie_min_n)
{
	constexpr int NW = NT / 32, ITER = CAP / NT, SEG = ITER * 32, RS = NW + 1, NH = 256 * RS, EPT = (NH + NT - 1) / NT;
	extern __shared__ __align__(16) uint8_t sm_raw[];
	uint32_t *kb0 = (uint32_t*)sm_raw, *kb1 = kb0 + CAP;
	uint16_t *ib0 = (uint16_t*)(kb1 + CAP), *ib1 = ib0 + CAP;
	uint16_t *hist = ib1 + CAP;
	__shared__ unsigned long long s_or;
	__shared__ int s_wsum[32];
	__shared__ int s_tie;
	const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
	const unsigned full = 0xffffffffu;
	const int n_list = *cnt_ptr;
	for (int li = blockIdx.x; li < n_list; li += gridDim.x) {
		const int rd = list[li];
		const int64_t off = a_off[rd];
		const int n = (int)(a_off[rd + 1] - off);
		// ---- stage the 64-bit keys (over both key buffers), find the varying bits ----
		uint64_t *X64 = (uint64_t*)kb0;
		if (tid == 0) s_or = 0, s_tie = 0;
		__syncthreads();
		const uint64_t x0 = a_in[off].x;
		uint64_t m = 0;
		for (int i = tid; i < n; i += NT) { const uint64_t x = a_in[off + i].x; X64[i] = x; m |= x ^ x0; }
		#pragma unroll
		for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(full, m, o);
		if (lane == 0 && m) atomicOr(&s_or, (unsigned long long)m);
		__syncthreads();
		const uint64_t M = s_or;
		const int nb = __popcll(M);
		if (nb > 33) { // cannot happen with < 2^32 distinct (contig, position) pairs per strand; kept exact by the network sort
			if (tid == 0) fallback_list[atomicAdd(fallback_cnt, 1)] = rd;
			__syncthreads();
			continue;
		}
		uint64_t xr[ITER];
		#pragma unroll
		for (int it = 0; it < ITER; ++it) { const int e = w * SEG + it * 32 + lane; xr[it] = e < n? X64[e] : 0; }
		__syncthreads();
		#pragma unroll
		for (int it = 0; it < ITER; ++it) {
			const int e = w * SEG + it * 32 + lane;
			if (e < n) { // squeeze the varying bits together, run by run (typically three runs: position, contig, strand)
				uint64_t mm = M, ck = 0; int sh = 0;
				while (mm) {
					const int st = __ffsll((long long)mm) - 1;
					const uint64_t r = mm >> st;
					const int len = r == ~0ULL? 64 : __ffsll((long long)~r) - 1;
					const uint64_t fm = len >= 64? ~0ULL : (1ULL << len) - 1;
					ck |= ((xr[it] >> st) & fm) << sh;
					sh += len;
					mm = len + st >= 64? 0 : mm & ~(fm << st);
				}
				kb0[e] = (uint32_t)ck;
				ib0[e] = (uint16_t)(e | (int)(ck >> 32 & 1) << 15);
			}
		}
		__syncthreads();
		uint32_t *kin = kb0, *kout = kb1;
		uint16_t *iin = ib0, *iout = ib1;
		const int n_pass = (min(nb, 32) + 7) / 8 + (nb > 32? 1 : 0);
		for (int pass = 0; pass < n_pass; ++pass) {
			const bool top = nb > 32 && pass == n_pass - 1;
			const int shift = pass * 8;
			for (int i = tid; i < NH; i += NT) hist[i] = 0;
			__syncthreads();
			int rank[ITER];
			#pragma unroll
			for (int it = 0; it < ITER; ++it) {
				const int e = w * SEG + it * 32 + lane;
				const bool valid = e < n;
				const unsigned d = !valid? (0x100u | (unsigned)lane) : top? (unsigned)(iin[e] >> 15) : (kin[e] >> shift & 0xffu);
				const unsigned peers = __match_any_sync(full, d);
				const unsigned lt = peers & ((1u << lane) - 1u);
				const int base = valid? hist[d * RS + w] : 0;
				rank[it] = base + __popc(lt);
				__syncwarp();
				if (valid && lt == 0) hist[d * RS + w] = (uint16_t)(base + __popc(peers));
				__syncwarp();
			}
			__syncthreads();
			{ // exclusive scan of the counters in (digit, warp) order
				int loc[EPT], sum = 0;
				#pragma unroll
				for (int k = 0; k < EPT; ++k) { const int i = tid * EPT + k; loc[k] = i < NH? hist[i] : 0; sum += loc[k]; }
				int x = sum;
				#pragma unroll
				for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(full, x, o); if (lane >= o) x += y; }
				if (lane == 31) s_wsum[w] = x;
				__syncthreads();
				if (w == 0) {
					int v = lane < NW? s_wsum[lane] : 0, z = v;
					#pragma unroll
					for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(full, z, o); if (lane >= o) z += y; }
					s_wsum[lane] = z - v;
				}
				__syncthreads();
				int run = s_wsum[w] + x - sum;
				#pragma unroll
				for (int k = 0; k < EPT; ++k) { const int i = tid * EPT + k; if (i < NH) hist[i] = (uint16_t)run; run += loc[k]; }
			}
			__syncthreads();
			#pragma unroll
			for (int it = 0; it < ITER; ++it) {
				const int e = w * SEG + it * 32 + lane;
				if (e < n) {
					const uint32_t k = kin[e]; const uint16_t ix = iin[e];
					const unsigned d = top? (unsigned)(ix >> 15) : (k >> shift & 0xffu);
					const int pos = hist[d * RS + w] + rank[it];
					kout[pos] = k, iout[pos] = ix;
				}
			}
			__syncthreads();
			{ uint32_t *t = kin; kin = kout; kout = t; uint16_t *u = iin; iin = iout; iout = u; }
		}
		int tie = 0;
		for (int i = tid; i < n; i += NT) {
			a_out[off + i] = a_in[off + (iin[i] & 0x3fff)];
			if (i + 1 < n && kin[i] == kin[i + 1] && (iin[i] >> 15) == (iin[i + 1] >> 15)) tie = 1;
		}
		if (tie) s_tie = 1;
		__syncthreads();
		if (tid == 0 && s_tie && n > tie_min_n) exact_list[atomicAdd(exact_cnt, 1)] = rd;
		__syncthreads();
	}
}

__global__ void __launch_bounds__(64) sort_exact_kernel(const m128 *a_in, m128 *a_out, const int64_t *a_off, const int *list, const int *cnt_ptr,
														int32_t *stk, const int64_t *stk_off)
{
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= *cnt_ptr) return;
	const int rd = list[t];
	const int64_t off = a_off[rd], n = a_off[rd + 1] - off;
	for (int64_t i = 0; i < n; ++i) a_out[off + i] = a_in[off + i];
	if (n > 1) mmx_rs_sort(a_out + off, n, stk + stk_off[rd], KeyX128());
}

// The reference's walk of one range over the buckets of one level (ksort.h:126-138): every word in pd is stamped with its digit
// (bits 16-23), head[b] and tail[b] bound bucket b. The cycle-leader permutation moves every word into its bucket; head ends equal to tail.
__device__ __forceinline__ void exact_permute(uint32_t *pd, uint16_t *head, const uint16_t *tail)
{
	for (int b = 0; b < 256;) {
		const uint32_t hb = head[b];
		if (hb != tail[b]) {
			const uint32_t w = pd[hb];
			uint32_t l = w >> 16;
			if (l != (uint32_t)b) {
				uint32_t tmp = w;
				do {
					const uint32_t sw = tmp, hl = head[l];
					tmp = pd[hl]; pd[hl] = sw; head[l] = (uint16_t)(hl + 1);
					l = tmp >> 16;
				} while (l != (uint32_t)b);
				pd[hb] = tmp;
			}
			head[b] = (uint16_t)(hb + 1);
		} else ++b;
	}
}

// What the reference does with one bucket [bb, be) after the walk (ksort.h:100-110): a range of more than 64 goes to the next level's
// task list, a smaller one is insertion-sorted on the full key.
__device__ __forceinline__ void exact_bucket(uint32_t *pd, const uint64_t *X, uint32_t bb, uint32_t be, uint32_t *nxt, int *n_next)
{
	if (be - bb > 64) nxt[atomicAdd(n_next, 1)] = bb | be << 16;
	else if (be - bb > 1) {
		for (uint32_t i = bb + 1; i < be; ++i) {
			const uint32_t wi = pd[i];
			const uint64_t ki = X[wi & 0xffffu];
			if (ki < X[pd[i - 1] & 0xffffu]) {
				uint32_t j;
				for (j = i; j > bb && ki < X[pd[j - 1] & 0xffffu]; --j) pd[j] = pd[j - 1];
				pd[j] = wi;
			}
		}
	}
}

// Exact emulation for the reads whose anchors contain equal keys. The American-flag walk of one bucket is sequential, but
// (1) buckets of one level are independent, so the 32 lanes of a warp each walk a different bucket, level by level;
// (2) the walk only needs an element's digit and identity, so it permutes 32-bit words (index | digit << 16) in shared
//     memory instead of 16-byte anchors, with the 64-bit keys kept in a read-only shared array;
// (3) a bucket whose elements all share the digit is left untouched by the reference's walk, so it is skipped.
// One warp (= one CTA) per read.
__global__ void __launch_bounds__(32) sort_exact_smem_kernel(const m128 *a_in, m128 *a_out, const int64_t *a_off, const int *list, const int *cnt_ptr,
															 int cap, int *over_cnt, int *over_list)
{
	extern __shared__ __align__(16) uint8_t sm_raw[];
	const int MAXT = 512;
	uint64_t *X = (uint64_t*)sm_raw;
	uint32_t *pd = (uint32_t*)(X + cap);
	uint16_t *head = (uint16_t*)(pd + cap) + (size_t)threadIdx.x * 512, *tail = head + 256;
	uint32_t *tasks0 = (uint32_t*)((uint16_t*)(pd + cap) + 32 * 512), *tasks1 = tasks0 + MAXT;
	__shared__ int s_next;
	const int lane = threadIdx.x;
	const int n_list = *cnt_ptr;
	for (int li = blockIdx.x; li < n_list; li += gridDim.x) {
		const int rd = list[li];
		const int64_t off = a_off[rd];
		const int n = (int)(a_off[rd + 1] - off);
		if (n > cap) { if (lane == 0) over_list[atomicAdd(over_cnt, 1)] = rd; continue; }
		uint64_t vary = 0; // bits in which the read's keys differ: a level whose byte of `vary` is zero leaves every range untouched
		{
			const uint64_t x0 = a_in[off].x;
			for (int i = lane; i < n; i += 32) { const uint64_t x = a_in[off + i].x; X[i] = x, pd[i] = (uint32_t)i; vary |= x ^ x0; }
			#pragma unroll
			for (int o = 16; o > 0; o >>= 1) vary |= __shfl_xor_sync(0xffffffffu, vary, o);
		}
		if (lane == 0) tasks0[0] = 0u | (uint32_t)n << 16, s_next = 0;
		__syncwarp();
		uint32_t *cur = tasks0, *nxt = tasks1;
		int n_task = 1;
		if (n <= 64) { // ksort.h:147: plain insertion sort
			if (lane == 0)
				for (int i = 1; i < n; ++i)
					if (X[pd[i]] < X[pd[i - 1]]) {
						const uint32_t tmp = pd[i]; int j;
						for (j = i; j > 0 && X[tmp] < X[pd[j - 1]]; --j) pd[j] = pd[j - 1];
						pd[j] = tmp;
					}
			n_task = 0;
		}
		for (int shift = 56; n_task > 0; shift = shift > 8? shift - 8 : 0) {
			if ((vary >> shift & 0xff) == 0) { // every key has the same digit here: the reference's pass counts, moves nothing and recurses on the same ranges
				if (shift == 0) break;
				continue;
			}
			// large ranges (the first levels: one or two ranges holding the whole read) are handled by the whole warp: digit stamping, counting
			// and the bucket post-processing run on all lanes, only the cycle-leader walk itself -- sequential by nature -- stays on lane 0
			for (int t = 0; t < n_task; ++t) {
				const int beg = cur[t] & 0xffff, end = cur[t] >> 16;
				if (end - beg < 1024) continue;
				uint16_t *h0 = head - (size_t)lane * 512, *t0 = h0 + 256; // lane 0's tables
				uint32_t *cnt = (uint32_t*)(h0 + 512 * 4); // lane 4's tables double as 256 32-bit counters (every lane rebuilds its tables before use)
				for (int b = lane; b < 256; b += 32) cnt[b] = 0;
				__syncwarp();
				for (int i = beg + lane; i < end; i += 32) {
					const uint32_t idx = pd[i] & 0xffffu, d = (uint32_t)(X[idx] >> shift) & 0xffu;
					pd[i] = idx | d << 16;
					atomicAdd(&cnt[d], 1u);
				}
				__syncwarp();
				uint32_t c8[8], sum = 0, mx = 0;
				#pragma unroll
				for (int k = 0; k < 8; ++k) { c8[k] = cnt[lane * 8 + k]; sum += c8[k]; mx = max(mx, c8[k]); }
				uint32_t inc = sum;
				#pragma unroll
				for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
				#pragma unroll
				for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
				__syncwarp();
				uint32_t run = (uint32_t)beg + inc - sum;
				#pragma unroll
				for (int k = 0; k < 8; ++k) { h0[lane * 8 + k] = (uint16_t)run; run += c8[k]; t0[lane * 8 + k] = (uint16_t)run; }
				__syncwarp();
				if (lane == 0 && mx != (uint32_t)(end - beg)) exact_permute(pd, h0, t0);
				__syncwarp();
				if (shift) for (int b = lane; b < 256; b += 32) exact_bucket(pd, X, b? t0[b - 1] : (uint32_t)beg, t0[b], nxt, &s_next);
				__syncwarp();
				if (lane == 0) cur[t] = 0; // done
				__syncwarp();
			}
			for (int t = lane; t < n_task; t += 32) {
				const int beg = cur[t] & 0xffff, end = cur[t] >> 16;
				if (end <= beg) continue;
				for (int b = 0; b < 256; b += 2) *(uint32_t*)(head + b) = 0;
				for (int i = beg; i < end; ++i) { // count, and stamp each word with its digit at this level
					const uint32_t idx = pd[i] & 0xffffu, d = (uint32_t)(X[idx] >> shift) & 0xffu;
					pd[i] = idx | d << 16;
					++head[d];
				}
				uint32_t run = (uint32_t)beg, mx = 0;
				for (int b = 0; b < 256; ++b) { const uint32_t c = head[b]; mx = max(mx, c); head[b] = (uint16_t)run; run += c; tail[b] = (uint16_t)run; }
				if (mx != (uint32_t)(end - beg)) exact_permute(pd, head, tail);
				if (shift) for (int b = 0; b < 256; ++b) exact_bucket(pd, X, b? tail[b - 1] : (uint32_t)beg, tail[b], nxt, &s_next);
			}
			__syncwarp();
			n_task = s_next;
			__syncwarp();
			if (lane == 0) s_next = 0;
			uint32_t *sw = cur; cur = nxt; nxt = sw;
			__syncwarp();
			if (shift == 0) break;
		}
		__syncwarp();
		for (int i = lane; i < n; i += 32) a_out[off + i] = a_in[off + (pd[i] & 0xffffu)];
		__syncwarp();
	}
}


// ---------------------------------------------------------------------------------------------------------
// Heap-ordered anchors (collect_seed_hits_heap, map.c:102-166; MM_F_HEAP_SORT). The reference merges the kept seeds' occurrence lists
// with a min-heap on the occurrence word r and writes forward hits in pop order, then reverse hits in pop order. Occurrence lists are
// ascending, so pops come in ascending r and both blocks are ascending in x: for a read whose anchors have distinct x this is the
// stable sort's order. Only the order of equal x depends on the heap's history (equal keys keep sifting down), so the reads with equal
// adjacent keys after the sort, and the oversize reads the sort kernels do not handle, are replayed here step by step.
// ---------------------------------------------------------------------------------------------------------
#define HEAP_SMEM 128 // heap entries per thread in shared memory; reads with more kept seeds keep their heap in global scratch

// ks_heapdown (ksort.h:44-56) with heap_lt(a, b) = a.x > b.x (map.c:74): the smaller child is taken, and the sift stops only below a
// strictly larger key -- equal keys keep sifting down
__device__ __forceinline__ void heap_sift_x(m128 *h, int i, int n)
{
	const m128 tmp = h[i];
	int k = i;
	while ((k = (k << 1) + 1) < n) {
		if (k != n - 1 && h[k].x > h[k + 1].x) ++k;
		if (h[k].x > tmp.x) break;
		h[i] = h[k]; i = k;
	}
	h[i] = tmp;
}

// The replay of one read into a_sorted; h holds n_keep entries {x = r, y = seed << 32 | occurrence}. Every occurrence takes its turn
// in the heap, also those skip_seed drops.
__device__ void heap_merge_read(const SeedArgs &A, int rd, m128 *h)
{
	const int64_t base = A.mz_off[rd], n = A.a_off[rd + 1] - A.a_off[rd];
	const int nk = A.n_keep[rd], qlen = A.qlen[rd];
	const uint32_t *kidx = A.k_idx + base;
	m128 *out = A.a_sorted + A.a_off[rd];
	const bool filtered = (A.flag & MMB_SKIP_FLAGS) != 0;
	for (int i = 0; i < nk; ++i) h[i].x = A.ix.pos[A.s_off[base + (kidx[i] & 0x7fffffffu)]], h[i].y = (uint64_t)i << 32;
	for (int i = (nk >> 1) - 1; i >= 0; --i) heap_sift_x(h, i, nk); // ks_heapmake
	int64_t n_for = 0, n_rev = 0;
	for (int hs = nk; hs > 0;) {
		const uint64_t r = h[0].x;
		const uint32_t e = kidx[h[0].y >> 32], mi = e & 0x7fffffffu, j = (uint32_t)h[0].y;
		const m128 q = A.mz[base + mi];
		bool is_self = false;
		if (!(filtered && skip_seed_dev(A, rd, r, (uint32_t)q.y, qlen, &is_self))) {
			const m128 p = make_anchor(A, r, q, e, is_self, qlen, false);
			if ((r & 1) == (q.y & 1)) out[n_for++] = p;
			else out[n - 1 - n_rev++] = p; // reverse hits from the back, in descending pop order
		}
		if (j + 1 < A.s_n[base + mi]) h[0].y += 1, h[0].x = A.ix.pos[A.s_off[base + mi] + j + 1];
		else h[0] = h[--hs];
		heap_sift_x(h, 0, hs);
	}
	for (int64_t k = 0; k < n_rev >> 1; ++k) { const m128 t = out[n_for + k]; out[n_for + k] = out[n - 1 - k]; out[n - 1 - k] = t; }
}

// One thread per read over two lists (the reads with equal keys, then the oversize reads); scratch: 16 B per minimizer of the batch
__global__ void __launch_bounds__(32) heap_merge_kernel(SeedArgs A, const int *list0, const int *cnt0, const int *list1, const int *cnt1, m128 *scratch)
{
	extern __shared__ __align__(16) uint8_t sm_raw[];
	m128 *mine = (m128*)sm_raw + (size_t)threadIdx.x * HEAP_SMEM;
	const int n0 = *cnt0, n_all = n0 + *cnt1;
	for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_all; t += gridDim.x * blockDim.x) {
		const int rd = t < n0? list0[t] : list1[t - n0];
		heap_merge_read(A, rd, A.n_keep[rd] <= HEAP_SMEM? mine : scratch + A.mz_off[rd]);
	}
}

} // namespace

// Runs mz-filter, lookup and selection; leaves A.n_a[] filled. Then the caller scans n_a into a_off, sizes the anchor
// buffer and calls mmb_seed_expand_sort.
void mmb_seed_select_device(mmb_ctx_t *ctx, SeedArgs &A, int64_t total_mz)
{
	if (A.n_reads <= 0) return;
	const int rb = (A.n_reads + 127) / 128;
	ProfScope prof(ctx, MMB_PROF_SEED, (uint64_t)total_mz);
	{
		const size_t smem = (size_t)MZFLT_SLOTS * 12 + 129 * 4 + 16;
		static std::once_flag once;
		std::call_once(once, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(mzflt_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); });
		mzflt_smem_kernel<<<ctx->n_sm * 4, 128, smem, ctx->stream>>>(A);
		++ctx->n_launch;
	}
	mzflt_kernel<<<rb, 128, 0, ctx->stream>>>(A);
	++ctx->n_launch;
	if (total_mz > 0) {
		lookup_kernel<<<(unsigned)((total_mz + 255) / 256), 256, 0, ctx->stream>>>(A, total_mz);
		++ctx->n_launch;
	}
	{
		const size_t smem = (size_t)SEL_CAP * 10 * 4;
		static std::once_flag once;
		std::call_once(once, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); });
		select_kernel<<<(unsigned)(((int64_t)A.n_reads * 32 + 127) / 128), 128, smem, ctx->stream>>>(A);
		++ctx->n_launch;
	}
	if ((A.flag & MMB_SKIP_FLAGS) && total_mz > 0) { // skip_seed changes the anchor counts (map.c:78-100)
		skip_count_kernel<<<(unsigned)((total_mz + 255) / 256), 256, 0, ctx->stream>>>(A, total_mz);
		skip_offsets_kernel<<<rb, 128, 0, ctx->stream>>>(A);
		ctx->n_launch += 2;
	}
	MMB_CUDA_CHECK(cudaGetLastError());
}

void mmb_seed_expand_sort_device(mmb_ctx_t *ctx, SeedArgs &A, int64_t total_mz, int64_t total_a, DevBuf &stkbuf)
{
	if (A.n_reads <= 0) return;
	{
		ProfScope prof(ctx, MMB_PROF_SEED, 0);
		if (total_mz > 0) {
			expand_kernel<<<(unsigned)((total_mz + 255) / 256), 256, 0, ctx->stream>>>(A, total_mz);
			++ctx->n_launch;
		}
	}
	// sort_exact_kernel's stacks, after the class counters and lists: 16 counters, then (N_CLS+3) lists of n_reads entries: classes,
	// oversize (index N_CLS), ties (N_CLS+1), fallback of the radix kernels (N_CLS+2)
	const int N_CLS = 5, CAP0 = 1024; // shared-memory classes: 1024, 2048, 4096, 8192, 16384 anchors
	// heap mode (MM_F_HEAP_SORT): the sort kernels list every read with equal keys, whatever its size, and those reads and the oversize
	// ones go to heap_merge_kernel instead of the exact emulation; its global-memory heaps (16 B per minimizer) follow the lists
	const bool heap = (A.flag & MM_F_HEAP_SORT) != 0;
	const size_t lists_bytes = ((size_t)A.n_reads * 8 + 64) * sizeof(int), heap_bytes = heap? (size_t)total_mz * sizeof(m128) + 16 : 0;
	int64_t *d_stk_off = mmb_sort_stacks_async(ctx, A.a_off, A.n_reads, total_a, stkbuf, lists_bytes + heap_bytes);
	int32_t *d_stk = mmb_sort_stacks(d_stk_off, A.n_reads);
	int *d_cls_cnt = (int*)stkbuf.p, *d_cls_list = d_cls_cnt + 16;
	const int tie_min_n = heap? 0 : 64; // the radix sort is the reference's order for n <= 64 (insertion sort), the heap merge's is not
	{
		ProfScope prof(ctx, MMB_PROF_SORT, (uint64_t)total_a);
		MMB_CUDA_CHECK(cudaMemsetAsync(d_cls_cnt, 0, 16 * sizeof(int), ctx->stream));
		sort_classify_kernel<<<(A.n_reads + 255) / 256, 256, 0, ctx->stream>>>(A.a_off, A.n_reads, d_cls_cnt, d_cls_list, N_CLS, CAP0);
		++ctx->n_launch;
		int *d_tie_cnt = d_cls_cnt + N_CLS + 1, *d_tie_list = d_cls_list + (size_t)(N_CLS + 1) * A.n_reads;
		int *d_fb_cnt = d_cls_cnt + N_CLS + 2, *d_fb_list = d_cls_list + (size_t)(N_CLS + 2) * A.n_reads;
		#define MMB_RADIX_LAUNCH(CAP_, NT_, c_) do { \
			const size_t smem_ = (size_t)(CAP_) * 12 + (size_t)256 * ((NT_) / 32 + 1) * 2; \
			{ static std::once_flag once_; std::call_once(once_, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(sort_radix_kernel<CAP_, NT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_)); }); } \
			int per_sm_ = 1; \
			MMB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_, sort_radix_kernel<CAP_, NT_>, NT_, smem_)); \
			sort_radix_kernel<CAP_, NT_><<<ctx->n_sm * (per_sm_ > 0? per_sm_ : 1), NT_, smem_, ctx->stream>>>(A.a, A.a_sorted, A.a_off, d_cls_list + (size_t)(c_) * A.n_reads, \
				d_cls_cnt + (c_), d_tie_cnt, d_tie_list, d_fb_cnt, d_fb_list, tie_min_n); \
			++ctx->n_launch; } while (0)
		MMB_RADIX_LAUNCH(1024, 128, 0);
		MMB_RADIX_LAUNCH(2048, 256, 1);
		MMB_RADIX_LAUNCH(4096, 512, 2);
		MMB_RADIX_LAUNCH(8192, 512, 3); // 16 elements per thread, 64 registers: two CTAs per SM instead of one 1024-thread CTA that owns the whole register file
		MMB_RADIX_LAUNCH(16384, 1024, 4);
		#undef MMB_RADIX_LAUNCH
		{ // network sort: the fallback of the radix kernels (keys differing in more than 33 bit positions), one launch sized for the largest class
			const int cap = CAP0 << (N_CLS - 1), threads = 1024;
			const size_t smem = (size_t)cap * 10;
			{ static std::once_flag once; std::call_once(once, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(sort_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024)); }); }
			int per_sm = 1;
			MMB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sort_block_kernel, threads, smem));
			const int grid = ctx->n_sm * (per_sm > 0? per_sm : 1);
			sort_block_kernel<<<grid, threads, smem, ctx->stream>>>(A.a, A.a_sorted, A.a_off, d_fb_list, d_fb_cnt, cap, d_tie_cnt, d_tie_list, tie_min_n);
			++ctx->n_launch;
		}
		if (heap) { // heap merge replay of the reads with equal keys and of the oversize reads
			const size_t smem = (size_t)32 * HEAP_SMEM * sizeof(m128);
			{ static std::once_flag once; std::call_once(once, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(heap_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); }); }
			m128 *scratch = (m128*)(((uintptr_t)stkbuf.p + lists_bytes + 15) & ~(uintptr_t)15);
			heap_merge_kernel<<<ctx->n_sm * 3, 32, smem, ctx->stream>>>(A, d_tie_list, d_tie_cnt, d_cls_list + (size_t)N_CLS * A.n_reads, d_cls_cnt + N_CLS, scratch);
			++ctx->n_launch;
		}
		// exact emulation: reads with equal keys go through the shared-memory walker (cap 15360 anchors: 12 B/entry + per-lane bucket tables);
		// whatever does not fit, and the oversize class, falls back to the global-memory walker (one thread per read)
		else {
			const int cap = 15360;
			const size_t smem = (size_t)cap * 12 + 32 * 512 * 2 + 2 * 512 * 4;
			{ static std::once_flag once; std::call_once(once, [&]() { MMB_CUDA_CHECK(cudaFuncSetAttribute(sort_exact_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ctx->smem_optin - 1024)); }); }
			sort_exact_smem_kernel<<<ctx->n_sm, 32, smem, ctx->stream>>>(A.a, A.a_sorted, A.a_off, d_cls_list + (size_t)(N_CLS + 1) * A.n_reads, d_cls_cnt + N_CLS + 1,
																		 cap, d_cls_cnt + N_CLS, d_cls_list + (size_t)N_CLS * A.n_reads);
			++ctx->n_launch;
			sort_exact_kernel<<<(A.n_reads + 63) / 64, 64, 0, ctx->stream>>>(A.a, A.a_sorted, A.a_off, d_cls_list + (size_t)N_CLS * A.n_reads, d_cls_cnt + N_CLS, d_stk, d_stk_off);
			++ctx->n_launch;
		}
		static const bool dbg = getenv("MM_B200_SORT_STATS") != nullptr;
		if (dbg) { // development aid: reads per class / oversize / with equal keys / fallback
			int h[16];
			MMB_CUDA_CHECK(cudaMemcpyAsync(h, d_cls_cnt, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
			MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
			fprintf(stderr, "[sort] reads=%d anchors=%lld classes=%d/%d/%d/%d/%d oversize=%d ties=%d fallback=%d\n", A.n_reads, (long long)total_a, h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7]);
		}
	}
	MMB_CUDA_CHECK(cudaGetLastError());
}
