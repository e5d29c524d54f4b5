// minimap2_b200/csrc/sketch.cu
//
// K1: symmetric (w,k)-minimizer sketch on sm_90a. Replaces mm_sketch (reference sketch.c:77-143).
//
// mm_sketch is a sequential state machine (ring of the last w slot values + current minimum + run length l).
// It is chunk-parallelised here: one thread owns the positions [cs, ce) of one sequence and replays the reference
// state machine from a warm-up point R0 = cs - WU with a cleared state. After the warm-up the state equals the
// sequential one provided (a) no ambiguous base lies in [R0, cs) and (b) at most 16 symmetric-k-mer skips occurred,
// because then the ring holds the true last w slot writes, the k-mer registers hold the true last k bases and the run
// length is saturated (>= w+k) in both runs, which is all the emission rules (sketch.c:117-139) look at. A chunk
// whose warm-up fails the check (N nearby, long ATAT.. stretch) or whose sequence uses HPC is replayed from the
// sequence start instead -- slower, still exact. Emissions are produced in position order per chunk, so a count pass,
// an exclusive scan and a write pass give exactly the reference's output order with no sort.
#include "mmb_internal.h"
#include "mm_algo.cuh"
#include "scan.cuh"

namespace {

struct SeqSrc {          // how bases are fetched: nt4/ASCII bytes, or the 4-bit packed index sequence
	const uint8_t *bytes;
	const uint32_t *packed;
	__device__ __forceinline__ int get(int64_t i) const {
		if (packed) return (int)mmx_seq4_get(packed, (uint64_t)i) > 3? 4 : (int)mmx_seq4_get(packed, (uint64_t)i);
		return mmx_nt4(bytes[i]);
	}
};

struct SketchArgs {
	SeqSrc src;
	const int64_t *seq_off;     // n_seq+1 base offsets of the sequences in src
	const int64_t *chunk_off;   // n_seq+1: first chunk id of each sequence
	const uint32_t *rid;        // optional per-sequence rid (NULL: rid0 + seq index)
	uint32_t rid0;
	int n_seq, w, k, is_hpc, chunk, same_rid;
	int64_t n_chunks;
	int64_t *cnt;               // per chunk count (pass 0) / exclusive offsets (pass 1 input)
	m128 *out;
};

// binary search: largest s with chunk_off[s] <= c
__device__ __forceinline__ int find_seq(const int64_t *chunk_off, int n_seq, int64_t c)
{
	int lo = 0, hi = n_seq;
	while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (chunk_off[mid] <= c) lo = mid; else hi = mid; }
	return lo;
}

#define MAXW 256

template<bool WRITE>
__global__ void __launch_bounds__(128) sketch_kernel(SketchArgs A)
{
	const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= A.n_chunks) return;
	const int s = find_seq(A.chunk_off, A.n_seq, c);
	const int64_t base = A.seq_off[s];
	const int len = (int)(A.seq_off[s + 1] - base);
	const int w = A.w, k = A.k;
	const uint32_t rid = A.rid? A.rid[s] : A.same_rid? A.rid0 : A.rid0 + (uint32_t)s;
	int cs, ce;
	if (A.is_hpc) { cs = 0, ce = len; }           // HPC: one chunk per sequence (positions jump over homopolymers)
	else { cs = (int)((c - A.chunk_off[s]) * A.chunk); ce = min(len, cs + A.chunk); }
	const uint64_t shift1 = 2 * (k - 1), mask = (1ULL << 2 * k) - 1;
	const uint64_t MAXV = ~0ULL;
	uint64_t bx[MAXW];      // ring: x values (hash<<8|span); y is rebuilt from (pos,strand) kept in bp
	uint32_t bp[MAXW];      // ring: pos<<1|strand, 0xffffffff for "no k-mer"
	int64_t n_out = 0;
	m128 *out = WRITE? A.out + A.cnt[c] : nullptr;

	const int WU = 2 * w + 2 * k + 15;
	int start = cs - WU;
	bool warm = start > 0 && !A.is_hpc;
	if (!warm) start = 0;

	for (int attempt = 0; attempt < 2; ++attempt) {
		uint64_t kmer0 = 0, kmer1 = 0, minx = MAXV;
		uint32_t minp = 0xffffffffu;
		int l = 0, buf_pos = 0, min_pos = 0, kmer_span = 0, nskip = 0, after = 0; // after: slot writes at positions >= ce
		int tq[32], tq_front = 0, tq_cnt = 0;
		bool bad = false, checked = false;
		n_out = 0;
		for (int j = 0; j < w; ++j) bx[j] = MAXV, bp[j] = 0xffffffffu;
#define EMIT(X, P) do { int pos__ = (int)((P) >> 1); if (pos__ >= cs && pos__ < ce) { \
			if (WRITE) { out[n_out].x = (X); out[n_out].y = (uint64_t)rid << 32 | (P); } ++n_out; } } while (0)
		int i;
		for (i = start; i < len; ++i) {
			if (warm && !checked && i >= cs) { // warm-up verdict: enough non-skipped k-mers => ring, k-mer registers and run length are exact
				checked = true;
				if (nskip > 16) { bad = true; break; }
				if (l < w + k) l = w + k; // the true run length is >= w+k here; every rule compares l with thresholds <= w+k
			}
			int cch = A.src.get(base + i);
			uint64_t ix = MAXV; uint32_t ip = 0xffffffffu;
			if (cch < 4) {
				if (A.is_hpc) { // sketch.c:94-104
					int skip_len = 1;
					if (i + 1 < len && A.src.get(base + i + 1) == cch) {
						for (skip_len = 2; i + skip_len < len; ++skip_len)
							if (A.src.get(base + i + skip_len) != cch) break;
						i += skip_len - 1;
					}
					tq[(tq_cnt++ + tq_front) & 0x1f] = skip_len;
					kmer_span += skip_len;
					if (tq_cnt > k) { kmer_span -= tq[tq_front++]; tq_front &= 0x1f; --tq_cnt; }
				} else kmer_span = l + 1 < k? l + 1 : k;
				kmer0 = (kmer0 << 2 | (uint64_t)cch) & mask;
				kmer1 = (kmer1 >> 2) | (3ULL ^ (uint64_t)cch) << shift1;
				if (kmer0 == kmer1) { if (warm && i < cs && i >= start + k - 1) ++nskip; continue; }
				int z = kmer0 < kmer1? 0 : 1;
				++l;
				if (l >= k && kmer_span < 256) {
					ix = mmx_hash64(z? kmer1 : kmer0, mask) << 8 | (uint64_t)kmer_span;
					ip = (uint32_t)i << 1 | (uint32_t)z;
				}
			} else {
				l = 0, tq_cnt = tq_front = 0, kmer_span = 0;
				if (warm && i < cs) { bad = true; break; }
			}
			bx[buf_pos] = ix, bp[buf_pos] = ip;
			const int leff = l;
			if (leff == w + k - 1 && minx != MAXV) { // sketch.c:117-122
				for (int j = buf_pos + 1; j < w; ++j) if (minx == bx[j] && bp[j] != minp) EMIT(bx[j], bp[j]);
				for (int j = 0; j < buf_pos; ++j)     if (minx == bx[j] && bp[j] != minp) EMIT(bx[j], bp[j]);
			}
			if (ix <= minx) { // sketch.c:123-125
				if (leff >= w + k && minx != MAXV) EMIT(minx, minp);
				minx = ix, minp = ip, min_pos = buf_pos;
			} else if (buf_pos == min_pos) { // sketch.c:126-138
				if (leff >= w + k - 1 && minx != MAXV) EMIT(minx, minp);
				minx = MAXV;
				for (int j = buf_pos + 1; j < w; ++j) if (minx >= bx[j]) minx = bx[j], minp = bp[j], min_pos = j;
				for (int j = 0; j <= buf_pos; ++j)    if (minx >= bx[j]) minx = bx[j], minp = bp[j], min_pos = j;
				if (leff >= w + k - 1 && minx != MAXV) {
					for (int j = buf_pos + 1; j < w; ++j) if (minx == bx[j] && minp != bp[j]) EMIT(bx[j], bp[j]);
					for (int j = 0; j <= buf_pos; ++j)    if (minx == bx[j] && minp != bp[j]) EMIT(bx[j], bp[j]);
				}
			}
			if (++buf_pos == w) buf_pos = 0;
			if (i >= ce && ++after > w) break; // everything with pos < ce has left the window
		}
		if (!bad) {
			if (i >= len && minx != MAXV) EMIT(minx, minp); // sketch.c:141-142
			break;
		}
		warm = false, start = 0; // replay from the sequence start: exact by construction
	}
#undef EMIT
	if (!WRITE) A.cnt[c] = n_out;
}

__global__ void chunk_count_kernel(const int64_t *seq_off, int n_seq, int chunk, int is_hpc, int64_t *nchunk)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n_seq) {
		int64_t len = seq_off[i + 1] - seq_off[i];
		nchunk[i] = len <= 0? 0 : is_hpc? 1 : (len + chunk - 1) / chunk;
	}
}

// per-sequence minimizer counts from per-chunk exclusive offsets
__global__ void seq_count_kernel(const int64_t *chunk_off, const int64_t *cnt_excl, int64_t total, int64_t n_chunks, int n_seq, int64_t *seq_mz_off)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i <= n_seq) {
		int64_t c = i < n_seq? chunk_off[i] : n_chunks;
		seq_mz_off[i] = c < n_chunks? cnt_excl[c] : total;
	}
}


// =====================================================================================================================
// K1, tile version (the production path for odd k, w + k <= 64, no HPC -- every preset): minimizers from 2-BIT-PACKED bases.
//
// For odd k a k-mer never equals its reverse complement (the middle base would have to be its own complement), so the
// `kmer[0] == kmer[1] -> continue` skip of sketch.c:108 never fires and the ring of mm_sketch holds exactly the last w POSITIONS.
// The state machine then has a closed form per position i (X[j] = hash of the canonical k-mer ending at j, or MAX when fewer than k
// unambiguous bases end at j; l(i) = unambiguous run length ending at i; A(i) = RIGHT-MOST arg-min of X over [i-w+1, i] -- the
// reference's `<=` update and `>=` rescan both keep the right-most of equal minima):
//   (a) l(i) == w+k-1 and X[A(i-1)] != MAX: emit every j in [i-w+1, i-1] with X[j] == X[A(i-1)], j != A(i-1)    (sketch.c:117-122)
//   (b) X[i] <= X[A(i-1)]: emit A(i-1) if l(i) >= w+k and X[A(i-1)] != MAX                                     (sketch.c:123-125)
//   (c) else if A(i-1) == i-w (the minimum leaves the window): emit A(i-1) if l(i) >= w+k-1 [and != MAX]; then, if l(i) >= w+k-1 and
//       X[A(i)] != MAX, every j in [i-w+1, i] with X[j] == X[A(i)], j != A(i)                                   (sketch.c:126-138)
//   (d) after the last position: emit A(len-1) if its X != MAX                                                 (sketch.c:141-142)
// in this order, for increasing i. Every quantity is a function of at most w+k bases before i, so all positions are independent:
// one CTA owns a tile of TILE positions of one read; the tile's packed bases and ambiguity bits arrive with one TMA bulk copy each
// (cp.async.bulk + mbarrier); the canonical k-mers come out of the packed words with funnel shifts (forward) and brev (reverse
// complement); the window minima are w shared-memory reads per position; emissions are counted, prefix-summed inside the CTA, and
// the tiles are chained with a single-pass decoupled look-back (one kernel: no count pass, no replay). Output order = reference order.
// =====================================================================================================================
#define SKT_TILE 2048
#define SKT_THREADS 256
#define SKT_HALO 64            // >= w + k; X is kept for [ts - SKT_HALO, te)
#define SKT_PAD_WORDS 4        // leading words of the staged arrays that are never TMA targets (look-behind of the first words)

struct TileArgs {
	const uint32_t *pk;         // 2-bit bases, 16 per word, base b at bits 30-2*(b&15) (oldest base most significant)
	const uint32_t *nm;         // ambiguity bits, 32 per word, base b at bit 31-(b&31)
	const int64_t *seq_off;     // n_seq+1
	const int64_t *tile_off;    // n_seq+1: first tile of each sequence
	const int32_t *tile_seq;    // n_tiles: sequence of each tile
	const uint32_t *rid;
	uint32_t rid0;
	int n_seq, w, k, same_rid;
	int64_t n_tiles, cap;
	m128 *out;
	int64_t *tile_excl;         // n_tiles+1: exclusive minimizer offset of each tile (+ total)
	unsigned long long *status; // n_tiles look-back words: flag<<62 | value (flag 1 = tile aggregate, 2 = inclusive prefix)
	unsigned int *ticket;
};

#ifndef MMB_EMU
__device__ __forceinline__ uint32_t skt_smem(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
#endif

// bases (ASCII / nt4 bytes, or the index's 4-bit words) -> 2-bit words + ambiguity bits; one thread per 32 bases
__global__ void pack2_kernel(SeqSrc src, int64_t total, uint32_t *pk, uint32_t *nm, int64_t n_words32)
{
	const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_words32) return;
	uint32_t a = 0, b = 0, m = 0;
	const int64_t b0 = t * 32;
	#pragma unroll 8
	for (int i = 0; i < 32; ++i) {
		const int64_t g = b0 + i;
		const int c = g < total? src.get(g) : 4;
		const uint32_t c2 = c < 4? (uint32_t)c : 0u;
		if (i < 16) a |= c2 << (30 - 2 * i); else b |= c2 << (30 - 2 * (i - 16));
		m |= (c < 4? 0u : 1u) << (31 - i);
	}
	pk[2 * t] = a, pk[2 * t + 1] = b, nm[t] = m;
}

__global__ void tile_seq_kernel(const int64_t *tile_off, int n_seq, int32_t *tile_seq)
{
	const int s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= n_seq) return;
	for (int64_t t = tile_off[s]; t < tile_off[s + 1]; ++t) tile_seq[t] = s;
}

template<bool K32> struct SktX;
template<> struct SktX<true>  { typedef uint32_t T; static __device__ __forceinline__ T maxv() { return 0xffffffffu; } };
template<> struct SktX<false> { typedef uint64_t T; static __device__ __forceinline__ T maxv() { return ~0ULL; } };

// K32: 2k <= 30, every hash step fits 32-bit arithmetic (all steps are mod 2^2k; the right shifts act on masked values)
template<bool K32>
__global__ void __launch_bounds__(SKT_THREADS) sketch_tile_kernel(TileArgs A)
{
	typedef typename SktX<K32>::T XT;
	const XT MAXV = SktX<K32>::maxv();
	__shared__ __align__(16) uint32_t s_pk[SKT_PAD_WORDS + (SKT_TILE + SKT_HALO + 128) / 16 + 8];
	__shared__ __align__(16) uint32_t s_nm[SKT_PAD_WORDS + (SKT_TILE + SKT_HALO + 128) / 32 + 8];
	__shared__ XT s_x[SKT_TILE + SKT_HALO];
	__shared__ uint8_t s_z[SKT_TILE + SKT_HALO];
	__shared__ uint16_t s_a[SKT_TILE + 1];
	__shared__ int s_seg[SKT_TILE / 32 + 1];
	__shared__ __align__(8) unsigned long long s_bar;
	__shared__ long long s_base;
	__shared__ unsigned int s_tile;
	__shared__ int s_any_n;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int w = A.w, k = A.k;

	if (tid == 0) s_tile = atomicAdd(A.ticket, 1u), s_any_n = 0;
#ifndef MMB_EMU
	if (tid == 0) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(skt_smem(&s_bar)) : "memory");
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
#endif
	if (tid < SKT_PAD_WORDS) s_pk[tid] = 0, s_nm[tid] = 0xffffffffu;
	__syncthreads();
	const int64_t tile = s_tile;
	const int sq = A.tile_seq[tile];
	const int64_t off = A.seq_off[sq];
	const int len = (int)(A.seq_off[sq + 1] - off);
	const int ts = (int)(tile - A.tile_off[sq]) * SKT_TILE, te = min(len, ts + SKT_TILE);
	const uint32_t rid = A.rid? A.rid[sq] : A.same_rid? A.rid0 : A.rid0 + (uint32_t)sq;
	// stream window [gA, gE): starts at a multiple of 128 bases (16 B of either array) at or before the first base needed
	int64_t g0 = off + ts - SKT_HALO;
	if (g0 < 0) g0 = 0;
	const int64_t gA = g0 & ~127LL, gE = off + te;
	const uint32_t pk_bytes = (uint32_t)((gE - gA + 63) / 64) * 16, nm_bytes = (uint32_t)((gE - gA + 127) / 128) * 16;
#ifndef MMB_EMU
	if (tid == 0) { // TMA 1-D bulk copies global -> shared, completion counted in bytes on the mbarrier
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(skt_smem(&s_bar)), "r"(pk_bytes + nm_bytes) : "memory");
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
					 :: "r"(skt_smem(s_pk + SKT_PAD_WORDS)), "l"(A.pk + gA / 16), "r"(pk_bytes), "r"(skt_smem(&s_bar)) : "memory");
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
					 :: "r"(skt_smem(s_nm + SKT_PAD_WORDS)), "l"(A.nm + gA / 32), "r"(nm_bytes), "r"(skt_smem(&s_bar)) : "memory");
	}
	{
		uint32_t ok;
		do {
			asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
						 : "=r"(ok) : "r"(skt_smem(&s_bar)), "r"(0) : "memory");
		} while (!ok);
	}
#else
	for (uint32_t i = tid; i < pk_bytes / 4; i += SKT_THREADS) s_pk[SKT_PAD_WORDS + i] = A.pk[gA / 16 + i];
	for (uint32_t i = tid; i < nm_bytes / 4; i += SKT_THREADS) s_nm[SKT_PAD_WORDS + i] = A.nm[gA / 32 + i];
	__syncthreads();
#endif
	{ // any ambiguous base in the staged window? (almost never: then l(i) = min(i+1, w+k) without looking at the bits)
		int any = 0;
		for (uint32_t i = tid; i < nm_bytes / 4; i += SKT_THREADS) any |= s_nm[SKT_PAD_WORDS + i] != 0;
		if (any) s_any_n = 1;
	}
	__syncthreads();
	const bool any_n = s_any_n != 0;
	const int wk = w + k;
	const uint64_t wk_mask = wk >= 64? ~0ULL : (1ULL << wk) - 1;
	// l(i) clipped to w+k: distance to the nearest ambiguous base at or before i, or to the sequence start
	auto run_len = [&](int i) -> int {
		int l = i + 1 < wk? i + 1 : wk;
		if (any_n) {
			const int64_t d = off + i - gA;                 // stream offset of base i inside the staged window
			const int wn = (int)(d >> 5) + SKT_PAD_WORDS, sh = 31 - (int)(d & 31);
			const uint64_t hi = s_nm[wn - 2], mid = s_nm[wn - 1], lo = s_nm[wn];
			uint64_t v = (mid << 32 | lo) >> sh;
			if (sh) v |= hi << (64 - sh);
			v &= wk_mask;                                      // bit j = base i-j is ambiguous
			if (v) { const int dist = __ffsll((long long)v) - 1; if (dist < l) l = dist; }
		}
		return l;
	};
	// ---- pass 1: X (canonical k-mer hash) and strand for positions [ts - SKT_HALO, te) ----
	const uint64_t mask = (1ULL << 2 * k) - 1;
	for (int idx = tid; idx < te - ts + SKT_HALO; idx += SKT_THREADS) {
		const int i = ts - SKT_HALO + idx;
		XT x = MAXV; uint8_t z = 0;
		if (i >= k - 1 && run_len(i) >= k) {
			const int64_t d = off + i - gA;
			const int wi = (int)(d >> 4) + SKT_PAD_WORDS, sh = 30 - 2 * (int)(d & 15);
			if (K32) {
				const uint32_t m32 = (uint32_t)mask;
				const uint32_t f = __funnelshift_r(s_pk[wi], s_pk[wi - 1], sh) & m32;           // forward k-mer, newest base in the low bits
				uint32_t r = __brev(f);                                                        // reverse the 2-bit groups ...
				r = ((r & 0xaaaaaaaau) >> 1) | ((r & 0x55555555u) << 1);
				r = (~r) >> (32 - 2 * k);                                                      // ... and complement: kmer[1] of sketch.c:107
				z = f < r? 0 : 1;
				uint32_t key = z? r : f;
				key = (~key + (key << 21)) & m32;                                              // hash64 (sketch.c:28-38) on 2k <= 30 bits
				key = key ^ key >> 24;
				key = ((key + (key << 3)) + (key << 8)) & m32;
				key = key ^ key >> 14;
				key = ((key + (key << 2)) + (key << 4)) & m32;
				key = key ^ key >> 28;
				key = (key + (key << 31)) & m32;
				x = (XT)key;
			} else {
				const uint64_t w2 = s_pk[wi - 2], w1 = s_pk[wi - 1], w0 = s_pk[wi];
				uint64_t f = (w1 << 32 | w0) >> sh;
				if (sh) f |= w2 << (64 - sh);
				f &= mask;
				uint64_t r = __brevll(f);
				r = ((r & 0xaaaaaaaaaaaaaaaaULL) >> 1) | ((r & 0x5555555555555555ULL) << 1);
				r = (~r) >> (64 - 2 * k);
				z = f < r? 0 : 1;
				x = (XT)mmx_hash64(z? r : f, mask);
			}
		}
		s_x[idx] = x, s_z[idx] = z;
	}
	__syncthreads();
	// ---- pass 2: right-most arg-min of every window, A(i) for i in [ts-1, te); stored as offset inside the window | tie flag ----
	for (int idx = tid; idx < te - ts + 1; idx += SKT_THREADS) {
		const int i = ts - 1 + idx;                          // window [i-w+1, i]; s_x index of position p is p - ts + SKT_HALO
		const int b = i - w + 1 - ts + SKT_HALO;
		XT best = s_x[b]; int bo = 0, ties = 0;
		for (int j = 1; j < w; ++j) {
			const XT v = s_x[b + j];
			if (v < best) best = v, bo = j, ties = 0;
			else if (v == best) bo = j, ties = 1;
		}
		s_a[idx] = (uint16_t)(bo | (ties << 15));
	}
	__syncthreads();
	// ---- pass 3: emission counts; thread handles positions ts + n*256 + tid ----
	const int NR = SKT_TILE / SKT_THREADS;
	int cnt[NR];
	uint8_t flg[NR];  // 1: emit A(i-1) (rules b/c); 2: slow path (rule a and/or ties of rule c); 4: final emission (rule d)
	#pragma unroll
	for (int n = 0; n < NR; ++n) {
		const int i = ts + n * SKT_THREADS + tid;
		cnt[n] = 0, flg[n] = 0;
		if (i >= te) continue;
		const int xi_idx = i - ts + SKT_HALO;
		const int ap = s_a[i - ts], ac = s_a[i - ts + 1];
		const int pm = i - w + (ap & 0x7fff), pn = i - w + 1 + (ac & 0x7fff);
		const XT xm = s_x[pm - ts + SKT_HALO], xn = s_x[pn - ts + SKT_HALO], xi = s_x[xi_idx];
		const int l = run_len(i);
		int c = 0, f = 0;
		if (l == wk - 1 && xm != MAXV && w > 1) { // rule (a): duplicates of the first full window's minimum
			const int b = i - w + 1 - ts + SKT_HALO;
			int e = 0;
			for (int j = 0; j < w - 1; ++j) e += s_x[b + j] == xm && i - w + 1 + j != pm;
			if (e) c += e, f |= 2;
		}
		if (xi <= xm) { if (l >= wk && xm != MAXV) ++c, f |= 1; }
		else if (pm == i - w) {
			if (l >= wk - 1 && xm != MAXV) ++c, f |= 1;
			if (l >= wk - 1 && xn != MAXV && (ac & 0x8000)) {
				const int b = i - w + 1 - ts + SKT_HALO;
				int e = 0;
				for (int j = 0; j < w; ++j) e += s_x[b + j] == xn && i - w + 1 + j != pn;
				if (e) c += e, f |= 2;
			}
		}
		if (i == len - 1 && xn != MAXV) ++c, f |= 4;
		cnt[n] = c, flg[n] = (uint8_t)f;
	}
	// ---- CTA-wide exclusive prefix in position order: segment = (row n, warp) = 32 consecutive positions ----
	int pre[NR];
	#pragma unroll
	for (int n = 0; n < NR; ++n) {
		int x = cnt[n];
		for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
		pre[n] = x - cnt[n];
		if (lane == 31) s_seg[n * (SKT_THREADS / 32) + wid] = x;
	}
	__syncthreads();
	if (wid == 0) { // 64 segment totals -> exclusive offsets (two per lane)
		const int NS = SKT_TILE / 32;
		int a0 = s_seg[2 * lane], a1 = s_seg[2 * lane + 1], sum = a0 + a1, x = sum;
		for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
		const int ex = x - sum;
		s_seg[2 * lane] = ex, s_seg[2 * lane + 1] = ex + a0;
		if (lane == 31) s_seg[NS] = x;
	}
	__syncthreads();
	const int tile_total = s_seg[SKT_TILE / 32];
	// ---- chain the tiles: decoupled look-back over the status words (warp 0) ----
	if (wid == 0) {
		const unsigned long long FLAG_A = 1ULL << 62, FLAG_P = 2ULL << 62, VMASK = (1ULL << 62) - 1;
		volatile unsigned long long *st = A.status;
		long long excl = 0;
		if (tile == 0) { if (lane == 0) st[0] = FLAG_P | (unsigned long long)tile_total; }
		else {
			if (lane == 0) st[tile] = FLAG_A | (unsigned long long)tile_total;
			int64_t j0 = tile - 1;
			for (;;) {
				const int64_t j = j0 - lane;
				unsigned long long v = j >= 0? st[j] : FLAG_P;   // before the first tile: prefix 0
				while (__any_sync(0xffffffffu, (v >> 62) == 0)) v = j >= 0? st[j] : FLAG_P;
				const unsigned pmask = __ballot_sync(0xffffffffu, (v >> 62) == 2);
				const int first = pmask? __ffs((int)pmask) - 1 : 32; // nearest predecessor that already knows its inclusive prefix
				long long x = lane <= first? (long long)(v & VMASK) : 0;
				for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
				excl += x;
				if (pmask) break;
				j0 -= 32;
			}
			if (lane == 0) st[tile] = FLAG_P | (unsigned long long)(excl + tile_total);
		}
		if (lane == 0) {
			s_base = excl;
			A.tile_excl[tile] = excl;
			if (tile == A.n_tiles - 1) A.tile_excl[A.n_tiles] = excl + tile_total;
		}
	}
	__syncthreads();
	if (tile_total == 0) return;
	const long long base = s_base;
	// ---- pass 4: write, in the reference's order within each position ----
	const uint64_t span = (uint64_t)k;
	auto put = [&](long long o, int p) {
		if (o < A.cap) {
			const int xi_ = p - ts + SKT_HALO;
			m128 v;
			v.x = (uint64_t)s_x[xi_] << 8 | span;
			v.y = (uint64_t)rid << 32 | (uint32_t)p << 1 | s_z[xi_];
			A.out[o] = v;
		}
	};
	#pragma unroll
	for (int n = 0; n < NR; ++n) {
		if (!cnt[n]) continue;
		const int i = ts + n * SKT_THREADS + tid;
		long long o = base + s_seg[n * (SKT_THREADS / 32) + wid] + pre[n];
		const int ap = s_a[i - ts], ac = s_a[i - ts + 1];
		const int pm = i - w + (ap & 0x7fff), pn = i - w + 1 + (ac & 0x7fff);
		if (flg[n] & 2) {
			const int l = run_len(i);
			const XT xm = s_x[pm - ts + SKT_HALO], xn = s_x[pn - ts + SKT_HALO], xi = s_x[i - ts + SKT_HALO];
			const int b = i - w + 1 - ts + SKT_HALO;
			if (l == wk - 1 && xm != MAXV && w > 1)
				for (int j = 0; j < w - 1; ++j) if (s_x[b + j] == xm && i - w + 1 + j != pm) put(o++, i - w + 1 + j);
			if (flg[n] & 1) put(o++, pm);
			if (!(xi <= xm) && pm == i - w && l >= wk - 1 && xn != MAXV && (ac & 0x8000))
				for (int j = 0; j < w; ++j) if (s_x[b + j] == xn && i - w + 1 + j != pn) put(o++, i - w + 1 + j);
		} else if (flg[n] & 1) put(o++, pm);
		if (flg[n] & 4) put(o++, pn);
	}
}

__global__ void tile_count_kernel(const int64_t *seq_off, int n_seq, int64_t *ntile)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n_seq) { const int64_t len = seq_off[i + 1] - seq_off[i]; ntile[i] = len <= 0? 0 : (len + SKT_TILE - 1) / SKT_TILE; }
}

} // namespace

// Device-level launcher. d_seq_off: n_seq+1 int64 base offsets. Results: *d_out (grown as needed) holds all
// minimizers in (sequence, position) order; d_mz_off (n_seq+1 int64, device) their per-sequence offsets.
// Returns the total count (synchronises the stream once to size the output).
int64_t mmb_sketch_device(mmb_ctx_t *ctx, const uint8_t *d_bytes, const uint32_t *d_packed, const int64_t *d_seq_off, int n_seq,
						  const uint32_t *d_rid, uint32_t rid0, int w, int k, int is_hpc, int64_t total_bases,
						  DevBuf &out, int64_t *d_mz_off, DevBuf &tmp_a, DevBuf &tmp_b, int same_rid)
{
	if (n_seq <= 0) return 0;
	if (!(w > 0 && w < 256 && k > 0 && k <= 28)) { fprintf(stderr, "[ERROR] mm_sketch: invalid w=%d k=%d\n", w, k); abort(); }
	ProfScope prof(ctx, MMB_PROF_SKETCH, (uint64_t)total_bases);
	if ((k & 1) && w + k <= SKT_HALO && !is_hpc && total_bases > 0) { // tile kernel over 2-bit-packed bases (see above)
		DevBuf &pkb = ctx->sk_pk, &nmb = ctx->sk_nm, &misc = ctx->sk_misc; // per context (= per scheduler group); sized once in steady state
		const int64_t nw32 = (total_bases + 31) / 32;
		uint32_t *d_pk = pkb.as<uint32_t>((size_t)nw32 * 2 + 64), *d_nm = nmb.as<uint32_t>((size_t)nw32 + 64);
		SeqSrc src; src.bytes = d_bytes, src.packed = d_packed;
		pack2_kernel<<<(unsigned)((nw32 + 255) / 256), 256, 0, ctx->stream>>>(src, total_bases, d_pk, d_nm, nw32);
		int64_t *d_tile_off = tmp_a.as<int64_t>((size_t)n_seq + 1);
		tile_count_kernel<<<(n_seq + 255) / 256, 256, 0, ctx->stream>>>(d_seq_off, n_seq, d_tile_off);
		ctx->n_launch += 2;
		const int64_t n_tiles = mmb_exclusive_scan_i64(ctx, d_tile_off, n_seq, true);
		if (n_tiles == 0) { MMB_CUDA_CHECK(cudaMemsetAsync(d_mz_off, 0, sizeof(int64_t) * (n_seq + 1), ctx->stream)); return 0; }
		// scratch: tile_excl (n_tiles+1 i64) | status (n_tiles u64) | ticket (u64 slot) | tile_seq (n_tiles i32)
		uint8_t *m = (uint8_t*)misc.reserve((size_t)n_tiles * 20 + 64);
		TileArgs A;
		A.pk = d_pk, A.nm = d_nm, A.seq_off = d_seq_off, A.tile_off = d_tile_off, A.rid = d_rid, A.rid0 = rid0;
		A.n_seq = n_seq, A.w = w, A.k = k, A.same_rid = same_rid, A.n_tiles = n_tiles;
		A.tile_excl = (int64_t*)m, A.status = (unsigned long long*)(m + 8 * (size_t)(n_tiles + 1));
		A.ticket = (unsigned int*)(m + 8 * (size_t)(2 * n_tiles + 1));
		int32_t *d_tile_seq = (int32_t*)(m + 8 * (size_t)(2 * n_tiles + 2));
		A.tile_seq = d_tile_seq;
		tile_seq_kernel<<<(n_seq + 127) / 128, 128, 0, ctx->stream>>>(d_tile_off, n_seq, d_tile_seq);
		++ctx->n_launch;
		// capacity: the expected density of (w,k)-minimizers is 2/(w+1); 1.5x of that plus slack almost always suffices and the kernel
		// reports the exact total, so a batch of low-complexity sequence only costs a second launch
		int64_t cap = (int64_t)((double)total_bases * 3.0 / (w + 1)) + 4096;
		if ((int64_t)(out.cap / sizeof(m128)) - 1 > cap) cap = (int64_t)(out.cap / sizeof(m128)) - 1; // use what the arena already holds (never grow it by this)
		if (getenv("MM_B200_SKETCH_CAP")) cap = atoll(getenv("MM_B200_SKETCH_CAP")); // test hook: force the overflow / relaunch path
		int64_t total = 0;
		for (int attempt = 0; attempt < 2; ++attempt) {
			A.out = out.as<m128>((size_t)cap + 1), A.cap = cap;
			MMB_CUDA_CHECK(cudaMemsetAsync(A.status, 0, 8 * (size_t)(n_tiles + 1), ctx->stream)); // status words + ticket
			if (k <= 15) sketch_tile_kernel<true><<<(unsigned)n_tiles, SKT_THREADS, 0, ctx->stream>>>(A);
			else sketch_tile_kernel<false><<<(unsigned)n_tiles, SKT_THREADS, 0, ctx->stream>>>(A);
			MMB_CUDA_CHECK(cudaGetLastError());
			++ctx->n_launch;
			MMB_CUDA_CHECK(cudaMemcpyAsync(&total, A.tile_excl + n_tiles, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
			mmb_stream_sync(ctx);
			if (total <= cap) break;
			cap = total + 16;
		}
		seq_count_kernel<<<(n_seq + 1 + 255) / 256, 256, 0, ctx->stream>>>(d_tile_off, A.tile_excl, total, n_tiles, n_seq, d_mz_off);
		++ctx->n_launch;
		return total;
	}
	const int WU = 2 * w + 2 * k + 15;
	int chunk = 512;
	while (chunk < 6 * WU) chunk <<= 1;
	// chunk table
	int64_t *d_chunk_off = tmp_a.as<int64_t>((size_t)n_seq + 1);
	chunk_count_kernel<<<(n_seq + 255) / 256, 256, 0, ctx->stream>>>(d_seq_off, n_seq, chunk, is_hpc, d_chunk_off);
	++ctx->n_launch;
	int64_t n_chunks = mmb_exclusive_scan_i64(ctx, d_chunk_off, n_seq, true);
	if (n_chunks == 0) { MMB_CUDA_CHECK(cudaMemsetAsync(d_mz_off, 0, sizeof(int64_t) * (n_seq + 1), ctx->stream)); return 0; }
	int64_t *d_cnt = tmp_b.as<int64_t>((size_t)n_chunks + 1);
	SketchArgs A;
	A.src.bytes = d_bytes, A.src.packed = d_packed;
	A.seq_off = d_seq_off, A.chunk_off = d_chunk_off, A.rid = d_rid, A.rid0 = rid0;
	A.n_seq = n_seq, A.w = w, A.k = k, A.is_hpc = is_hpc, A.chunk = chunk, A.n_chunks = n_chunks, A.cnt = d_cnt, A.out = nullptr, A.same_rid = same_rid;
	const int threads = 128;
	const unsigned grid = (unsigned)((n_chunks + threads - 1) / threads);
	sketch_kernel<false><<<grid, threads, 0, ctx->stream>>>(A);
	MMB_CUDA_CHECK(cudaGetLastError());
	++ctx->n_launch;
	int64_t total = mmb_exclusive_scan_i64(ctx, d_cnt, n_chunks, true);
	A.out = out.as<m128>((size_t)total + 1);
	if (total > 0) {
		sketch_kernel<true><<<grid, threads, 0, ctx->stream>>>(A);
		MMB_CUDA_CHECK(cudaGetLastError());
		++ctx->n_launch;
	}
	seq_count_kernel<<<(n_seq + 1 + 255) / 256, 256, 0, ctx->stream>>>(d_chunk_off, d_cnt, total, n_chunks, n_seq, d_mz_off);
	++ctx->n_launch;
	return total;
}

extern "C" int64_t mmb_sketch_batch_host(mmb_ctx_t *ctx, int n_seq, const char *seqs, const int64_t *off, int w, int k, int is_hpc,
										 uint32_t rid0, uint64_t *out_xy, int64_t out_cap, int64_t *n_out)
{
	if (n_seq <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	const int64_t tot = off[n_seq];
	uint8_t *d_seq = ctx->d_a.as<uint8_t>((size_t)tot + 16);
	int64_t *d_off = ctx->d_b.as<int64_t>((size_t)n_seq + 1);
	int64_t *d_mz_off = ctx->d_c.as<int64_t>((size_t)n_seq + 1);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_seq, seqs, tot, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, off, sizeof(int64_t) * (n_seq + 1), cudaMemcpyHostToDevice, ctx->stream));
	int64_t total = mmb_sketch_device(ctx, d_seq, nullptr, d_off, n_seq, nullptr, rid0, w, k, is_hpc, tot, ctx->d_d, d_mz_off, ctx->d_e, ctx->d_f, 0);
	if (n_out) {
		std::vector<int64_t> mo(n_seq + 1);
		MMB_CUDA_CHECK(cudaMemcpyAsync(mo.data(), d_mz_off, sizeof(int64_t) * (n_seq + 1), cudaMemcpyDeviceToHost, ctx->stream));
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
		for (int i = 0; i < n_seq; ++i) n_out[i] = mo[i + 1] - mo[i];
	}
	if (out_xy && total <= out_cap && total > 0) {
		MMB_CUDA_CHECK(cudaMemcpyAsync(out_xy, ctx->d_d.p, sizeof(m128) * total, cudaMemcpyDeviceToHost, ctx->stream));
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	}
	return total;
}
