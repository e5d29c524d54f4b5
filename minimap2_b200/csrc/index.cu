// minimap2_b200/csrc/index.cu -- index construction on the GPU, .mmi I/O and the mm_idx_* part of the minimap.h API.
//
// Replaces index.c:222-640 (mm_idx_gen / worker_post / mm_idx_str / dump / load / reader) and the query side
// index.c:93-110,164-220. The build is GPU-first (SURVEY 8 row f1): the whole reference is sketched by the K1 kernel
// straight from the 4-bit packed S array, (hash, position) pairs are radix-sorted on the device (CUB DeviceRadixSort --
// library plumbing for this one-off stage, not part of the per-read hot path), runs are collapsed into keys and an
// open-addressing table is filled with atomicCAS. Occurrence lists come out ordered by position inside a key, the
// order the reference establishes with radix_sort_64 (index.c:264-266), so mm_idx_get-dependent results are identical.
#include "index.h"
#include "annot.h"
#include <emmintrin.h>
#include "mm_algo.cuh"
#include "fastx.h"
#include "scan.cuh"
#include <cub/cub.cuh>
#include <cstring>
#include <algorithm>
#include <unistd.h>
#include <fcntl.h>
#include <sys/time.h>
#include <sys/resource.h>

extern "C" {
int mm_verbose = 1;
int mm_dbg_flag = 0;
double mm_realtime0;
}

static double realtime_now(void)
{
	struct timeval tp;
	gettimeofday(&tp, NULL);
	return tp.tv_sec + tp.tv_usec * 1e-6;
}
static double cputime_now(void)
{
	struct rusage r;
	getrusage(RUSAGE_SELF, &r);
	return r.ru_utime.tv_sec + r.ru_stime.tv_sec + 1e-6 * (r.ru_utime.tv_usec + r.ru_stime.tv_usec);
}
extern "C" double realtime(void) { return realtime_now(); }
extern "C" double cputime(void) { return cputime_now(); }

static mmb_ctx_t *g_ctx = nullptr;
static std::mutex g_ctx_mu;

mmb_ctx_t *mmb_default_ctx(void)
{
	std::lock_guard<std::mutex> lk(g_ctx_mu);
	if (!g_ctx) {
		int dev = 0;
		const char *e = getenv("MM_B200_DEVICE");
		if (!e) e = getenv("LOCAL_RANK");
		if (e) dev = atoi(e);
		int n = mmb_device_count();
		if (n <= 0) { fprintf(stderr, "[ERROR] minimap2_b200 needs a CUDA device (sm_90a); no CPU path exists\n"); abort(); }
		g_ctx = mmb_ctx_create(dev % n);
		if (!g_ctx) abort();
	}
	return g_ctx;
}

// ---------------------------------------------------------------------------------------------------------
// device build
// ---------------------------------------------------------------------------------------------------------
namespace {

__global__ void split_kernel(const m128 *mz, int64_t n, uint64_t *keys, uint64_t *vals)
{
	int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) { m128 v = mz[i]; keys[i] = v.x >> 8, vals[i] = v.y; }
}

__global__ void tab_clear_kernel(IdxSlot *tab, uint64_t n)
{
	uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) tab[i].key = MMB_IDX_EMPTY, tab[i].val = 0;
}

__global__ void tab_insert_kernel(IdxSlot *tab, int bits, const uint64_t *keys, const uint32_t *cnt, const int64_t *off, int64_t n)
{
	int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint64_t key = keys[i], mask = (1ULL << bits) - 1;
	uint64_t s = idx_slot_of(key, bits);
	for (;;) {
		unsigned long long old = atomicCAS((unsigned long long*)&tab[s].key, (unsigned long long)MMB_IDX_EMPTY, (unsigned long long)key);
		if (old == MMB_IDX_EMPTY) { tab[s].val = (uint64_t)off[i] << MMB_IDX_NBITS | cnt[i]; return; }
		s = (s + 1) & mask;
	}
}



void finish_table(mm_idx_t *mi, mmb_ctx_t *ctx, const uint64_t *d_keys, const uint32_t *d_cnt, const int64_t *d_off, int64_t n_keys)
{
	mm_idx_bucket_s *B = mi->B;
	int bits = 10;
	while ((1ULL << bits) < (uint64_t)n_keys * 2) ++bits;
	B->tab_bits = bits;
	MMB_CUDA_CHECK(cudaMalloc(&B->d_tab, sizeof(IdxSlot) << bits));
	const uint64_t ns = 1ULL << bits;
	tab_clear_kernel<<<(unsigned)((ns + 255) / 256), 256, 0, ctx->stream>>>(B->d_tab, ns);
	if (n_keys > 0)
		tab_insert_kernel<<<(unsigned)((n_keys + 255) / 256), 256, 0, ctx->stream>>>(B->d_tab, bits, d_keys, d_cnt, d_off, n_keys);
	MMB_CUDA_CHECK(cudaGetLastError());
	// ascending counts for mm_idx_cal_max_occ (order statistics only depend on the multiset, index.c:198-220)
	MMB_CUDA_CHECK(cudaMalloc(&B->d_cnt_sorted, sizeof(uint32_t) * (size_t)(n_keys + 1)));
	if (n_keys > 0) {
		size_t tb = 0;
		cub::DeviceRadixSort::SortKeys(nullptr, tb, d_cnt, B->d_cnt_sorted, (int64_t)n_keys, 0, 32, ctx->stream);
		void *tmp = nullptr;
		MMB_CUDA_CHECK(cudaMalloc(&tmp, tb + 16));
		cub::DeviceRadixSort::SortKeys(tmp, tb, d_cnt, B->d_cnt_sorted, (int64_t)n_keys, 0, 32, ctx->stream);
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
		MMB_CUDA_CHECK(cudaFree(tmp));
	}
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

void upload_seqs(mm_idx_t *mi, mmb_ctx_t *ctx)
{
	mm_idx_bucket_s *B = mi->B;
	uint64_t sum_len = 0;
	std::vector<uint64_t> off(mi->n_seq + 1);
	std::vector<uint32_t> len(mi->n_seq + 1);
	for (uint32_t i = 0; i < mi->n_seq; ++i) off[i] = mi->seq[i].offset, len[i] = mi->seq[i].len, sum_len += mi->seq[i].len;
	off[mi->n_seq] = sum_len;
	const size_t nw = (sum_len + 7) / 8;
	MMB_CUDA_CHECK(cudaMalloc(&B->d_S, (nw + 4) * 4));
	MMB_CUDA_CHECK(cudaMemset(B->d_S, 0, (nw + 4) * 4));
	if (mi->S && nw) MMB_CUDA_CHECK(cudaMemcpy(B->d_S, mi->S, nw * 4, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMalloc(&B->d_seq_off, sizeof(uint64_t) * (mi->n_seq + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&B->d_seq_len, sizeof(uint32_t) * (mi->n_seq + 1)));
	MMB_CUDA_CHECK(cudaMemcpy(B->d_seq_off, off.data(), sizeof(uint64_t) * (mi->n_seq + 1), cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(B->d_seq_len, len.data(), sizeof(uint32_t) * (mi->n_seq + 1), cudaMemcpyHostToDevice));
}

} // namespace

void mmb_idx_build_device(mm_idx_t *mi)
{
	mmb_ctx_t *ctx = mmb_default_ctx();
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	mm_idx_bucket_s *B = mi->B;
	B->ctx = ctx;
	upload_seqs(mi, ctx);
	uint64_t sum_len = 0;
	for (uint32_t i = 0; i < mi->n_seq; ++i) sum_len += mi->seq[i].len;
	// 1. sketch every sequence straight from the packed S
	DevBuf mz, t1, t2, t3;
	int64_t *d_seq_off64 = t3.as<int64_t>((size_t)mi->n_seq * 2 + 4), *d_mz_off = d_seq_off64 + mi->n_seq + 2;
	static_assert(sizeof(int64_t) == sizeof(uint64_t), "");
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_seq_off64, B->d_seq_off, sizeof(int64_t) * (mi->n_seq + 1), cudaMemcpyDeviceToDevice, ctx->stream));
	int64_t n_mz = mi->n_seq? mmb_sketch_device(ctx, nullptr, B->d_S, d_seq_off64, (int)mi->n_seq, nullptr, 0, mi->w, mi->k, mi->flag & MM_I_HPC,
												(int64_t)sum_len, mz, d_mz_off, t1, t2) : 0;
	t1.release(); t2.release();
	// 2. sort (hash, position) by hash; the input is in (rid, pos) order and the LSD radix sort is stable, so positions
	//    end up ascending inside each key exactly as after index.c:264-266
	uint64_t *k_in, *k_out, *v_in, *v_out;
	MMB_CUDA_CHECK(cudaMalloc(&k_in, sizeof(uint64_t) * (size_t)(n_mz + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&v_in, sizeof(uint64_t) * (size_t)(n_mz + 1)));
	if (n_mz > 0) split_kernel<<<(unsigned)((n_mz + 255) / 256), 256, 0, ctx->stream>>>((const m128*)mz.p, n_mz, k_in, v_in);
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	mz.release();
	MMB_CUDA_CHECK(cudaMalloc(&k_out, sizeof(uint64_t) * (size_t)(n_mz + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&v_out, sizeof(uint64_t) * (size_t)(n_mz + 1)));
	uint64_t *d_ukeys = nullptr; uint32_t *d_cnt = nullptr; int64_t *d_off = nullptr;
	int64_t n_keys = 0;
	if (n_mz > 0) {
		size_t tb = 0; void *tmp = nullptr;
		cub::DeviceRadixSort::SortPairs(nullptr, tb, k_in, k_out, v_in, v_out, n_mz, 0, 2 * mi->k, ctx->stream);
		MMB_CUDA_CHECK(cudaMalloc(&tmp, tb + 16));
		cub::DeviceRadixSort::SortPairs(tmp, tb, k_in, k_out, v_in, v_out, n_mz, 0, 2 * mi->k, ctx->stream);
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
		MMB_CUDA_CHECK(cudaFree(tmp));
		MMB_CUDA_CHECK(cudaFree(k_in)); MMB_CUDA_CHECK(cudaFree(v_in));
		// 3. collapse runs
		int64_t *d_nruns;
		MMB_CUDA_CHECK(cudaMalloc(&d_ukeys, sizeof(uint64_t) * (size_t)(n_mz + 1)));
		MMB_CUDA_CHECK(cudaMalloc(&d_cnt, sizeof(uint32_t) * (size_t)(n_mz + 1)));
		MMB_CUDA_CHECK(cudaMalloc(&d_nruns, sizeof(int64_t)));
		tb = 0;
		cub::DeviceRunLengthEncode::Encode(nullptr, tb, k_out, d_ukeys, d_cnt, d_nruns, n_mz, ctx->stream);
		MMB_CUDA_CHECK(cudaMalloc(&tmp, tb + 16));
		cub::DeviceRunLengthEncode::Encode(tmp, tb, k_out, d_ukeys, d_cnt, d_nruns, n_mz, ctx->stream);
		MMB_CUDA_CHECK(cudaMemcpyAsync(&n_keys, d_nruns, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
		MMB_CUDA_CHECK(cudaFree(tmp)); MMB_CUDA_CHECK(cudaFree(d_nruns)); MMB_CUDA_CHECK(cudaFree(k_out));
		// 4. offsets
		MMB_CUDA_CHECK(cudaMalloc(&d_off, sizeof(int64_t) * (size_t)(n_keys + 1)));
		tb = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tb, d_cnt, d_off, n_keys, ctx->stream);
		MMB_CUDA_CHECK(cudaMalloc(&tmp, tb + 16));
		cub::DeviceScan::ExclusiveSum(tmp, tb, d_cnt, d_off, n_keys, ctx->stream);
		MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
		MMB_CUDA_CHECK(cudaFree(tmp));
	} else {
		MMB_CUDA_CHECK(cudaFree(k_in)); MMB_CUDA_CHECK(cudaFree(v_in)); MMB_CUDA_CHECK(cudaFree(k_out));
	}
	B->n_keys = n_keys, B->n_pos = n_mz, B->d_pos = v_out;
	finish_table(mi, ctx, d_ukeys, d_cnt, d_off, n_keys);
	B->d_ukeys = d_ukeys, B->d_ucnt = d_cnt, B->d_uoff = d_off; // kept for the lazy host mirror (mm_idx_get on the host, stat, dump)
	t3.release();
}

void mmb_idx_build_from_lists(mm_idx_t *mi, std::vector<uint64_t> &keys, std::vector<uint32_t> &cnt, std::vector<uint64_t> &pos)
{
	mmb_ctx_t *ctx = mmb_default_ctx();
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	mm_idx_bucket_s *B = mi->B;
	B->ctx = ctx;
	upload_seqs(mi, ctx);
	const int64_t n_keys = (int64_t)keys.size(), n_pos = (int64_t)pos.size();
	std::vector<int64_t> off(n_keys + 1);
	int64_t run = 0;
	for (int64_t i = 0; i < n_keys; ++i) off[i] = run, run += cnt[i];
	uint64_t *d_keys; uint32_t *d_cnt; int64_t *d_off;
	MMB_CUDA_CHECK(cudaMalloc(&d_keys, 8 * (size_t)(n_keys + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&d_cnt, 4 * (size_t)(n_keys + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&d_off, 8 * (size_t)(n_keys + 1)));
	MMB_CUDA_CHECK(cudaMalloc(&B->d_pos, 8 * (size_t)(n_pos + 1)));
	MMB_CUDA_CHECK(cudaMemcpy(d_keys, keys.data(), 8 * (size_t)n_keys, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(d_cnt, cnt.data(), 4 * (size_t)n_keys, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(d_off, off.data(), 8 * (size_t)n_keys, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(B->d_pos, pos.data(), 8 * (size_t)n_pos, cudaMemcpyHostToDevice));
	B->n_keys = n_keys, B->n_pos = n_pos;
	finish_table(mi, ctx, d_keys, d_cnt, d_off, n_keys);
	B->h_keys.swap(keys);
	B->h_val.resize(n_keys);
	for (int64_t i = 0; i < n_keys; ++i) B->h_val[i] = (uint64_t)off[i] << MMB_IDX_NBITS | cnt[i];
	B->h_pos.swap(pos);
	MMB_CUDA_CHECK(cudaFree(d_keys)); MMB_CUDA_CHECK(cudaFree(d_cnt)); MMB_CUDA_CHECK(cudaFree(d_off));
}

void mmb_idx_host_sync(const mm_idx_t *mi)
{
	mm_idx_bucket_s *B = mi->B;
	std::lock_guard<std::mutex> lk(B->mu);
	if (B->host_ready) return;
	if (B->h_keys.size() != (size_t)B->n_keys) {
		const int64_t n_keys = B->n_keys;
		B->h_keys.resize(n_keys); B->h_val.resize(n_keys);
		std::vector<uint32_t> hc(n_keys); std::vector<int64_t> ho(n_keys);
		MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
		if (n_keys) {
			MMB_CUDA_CHECK(cudaMemcpy(B->h_keys.data(), B->d_ukeys, sizeof(uint64_t) * n_keys, cudaMemcpyDeviceToHost));
			MMB_CUDA_CHECK(cudaMemcpy(hc.data(), B->d_ucnt, sizeof(uint32_t) * n_keys, cudaMemcpyDeviceToHost));
			MMB_CUDA_CHECK(cudaMemcpy(ho.data(), B->d_uoff, sizeof(int64_t) * n_keys, cudaMemcpyDeviceToHost));
		}
		for (int64_t i = 0; i < n_keys; ++i) B->h_val[i] = (uint64_t)ho[i] << MMB_IDX_NBITS | hc[i];
	}
	if (B->h_pos.size() != (size_t)B->n_pos) {
		B->h_pos.resize(B->n_pos);
		MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
		if (B->n_pos) MMB_CUDA_CHECK(cudaMemcpy(B->h_pos.data(), B->d_pos, 8 * (size_t)B->n_pos, cudaMemcpyDeviceToHost));
	}
	B->h_map = new std::unordered_map<uint64_t, uint32_t>();
	B->h_map->reserve(B->h_keys.size() * 2);
	for (size_t i = 0; i < B->h_keys.size(); ++i) (*B->h_map)[B->h_keys[i]] = (uint32_t)i;
	B->host_ready = true;
}

// ---------------------------------------------------------------------------------------------------------
// minimap.h API: index
// ---------------------------------------------------------------------------------------------------------
static mm_idx_t *idx_init(int w, int k, int b, int flag) // index.c:52-61
{
	if (k * 2 < b) b = k * 2;
	if (w < 1) w = 1;
	mm_idx_t *mi = (mm_idx_t*)calloc(1, sizeof(mm_idx_t));
	mi->w = w, mi->k = k, mi->b = b, mi->flag = flag;
	mi->B = new mm_idx_bucket_s();
	return mi;
}

extern "C" void mm_idx_destroy(mm_idx_t *mi) // index.c:62-91
{
	if (mi == 0) return;
	if (mi->h) delete (std::unordered_map<std::string, uint32_t>*)mi->h;
	if (mi->B) {
		mm_idx_bucket_s *B = mi->B;
		if (B->ctx) cudaSetDevice(B->ctx->device);
		if (!B->external) { cudaFree(B->d_tab); cudaFree(B->d_pos); cudaFree(B->d_S); cudaFree(B->d_seq_off); cudaFree(B->d_seq_len); cudaFree(B->d_cnt_sorted); } cudaFree(B->d_name_rank); cudaFree(B->d_ukeys); cudaFree(B->d_ucnt); cudaFree(B->d_uoff);
		if (B->d_junc) cudaFree(B->d_junc);
		if (B->d_jump_off) cudaFree(B->d_jump_off);
		for (int t = 0; t < 2; ++t) if (B->d_spsc[t]) cudaFree(B->d_spsc[t]);
		delete B->h_map;
		delete B;
	}
	if (mi->I) { for (uint32_t i = 0; i < mi->n_seq; ++i) free(mi->I[i].a); free(mi->I); }
	if (mi->spsc) { for (uint32_t i = 0; i < mi->n_seq * 2; ++i) free(mi->spsc[i].a); free(mi->spsc); }
	if (mi->J) { for (uint32_t i = 0; i < mi->n_seq; ++i) free(mi->J[i].a); free(mi->J); }
	for (uint32_t i = 0; i < mi->n_seq; ++i) free(mi->seq[i].name);
	free(mi->seq); free(mi->S); free(mi);
}

extern "C" const uint64_t *mm_idx_get(const mm_idx_t *mi, uint64_t minier, int *n) // index.c:93-110 (host mirror)
{
	mm_idx_bucket_s *B = mi->B;
	if (!B->host_ready) mmb_idx_host_sync(mi);
	*n = 0;
	auto it = B->h_map->find(minier);
	if (it == B->h_map->end()) return 0;
	uint64_t v = B->h_val[it->second];
	*n = (int)(v & ((1ULL << MMB_IDX_NBITS) - 1));
	return &B->h_pos[v >> MMB_IDX_NBITS];
}

extern "C" void mm_idx_stat(const mm_idx_t *mi) // index.c:112-134
{
	mm_idx_bucket_s *B = mi->B;
	int64_t n = B->n_keys, n1 = 0;
	uint64_t sum = 0, len = 0;
	fprintf(stderr, "[M::%s] kmer size: %d; skip: %d; is_hpc: %d; #seq: %d\n", __func__, mi->k, mi->w, mi->flag&MM_I_HPC, mi->n_seq);
	for (uint32_t i = 0; i < mi->n_seq; ++i) len += mi->seq[i].len;
	mmb_idx_host_sync(mi);
	for (size_t i = 0; i < B->h_val.size(); ++i) {
		uint32_t c = (uint32_t)(B->h_val[i] & ((1ULL << MMB_IDX_NBITS) - 1));
		sum += c;
		if (c == 1) ++n1;
	}
	fprintf(stderr, "[M::%s::%.3f*%.2f] distinct minimizers: %ld (%.2f%% are singletons); average occurrences: %.3lf; average spacing: %.3lf; total length: %ld\n",
			__func__, realtime_now() - mm_realtime0, cputime_now() / (realtime_now() - mm_realtime0), (long)n, 100.0*n1/n, (double)sum / n, (double)len / sum, (long)len);
}

extern "C" int mm_idx_index_name(mm_idx_t *mi) // index.c:136-153
{
	if (mi->h) return 0;
	auto *h = new std::unordered_map<std::string, uint32_t>();
	int has_dup = 0;
	for (uint32_t i = 0; i < mi->n_seq; ++i) {
		if (!mi->seq[i].name) continue;
		auto r = h->emplace(mi->seq[i].name, i);
		if (!r.second) has_dup = 1;
	}
	mi->h = h;
	if (has_dup && mm_verbose >= 2) fprintf(stderr, "[WARNING] some database sequences have identical sequence names\n");
	return has_dup;
}

extern "C" int mm_idx_name2id(const mm_idx_t *mi, const char *name) // index.c:155-162
{
	auto *h = (std::unordered_map<std::string, uint32_t>*)mi->h;
	if (h == 0) return -2;
	auto it = h->find(name);
	return it == h->end()? -1 : (int)it->second;
}

extern "C" int mm_idx_getseq(const mm_idx_t *mi, uint32_t rid, uint32_t st, uint32_t en, uint8_t *seq) // index.c:164-175
{
	if (rid >= mi->n_seq || st >= mi->seq[rid].len) return -1;
	if (en > mi->seq[rid].len) en = mi->seq[rid].len;
	const uint64_t st1 = mi->seq[rid].offset + st, en1 = mi->seq[rid].offset + en;
	uint64_t i = st1;
	for (; i < en1 && (i & 7); ++i) seq[i - st1] = (uint8_t)mmx_seq4_get(mi->S, i);
	const __m128i m0f = _mm_set1_epi8(0x0f);
	for (; i + 16 <= en1; i += 16) { // two 32-bit words = 16 bases: split the nibbles and interleave them back in order
		uint64_t w;
		memcpy(&w, &mi->S[i >> 3], 8);
		const __m128i v = _mm_cvtsi64_si128((long long)w);
		const __m128i lo = _mm_and_si128(v, m0f), hi = _mm_and_si128(_mm_srli_epi16(v, 4), m0f);
		_mm_storeu_si128((__m128i*)(seq + (i - st1)), _mm_unpacklo_epi8(lo, hi));
	}
	for (; i + 8 <= en1; i += 8) { // one 32-bit word = 8 bases
		uint32_t w = mi->S[i >> 3];
		uint8_t *o = seq + (i - st1);
		o[0] = w & 0xf, o[1] = w >> 4 & 0xf, o[2] = w >> 8 & 0xf, o[3] = w >> 12 & 0xf;
		o[4] = w >> 16 & 0xf, o[5] = w >> 20 & 0xf, o[6] = w >> 24 & 0xf, o[7] = w >> 28 & 0xf;
	}
	for (; i < en1; ++i) seq[i - st1] = (uint8_t)mmx_seq4_get(mi->S, i);
	return (int)(en - st);
}

extern "C" int32_t mm_idx_cal_max_occ(const mm_idx_t *mi, float f) // index.c:198-220
{
	mm_idx_bucket_s *B = mi->B;
	if (f <= 0.) return INT32_MAX;
	size_t n = (size_t)B->n_keys;
	if (n == 0) return INT32_MAX;
	uint32_t kk = (uint32_t)((1. - f) * n), v = 0;
	MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
	MMB_CUDA_CHECK(cudaMemcpy(&v, B->d_cnt_sorted + kk, 4, cudaMemcpyDeviceToHost)); // k-th smallest of the counts
	return (int32_t)(v + 1);
}

// pack ASCII into the 4-bit array (index.c:351-357)
static void pack_seq(uint32_t *S, uint64_t off, const char *s, uint32_t len)
{
	for (uint32_t j = 0; j < len; ++j) {
		uint64_t o = off + j;
		uint32_t c = mmx_nt4((uint8_t)s[j]);
		S[o >> 3] |= c << ((o & 7) << 2);
	}
}

extern "C" mm_idx_t *mm_idx_str(int w, int k, int is_hpc, int bucket_bits, int n, const char **seq, const char **name) // index.c:421-469
{
	uint64_t sum_len = 0;
	int flag = 0;
	if (n <= 0) return 0;
	for (int i = 0; i < n; ++i) sum_len += strlen(seq[i]);
	if (is_hpc) flag |= MM_I_HPC;
	if (name == 0) flag |= MM_I_NO_NAME;
	if (bucket_bits < 0) bucket_bits = 14;
	mm_idx_t *mi = idx_init(w, k, bucket_bits, flag);
	mi->n_seq = n;
	mi->seq = (mm_idx_seq_t*)calloc(n, sizeof(mm_idx_seq_t));
	mi->S = (uint32_t*)calloc((sum_len + 7) / 8 + 1, 4);
	sum_len = 0;
	for (int i = 0; i < n; ++i) {
		mm_idx_seq_t *p = &mi->seq[i];
		if (name && name[i]) p->name = strdup(name[i]);
		p->offset = sum_len, p->len = (uint32_t)strlen(seq[i]), p->is_alt = 0;
		pack_seq(mi->S, sum_len, seq[i], p->len);
		sum_len += p->len;
	}
	if (name) mm_idx_index_name(mi);
	mmb_idx_build_device(mi);
	return mi;
}

struct mm_bseq_file_s { FastxReader *rd; FastxRecord pending; bool has_pending; };

static mm_idx_t *idx_gen(mm_bseq_file_s *fp, int w, int k, int b, int flag, int64_t mini_batch_size, uint64_t batch_size) // index.c:389-408
{
	if (fp == 0 || fp->rd->eof()) return 0;
	mm_idx_t *mi = idx_init(w, k, b, flag);
	std::vector<mm_idx_seq_t> seqs;
	std::vector<uint32_t> S;
	uint64_t sum_len = 0;
	FastxRecord r;
	// the reference reads whole mini-batches (mm_bseq_read stops at the first record that brings the mini-batch to mini_batch_size bases,
	// bseq.c:80-119) and tests the running total only between them (index.c:322,326): a part ends at the first mini-batch boundary
	// past batch_size
	const uint64_t mbs = (uint64_t)mini_batch_size < batch_size? (uint64_t)mini_batch_size : batch_size;
	uint64_t in_mb = 0;
	for (;;) {
		if (in_mb >= mbs) { in_mb = 0; if (sum_len > batch_size) break; }
		int ret = fp->rd->next(r, false, false);
		if (ret <= 0) break;
		in_mb += r.seq.size();
		mm_idx_seq_t s;
		s.name = (flag & MM_I_NO_NAME)? 0 : strdup(r.name.c_str());
		s.len = (uint32_t)r.seq.size(), s.offset = sum_len, s.is_alt = 0;
		if (r.seq.empty() && mm_verbose >= 2) fprintf(stderr, "[WARNING] the length database sequence '%s' is 0\n", r.name.c_str());
		size_t need = (sum_len + s.len + 7) / 8 + 1;
		if (S.size() < need) S.resize(std::max(need, S.size() * 2), 0);
		pack_seq(S.data(), sum_len, r.seq.data(), s.len);
		sum_len += s.len;
		seqs.push_back(s);
	}
	mi->n_seq = (uint32_t)seqs.size();
	mi->seq = (mm_idx_seq_t*)calloc(seqs.size() + 1, sizeof(mm_idx_seq_t));
	memcpy(mi->seq, seqs.data(), seqs.size() * sizeof(mm_idx_seq_t));
	mi->S = (uint32_t*)calloc((sum_len + 7) / 8 + 1, 4);
	memcpy(mi->S, S.data(), ((sum_len + 7) / 8) * 4);
	if (mm_verbose >= 3) fprintf(stderr, "[M::%s::%.3f*%.2f] loaded %u sequences\n", __func__, realtime_now() - mm_realtime0, cputime_now() / (realtime_now() - mm_realtime0), mi->n_seq);
	mmb_idx_build_device(mi);
	if (mm_verbose >= 3) fprintf(stderr, "[M::%s::%.3f*%.2f] sorted minimizers (GPU)\n", __func__, realtime_now() - mm_realtime0, cputime_now() / (realtime_now() - mm_realtime0));
	return mi;
}

extern "C" mm_idx_t *mm_idx_build(const char *fn, int w, int k, int flag, int n_threads) // index.c:410-419
{
	(void)n_threads;
	mm_bseq_file_s fp;
	fp.rd = new FastxReader(fn); fp.has_pending = false;
	if (!fp.rd->ok()) { delete fp.rd; return 0; }
	mm_idx_t *mi = idx_gen(&fp, w, k, 14, flag, 1 << 18, UINT64_MAX); // index.c:417
	delete fp.rd;
	return mi;
}

// ---- .mmi I/O, byte-compatible with the reference reader/writer (index.c:475-569) ----
extern "C" void mm_idx_dump(FILE *fp, const mm_idx_t *mi)
{
	mm_idx_bucket_s *B = mi->B;
	mmb_idx_host_sync(mi);
	uint64_t sum_len = 0;
	uint32_t x[5];
	x[0] = mi->w, x[1] = mi->k, x[2] = mi->b, x[3] = mi->n_seq, x[4] = mi->flag;
	fwrite(MM_IDX_MAGIC, 1, 4, fp);
	fwrite(x, 4, 5, fp);
	for (uint32_t i = 0; i < mi->n_seq; ++i) {
		uint8_t l = mi->seq[i].name? (uint8_t)strlen(mi->seq[i].name) : 0;
		fwrite(&l, 1, 1, fp);
		if (l) fwrite(mi->seq[i].name, 1, l, fp);
		fwrite(&mi->seq[i].len, 4, 1, fp);
		sum_len += mi->seq[i].len;
	}
	// group keys by the low b bits (the reference's first-level bucket)
	const int b = mi->b;
	const uint64_t mask = (1ULL << b) - 1, nmask = (1ULL << MMB_IDX_NBITS) - 1;
	std::vector<uint32_t> bstart((size_t)(1ULL << b) + 1, 0);
	for (uint64_t key : B->h_keys) ++bstart[(key & mask) + 1];
	for (size_t i = 1; i < bstart.size(); ++i) bstart[i] += bstart[i - 1];
	std::vector<uint32_t> order(B->h_keys.size()), fill(bstart.begin(), bstart.end() - 1);
	for (size_t i = 0; i < B->h_keys.size(); ++i) order[fill[B->h_keys[i] & mask]++] = (uint32_t)i;
	std::vector<uint64_t> pbuf;
	for (uint64_t bi = 0; bi < (1ULL << b); ++bi) {
		int32_t np = 0;
		uint32_t size = bstart[bi + 1] - bstart[bi];
		pbuf.clear();
		for (uint32_t j = bstart[bi]; j < bstart[bi + 1]; ++j) {
			uint64_t v = B->h_val[order[j]], c = v & nmask;
			if (c > 1) { for (uint64_t t = 0; t < c; ++t) pbuf.push_back(B->h_pos[(v >> MMB_IDX_NBITS) + t]); np += (int32_t)c; }
		}
		fwrite(&np, 4, 1, fp);
		if (np) fwrite(pbuf.data(), 8, np, fp);
		fwrite(&size, 4, 1, fp);
		if (size == 0) continue;
		uint64_t start_p = 0;
		for (uint32_t j = bstart[bi]; j < bstart[bi + 1]; ++j) {
			uint64_t key = B->h_keys[order[j]], v = B->h_val[order[j]], c = v & nmask, kv[2];
			kv[0] = key >> b << 1;
			if (c == 1) kv[0] |= 1, kv[1] = B->h_pos[v >> MMB_IDX_NBITS];
			else kv[1] = start_p << 32 | c, start_p += c;
			fwrite(kv, 8, 2, fp);
		}
	}
	if (!(mi->flag & MM_I_NO_SEQ)) fwrite(mi->S, 4, (sum_len + 7) / 8, fp);
	fflush(fp);
}

extern "C" mm_idx_t *mm_idx_load(FILE *fp)
{
	char magic[4];
	uint32_t x[5];
	uint64_t sum_len = 0;
	if (fread(magic, 1, 4, fp) != 4) return 0;
	if (strncmp(magic, MM_IDX_MAGIC, 4) != 0) return 0;
	if (fread(x, 4, 5, fp) != 5) return 0;
	mm_idx_t *mi = idx_init(x[0], x[1], x[2], x[4]);
	mi->n_seq = x[3];
	mi->seq = (mm_idx_seq_t*)calloc(mi->n_seq + 1, sizeof(mm_idx_seq_t));
	for (uint32_t i = 0; i < mi->n_seq; ++i) {
		uint8_t l;
		mm_idx_seq_t *s = &mi->seq[i];
		if (fread(&l, 1, 1, fp) != 1) goto fail;
		if (l) {
			s->name = (char*)malloc(l + 1);
			if (fread(s->name, 1, l, fp) != l) goto fail;
			s->name[l] = 0;
		}
		if (fread(&s->len, 4, 1, fp) != 1) goto fail;
		s->offset = sum_len, s->is_alt = 0;
		sum_len += s->len;
	}
	{
		std::vector<uint64_t> keys, pos, p, kvbuf;
		std::vector<uint32_t> cnt;
		const int b = mi->b;
		for (uint64_t bi = 0; bi < (1ULL << b); ++bi) {
			int32_t np; uint32_t size;
			if (fread(&np, 4, 1, fp) != 1) goto fail;
			p.resize(np);
			if (np && fread(p.data(), 8, np, fp) != (size_t)np) goto fail;
			if (fread(&size, 4, 1, fp) != 1) goto fail;
			kvbuf.resize((size_t)size * 2); // the bucket's (key, value) pairs in one read
			if (size && fread(kvbuf.data(), 16, size, fp) != size) goto fail;
			for (uint32_t j = 0; j < size; ++j) {
				const uint64_t *kv = &kvbuf[(size_t)j * 2];
				keys.push_back((kv[0] >> 1) << b | bi);
				if (kv[0] & 1) cnt.push_back(1), pos.push_back(kv[1]);
				else {
					uint32_t c = (uint32_t)kv[1]; uint64_t o = kv[1] >> 32;
					cnt.push_back(c);
					for (uint32_t t = 0; t < c; ++t) pos.push_back(p[o + t]);
				}
			}
		}
		if (!(mi->flag & MM_I_NO_SEQ)) {
			mi->S = (uint32_t*)malloc(((sum_len + 7) / 8 + 1) * 4);
			if (fread(mi->S, 4, (sum_len + 7) / 8, fp) != (sum_len + 7) / 8) goto fail;
		}
		mmb_idx_build_from_lists(mi, keys, cnt, pos);
	}
	return mi;
fail:
	if (mm_verbose >= 1) fprintf(stderr, "[ERROR] truncated or corrupt index file\n");
	mm_idx_destroy(mi);
	return 0;
}

extern "C" int64_t mm_idx_is_idx(const char *fn) // index.c:571-593
{
	int fd, is_idx = 0;
	int64_t ret, off_end;
	char magic[4];
	if (strcmp(fn, "-") == 0) return 0;
	fd = open(fn, O_RDONLY);
	if (fd < 0) return -1;
	if ((off_end = lseek(fd, 0, SEEK_END)) >= 4) {
		lseek(fd, 0, SEEK_SET);
		ret = read(fd, magic, 4);
		if (ret == 4 && strncmp(magic, MM_IDX_MAGIC, 4) == 0) is_idx = 1;
	}
	close(fd);
	return is_idx? off_end : 0;
}

extern "C" void mm_idxopt_init(mm_idxopt_t *opt);

extern "C" mm_idx_reader_t *mm_idx_reader_open(const char *fn, const mm_idxopt_t *opt, const char *fn_out) // index.c:595-613
{
	int64_t is_idx = mm_idx_is_idx(fn);
	if (is_idx < 0) return 0;
	mm_idx_reader_t *r = (mm_idx_reader_t*)calloc(1, sizeof(mm_idx_reader_t));
	r->is_idx = (int)is_idx;
	if (opt) r->opt = *opt; else mm_idxopt_init(&r->opt);
	if (r->is_idx) {
		r->fp.idx = fopen(fn, "rb");
		r->idx_size = is_idx;
	} else {
		mm_bseq_file_s *f = new mm_bseq_file_s();
		f->rd = new FastxReader(fn); f->has_pending = false;
		if (!f->rd->ok()) { delete f->rd; delete f; free(r); return 0; }
		r->fp.seq = f;
	}
	if (fn_out) r->fp_out = fopen(fn_out, "wb");
	return r;
}

extern "C" void mm_idx_reader_close(mm_idx_reader_t *r) // index.c:615-621
{
	if (r->is_idx) fclose(r->fp.idx);
	else { delete r->fp.seq->rd; delete r->fp.seq; }
	if (r->fp_out) fclose(r->fp_out);
	free(r);
}

extern "C" mm_idx_t *mm_idx_reader_read(mm_idx_reader_t *r, int n_threads) // index.c:623-637
{
	(void)n_threads;
	mm_idx_t *mi;
	if (r->is_idx) {
		mi = mm_idx_load(r->fp.idx);
		if (mi && mm_verbose >= 2 && (mi->k != r->opt.k || mi->w != r->opt.w || (mi->flag&MM_I_HPC) != (r->opt.flag&MM_I_HPC)))
			fprintf(stderr, "[WARNING]\033[1;31m Indexing parameters (-k, -w or -H) overridden by parameters used in the prebuilt index.\033[0m\n");
	} else mi = idx_gen(r->fp.seq, r->opt.w, r->opt.k, r->opt.bucket_bits, r->opt.flag, r->opt.mini_batch_size, r->opt.batch_size);
	if (mi) {
		if (r->fp_out) mm_idx_dump(r->fp_out, mi);
		mi->index = r->n_parts++;
	}
	return mi;
}

extern "C" int mm_idx_reader_eof(const mm_idx_reader_t *r) // index.c:639-642
{
	return r->is_idx? (feof(r->fp.idx) || ftell(r->fp.idx) == r->idx_size) : r->fp.seq->rd->eof();
}

extern "C" int mm_idx_alt_read(mm_idx_t *mi, const char *fn) // index.c:648-670: one contig name per line (first token), plain or gzipped
{
	gzFile fp = fn && strcmp(fn, "-")? gzopen(fn, "r") : gzdopen(0, "r");
	if (fp == 0) return -1;
	if (mi->h == 0) mm_idx_index_name(mi);
	int n_alt = 0, c;
	std::string tok;
	bool in_tok = true; // still inside the first token of the current line
	auto flush = [&]() {
		const int id = mm_idx_name2id(mi, tok.c_str());
		if (id >= 0) mi->seq[id].is_alt = 1, ++n_alt;
		tok.clear(), in_tok = true;
	};
	bool any = false;
	while ((c = gzgetc(fp)) >= 0) {
		any = true;
		if (c == '\n') { flush(); any = false; }
		else if (in_tok) { if (isspace(c)) in_tok = false; else tok += (char)c; }
	}
	if (any) flush(); // last line without a newline
	gzclose(fp);
	mi->n_alt = n_alt;
	if (mm_verbose >= 3) fprintf(stderr, "[M::%s] found %d ALT contigs\n", __func__, n_alt);
	return n_alt;
}
// index.c:903-930 + the device copy K5 (jump.cuh) reads. Where the reference dereferences NULL (a file that cannot be opened), this
// returns -1 and leaves mi->J as it was.
extern "C" int mm_idx_jjump_read(mm_idx_t *mi, const char *fn, int flag, int min_sc)
{
	if (mi->h == 0) mm_idx_index_name(mi);
	mm_idx_intv_s *I = mmx_bed_read(fn, mi->n_seq, 1, min_sc, [&](const char *name) { return mm_idx_name2id(mi, name); }, nullptr, nullptr);
	if (I == 0) return -1;
	mm_idx_jjump_s *J = mmx_bed2jjump(I, mi->n_seq, (uint16_t)flag);
	for (uint32_t i = 0; i < mi->n_seq; ++i) free(I[i].a);
	free(I);
	mi->J = mi->J? mmx_jjump_merge(mi->J, J, mi->n_seq) : J;
	int64_t n_anno = 0, n_misc = 0;
	std::vector<int64_t> off((size_t)mi->n_seq + 1, 0);
	for (uint32_t i = 0; i < mi->n_seq; ++i) {
		for (int32_t j = 0; j < mi->J[i].n; ++j)
			if (mi->J[i].a[j].flag & MM_JUNC_ANNO) ++n_anno;
			else ++n_misc;
		off[i + 1] = off[i] + mi->J[i].n;
	}
	if (mm_verbose >= 3)
		fprintf(stderr, "[%s] there are %d annotated and %d other splice positions in the index\n", __func__, (int)n_anno, (int)n_misc);
	mm_idx_bucket_s *B = mi->B;
	if (B) {
		if (B->ctx) MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
		if (B->d_jump_off) { MMB_CUDA_CHECK(cudaFree(B->d_jump_off)); B->d_jump_off = nullptr, B->d_jump = nullptr; }
		const size_t n = (size_t)off[mi->n_seq], head = ((size_t)mi->n_seq + 1) * 8;
		MMB_CUDA_CHECK(cudaMalloc((void**)&B->d_jump_off, head + n * sizeof(mm_idx_jjump1_t) + 16));
		B->d_jump = (mm_idx_jjump1_t*)((uint8_t*)B->d_jump_off + head);
		MMB_CUDA_CHECK(cudaMemcpy(B->d_jump_off, off.data(), head, cudaMemcpyHostToDevice));
		for (uint32_t i = 0; i < mi->n_seq; ++i)
			if (mi->J[i].n) MMB_CUDA_CHECK(cudaMemcpy(B->d_jump + off[i], mi->J[i].a, sizeof(mm_idx_jjump1_t) * mi->J[i].n, cudaMemcpyHostToDevice));
	}
	return 0;
}
// index.c:946-959
extern "C" const mm_idx_jjump1_t *mm_idx_jump_get(const mm_idx_t *mi, int32_t cid, int32_t st, int32_t en, int32_t *n)
{
	*n = 0;
	if (cid >= (int32_t)mi->n_seq || cid < 0 || mi->J == 0) return 0;
	return mmx_jump_get(mi->J[cid].n, mi->J[cid].a, (int32_t)mi->seq[cid].len, st, en, n);
}
// index.c:796-800 + the device copy the spliced kernel reads: introns of all contigs in global S coordinates, sorted by start
extern "C" int mm_idx_bed_read(mm_idx_t *mi, const char *fn, int read_junc)
{
	if (mi->h == 0) mm_idx_index_name(mi);
	long n0 = 0, n = 0;
	if (mi->I) { for (uint32_t i = 0; i < mi->n_seq; ++i) free(mi->I[i].a); free(mi->I); mi->I = 0; }
	mi->I = mmx_bed_read(fn, mi->n_seq, read_junc, -1, [&](const char *name) { return mm_idx_name2id(mi, name); }, &n0, &n);
	mm_idx_bucket_s *B = mi->B;
	if (B) {
		if (B->ctx) MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
		if (B->d_junc) { MMB_CUDA_CHECK(cudaFree(B->d_junc)); B->d_junc = nullptr; }
		B->n_junc = 0;
	}
	if (mi->I == 0) return 0;
	if (mm_verbose >= 3) fprintf(stderr, "[%s] read %ld introns, %ld of which are non-redundant\n", __func__, n0, n);
	if (B && n > 0) {
		std::vector<int64_t> h((size_t)n * 2 + ((size_t)n + 7) / 8);
		int8_t *hs = (int8_t*)(h.data() + (size_t)n * 2);
		int64_t k = 0;
		for (uint32_t i = 0; i < mi->n_seq; ++i)
			for (int32_t j = 0; j < mi->I[i].n; ++j, ++k) {
				const mm_idx_intv1_t &t = mi->I[i].a[j];
				h[k] = (int64_t)mi->seq[i].offset + t.st, h[n + k] = (int64_t)mi->seq[i].offset + t.en, hs[k] = (int8_t)t.strand;
			}
		MMB_CUDA_CHECK(cudaMalloc((void**)&B->d_junc, h.size() * 8));
		MMB_CUDA_CHECK(cudaMemcpy(B->d_junc, h.data(), h.size() * 8, cudaMemcpyHostToDevice));
		B->n_junc = n;
	}
	return 0;
}
extern "C" int mm_idx_bed_junc(const mm_idx_t *mi, int32_t ctg, int32_t st, int32_t en, uint8_t *s) { return mmx_bed_junc(mi->I, (int32_t)mi->n_seq, ctg, st, en, s); }
// index.c:968-1040 + the device copy the spliced kernel reads: per strand, one entry per position (the largest byte, which is what
// the reference's in-window scan keeps), in global S coordinates
extern "C" int32_t mm_idx_spsc_read2(mm_idx_t *mi, const char *fn, int32_t max_sc, float scale)
{
	if (mi->h == 0) mm_idx_index_name(mi);
	if (mi->spsc) { for (uint32_t i = 0; i < mi->n_seq * 2; ++i) free(mi->spsc[i].a); free(mi->spsc); mi->spsc = 0; }
	long n_read = 0;
	mi->spsc = mmx_spsc_read(fn, mi->n_seq, max_sc, scale, [&](const char *name) { return mm_idx_name2id(mi, name); }, [&](int cid) { return mi->seq[cid].len; }, &n_read);
	mm_idx_bucket_s *B = mi->B;
	if (B) {
		if (B->ctx) MMB_CUDA_CHECK(cudaSetDevice(B->ctx->device));
		for (int t = 0; t < 2; ++t) { if (B->d_spsc[t]) MMB_CUDA_CHECK(cudaFree(B->d_spsc[t])); B->d_spsc[t] = nullptr, B->n_spsc[t] = 0; }
	}
	if (mi->spsc == 0) return -1;
	if (mm_verbose >= 3) fprintf(stderr, "[M::%s] read %ld splice scores\n", __func__, n_read);
	for (int t = 0; B && t < 2; ++t) {
		std::vector<int64_t> pos; std::vector<uint8_t> val;
		for (uint32_t i = 0; i < mi->n_seq; ++i) {
			const mm_idx_spsc_s *s = &mi->spsc[i << 1 | t];
			for (uint32_t j = 0; j < s->n; ++j) {
				const int64_t p = (int64_t)mi->seq[i].offset + (int64_t)(s->a[j] >> 8);
				const uint8_t v = (uint8_t)(s->a[j] & 0xff);
				if (!pos.empty() && pos.back() == p) { if (val.back() == 0xff || val.back() < v) val.back() = v; } // index.c:1070
				else pos.push_back(p), val.push_back(v);
			}
		}
		if (pos.empty()) continue;
		const size_t n = pos.size();
		MMB_CUDA_CHECK(cudaMalloc((void**)&B->d_spsc[t], n * 9 + 64));
		MMB_CUDA_CHECK(cudaMemcpy(B->d_spsc[t], pos.data(), n * 8, cudaMemcpyHostToDevice));
		MMB_CUDA_CHECK(cudaMemcpy(B->d_spsc[t] + n * 8, val.data(), n, cudaMemcpyHostToDevice));
		B->n_spsc[t] = (int64_t)n;
	}
	return 0;
}
extern "C" int32_t mm_idx_spsc_read(mm_idx_t *mi, const char *fn, int32_t max_sc) { return mm_idx_spsc_read2(mi, fn, max_sc, 1.0f); }
extern "C" int64_t mm_idx_spsc_get(const mm_idx_t *mi, int32_t cid, int64_t st0, int64_t en0, int32_t rev, uint8_t *sc) // index.c:1055-1075
{
	return mmx_spsc_get(mi->spsc, (int32_t)mi->n_seq, cid, cid >= 0 && cid < (int32_t)mi->n_seq? (int64_t)mi->seq[cid].len : 0, st0, en0, rev, sc);
}

// ---------------------------------------------------------------------------------------------------------
// Multi-GPU: the device index is replicated, not sharded (reads shard; SURVEY 8e). Rank 0 exports the device arrays,
// torch.distributed (NCCL over NVLink) broadcasts them into buffers on the other ranks, which adopt them here.
// ---------------------------------------------------------------------------------------------------------

extern "C" void mmb_idx_export(const mm_idx_t *mi, mmb_idx_desc_t *d)
{
	mm_idx_bucket_s *B = mi->B;
	uint64_t sum_len = 0;
	for (uint32_t i = 0; i < mi->n_seq; ++i) sum_len += mi->seq[i].len;
	d->ptr[0] = B->d_tab, d->bytes[0] = sizeof(IdxSlot) << B->tab_bits;
	d->ptr[1] = B->d_pos, d->bytes[1] = 8ull * (uint64_t)(B->n_pos + 1);
	d->ptr[2] = B->d_S, d->bytes[2] = ((sum_len + 7) / 8 + 4) * 4;
	d->ptr[3] = B->d_seq_off, d->bytes[3] = 8ull * (mi->n_seq + 1);
	d->ptr[4] = B->d_seq_len, d->bytes[4] = 4ull * (mi->n_seq + 1);
	d->n_keys = B->n_keys, d->n_pos = B->n_pos, d->tab_bits = B->tab_bits;
	d->w = mi->w, d->k = mi->k, d->b = mi->b, d->flag = mi->flag, d->n_seq = mi->n_seq, d->sum_len = sum_len;
}

// Build an mm_idx_t around device buffers that already hold a broadcast copy (the buffers stay owned by the caller and
// must outlive the index). names: n_seq NUL-terminated strings; lens: n_seq lengths. The host 4-bit S is copied back
// from the device for the host-side alignment driver.
extern "C" mm_idx_t *mmb_idx_adopt(const mmb_idx_desc_t *d, const char **names, const uint32_t *lens, const uint32_t *cnt_sorted_dev)
{
	mmb_ctx_t *ctx = mmb_default_ctx();
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	mm_idx_t *mi = (mm_idx_t*)calloc(1, sizeof(mm_idx_t));
	mi->w = d->w, mi->k = d->k, mi->b = d->b, mi->flag = d->flag, mi->n_seq = d->n_seq;
	mi->B = new mm_idx_bucket_s();
	mm_idx_bucket_s *B = mi->B;
	B->ctx = ctx, B->external = true;
	B->d_tab = (IdxSlot*)d->ptr[0], B->tab_bits = d->tab_bits, B->d_pos = (uint64_t*)d->ptr[1], B->d_S = (uint32_t*)d->ptr[2];
	B->d_seq_off = (uint64_t*)d->ptr[3], B->d_seq_len = (uint32_t*)d->ptr[4];
	B->n_keys = d->n_keys, B->n_pos = d->n_pos;
	B->d_cnt_sorted = (uint32_t*)cnt_sorted_dev;
	mi->seq = (mm_idx_seq_t*)calloc(d->n_seq + 1, sizeof(mm_idx_seq_t));
	uint64_t off = 0;
	for (uint32_t i = 0; i < d->n_seq; ++i) {
		mi->seq[i].name = names && names[i]? strdup(names[i]) : 0;
		mi->seq[i].len = lens[i], mi->seq[i].offset = off, off += lens[i];
	}
	mi->S = (uint32_t*)calloc((d->sum_len + 7) / 8 + 1, 4);
	MMB_CUDA_CHECK(cudaMemcpy(mi->S, B->d_S, ((d->sum_len + 7) / 8) * 4, cudaMemcpyDeviceToHost));
	mm_idx_index_name(mi);
	return mi;
}

extern "C" const void *mmb_idx_cnt_sorted(const mm_idx_t *mi, uint64_t *bytes)
{
	*bytes = 4ull * (uint64_t)(mi->B->n_keys + 1);
	return mi->B->d_cnt_sorted;
}
