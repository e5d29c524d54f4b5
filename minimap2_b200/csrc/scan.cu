// minimap2_b200/csrc/scan.cu -- three-phase exclusive scan (tile sums -> scan of sums -> add), int64.
#include "scan.cuh"
#include "mm_algo.cuh"

namespace {
const int TILE = 2048;      // elements per CTA (256 threads x 8)

__device__ __forceinline__ int64_t block_exclusive(int64_t v, int64_t *total, int64_t *sh)
{
	// 256-thread exclusive scan of one value per thread via warp shuffles
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	int64_t x = v;
	for (int o = 1; o < 32; o <<= 1) { int64_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
	if (lane == 31) sh[wid] = x;
	__syncthreads();
	if (wid == 0) {
		int64_t s = lane < 8? sh[lane] : 0;
		for (int o = 1; o < 8; o <<= 1) { int64_t y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
		if (lane < 8) sh[lane] = s;
	}
	__syncthreads();
	int64_t off = wid > 0? sh[wid - 1] : 0;
	*total = sh[7];
	__syncthreads();
	return off + x - v;
}

__global__ void __launch_bounds__(256) scan_tile_kernel(int64_t *d, int64_t n, int64_t *tile_sum, int phase)
{
	__shared__ int64_t sh[8];
	const int64_t t0 = (int64_t)blockIdx.x * TILE + threadIdx.x * 8;
	int64_t v[8], s = 0;
	#pragma unroll
	for (int i = 0; i < 8; ++i) { v[i] = t0 + i < n? d[t0 + i] : 0; s += v[i]; }
	int64_t total, ex = block_exclusive(s, &total, sh);
	if (phase == 0) { if (threadIdx.x == 0) tile_sum[blockIdx.x] = total; return; }
	int64_t run = ex + tile_sum[blockIdx.x];
	#pragma unroll
	for (int i = 0; i < 8; ++i) { if (t0 + i < n) d[t0 + i] = run; run += v[i]; }
}

__global__ void __launch_bounds__(256) scan_sums_kernel(int64_t *tile_sum, int64_t n_tiles, int64_t *d, int64_t n)
{
	// single CTA: exclusive scan of tile sums (sequential over blocks of 256)
	__shared__ int64_t sh[8];
	__shared__ int64_t carry;
	if (threadIdx.x == 0) carry = 0;
	__syncthreads();
	for (int64_t b = 0; b < n_tiles; b += 256) {
		int64_t i = b + threadIdx.x, v = i < n_tiles? tile_sum[i] : 0, total;
		int64_t ex = block_exclusive(v, &total, sh);
		if (i < n_tiles) tile_sum[i] = ex + carry;
		__syncthreads();
		if (threadIdx.x == 0) carry += total;
		__syncthreads();
	}
	if (threadIdx.x == 0 && d) d[n] = carry;
}

__global__ void stk_len_kernel(const int64_t *a_off, int n_reads, int64_t *stk_off)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n_reads) stk_off[i] = mmx_rs_stack_len(a_off[i + 1] - a_off[i]);
}
} // namespace

void mmb_exclusive_scan_i64_async(mmb_ctx_t *ctx, int64_t *d, int64_t n)
{
	if (n <= 0) { MMB_CUDA_CHECK(cudaMemsetAsync(d, 0, sizeof(int64_t), ctx->stream)); return; }
	const int64_t n_tiles = (n + TILE - 1) / TILE;
	DevBuf &sums = ctx->scan_sums;
	int64_t *ts = sums.as<int64_t>((size_t)n_tiles + 1);
	scan_tile_kernel<<<(unsigned)n_tiles, 256, 0, ctx->stream>>>(d, n, ts, 0);
	scan_sums_kernel<<<1, 256, 0, ctx->stream>>>(ts, n_tiles, d, n);
	scan_tile_kernel<<<(unsigned)n_tiles, 256, 0, ctx->stream>>>(d, n, ts, 1);
	MMB_CUDA_CHECK(cudaGetLastError());
	ctx->n_launch += 3;
}

int64_t *mmb_sort_stacks_async(mmb_ctx_t *ctx, const int64_t *a_off, int n_reads, int64_t n_tot, DevBuf &buf, size_t head_bytes)
{
	const size_t n_stk = (size_t)n_tot / 65 * 24 + (size_t)n_reads * 48 + 64; // >= the sum of mmx_rs_stack_len over the reads
	int64_t *stk_off = (int64_t*)((uint8_t*)buf.reserve(head_bytes + ((size_t)n_reads + 1) * 8 + n_stk * 4) + head_bytes);
	stk_len_kernel<<<(n_reads + 255) / 256, 256, 0, ctx->stream>>>(a_off, n_reads, stk_off);
	++ctx->n_launch;
	mmb_exclusive_scan_i64_async(ctx, stk_off, n_reads);
	return stk_off;
}

int64_t mmb_exclusive_scan_i64(mmb_ctx_t *ctx, int64_t *d, int64_t n, bool with_total)
{
	(void)with_total;
	mmb_exclusive_scan_i64_async(ctx, d, n);
	int64_t total = 0;
	MMB_CUDA_CHECK(cudaMemcpyAsync(&total, d + (n > 0? n : 0), sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
	mmb_stream_sync(ctx);
	return total;
}
