// minimap2_b200/csrc/mmb_ctx.cu -- device context + kernel-level C-ABI entry points with host buffers (mm_b200.h).
#include "mmb_internal.h"
#include <cstring>
#include <ctime>

int mm_verbose_dummy_anchor = 0;

extern "C" int mmb_device_count(void)
{
	int n = 0;
	cudaError_t err = cudaGetDeviceCount(&n);
	if (err != cudaSuccess) {
		fprintf(stderr, "[ERROR] minimap2_b200: no usable CUDA device (%s); there is no CPU fallback\n", cudaGetErrorString(err));
		return -1;
	}
	return n;
}

bool g_mmb_tl_on = false;
double mmb_tl_now()
{
	timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}
extern "C" void mmb_timeline_enable(int on) { g_mmb_tl_on = on != 0; }
extern "C" double mmb_timeline_now(void) { return mmb_tl_now(); }

#include <mutex>
static std::vector<mmb_ctx_t*> g_all_ctx;
static std::mutex g_all_mu;
void mmb_register_ctx(mmb_ctx_t *c) { std::lock_guard<std::mutex> lk(g_all_mu); g_all_ctx.push_back(c); }

extern "C" mmb_ctx_t *mmb_ctx_create(int device)
{
	int n = mmb_device_count();
	if (n <= 0 || device < 0 || device >= n) {
		fprintf(stderr, "[ERROR] minimap2_b200: cannot create a context on device %d (%d visible)\n", device, n);
		return nullptr;
	}
	mmb_ctx_t *c = new mmb_ctx_t();
	c->device = device;
	MMB_CUDA_CHECK(cudaSetDevice(device));
	cudaDeviceProp prop;
	MMB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
	c->n_sm = prop.multiProcessorCount;
	c->smem_optin = prop.sharedMemPerBlockOptin;
	MMB_CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	MMB_CUDA_CHECK(cudaEventCreate(&c->ev0));
	MMB_CUDA_CHECK(cudaEventCreate(&c->ev1));
	MMB_CUDA_CHECK(cudaEventCreate(&c->ev_sync));
	return c;
}

extern "C" void mmb_ctx_destroy(mmb_ctx_t *c)
{
	if (!c) return;
	cudaSetDevice(c->device);
	cudaStreamSynchronize(c->stream);
	c->d_a.release(); c->d_b.release(); c->d_c.release(); c->d_d.release();
	c->d_e.release(); c->d_f.release(); c->d_g.release(); c->d_h.release(); c->sk_pk.release(); c->sk_nm.release(); c->sk_misc.release(); c->scan_sums.release(); c->d_junc.release(); c->d_spsc[0].release(); c->d_spsc[1].release();
	cudaEventDestroy(c->ev0); cudaEventDestroy(c->ev1); cudaEventDestroy(c->ev_sync);
	cudaStreamDestroy(c->stream);
	delete c;
}

extern "C" void *mmb_ctx_stream(mmb_ctx_t *c) { return (void*)c->stream; }

// Splice scores for MMB_JOB_SPLICE jobs carrying MMB_KSW_SPLICE_SCORE (host arrays; pos strictly ascending, in the coordinates of
// the target array; val = (score+64)<<1 | acceptor). strand 0: jobs without MMB_KSW_SPLICE_REV, 1: with. n = 0 clears the table.
extern "C" int mmb_ctx_set_splice_scores(mmb_ctx_t *c, int strand, int64_t n, const int64_t *pos, const uint8_t *val)
{
	if (strand < 0 || strand > 1) return -1;
	MMB_CUDA_CHECK(cudaSetDevice(c->device));
	MMB_CUDA_CHECK(cudaStreamSynchronize(c->stream));
	c->spsc_pos[strand] = nullptr, c->spsc_val[strand] = nullptr, c->n_spsc[strand] = 0;
	if (n <= 0) return 0;
	for (int64_t i = 1; i < n; ++i) if (pos[i] <= pos[i - 1]) return -1;
	uint8_t *d = (uint8_t*)c->d_spsc[strand].reserve((size_t)n * 9 + 64);
	MMB_CUDA_CHECK(cudaMemcpy(d, pos, (size_t)n * 8, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(d + (size_t)n * 8, val, (size_t)n, cudaMemcpyHostToDevice));
	c->spsc_pos[strand] = (const int64_t*)d, c->spsc_val[strand] = d + (size_t)n * 8, c->n_spsc[strand] = n;
	return 0;
}

// Annotated introns for MMB_JOB_SPLICE jobs of the kernel-level entry points (host arrays, sorted by st; coordinates index the
// target array passed to mmb_ksw_batch_host). n = 0 removes the annotation.
extern "C" int mmb_ctx_set_junctions(mmb_ctx_t *c, int64_t n, const int64_t *st, const int64_t *en, const int8_t *strand)
{
	MMB_CUDA_CHECK(cudaSetDevice(c->device));
	MMB_CUDA_CHECK(cudaStreamSynchronize(c->stream));
	c->junc_st = c->junc_en = nullptr, c->junc_strand = nullptr, c->n_junc = 0;
	if (n <= 0) return 0;
	for (int64_t i = 1; i < n; ++i) if (st[i] < st[i - 1]) return -1;
	uint8_t *d = (uint8_t*)c->d_junc.reserve((size_t)n * 17 + 64);
	MMB_CUDA_CHECK(cudaMemcpy(d, st, (size_t)n * 8, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(d + (size_t)n * 8, en, (size_t)n * 8, cudaMemcpyHostToDevice));
	MMB_CUDA_CHECK(cudaMemcpy(d + (size_t)n * 16, strand, (size_t)n, cudaMemcpyHostToDevice));
	c->junc_st = (const int64_t*)d, c->junc_en = (const int64_t*)(d + (size_t)n * 8), c->junc_strand = (const int8_t*)(d + (size_t)n * 16), c->n_junc = n;
	return 0;
}

extern "C" uint64_t mmb_launch_count(mmb_ctx_t *c, int reset)
{
	uint64_t n = c->n_launch;
	if (reset) c->n_launch = 0;
	return n;
}

extern "C" void mmb_profile_enable(mmb_ctx_t *c, int on) { c->profiling = on; }
extern "C" double mmb_profile_ms(mmb_ctx_t *c, int which, int reset)
{
	if (which < 0 || which >= MMB_PROF_N) return 0.0;
	if (!c->ev_pending[which].empty()) { // resolve queued event pairs
		MMB_CUDA_CHECK(cudaStreamSynchronize(c->stream));
		for (auto &pr : c->ev_pending[which]) {
			float ms = 0;
			MMB_CUDA_CHECK(cudaEventElapsedTime(&ms, pr.first, pr.second));
			c->prof_ms[which] += ms;
			++c->prof_launches[which];
			c->ev_pool.push_back(pr.first); c->ev_pool.push_back(pr.second);
		}
		c->ev_pending[which].clear();
	}
	double v = c->prof_ms[which];
	if (reset) c->prof_ms[which] = 0;
	return v;
}
extern "C" uint64_t mmb_profile_units(mmb_ctx_t *c, int which, int reset)
{
	if (which < 0 || which >= MMB_PROF_N) return 0;
	uint64_t v = c->prof_units[which];
	if (reset) c->prof_units[which] = 0;
	return v;
}

extern "C" int64_t mmb_ksw_batch_host(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *jobs,
									  const uint8_t *query, int64_t query_len, const uint8_t *target, int64_t target_len,
									  mmb_ksw_res_t *res, uint32_t *cigar_buf, int64_t cigar_cap)
{
	if (n_jobs <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	uint8_t *d_q = ctx->d_a.as<uint8_t>(query_len + 16), *d_t = ctx->d_b.as<uint8_t>(target_len + 16);
	mmb_ksw_job_t *d_jobs = ctx->d_c.as<mmb_ksw_job_t>(n_jobs);
	mmb_ksw_res_t *d_res = ctx->d_d.as<mmb_ksw_res_t>(n_jobs);
	uint32_t *d_cig = (uint32_t*)ctx->d_h.reserve((size_t)(cigar_cap + 2) * 4 + 16);
	unsigned long long *d_used = (unsigned long long*)(d_cig); // first 8 bytes: counter; ops start at +2
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_q, query, query_len, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_t, target, target_len, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_jobs, jobs, sizeof(mmb_ksw_job_t) * n_jobs, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemsetAsync(d_used, 0, 8, ctx->stream));
	mmb_ksw_launch(ctx, sc, n_jobs, jobs, d_jobs, d_q, d_t, 0, d_res, d_cig + 2, cigar_cap, d_used);
	unsigned long long used = 0;
	MMB_CUDA_CHECK(cudaMemcpyAsync(res, d_res, sizeof(mmb_ksw_res_t) * n_jobs, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(&used, d_used, 8, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	if ((int64_t)used > cigar_cap) return -(int64_t)used;
	MMB_CUDA_CHECK(cudaMemcpyAsync(cigar_buf, d_cig + 2, used * 4, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return (int64_t)used;
}

mmb_ctx_t *mmb_default_ctx(void);
extern "C" void *mmb_default_ctx_c(void) { return (void*)mmb_default_ctx(); }
extern "C" void mmb_free(void *p) { free(p); }

extern "C" uint64_t mmb_profile_scopes(mmb_ctx_t *c, int which, int reset)
{
	if (which < 0 || which >= MMB_PROF_N) return 0;
	mmb_profile_ms(c, which, 0);
	uint64_t v = c->prof_launches[which];
	if (reset) c->prof_launches[which] = 0;
	return v;
}

extern "C" uint64_t mmb_profile_bytes(mmb_ctx_t *c, int which, int reset)
{
	if (which < 0 || which >= MMB_PROF_N) return 0;
	uint64_t v = c->prof_bytes[which];
	if (reset) c->prof_bytes[which] = 0;
	return v;
}
static int g_resident_reads = 0;
extern "C" void mmb_set_resident_reads(int on) { g_resident_reads = on; }
int mmb_resident_reads(void) { return g_resident_reads; }
extern "C" uint64_t mmb_last_d2h_bytes_all(void);
extern "C" uint64_t mmb_last_d2h_bytes(void) { return mmb_last_d2h_bytes_all(); }

// aggregated over every context of this process (default context + the scheduler's group contexts); which as in mmb_profile_ms
extern "C" void mmb_profile_enable_all(int on)
{
	mmb_default_ctx()->profiling = on;
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) c->profiling = on;
}
extern "C" double mmb_profile_ms_all(int which, int reset)
{
	double v = mmb_profile_ms(mmb_default_ctx(), which, reset);
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += mmb_profile_ms(c, which, reset);
	return v;
}
extern "C" uint64_t mmb_profile_units_all(int which, int reset)
{
	uint64_t v = mmb_profile_units(mmb_default_ctx(), which, reset);
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += mmb_profile_units(c, which, reset);
	return v;
}
extern "C" uint64_t mmb_profile_bytes_all(int which, int reset)
{
	uint64_t v = mmb_profile_bytes(mmb_default_ctx(), which, reset);
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += mmb_profile_bytes(c, which, reset);
	return v;
}
extern "C" uint64_t mmb_profile_scopes_all(int which, int reset)
{
	uint64_t v = mmb_profile_scopes(mmb_default_ctx(), which, reset);
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += mmb_profile_scopes(c, which, reset);
	return v;
}
extern "C" uint64_t mmb_launch_count_all(int reset)
{
	uint64_t v = mmb_launch_count(mmb_default_ctx(), reset);
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += mmb_launch_count(c, reset);
	return v;
}
extern "C" uint64_t mmb_last_d2h_bytes_all(void)
{
	uint64_t v = mmb_default_ctx()->last_d2h_bytes;
	std::lock_guard<std::mutex> lk(g_all_mu);
	for (auto *c : g_all_ctx) v += c->last_d2h_bytes;
	return v;
}
