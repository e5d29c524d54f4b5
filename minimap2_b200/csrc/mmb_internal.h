// minimap2_b200/csrc/mmb_internal.h -- internal declarations shared by the CUDA translation units.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <utility>
#include <chrono>
#include <thread>
#include "mm_b200.h"

extern "C" int mm_verbose;

#define MMB_CUDA_CHECK(expr) do { \
	cudaError_t err__ = (expr); \
	if (err__ != cudaSuccess) { \
		fprintf(stderr, "[ERROR] CUDA failure '%s' at %s:%d: %s\n", #expr, __FILE__, __LINE__, cudaGetErrorString(err__)); \
		abort(); \
	} } while (0)

enum { MMB_PROF_SKETCH = 0, MMB_PROF_SEED = 1, MMB_PROF_SORT = 2, MMB_PROF_CHAIN = 3, MMB_PROF_KSW = 4, MMB_PROF_OTHER = 5, MMB_PROF_N = 6 };

// A grow-only device buffer (arena slice): avoids cudaMalloc on the per-batch path.
struct DevBuf {
	void *p = nullptr;
	size_t cap = 0;
	void *reserve(size_t bytes) {
		if (bytes > cap) {
			if (p) MMB_CUDA_CHECK(cudaFree(p));
			size_t ncap = bytes + (bytes > ((size_t)64 << 20)? bytes >> 3 : bytes >> 2) + 256; // growth headroom: 1/8 for the large arenas (twelve groups own a set each), 1/4 below 64 MB
			MMB_CUDA_CHECK(cudaMalloc(&p, ncap));
			cap = ncap;
		}
		return p;
	}
	template<class T> T *as(size_t n) { return (T*)reserve(n * sizeof(T)); }
	void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct PinBuf { // pinned host staging buffer
	void *p = nullptr;
	size_t cap = 0;
	void *reserve(size_t bytes) {
		if (bytes > cap) {
			if (p) MMB_CUDA_CHECK(cudaFreeHost(p));
			size_t ncap = bytes + (bytes >> 2) + 256;
			MMB_CUDA_CHECK(cudaMallocHost(&p, ncap));
			cap = ncap;
		}
		return p;
	}
	template<class T> T *as(size_t n) { return (T*)reserve(n * sizeof(T)); }
	void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

struct mmb_ctx_s {
	int device = 0;
	int group_id = 0;
	int n_sm = 0;
	size_t smem_optin = 0;
	cudaStream_t stream = nullptr;
	uint64_t n_launch = 0;
	int profiling = 0;
	double prof_ms[MMB_PROF_N] = {0};
	uint64_t prof_units[MMB_PROF_N] = {0};
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	std::vector<cudaEvent_t> ev_pool;
	std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pending[MMB_PROF_N];
	uint64_t prof_launches[MMB_PROF_N] = {0};
	uint64_t prof_bytes[MMB_PROF_N] = {0};   // algorithmic bytes (SURVEY 8d definitions)
	uint64_t last_d2h_bytes = 0, last_h2d_bytes = 0;
	// scratch used by the kernel-level host entry points
	DevBuf d_a, d_b, d_c, d_d, d_e, d_f, d_g, d_h;
	DevBuf sk_pk, sk_nm, sk_misc, scan_sums;   // stage scratch that lives with the context (2-bit bases / ambiguity bits / tile chaining of K1; tile sums of the scans)
	// annotated introns for the spliced kernel (mm_idx_bed_junc semantics, index.c:802-826), sorted by start, in the coordinates
	// of the target array the jobs address: first base, one past the last base, strand (+1/-1). Null: no annotation.
	const int64_t *junc_st = nullptr, *junc_en = nullptr; const int8_t *junc_strand = nullptr; int64_t n_junc = 0;
	DevBuf d_junc;                            // backing store when set through mmb_ctx_set_junctions
	// splice scores (mm_idx_spsc_get semantics, index.c:1055-1075), one table per strand [0: '+', 1: '-']: positions (sorted, one
	// entry per position: the largest byte) in target coordinates and their bytes (score+64)<<1 | acceptor
	const int64_t *spsc_pos[2] = {nullptr, nullptr}; const uint8_t *spsc_val[2] = {nullptr, nullptr}; int64_t n_spsc[2] = {0, 0};
	DevBuf d_spsc[2];
	std::vector<double> tl;                   // scheduler timeline of the current batch: (time, event, argument) triples, see mmb_tl
	cudaEvent_t ev_sync = nullptr;            // the event mmb_stream_sync polls
	bool sleepy_sync = false;                 // mmb_stream_sync sleeps between polls (a scheduler group running next to others)
};

// Scheduler timeline (mmb_timeline_enable): the host clock (CLOCK_MONOTONIC, seconds) at each phase boundary of a group's batch.
// Recording takes no lock and never synchronises, so the schedule it observes is the one that runs without it.
enum {
	MMB_TL_GATE_REQ = 0,   // argument: gate class (0 stage 1, 1 alignment wave)
	MMB_TL_GATE_GRANT = 1, // argument: gate class
	MMB_TL_GATE_REL = 2,   // argument: gate class
	MMB_TL_ENQUEUED = 3,   // the device work of a phase is on the stream; argument: 0 stage 1, 1 wave chunk, 2 device tail
	MMB_TL_SYNC = 4,       // a stream synchronise returned
	MMB_TL_HOST_BEGIN = 5, // argument: host phase (map.cu, HostPhase)
	MMB_TL_HOST_END = 6,
};
extern bool g_mmb_tl_on;
double mmb_tl_now();
inline void mmb_tl(mmb_ctx_t *c, int ev, int arg = 0)
{
	if (g_mmb_tl_on) c->tl.push_back(mmb_tl_now()), c->tl.push_back(ev), c->tl.push_back(arg);
}
// Waits until the work on the context's stream is done, recorded on the timeline. A scheduler group that runs next to others
// (sleepy_sync) sleeps between polls instead of spinning as cudaStreamSynchronize does: the groups that hold a device slot wait here
// most of the time, and spinning threads would take the host CPUs the other groups' host phases run on. A wait then ends up to
// about 1 ms late (measured on an H100 host), which the concurrent groups cover; a context running alone spins, so that the
// per-kernel CUDA-event times of a serialised run do not take in the late wake-ups.
inline void mmb_stream_sync(mmb_ctx_t *c)
{
	if (c->sleepy_sync) {
		MMB_CUDA_CHECK(cudaEventRecord(c->ev_sync, c->stream));
		cudaError_t st;
		while ((st = cudaEventQuery(c->ev_sync)) == cudaErrorNotReady) std::this_thread::sleep_for(std::chrono::microseconds(20));
		MMB_CUDA_CHECK(st);
	} else MMB_CUDA_CHECK(cudaStreamSynchronize(c->stream));
	mmb_tl(c, MMB_TL_SYNC);
}

// Timing of one kernel family on the ctx stream with CUDA events (only when profiling is enabled). Asynchronous: the event
// pairs are queued and resolved by mmb_profile_ms(), so enabling profiling does not serialise the pipeline.
struct ProfScope {
	mmb_ctx_t *c; int which; cudaEvent_t e0 = nullptr, e1 = nullptr;
	ProfScope(mmb_ctx_t *ctx, int w, uint64_t units) : c(ctx), which(w) {
		if (c->profiling) {
			c->prof_units[w] += units;
			if (!c->ev_pool.empty()) { e0 = c->ev_pool.back(); c->ev_pool.pop_back(); } else MMB_CUDA_CHECK(cudaEventCreate(&e0));
			if (!c->ev_pool.empty()) { e1 = c->ev_pool.back(); c->ev_pool.pop_back(); } else MMB_CUDA_CHECK(cudaEventCreate(&e1));
			MMB_CUDA_CHECK(cudaEventRecord(e0, c->stream));
		}
	}
	~ProfScope() {
		if (e0) {
			MMB_CUDA_CHECK(cudaEventRecord(e1, c->stream));
			c->ev_pending[which].push_back(std::make_pair(e0, e1));
		}
	}
};

// ---- device-side launchers (all asynchronous on ctx->stream) ----

// map.cu / jump.cuh: K5 on n_hits descriptors (device), reads d_seq (nt4) and mi's device jump table; decisions to d_out
void mmb_jump_device(mmb_ctx_t *ctx, const mm_idx_t *mi, const mm_mapopt_t *opt, int n_hits, const mmb_jump_hit_t *d_hits, const uint8_t *d_seq, mmb_jump_dec_t *d_out);
bool mmb_jump_wanted(const mm_idx_t *mi, const mm_mapopt_t *opt, int qlen, const mm_reg1_t *r); // mm_jump_check of either end

// ksw_extd2.cu: d_jobs/d_res are device arrays; query is a device byte array (nt4), target either bytes or 4-bit packed words.
// h_jobs is the host copy (used for tiering). cigar ops go to d_cigar (capacity cigar_cap), *d_cigar_used counts them.
void mmb_ksw_launch(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
					const uint8_t *d_query, const void *d_target, int t_packed,
					mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap, unsigned long long *d_cigar_used);
