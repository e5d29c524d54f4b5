// minimap2_b200/csrc/ksw_plan.h -- a prepared K3 kernel launch: all host-side preparation (queue order, sizes) is done before
// anything goes on the stream, so that a scheduler group plans without holding a device slot and the kernels of one batch run
// back to back.
#pragma once
#include <functional>
#include <vector>
#include <cstdint>
#include <cstddef>
struct KswPlan {
	size_t pws_bytes = 0, cigws_bytes = 0;                 // traceback / CIGAR workspace this launch needs
	std::vector<int> order;                                // the job queue: batch indices in the order the workers take them
	int *d_order = nullptr;                                // its device copy: a counter word, then the order
	std::function<void(uint8_t *pws, uint32_t *cigws)> go; // enqueue the kernel on the context's stream
};
struct KswLaunch { // one K3 launch set: mmb_ksw_plan fills it on the host, mmb_ksw_enqueue puts it on the stream
	KswPlan ll;                 // the ksw_ll probes (no go without any); they run first and are timed apart from the rest
	std::vector<KswPlan> plans; // the fast-path classes and the universal tiers
	uint64_t cells = 0;
};
void mmb_order_by_cells(std::vector<int> &v, const mmb_ksw_job_t *h_jobs);
// mmb_ksw_launch in two halves (ksw_extd2.cu): the host planning, then the uploads and kernels on ctx->stream
void mmb_ksw_plan(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *h_jobs, const mmb_ksw_job_t *d_jobs,
				  const uint8_t *d_query, const void *d_target, int t_packed,
				  mmb_ksw_res_t *d_res, uint32_t *d_cigar, int64_t cigar_cap, unsigned long long *d_cigar_used, KswLaunch &K);
void mmb_ksw_enqueue(mmb_ctx_t *ctx, const KswLaunch &K);
