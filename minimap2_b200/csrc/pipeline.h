// minimap2_b200/csrc/pipeline.h -- device-side stage interfaces of the batch mapper (K1 -> K2a/b -> K2c -> K3).
#pragma once
#include "index.h"
#include "mm_algo.cuh"

struct SeedArgs {
	DevIndexView ix;
	int n_reads;
	m128 *mz;                 // minimizers of all reads (sketch output), per-read slices at mz_off
	const int64_t *mz_off;    // n_reads+1
	int32_t *n_mz;            // live count per read (shrinks after the query-side filter)
	const int32_t *qlen;
	int q_occ_max; float q_occ_frac;
	int max_occ, max_max_occ, occ_dist;
	int64_t flag;
	// per minimizer (same offsets as mz)
	uint32_t *s_n; uint64_t *s_off;
	uint32_t *k_idx, *k_aoff; uint8_t *flt; uint64_t *mini_pos;
	// per read
	int32_t *n_keep, *rep_len; int64_t *n_a;
	// anchors
	m128 *a; const int64_t *a_off;
	m128 *a_sorted;           // output of the anchor sort (a stays in expansion order for the exact-sort fallback)
	// skip_seed (map.c:78-100), only when MM_F_NO_DIAG/NO_DUAL/FOR_ONLY/REV_ONLY is set: names are compared through their
	// rank in the sorted list of reference names; a query name equals the references ranked [q_name_lo, q_name_hi)
	const uint32_t *name_rank = nullptr;  // per reference sequence (null: no query names => no name tests, as in the reference)
	const uint32_t *q_name_lo = nullptr, *q_name_hi = nullptr; // per read
	uint32_t *k_cnt = nullptr;            // per kept seed: occurrences that survive skip_seed
};

void mmb_seed_select_device(mmb_ctx_t *ctx, SeedArgs &A, int64_t total_mz);
void mmb_seed_expand_sort_device(mmb_ctx_t *ctx, SeedArgs &A, int64_t total_mz, int64_t total_a, DevBuf &stkbuf);

// The anchor sort (radix_sort_128x, map.c:202) of n_reads reads: a_in[a_off[i], a_off[i+1]) sorted by x into a_out at the same offsets.
// Each read goes by its anchor count to one of the shared-memory radix classes or to the oversize list. The radix kernels hand reads
// whose keys vary in more than 33 bits to the network sort, and list the reads with equal keys and more than tie_min_n anchors. With
// run_exact, the listed reads and the oversize ones are then re-sorted by the exact emulation of the reference's unstable sort; without
// it the caller orders them (heap mode). The returned counters and lists live in stkbuf, in device memory: cnt[c] reads in
// list + c * n_reads, for c = 0..4 (radix class of at most 1024 << c anchors), MMB_SORT_OVERSIZE (more than 16384 anchors, and the
// listed reads the shared-memory exact walker passes on), MMB_SORT_TIES and MMB_SORT_FALLBACK (network sort). extra: extra_bytes of
// 16-byte aligned device scratch for the caller, after the lists.
enum { MMB_SORT_N_CLS = 5, MMB_SORT_OVERSIZE = 5, MMB_SORT_TIES = 6, MMB_SORT_FALLBACK = 7 };
// tie_min_n of the sorted order: the reference sorts up to 64 anchors by a stable insertion sort (ksort.h:147), so only larger reads with
// equal keys need the exact emulation
enum { MMB_SORT_TIE_MIN_N = 64 };
struct AnchorSortLists { int *cnt, *list; void *extra; };
AnchorSortLists mmb_anchor_sort_device(mmb_ctx_t *ctx, const m128 *a_in, m128 *a_out, const int64_t *d_a_off, int n_reads, int64_t total_a,
										int tie_min_n, bool run_exact, DevBuf &stkbuf, size_t extra_bytes);

void mmb_chain_device(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const m128 *d_a, const int64_t *d_a_off, int64_t n_tot,
					  int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2);

struct RescuePar {            // long-join rescue with mg_lchain_rmq (map.c:283-292)
	const int32_t *qlen;
	int32_t rescue_size; float rescue_ratio;
	int32_t max_dist, max_dist_inner, bw, max_skip, rmq_size_cap, min_cnt, min_sc;
	float pen_gap, pen_skip;
	uint8_t *tree; const int64_t *tree_off;
	int32_t primary;              // 1: mg_lchain_rmq as the first chainer (map.c:275-276): every read, anchors taken as they are (no re-sort)
};
// mg_lchain_rmq as the primary chainer (MM_F_RMQ, map.c:275-276); same outputs as mmb_chain_device
void mmb_chain_rmq_primary_device(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const m128 *d_a, const int64_t *d_a_off, int64_t n_tot,
								  int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf);
void mmb_chain_rescue_device(mmb_ctx_t *ctx, const RescuePar *rp, int n_reads, const int64_t *d_a_off, int64_t n_tot,
							 int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf, int64_t tot_v);
// The chaining stage of a batch (map.c:262-292): the first chainer (mmb_chain_rmq_primary_device when par->use_rmq, else
// mmb_chain_device), then, when rp is given, the long-join rescue. d_vo (n_reads+1) receives the rescue's tree offsets.
void mmb_chain_stage(mmb_ctx_t *ctx, const mmb_chain_par_t *par, const RescuePar *rp, int n_reads, const m128 *d_a, const int64_t *d_a_off,
					 int64_t n_tot, int32_t *d_n_u, int32_t *d_n_v, uint64_t *d_u, m128 *d_a_out, int64_t *d_vo,
					 DevBuf &scratch, DevBuf &scratch2, DevBuf &treebuf);

// ---- K4 (finalize.cu): CIGAR assembly + mm_fix_cigar + mm_update_extra of finished hits on the device (align.c:105-181,254-334) ----
struct FinJobRef { const uint32_t *cig; uint32_t n, pad; }; // one ksw2 result: its CIGAR in the device arena of the wave that ran it
struct FinReg {
	int64_t q0;               // offset of the read's first base in the device query array (nt4)
	int64_t t0;               // offset (in bases) of target position rs in the packed reference
	int64_t out_off;          // where the hit's CIGAR goes in the output arena (room for the sum of its pieces)
	int32_t qlen, qs, rev;    // read length; start of the aligned piece on the strand it is read on; 1: reverse complement
	int32_t qspan, tspan;     // query / target bases the CIGAR must consume (consistency check)
	int32_t job_first, n_jobs;
	int32_t pad;
};
struct FinOut { int32_t n_cigar, blen, mlen, n_ambi, dp_max, qshift, tshift, status, is_spliced, pad[3]; }; // status 0: done; 2: the CIGAR does not consume qspan / tspan, the host driver redoes the read
struct FinPar { int8_t mat[25]; int8_t q, e, log_gap; };
void mmb_finalize_device(mmb_ctx_t *ctx, const FinReg *d_regs, const FinJobRef *d_jobs, int n_regs, const uint8_t *d_query, const uint32_t *d_S,
						 uint32_t *d_out, FinOut *d_res, const FinPar &par);
