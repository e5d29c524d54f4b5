/* include/mm_b200.h -- the C-ABI boundary between host C (the minimap.h API, include/minimap.h) and the
 * hand-written sm_90a CUDA kernels of the seed-chain-extend hot path.
 *
 * Plain C: pointers, sizes, PODs. No C++/torch types cross this line. Every entry point names the reference
 * interface it replaces (file:line under lh3/minimap2 v2.30). The library is libminimap2_b200.so
 * (minimap2_b200/csrc). A CUDA failure prints to stderr (when mm_verbose>=1) and abort()s, matching the
 * reference's no-error-code convention on the map path (misc.c:123-151, kalloc.c:32-36). If no CUDA device is
 * present every entry point below fails loudly (returns <0 from mmb_init / aborts elsewhere); there is NO CPU fallback.
 */
#ifndef MM_B200_H
#define MM_B200_H

#include <stdint.h>
#include <stddef.h>
#include "minimap.h" /* mm_idx_t */

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------
 * Device / context
 * --------------------------------------------------------------------------------------------------------- */
typedef struct mmb_ctx_s mmb_ctx_t; /* one per GPU (one process per GPU); owns streams and arenas */

/* returns 0 on success, <0 when no usable CUDA device (fails loudly; nothing else may be called) */
int  mmb_device_count(void);
mmb_ctx_t *mmb_ctx_create(int device);          /* NULL + message on failure */
void mmb_ctx_destroy(mmb_ctx_t *ctx);
void *mmb_ctx_stream(mmb_ctx_t *ctx);           /* cudaStream_t the kernels are launched on (for CUDA-event timing) */
/* counters: kernels launched by this library since creation / last reset (bench.py "gpu_launches") */
uint64_t mmb_launch_count(mmb_ctx_t *ctx, int reset);
/* accumulated device time (ms, CUDA events on the launch stream) per kernel family since last reset;
 * which: 0 sketch, 1 seed, 2 sort, 3 chain, 4 ksw(extd2), 5 other. Only valid when profiling was enabled. */
void  mmb_profile_enable(mmb_ctx_t *ctx, int on);
double mmb_profile_ms(mmb_ctx_t *ctx, int which, int reset);
uint64_t mmb_profile_units(mmb_ctx_t *ctx, int which, int reset); /* algorithmic units: bases, anchors, DP cells.. */

/* ---------------------------------------------------------------------------------------------------------
 * K3: ksw2 extension kernels   (replaces ksw_extd2_sse ksw2_extd2_sse.c:27-401, ksw_ll_i16 ksw2_ll_sse.c:85-152,
 *                                dispatched like mm_align_pair align.c:336-368)
 * --------------------------------------------------------------------------------------------------------- */
#define MMB_KSW_SCORE_ONLY   0x01   /* = KSW_EZ_* (ksw2.h:8-20) */
#define MMB_KSW_RIGHT        0x02
#define MMB_KSW_GENERIC_SC   0x04
#define MMB_KSW_APPROX_MAX   0x08
#define MMB_KSW_APPROX_DROP  0x10
#define MMB_KSW_EXTZ_ONLY    0x40
#define MMB_KSW_REV_CIGAR    0x80
#define MMB_KSW_SPLICE_FOR   0x100  /* spliced alignment (ksw_exts2_sse, ksw2_exts2_sse.c:26): KSW_EZ_SPLICE_* of ksw2.h:15-19 */
#define MMB_KSW_SPLICE_REV   0x200
#define MMB_KSW_SPLICE_FLANK 0x400
#define MMB_KSW_SPLICE_CMPLX 0x800
#define MMB_KSW_SPLICE_SCORE 0x1000
/* job-level addressing flags (how the kernel walks the resident sequences) */
#define MMB_JOB_Q_COMP       0x10000 /* complement query bases (3-c, N stays 4): reverse strand (align.c:1056-1061) */
#define MMB_JOB_LL           0x20000 /* run ksw_ll_i16 (local score) instead of extd2 */
#define MMB_JOB_SPLICE       0x80000 /* the job is a ksw_exts2 call (align.c:352-355): q/e = gap open/extend, q2 = intron open, MMB_KSW_SPLICE_* select the model */
#define MMB_JOB_T_COMP       0x100000 /* the target is read complemented (query-strand mode, mm_idx_getseq_rev index.c:176-190: with t_step = -1 the job sees the reverse complement) */
#define MMB_JOB_ZDROP        0x40000 /* also run mm_test_zdrop's scan over the resulting CIGAR (align.c:61-89); see zd_* below */

typedef struct {
	int64_t q_start;   /* index of the first query base of this job in the query byte array (nt4 codes, 1 B/base) */
	int64_t t_start;   /* index of the first target base (bases; 4-bit packed S or byte array, see t_packed) */
	int32_t q_step;    /* +1 or -1: direction the query is walked (mm_seq_rev for left extension, align.c:787) */
	int32_t t_step;    /* +1 or -1 */
	int32_t qlen, tlen;
	int32_t w, zdrop, end_bonus;
	int32_t flag;      /* MMB_KSW_* | MMB_JOB_* */
} mmb_ksw_job_t;

typedef struct {      /* ksw_extz_t (ksw2.h:34-43) without the pointer */
	int32_t max, zdropped;
	int32_t max_q, max_t;
	int32_t mqe, mqe_t;
	int32_t mte, mte_q;
	int32_t score;
	int32_t n_cigar, reach_end;
	uint32_t cigar_off; /* offset (in uint32 ops) of this job's CIGAR in the batch cigar buffer */
	/* MMB_JOB_ZDROP: max_zdrop and pos[0][0], pos[0][1], pos[1][0], pos[1][1] of mm_test_zdrop (align.c:61-89), i.e. the
	 * largest score drop along the alignment path and where it starts/ends on target and query. zd_max = -1: not evaluated
	 * by the kernel that ran the job (the caller scans the CIGAR itself). */
	int32_t zd_max, zd_t0, zd_t1, zd_q0, zd_q1;
} mmb_ksw_res_t;

typedef struct {      /* scoring: what align.c:655 ksw_gen_ts_mat + mm_mapopt_t a,b,q,e,q2,e2 give */
	int8_t mat[25];
	int8_t q, e, q2, e2;
	int8_t noncan, junc_bonus, junc_pen; /* spliced alignment only (MMB_JOB_SPLICE): mm_mapopt_t noncan / junc_bonus / junc_pen */
	int16_t zd_skip; /* MMB_JOB_ZDROP jobs: if > 0, the kernel may skip the mm_test_zdrop scan (and report max drop 0) when the alignment's total
	                  * penalty under that function's scoring provably cannot exceed this value; the caller passes the smallest threshold it compares the
	                  * drop with (min(zdrop, zdrop_inv), align.c:92-102). 0: always scan */
} mmb_ksw_score_t;

/* Kernel-level entry with HOST buffers (used by the parity tests and for single calls):
 * query/target are byte arrays of nt4 codes (0..4). res[n_jobs]; cigar ops are appended to cigar_buf (capacity
 * cigar_cap uint32s); returns the number of cigar ops written, or <0 if cigar_cap was too small (-needed). */
int64_t mmb_ksw_batch_host(mmb_ctx_t *ctx, const mmb_ksw_score_t *sc, int n_jobs, const mmb_ksw_job_t *jobs,
						   const uint8_t *query, int64_t query_len, const uint8_t *target, int64_t target_len,
						   mmb_ksw_res_t *res, uint32_t *cigar_buf, int64_t cigar_cap);

/* ---------------------------------------------------------------------------------------------------------
 * K1: minimizer sketch   (replaces mm_sketch, sketch.c:77-143)
 * --------------------------------------------------------------------------------------------------------- */
/* Kernel-level entry with HOST buffers. seqs: concatenated ASCII (or nt4) sequences; off[n_seq+1] offsets.
 * out must hold the total number of minimizers; call with out==NULL to get the count. rid of sequence i is rid0+i.
 * Returns total minimizers; n_out[i] (optional) receives the per-sequence counts. */
int64_t mmb_sketch_batch_host(mmb_ctx_t *ctx, int n_seq, const char *seqs, const int64_t *off, int w, int k, int is_hpc,
							  uint32_t rid0, uint64_t *out_xy /* mm128_t pairs */, int64_t out_cap, int64_t *n_out);

/* Junction annotation for MMB_JOB_SPLICE jobs (replaces the junc[] argument of ksw_exts2_sse, ksw2_exts2_sse.c:26-31, that
 * align.c:638-643 fills with mm_idx_bed_junc, index.c:802-826): n annotated introns sorted by st, [st,en) in the coordinates of the
 * target array the jobs address, strand +1/-1. A job marks exactly the introns that lie entirely inside its target window, as
 * mm_idx_bed_junc does for the window mm_align1 passes. n = 0 clears it. Returns -1 if st[] is not sorted. */
int mmb_ctx_set_junctions(mmb_ctx_t *ctx, int64_t n, const int64_t *st, const int64_t *en, const int8_t *strand);

/* Splice scores for MMB_JOB_SPLICE | MMB_KSW_SPLICE_SCORE jobs (the junc[] bytes mm_idx_spsc_get, index.c:1055-1075, hands to
 * ksw_exts2_sse, ksw2_exts2_sse.c:213-219): per strand (0: jobs without MMB_KSW_SPLICE_REV, 1: with) n positions in strictly
 * ascending order, in the coordinates of the target array, with their bytes (score+64)<<1 | acceptor. A job sees the entries strictly
 * inside its target window. n = 0 clears the strand's table. Returns -1 on unsorted input. */
int mmb_ctx_set_splice_scores(mmb_ctx_t *ctx, int strand, int64_t n, const int64_t *pos, const uint8_t *val);

/* ---------------------------------------------------------------------------------------------------------
 * K2c: chaining   (replaces mg_lchain_dp lchain.c:148-217 incl. mg_chain_backtrack/compact_a, and mg_lchain_rmq :250-368)
 * --------------------------------------------------------------------------------------------------------- */
typedef struct {
	int32_t max_dist_x, max_dist_y, bw, max_skip, max_iter, min_cnt, min_sc;
	float chn_pen_gap, chn_pen_skip;
	int32_t is_cdna, n_seg;
	/* rmq variant */
	int32_t use_rmq, max_dist_inner, rmq_size_cap;
} mmb_chain_par_t;

/* Kernel-level entry with HOST buffers. anchors: concatenated mm128_t (x,y) per read, a_off[n_reads+1].
 * Output: for read i, n_u[i] chains; u values appended at u_off[i]; compacted anchors overwrite a_out at a_off[i]
 * (n_v[i] of them). u_out capacity must be >= total anchors/ min_cnt... (pass total anchors to be safe). */
int mmb_chain_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const uint64_t *anchors_xy, const int64_t *a_off,
						 int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy);
/* Same layout, but every read goes through mg_lchain_rmq (lchain.c:251-357; the MM_F_RMQ chainer of map.c:275-276 and the long-join rescue chainer of map.c:283-292).
 * par: max_dist_x = max_dist, max_dist_inner, bw, max_skip, rmq_size_cap, min_cnt, min_sc, chn_pen_gap, chn_pen_skip. */
int mmb_chain_rmq_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, int n_reads, const uint64_t *anchors_xy, const int64_t *a_off,
							 int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy);
/* The long-join rescue (map.c:283-292): its selection rule and its mg_lchain_rmq parameters. max_skip, min_cnt, min_sc and the
 * penalties are the first chainer's. */
typedef struct {
	int32_t bw_long, rescue_size;
	float rescue_ratio;
	int32_t max_dist, max_dist_inner, rmq_size_cap;
} mmb_rescue_par_t;
/* Same layout: the mapper's whole chaining stage. The first chainer (mg_lchain_dp, or mg_lchain_rmq when par->use_rmq) runs on
 * every read, then the reads with more than one chain whose best chain passes the rescue test on qlen[i] are re-sorted and
 * re-chained with mg_lchain_rmq at rp->bw_long. */
int mmb_chain_rescue_batch_host(mmb_ctx_t *ctx, const mmb_chain_par_t *par, const mmb_rescue_par_t *rp, int n_reads, const uint64_t *anchors_xy,
								const int64_t *a_off, const int32_t *qlen, int32_t *n_u, int32_t *n_v, uint64_t *u_out, uint64_t *a_out_xy);

/* ---------------------------------------------------------------------------------------------------------
 * K4: per-hit tail of the alignment driver on the device   (replaces mm_append_cigar align.c:317-334, mm_fix_cigar
 * align.c:105-181 and mm_update_extra align.c:254-303 for finished hits; SURVEY 8 row f4)
 * --------------------------------------------------------------------------------------------------------- */
typedef struct {
	int64_t q0;            /* offset of the read's first base in `query` */
	int64_t t0;            /* offset of the hit's first target base in `target` */
	int32_t qlen;          /* read length */
	int32_t qs;            /* start of the aligned query piece on the strand it is read on */
	int32_t rev;           /* 1: the query piece is read on the reverse-complement strand */
	int32_t qspan, tspan;  /* query / target bases the hit's CIGAR consumes */
	int32_t piece_first, n_pieces; /* the hit's ksw2 pieces, in driver order */
	int32_t pad;
} mmb_tail_hit_t;
typedef struct { int32_t n_cigar, blen, mlen, n_ambi, dp_max, qshift, tshift, status, is_spliced, pad[3]; } mmb_tail_out_t;
/* Kernel-level entry with HOST buffers. query / target: nt4 codes (0..4), one byte per base (the target is packed to the index's
 * 4-bit layout on the way in). piece_len[n_pieces_total] operations per piece, stored back to back in ops[]. mat: the 5x5 scoring
 * matrix; q, e: opt->q / opt->e. out[n_hits]; hit i's final CIGAR goes to cigar_out + cig_off[i] (cig_off[n_hits+1]: prefix sums of the
 * hits' piece totals, computed by the caller). Returns 0. */
int mmb_tail_batch_host(mmb_ctx_t *ctx, int n_hits, const mmb_tail_hit_t *hits, int64_t n_pieces_total, const uint32_t *piece_len, const uint32_t *ops,
						const uint8_t *query, int64_t query_len, const uint8_t *target, int64_t target_len, const int8_t *mat, int q, int e,
						const int64_t *cig_off, mmb_tail_out_t *out, uint32_t *cigar_out);

/* ---------------------------------------------------------------------------------------------------------
 * K5: junction jumps of spliced hits on the device   (the decisions of mm_jump_split, jump.c:50-201)
 * --------------------------------------------------------------------------------------------------------- */
typedef struct {
	int32_t rid, rs, re, qs, qe, rev; /* the hit (mm_reg1_t fields) */
	int32_t qlen, n_cigar;            /* read length; the hit's CIGAR length */
	int64_t q_off;                    /* offset of the read's first base in the batch's bases */
	uint32_t cig_first, cig_last;     /* first and last CIGAR words */
} mmb_jump_hit_t;
typedef struct {
	int32_t act;          /* 0: nothing, 1: trim the end back to the splice site, 2: add an exon across the junction */
	int32_t l, off, off2; /* l as jump.c computes it; the chosen jump-table entry */
	int32_t mm0;          /* mismatches of the chosen candidate */
} mmb_jump_side_t;
typedef struct { mmb_jump_side_t side[2]; } mmb_jump_dec_t; /* [0]: left end of the alignment, [1]: right end (decided after [0]) */
/* Kernel-level entry: K5 on n_hits hits against the jump table of mi (mm_idx_jjump_read), reads given as ASCII back to back
 * (off[n_reads+1]); opt supplies a, b and jump_min_match. Returns 0, or -1 when mi has no jump table. */
int mmb_jump_batch_host(mmb_ctx_t *ctx, const mm_idx_t *mi, const mm_mapopt_t *opt, int n_reads, const char *seqs, const int64_t *off,
						int n_hits, const mmb_jump_hit_t *hits, mmb_jump_dec_t *out);
/* The host half of mm_jump_split: applies one hit's decisions (left, then right) to r and its libc-owned r->p. */
void mmb_jump_apply(const mm_mapopt_t *opt, int qlen, mm_reg1_t *r, const mmb_jump_dec_t *d);

/* ---------------------------------------------------------------------------------------------------------
 * Index on device + whole-path batch mapping are driven through the minimap.h API (include/minimap.h):
 * mm_idx_* builds/loads the index on the GPU (side table keyed by mm_idx_t*), mm_map_file / mm_map_batch run the GPU
 * batch scheduler that replaces worker_pipeline/kt_for (map.c:403-691). The entries below are the knobs and hand-off
 * points around it; none has a counterpart in the reference (single process, CPU threads).
 * --------------------------------------------------------------------------------------------------------- */

/* scheduler: the batch is cut into `n` groups that run the pipeline concurrently (n < 0: the same |n| groups one after
 * another -- clean per-kernel timing); at most `slots` groups are inside a device phase at a time. 0 / defaults:
 * MM_B200_GROUPS (12) and MM_B200_GPU_SLOTS (4). */
void mmb_set_groups(int n);
void mmb_set_gpu_slots(int slots);
/* benchmark aid: when on, a batch whose first read pointer / count / bases equal the previous batch's of the same group
 * reuses the reads already in HBM (no H2D, no re-encode): the "inputs resident" timing of bench.py. */
void mmb_set_resident_reads(int on);

/* process-wide variants of the per-context counters above (sum over the default context and every scheduler group) */
void *mmb_default_ctx_c(void);
void mmb_profile_enable_all(int on);
double mmb_profile_ms_all(int which, int reset);
uint64_t mmb_profile_units_all(int which, int reset);
uint64_t mmb_profile_bytes_all(int which, int reset);   /* algorithmic bytes per kernel family (DESIGN.md section 5) */
uint64_t mmb_profile_scopes_all(int which, int reset);  /* timed launch groups per family */
uint64_t mmb_profile_bytes(mmb_ctx_t *ctx, int which, int reset);
uint64_t mmb_profile_scopes(mmb_ctx_t *ctx, int which, int reset);
uint64_t mmb_launch_count_all(int reset);
uint64_t mmb_last_d2h_bytes(void);                      /* device->host bytes of the last mm_map_batch call */
uint64_t mmb_last_d2h_bytes_all(void);
void mmb_free(void *p);                                 /* free() for buffers handed out by this library */

/* one-process-per-GPU replication of the device index (index.c has no counterpart; SURVEY 8e): rank 0 exports the device
 * arrays, the caller broadcasts them (NCCL) into its own device buffers and adopts them as an mm_idx_t on each rank.
 * ptr/bytes order: hash table, positions, 4-bit sequence, sequence offsets, sequence lengths. */
typedef struct {
	void *ptr[5];
	uint64_t bytes[5];
	int64_t n_keys, n_pos;
	int32_t tab_bits, w, k, b, flag;
	uint32_t n_seq;
	uint64_t sum_len;
} mmb_idx_desc_t;
void mmb_idx_export(const mm_idx_t *mi, mmb_idx_desc_t *d);
mm_idx_t *mmb_idx_adopt(const mmb_idx_desc_t *d, const char **names, const uint32_t *lens, const uint32_t *cnt_sorted_dev);
const void *mmb_idx_cnt_sorted(const mm_idx_t *mi, uint64_t *bytes); /* sorted occurrence counts (mm_idx_cal_max_occ, index.c:158) */
/* Kernel-level probe of the device index for tests: one thread per key looks it up in the device hash table with the seeding kernels'
 * lookup (mm_idx_get, index.c:93-110) and gathers its occurrences. cnt[i]: occurrences of keys[i] (0: absent); occ_off[n+1]: where
 * they start in occ (prefix sums of cnt); occ receives the first occ_cap of them. Returns the total. */
int64_t mmb_idx_lookup_host(const mm_idx_t *mi, int64_t n, const uint64_t *keys, uint32_t *cnt, uint64_t *occ, int64_t occ_cap, int64_t *occ_off);

/* K2a/K2b as one stage for kernel-level tests: sketch -> mm_seed_mz_flt -> mm_idx_get -> mm_seed_select -> collect_seed_hits incl.
 * radix_sort_128x (seed.c:5-132, map.c:59-72,168-204) of a batch of reads against a device-resident index. With MM_F_HEAP_SORT in
 * flag the anchors come in the order of collect_seed_hits_heap (map.c:102-166) instead. See csrc/map.cu. */
int64_t mmb_seed_batch_host(mmb_ctx_t *ctx, const mm_idx_t *mi, int n_reads, const char *seqs, const int64_t *off, int64_t flag, int mid_occ,
							float q_occ_frac, int max_max_occ, int occ_dist, int64_t *a_off_out, int32_t *rep_len_out, int32_t *n_mini_out,
							uint64_t *anchors_xy, int64_t a_cap, uint64_t *mini_pos, int64_t mp_cap);

/* synthetic workload for bench.py (BASELINE.json configs[1] shape; there is no network for real genomes): a random
 * genome of total_len bases in n_contigs contigs indexed on the device, and reads sampled from it with the given
 * error profile (err = per-base error rate, split into substitutions / insertions / deletions by sub, ins, 1-sub-ins). */
mm_idx_t *mmb_synth_index(uint64_t total_len, int n_contigs, uint64_t seed, int w, int k, int bucket_bits);
int mmb_synth_reads(const mm_idx_t *mi, int n_reads, int read_len, uint64_t seed, float err, float sub, float ins, char *out);
int mmb_idx_write_fasta(const mm_idx_t *mi, const char *fn); /* dump the indexed sequences (to feed the reference arm) */
int mmb_synth_cdna_reads(const mm_idx_t *mi, int n_reads, int read_len, uint64_t seed, float err, char *out); /* spliced transcripts: exons joined over GT..AG introns */
int64_t mmb_aligned_bases(int n, const int32_t *n_regs, mm_reg1_t *const *regs, int all_records); /* sum of qe-qs over primary (or all) hits: bench metric */

#ifdef __cplusplus
}
#endif
#endif
