/* include/minimap.h -- public C API of the H100-native (sm_90a) mapper.
 *
 * This is the drop-in boundary: it declares the same symbols, with the same argument meaning, ownership and
 * error behaviour, and the same struct layouts (field order, widths, bit-fields) as lh3/minimap2 v2.30's
 * minimap.h (reference minimap.h:77-430), so that main.c / example.c / mappy-style bindings written against the
 * reference compile and link against libminimap2_b200.so unchanged. The implementation behind it is new:
 * the per-read hot path (mm_sketch -> seed collection -> mg_lchain_* -> ksw2) runs as sm_90a CUDA kernels and
 * mm_map_file*'s pthread pipeline (map.c:541-691) is replaced by a GPU batch scheduler. See DESIGN.md.
 *
 * Each declaration cites the reference line it mirrors. Layout identity is asserted by tests/test_abi.py against
 * the reference build (oracle/_ref).
 */
#ifndef MINIMAP2_H
#define MINIMAP2_H

#include <stdint.h>
#include <stdio.h>
#include <sys/types.h>

#define MM_VERSION "2.30-b200-r1"

/* mapping flags, mm_mapopt_t::flag (reference minimap.h:10-50; same bit positions) */
#define MM_F_NO_DIAG       (0x001LL)
#define MM_F_NO_DUAL       (0x002LL)
#define MM_F_CIGAR         (0x004LL)
#define MM_F_OUT_SAM       (0x008LL)
#define MM_F_NO_QUAL       (0x010LL)
#define MM_F_OUT_CG        (0x020LL)
#define MM_F_OUT_CS        (0x040LL)
#define MM_F_SPLICE        (0x080LL)
#define MM_F_SPLICE_FOR    (0x100LL)
#define MM_F_SPLICE_REV    (0x200LL)
#define MM_F_NO_LJOIN      (0x400LL)
#define MM_F_OUT_CS_LONG   (0x800LL)
#define MM_F_SR            (0x1000LL)
#define MM_F_FRAG_MODE     (0x2000LL)
#define MM_F_NO_PRINT_2ND  (0x4000LL)
#define MM_F_2_IO_THREADS  (0x8000LL)
#define MM_F_LONG_CIGAR    (0x10000LL)
#define MM_F_INDEPEND_SEG  (0x20000LL)
#define MM_F_SPLICE_FLANK  (0x40000LL)
#define MM_F_SOFTCLIP      (0x80000LL)
#define MM_F_FOR_ONLY      (0x100000LL)
#define MM_F_REV_ONLY      (0x200000LL)
#define MM_F_HEAP_SORT     (0x400000LL)
#define MM_F_ALL_CHAINS    (0x800000LL)
#define MM_F_OUT_MD        (0x1000000LL)
#define MM_F_COPY_COMMENT  (0x2000000LL)
#define MM_F_EQX           (0x4000000LL)
#define MM_F_PAF_NO_HIT    (0x8000000LL)
#define MM_F_NO_END_FLT    (0x10000000LL)
#define MM_F_HARD_MLEVEL   (0x20000000LL)
#define MM_F_SAM_HIT_ONLY  (0x40000000LL)
#define MM_F_RMQ           (0x80000000LL)
#define MM_F_QSTRAND       (0x100000000LL)
#define MM_F_NO_INV        (0x200000000LL)
#define MM_F_NO_HASH_NAME  (0x400000000LL)
#define MM_F_SPLICE_OLD    (0x800000000LL)
#define MM_F_SECONDARY_SEQ (0x1000000000LL)
#define MM_F_OUT_DS        (0x2000000000LL)
#define MM_F_WEAK_PAIRING  (0x4000000000LL)
#define MM_F_SR_RNA        (0x8000000000LL)
#define MM_F_OUT_JUNC      (0x10000000000LL)

/* index flags, mm_idx_t::flag (minimap.h:52-54) */
#define MM_I_HPC          0x1
#define MM_I_NO_SEQ       0x2
#define MM_I_NO_NAME      0x4

#define MM_IDX_MAGIC   "MMI\2"   /* .mmi files are interchangeable with the reference (index.c:475-569) */
#define MM_MAX_SEG       255

/* CIGAR operators (minimap.h:60-70) */
#define MM_CIGAR_MATCH      0
#define MM_CIGAR_INS        1
#define MM_CIGAR_DEL        2
#define MM_CIGAR_N_SKIP     3
#define MM_CIGAR_SOFTCLIP   4
#define MM_CIGAR_HARDCLIP   5
#define MM_CIGAR_PADDING    6
#define MM_CIGAR_EQ_MATCH   7
#define MM_CIGAR_X_MISMATCH 8
#define MM_CIGAR_STR  "MIDNSHP=XB"

#ifdef __cplusplus
extern "C" {
#endif

/* 128-bit pair used for minimizers, anchors and sort records (minimap.h:77-78) */
typedef struct { uint64_t x, y; } mm128_t;
typedef struct { size_t n, m; mm128_t *a; } mm128_v;

/* one reference sequence (minimap.h:81-86) */
typedef struct {
	char *name;
	uint64_t offset;   /* first base in mm_idx_t::S */
	uint32_t len;
	uint32_t is_alt;
} mm_idx_seq_t;

/* the index (minimap.h:88-100). B is opaque: here it points at the device index object (host lookup arrays + the
 * HBM-resident mirror); I, spsc and J are the annotation tables of mm_idx_bed_read, mm_idx_spsc_read2 and mm_idx_jjump_read. */
typedef struct {
	int32_t b, w, k, flag;
	uint32_t n_seq;
	int32_t index;
	int32_t n_alt;
	mm_idx_seq_t *seq;
	uint32_t *S;                 /* 4-bit packed bases, 8 per word */
	struct mm_idx_bucket_s *B;
	struct mm_idx_intv_s *I;
	struct mm_idx_spsc_s *spsc;
	struct mm_idx_jjump_s *J;
	void *km, *h;
} mm_idx_t;

/* base-level alignment attached to a hit (minimap.h:103-110) */
typedef struct {
	uint32_t capacity;
	int32_t dp_score, dp_max, dp_max2;
	int32_t dp_max0;
	uint32_t n_ambi:30, trans_strand:2;
	uint32_t n_cigar;
	uint32_t cigar[];
} mm_extra_t;

/* one hit (minimap.h:112-127) */
typedef struct {
	int32_t id;
	int32_t cnt;
	int32_t rid;
	int32_t score;
	int32_t qs, qe, rs, re;
	int32_t parent, subsc;
	int32_t as;
	int32_t mlen, blen;
	int32_t n_sub;
	int32_t score0;
	uint32_t mapq:8, split:2, rev:1, inv:1, sam_pri:1, proper_frag:1, pe_thru:1, seg_split:1, seg_id:8, split_inv:1, is_alt:1, strand_retained:1, is_spliced:1, dummy:4;
	uint32_t hash;
	float div;
	mm_extra_t *p;
} mm_reg1_t;

/* indexing options (minimap.h:130-134) */
typedef struct {
	short k, w, flag, bucket_bits;
	int64_t mini_batch_size;
	uint64_t batch_size;
} mm_idxopt_t;

/* mapping options (minimap.h:136-192) */
typedef struct {
	int64_t flag;
	int seed;
	int sdust_thres;

	int max_qlen;

	int bw, bw_long;
	int max_gap, max_gap_ref;
	int max_frag_len;
	int max_chain_skip, max_chain_iter;
	int min_cnt;
	int min_chain_score;
	float chain_gap_scale;
	float chain_skip_scale;
	int rmq_size_cap, rmq_inner_dist;
	int rmq_rescue_size;
	float rmq_rescue_ratio;

	float mask_level;
	int mask_len;
	float pri_ratio;
	int best_n;

	float alt_drop;

	int a, b, q, e, q2, e2;
	int transition;
	int sc_ambi;
	int noncan;
	int junc_bonus;
	int junc_pen;
	int zdrop, zdrop_inv;
	int end_bonus;
	int min_dp_max;
	int min_ksw_len;
	int anchor_ext_len, anchor_ext_shift;
	float max_clip_ratio;

	int rank_min_len;
	float rank_frac;

	int pe_ori, pe_bonus;

	int32_t jump_min_match;

	float mid_occ_frac;
	float q_occ_frac;
	int32_t min_mid_occ, max_mid_occ;
	int32_t mid_occ;
	int32_t max_occ, max_max_occ, occ_dist;
	int64_t mini_batch_size;
	int64_t max_sw_mat;
	int64_t cap_kalloc;

	const char *split_prefix;
} mm_mapopt_t;

/* index reader (minimap.h:195-204) */
typedef struct {
	int is_idx, n_parts;
	int64_t idx_size;
	mm_idxopt_t opt;
	FILE *fp_out;
	union {
		struct mm_bseq_file_s *seq;
		FILE *idx;
	} fp;
} mm_idx_reader_t;

/* per-thread buffer (minimap.h:207-212); km is unused here (scratch lives in per-batch arenas) */
struct mm_tbuf_s {
	void *km;
	int rep_len, frag_gap;
};
typedef struct mm_tbuf_s mm_tbuf_t;

extern int mm_verbose, mm_dbg_flag;   /* minimap.h:215 */
extern double mm_realtime0;           /* minimap.h:216 */

/* options (options.c) */
int mm_set_opt(const char *preset, mm_idxopt_t *io, mm_mapopt_t *mo);                 /* minimap.h:227, options.c:91 */
int mm_check_opt(const mm_idxopt_t *io, const mm_mapopt_t *mo);                       /* minimap.h:228, options.c:202 */
void mm_mapopt_update(mm_mapopt_t *opt, const mm_idx_t *mi);                          /* minimap.h:240, options.c:69 */
void mm_mapopt_max_intron_len(mm_mapopt_t *opt, int max_intron_len);                  /* minimap.h:242 */
void mm_mapopt_init(mm_mapopt_t *opt);                                                /* minimap.h:426 (deprecated) */
void mm_idxopt_init(mm_idxopt_t *opt);                                                /* mmpriv.h:95 */

/* index construction / IO (index.c) */
mm_idx_reader_t *mm_idx_reader_open(const char *fn, const mm_idxopt_t *opt, const char *fn_out); /* minimap.h:253 */
mm_idx_t *mm_idx_reader_read(mm_idx_reader_t *r, int n_threads);                      /* minimap.h:270 */
void mm_idx_reader_close(mm_idx_reader_t *r);                                         /* minimap.h:277 */
int mm_idx_reader_eof(const mm_idx_reader_t *r);                                      /* minimap.h:279 */
int64_t mm_idx_is_idx(const char *fn);                                                /* minimap.h:288 */
mm_idx_t *mm_idx_load(FILE *fp);                                                      /* minimap.h:301 */
void mm_idx_dump(FILE *fp, const mm_idx_t *mi);                                       /* minimap.h:309 */
mm_idx_t *mm_idx_str(int w, int k, int is_hpc, int bucket_bits, int n, const char **seq, const char **name); /* minimap.h:324 */
mm_idx_t *mm_idx_build(const char *fn, int w, int k, int flag, int n_threads);        /* minimap.h:427 (deprecated) */
void mm_idx_stat(const mm_idx_t *idx);                                                /* minimap.h:331 */
void mm_idx_destroy(mm_idx_t *mi);                                                    /* minimap.h:338 */
int mm_idx_index_name(mm_idx_t *mi);                                                  /* minimap.h:409 */
int mm_idx_name2id(const mm_idx_t *mi, const char *name);                             /* minimap.h:410 */
int mm_idx_getseq(const mm_idx_t *mi, uint32_t rid, uint32_t st, uint32_t en, uint8_t *seq); /* minimap.h:411 */
const uint64_t *mm_idx_get(const mm_idx_t *mi, uint64_t minier, int *n);              /* mmpriv.h:96, index.c:93 */
int32_t mm_idx_cal_max_occ(const mm_idx_t *mi, float f);                              /* mmpriv.h:97, index.c:198 */

/* optional index annotations (index.c:642-1074) */
int mm_idx_alt_read(mm_idx_t *mi, const char *fn);                                    /* minimap.h:413 */
int mm_idx_bed_read(mm_idx_t *mi, const char *fn, int read_junc);                     /* minimap.h:414 */
int mm_idx_bed_junc(const mm_idx_t *mi, int32_t ctg, int32_t st, int32_t en, uint8_t *s); /* minimap.h:415 */
int mm_max_spsc_bonus(const mm_mapopt_t *mo);                                         /* minimap.h:417 */
int32_t mm_idx_spsc_read(mm_idx_t *idx, const char *fn, int32_t max_sc);              /* minimap.h:418 */
int32_t mm_idx_spsc_read2(mm_idx_t *idx, const char *fn, int32_t max_sc, float scale);/* minimap.h:419 */
int64_t mm_idx_spsc_get(const mm_idx_t *db, int32_t cid, int64_t st0, int64_t en0, int32_t rev, uint8_t *sc); /* minimap.h:420 */
/* junctions that spliced hits may jump across (index.c:903-930): flag MM_JUNC_ANNO for annotation, MM_JUNC_MISC for junctions of a
 * first pass (--write-junc output, lines scoring at least min_sc). A second call merges into the table. -1: the file cannot be read. */
#define MM_JUNC_ANNO 0x1 /* mmpriv.h:27-28 */
#define MM_JUNC_MISC 0x2
int mm_idx_jjump_read(mm_idx_t *mi, const char *fn, int flag, int min_sc);             /* mmpriv.h:95 */

/* thread buffers (map.c:13-31) */
mm_tbuf_t *mm_tbuf_init(void);                                                        /* minimap.h:351 */
void mm_tbuf_destroy(mm_tbuf_t *b);                                                   /* minimap.h:358 */
void *mm_tbuf_get_km(mm_tbuf_t *b);                                                   /* minimap.h:360 */

/* mapping. Results are libc-malloc'd (array and each ->p); the caller frees them (minimap.h:364-377). */
mm_reg1_t *mm_map(const mm_idx_t *mi, int l_seq, const char *seq, int *n_regs, mm_tbuf_t *b, const mm_mapopt_t *opt, const char *name); /* minimap.h:379 */
void mm_map_frag(const mm_idx_t *mi, int n_segs, const int *qlens, const char **seqs, int *n_regs, mm_reg1_t **regs, mm_tbuf_t *b, const mm_mapopt_t *opt, const char *qname); /* minimap.h:381 */
int mm_map_file(const mm_idx_t *idx, const char *fn, const mm_mapopt_t *opt, int n_threads);   /* minimap.h:393 */
int mm_map_file_frag(const mm_idx_t *idx, int n_segs, const char **fn, const mm_mapopt_t *opt, int n_threads); /* minimap.h:395 */

/* Extension (not in the reference): map a whole in-memory batch through the GPU scheduler. seqs[i]/names[i]
 * are NUL-terminated; regs_out[i] / n_regs_out[i] follow mm_map()'s ownership rules; rep_len_out may be NULL.
 * Thread-safe: concurrent callers are served one batch at a time (the scheduler's streams and arenas are process-wide);
 * mm_map()/mm_map_frag() are batches of one and share that queue. */
int mm_map_batch(const mm_idx_t *mi, int n_reads, const int *qlens, const char **seqs, const char **names,
				 int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out, const mm_mapopt_t *opt, int n_threads);

/* tags (format.c:364-395) */
int mm_gen_cs(void *km, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq, int no_iden); /* minimap.h:404 */
int mm_gen_ds(void *km, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq, int no_iden); /* minimap.h:405 */
int mm_gen_MD(void *km, char **buf, int *max_len, const mm_idx_t *mi, const mm_reg1_t *r, const char *seq);             /* minimap.h:406 */

#ifdef __cplusplus
}
#endif

#endif
