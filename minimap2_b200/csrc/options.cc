// minimap2_b200/csrc/options.cc -- option defaults, presets and validation (minimap.h API).
// Mirrors the VALUES of reference options.c (defaults :5-67, presets :91-193, checks :202-277): the kernels are driven by
// these numbers and output parity depends on them being identical.
#include <cstring>
#include <cstdio>
#include <climits>
#include <string>
#include "minimap.h"

extern "C" double realtime(void);
extern "C" double cputime(void);

extern "C" void mm_idxopt_init(mm_idxopt_t *o) // options.c:5-12
{
	memset(o, 0, sizeof(*o));
	o->k = 15, o->w = 10, o->flag = 0, o->bucket_bits = 14;
	o->mini_batch_size = 50000000;
	o->batch_size = 8000000000ULL;
}

extern "C" void mm_mapopt_init(mm_mapopt_t *o) // options.c:14-67
{
	memset(o, 0, sizeof(*o));
	o->seed = 11;
	// seeding
	o->mid_occ_frac = 2e-4f, o->min_mid_occ = 10, o->max_mid_occ = 1000000;
	o->sdust_thres = 0, o->q_occ_frac = 0.01f;
	o->max_max_occ = 4095, o->occ_dist = 500;
	// chaining
	o->min_cnt = 3, o->min_chain_score = 40;
	o->bw = 500, o->bw_long = 20000;
	o->max_gap = 5000, o->max_gap_ref = -1;
	o->max_chain_skip = 25, o->max_chain_iter = 5000;
	o->rmq_inner_dist = 1000, o->rmq_size_cap = 100000, o->rmq_rescue_size = 1000, o->rmq_rescue_ratio = 0.1f;
	o->chain_gap_scale = 0.8f, o->chain_skip_scale = 0.0f;
	// hit selection
	o->mask_level = 0.5f, o->mask_len = INT_MAX, o->pri_ratio = 0.8f, o->best_n = 5;
	o->alt_drop = 0.15f;
	// base alignment
	o->a = 2, o->b = 4, o->q = 4, o->e = 2, o->q2 = 24, o->e2 = 1;
	o->transition = 0, o->sc_ambi = 1;
	o->zdrop = 400, o->zdrop_inv = 200;
	o->end_bonus = -1;
	o->min_dp_max = o->min_chain_score * o->a;
	o->min_ksw_len = 200;
	o->anchor_ext_len = 20, o->anchor_ext_shift = 6;
	o->max_clip_ratio = 1.0f;
	// batching
	o->mini_batch_size = 500000000;
	o->max_sw_mat = 100000000;
	o->cap_kalloc = 500000000;
	o->rank_min_len = 500, o->rank_frac = 0.9f;
	o->pe_ori = 0, o->pe_bonus = 33;
	o->jump_min_match = 3;
}

extern "C" void mm_mapopt_update(mm_mapopt_t *opt, const mm_idx_t *mi) // options.c:69-83
{
	if ((opt->flag & MM_F_SPLICE_FOR) || (opt->flag & MM_F_SPLICE_REV)) opt->flag |= MM_F_SPLICE;
	if (opt->mid_occ <= 0) {
		opt->mid_occ = mm_idx_cal_max_occ(mi, opt->mid_occ_frac);
		if (opt->mid_occ < opt->min_mid_occ) opt->mid_occ = opt->min_mid_occ;
		if (opt->max_mid_occ > opt->min_mid_occ && opt->mid_occ > opt->max_mid_occ) opt->mid_occ = opt->max_mid_occ;
	}
	if (opt->bw_long < opt->bw) opt->bw_long = opt->bw;
	if (mm_verbose >= 3)
		fprintf(stderr, "[M::%s::%.3f*%.2f] mid_occ = %d\n", __func__, realtime() - mm_realtime0, cputime() / (realtime() - mm_realtime0), opt->mid_occ);
}

extern "C" void mm_mapopt_max_intron_len(mm_mapopt_t *opt, int max_intron_len) // options.c:85-89
{
	if ((opt->flag & MM_F_SPLICE) && max_intron_len > 0)
		opt->max_gap_ref = opt->bw = opt->bw_long = max_intron_len;
}

static void set_gap_scores(mm_mapopt_t *mo, int a, int b, int q, int e, int q2, int e2)
{
	mo->a = a, mo->b = b, mo->q = q, mo->e = e, mo->q2 = q2, mo->e2 = e2;
}

static void set_ava(mm_mapopt_t *mo)
{
	mo->flag |= MM_F_ALL_CHAINS | MM_F_NO_DIAG | MM_F_NO_DUAL | MM_F_NO_LJOIN;
	mo->min_chain_score = 100, mo->pri_ratio = 0.0f, mo->max_chain_skip = 25;
	mo->occ_dist = 0;
}

extern "C" int mm_set_opt(const char *preset, mm_idxopt_t *io, mm_mapopt_t *mo) // options.c:91-193
{
	if (preset == 0) {
		mm_idxopt_init(io);
		mm_mapopt_init(mo);
		return 0;
	}
	const std::string p(preset);
	if (p == "lr" || p == "map-ont") {
		// the defaults
	} else if (p == "ava-ont") {
		io->flag = 0, io->k = 15, io->w = 5;
		set_ava(mo);
		mo->bw = mo->bw_long = 2000;
	} else if (p == "map10k" || p == "map-pb") {
		io->flag |= MM_I_HPC, io->k = 19;
	} else if (p == "ava-pb") {
		io->flag |= MM_I_HPC, io->k = 19, io->w = 5;
		set_ava(mo);
		mo->bw_long = mo->bw;
	} else if (p == "lr:hq" || p == "map-hifi" || p == "map-ccs") {
		io->flag = 0, io->k = 19, io->w = 19;
		mo->max_gap = 10000;
		mo->min_mid_occ = 50, mo->max_mid_occ = 500;
		if (p != "lr:hq") {
			set_gap_scores(mo, 1, 4, 6, 2, 26, 1);
			mo->min_dp_max = 200;
		}
	} else if (p == "lr:hqae") {
		io->flag = 0, io->k = 25, io->w = 51;
		mo->flag |= MM_F_RMQ;
		mo->min_mid_occ = 50, mo->max_mid_occ = 500;
		mo->rmq_inner_dist = 5000;
		mo->occ_dist = 200;
		mo->best_n = 100;
		mo->chain_gap_scale = 5.0f;
	} else if (p == "map-iclr-prerender") {
		io->flag = 0, io->k = 15;
		mo->b = 6, mo->transition = 1;
		mo->q = 10, mo->q2 = 50;
	} else if (p == "map-iclr") {
		io->flag = 0, io->k = 19;
		mo->b = 6, mo->transition = 4;
		mo->q = 10, mo->q2 = 50;
	} else if (p.compare(0, 3, "asm") == 0) {
		io->flag = 0, io->k = 19, io->w = 19;
		mo->bw = 1000, mo->bw_long = 100000;
		mo->max_gap = 10000;
		mo->flag |= MM_F_RMQ;
		mo->min_mid_occ = 50, mo->max_mid_occ = 500;
		mo->min_dp_max = 200;
		mo->best_n = 50;
		if (p == "asm5") set_gap_scores(mo, 1, 19, 39, 3, 81, 1), mo->zdrop = mo->zdrop_inv = 200;
		else if (p == "asm10") set_gap_scores(mo, 1, 9, 16, 2, 41, 1), mo->zdrop = mo->zdrop_inv = 200;
		else if (p == "asm20") set_gap_scores(mo, 1, 4, 6, 2, 26, 1), mo->zdrop = mo->zdrop_inv = 200, io->w = 10;
		else return -1;
	} else if (p == "short" || p == "sr") {
		io->flag = 0, io->k = 21, io->w = 11;
		mo->flag |= MM_F_SR | MM_F_FRAG_MODE | MM_F_NO_PRINT_2ND | MM_F_2_IO_THREADS | MM_F_HEAP_SORT;
		mo->pe_ori = 0<<1|1;
		set_gap_scores(mo, 2, 8, 12, 2, 24, 1);
		mo->zdrop = mo->zdrop_inv = 100;
		mo->end_bonus = 10;
		mo->max_frag_len = 800;
		mo->max_gap = 100;
		mo->bw = mo->bw_long = 100;
		mo->pri_ratio = 0.5f;
		mo->min_cnt = 2;
		mo->min_chain_score = 25;
		mo->min_dp_max = 40;
		mo->best_n = 20;
		mo->mid_occ = 1000;
		mo->max_occ = 5000;
		mo->mini_batch_size = 50000000;
	} else if (p == "splice" || p == "splice:hq" || p == "splice:sr" || p == "cdna") {
		io->flag = 0, io->k = 15, io->w = 5;
		mo->flag |= MM_F_SPLICE | MM_F_SPLICE_FOR | MM_F_SPLICE_REV | MM_F_SPLICE_FLANK;
		mo->max_sw_mat = 0;
		mo->max_gap = 2000, mo->max_gap_ref = mo->bw = mo->bw_long = 200000;
		set_gap_scores(mo, 1, 2, 2, 1, 32, 0);
		mo->noncan = 9;
		mo->junc_bonus = 9;
		mo->junc_pen = 5;
		mo->zdrop = 200, mo->zdrop_inv = 100;
		if (p == "splice:hq") {
			mo->noncan = 5, mo->b = 4, mo->q = 6, mo->q2 = 24;
		} else if (p == "splice:sr") {
			mo->flag |= MM_F_NO_PRINT_2ND | MM_F_2_IO_THREADS | MM_F_HEAP_SORT | MM_F_FRAG_MODE | MM_F_WEAK_PAIRING | MM_F_SR_RNA;
			mo->noncan = 5, mo->b = 4, mo->q = 6, mo->q2 = 24;
			mo->min_chain_score = 25;
			mo->min_dp_max = 40;
			mo->min_ksw_len = 20;
			mo->pe_ori = 0<<1|1;
			mo->best_n = 10;
			mo->mini_batch_size = 100000000;
		}
	} else return -1;
	return 0;
}

extern "C" int mm_max_spsc_bonus(const mm_mapopt_t *mo) // options.c:195-200
{
	int max_sc = (mo->q2 + 1) / 2 - 1;
	return max_sc > mo->q2 - mo->q? max_sc : mo->q2 - mo->q;
}

static int opt_err(int code, const char *msg)
{
	if (mm_verbose >= 1) fprintf(stderr, "[ERROR]\033[1;31m %s\033[0m\n", msg);
	return code;
}

extern "C" int mm_check_opt(const mm_idxopt_t *io, const mm_mapopt_t *mo) // options.c:202-277 (same codes, same order)
{
	if (mo->bw > mo->bw_long) {
		if (mm_verbose >= 1)
			fprintf(stderr, "[ERROR]\033[1;31m with '-rNUM1,NUM2', NUM1 (%d) can't be larger than NUM2 (%d)\033[0m\n", mo->bw, mo->bw_long);
		return -8;
	}
	if ((mo->flag & MM_F_RMQ) && (mo->flag & (MM_F_SR|MM_F_SPLICE))) return opt_err(-7, "--rmq doesn't work with --sr or --splice");
	if (mo->split_prefix && (mo->flag & (MM_F_OUT_CS|MM_F_OUT_MD))) return opt_err(-6, "--cs or --MD doesn't work with --split-prefix");
	if (io->k <= 0 || io->w <= 0) return opt_err(-5, "-k and -w must be positive");
	if (mo->best_n < 0) return opt_err(-4, "-N must be no less than 0");
	if (mo->best_n == 0 && mm_verbose >= 2)
		fprintf(stderr, "[WARNING]\033[1;31m '-N 0' reduces mapping accuracy. Please use '--secondary=no' instead.\033[0m\n");
	if (mo->pri_ratio < 0.0f || mo->pri_ratio > 1.0f) return opt_err(-4, "-p must be within 0 and 1 (including 0 and 1)");
	if ((mo->flag & MM_F_FOR_ONLY) && (mo->flag & MM_F_REV_ONLY)) return opt_err(-3, "--for-only and --rev-only can't be applied at the same time");
	if (mo->e <= 0 || mo->q <= 0) return opt_err(-1, "-O and -E must be positive");
	if ((mo->q != mo->q2 || mo->e != mo->e2) && !(mo->e > mo->e2 && mo->q + mo->e < mo->q2 + mo->e2))
		return opt_err(-2, "dual gap penalties violating E1>E2 and O1+E1<O2+E2");
	if ((mo->q + mo->e) + (mo->q2 + mo->e2) > 127) return opt_err(-1, "scoring system violating ({-O}+{-E})+({-O2}+{-E2}) <= 127");
	if (mo->sc_ambi < 0 || mo->sc_ambi >= mo->b) return opt_err(-1, "--score-N should be within [0,{-B})");
	if (mo->zdrop < mo->zdrop_inv) return opt_err(-5, "Z-drop should not be less than inversion-Z-drop");
	if ((mo->flag & MM_F_NO_PRINT_2ND) && (mo->flag & MM_F_ALL_CHAINS)) return opt_err(-5, "-X/-P and --secondary=no can't be applied at the same time");
	if ((mo->flag & MM_F_QSTRAND) && ((mo->flag & (MM_F_OUT_SAM|MM_F_SPLICE|MM_F_FRAG_MODE)) || (io->flag & MM_I_HPC)))
		return opt_err(-5, "--qstrand doesn't work with -a, -H, --frag or --splice");
	return 0;
}

// ---- symbols of the reference's private header that its own main.c links against (mmpriv.h:55,104,118,132) ----
#include <sys/resource.h>
extern "C" long peakrss(void) // misc.c:35-44
{
	struct rusage r;
	getrusage(RUSAGE_SELF, &r);
	return r.ru_maxrss * 1024;
}
// split-index merging (main.c:511, --split-prefix) is outside the hot-path scope: the entry point exists so that main.c links unchanged;
// it refuses instead of pretending.
extern "C" int mm_split_merge(int n_segs, const char **fn, const mm_mapopt_t *opt, int n_split_idx)
{
	(void)n_segs; (void)fn; (void)opt; (void)n_split_idx;
	fprintf(stderr, "[ERROR] minimap2_b200: --split-prefix (multi-part index merging) is not supported\n");
	return -1;
}
