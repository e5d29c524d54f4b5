// minimap2_b200/cli/main.cc -- command-line front end linked against libminimap2_b200.so through include/minimap.h only.
// Option letters/long names and their effect on mm_idxopt_t/mm_mapopt_t follow reference main.c:24-351 (presets are
// applied first, then the other options); the run loop follows main.c:437-524.
#include <getopt.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cerrno>
#include <string>
#include "minimap.h"

extern "C" double realtime(void);
extern "C" double cputime(void);

static int64_t parse_num2(const char *str, char **q) // main.c:104-116
{
	char *p;
	double x = strtod(str, &p);
	if (*p == 'G' || *p == 'g') x *= 1e9, ++p;
	else if (*p == 'M' || *p == 'm') x *= 1e6, ++p;
	else if (*p == 'K' || *p == 'k') x *= 1e3, ++p;
	if (q) *q = p;
	return (int64_t)(x + .499);
}
static int64_t parse_num(const char *s) { return parse_num2(s, 0); }

static void yes_or_no(mm_mapopt_t *opt, int64_t flag, const char *name, const char *arg, int yes_to_set)
{
	bool yes = strcmp(arg, "yes") == 0 || strcmp(arg, "y") == 0, no = strcmp(arg, "no") == 0 || strcmp(arg, "n") == 0;
	if (!yes && !no) { fprintf(stderr, "[WARNING]\033[1;31m option '--%s' only accepts 'yes' or 'no'.\033[0m\n", name); return; }
	if ((yes && yes_to_set) || (no && !yes_to_set)) opt->flag |= flag; else opt->flag &= ~flag;
}

static struct option long_options[] = {
	{ "splice-flank", required_argument, 0, 319 }, { "end-seed-pen", required_argument, 0, 321 }, { "cost-non-gt-ag", required_argument, 0, 'C' },
	{ "max-intron-len", required_argument, 0, 'G' }, { "lj-min-ratio", required_argument, 0, 330 }, { "cap-kalloc", required_argument, 0, 349 }, { "no-kalloc", no_argument, 0, 303 },
	{ "bucket-bits", required_argument, 0, 300 }, { "mb-size", required_argument, 0, 'K' }, { "seed", required_argument, 0, 302 },
	{ "no-self", no_argument, 0, 'D' }, { "max-chain-skip", required_argument, 0, 307 }, { "min-dp-len", required_argument, 0, 308 },
	{ "splice", no_argument, 0, 310 }, { "no-long-join", no_argument, 0, 312 }, { "secondary", required_argument, 0, 315 },
	{ "cs", optional_argument, 0, 316 }, { "end-bonus", required_argument, 0, 317 }, { "for-only", no_argument, 0, 322 }, { "qstrand", no_argument, 0, 348 },
	{ "heap-sort", required_argument, 0, 324 },
	{ "rev-only", no_argument, 0, 323 }, { "all-chain", no_argument, 0, 'P' }, { "dual", required_argument, 0, 326 },
	{ "max-clip-ratio", required_argument, 0, 327 }, { "min-occ-floor", required_argument, 0, 328 }, { "MD", no_argument, 0, 329 },
	{ "score-N", required_argument, 0, 331 }, { "eqx", no_argument, 0, 332 }, { "paf-no-hit", no_argument, 0, 333 },
	{ "no-end-flt", no_argument, 0, 335 }, { "hard-mask-level", no_argument, 0, 336 }, { "cap-sw-mem", required_argument, 0, 337 },
	{ "max-qlen", required_argument, 0, 338 }, { "max-chain-iter", required_argument, 0, 339 }, { "sam-hit-only", no_argument, 0, 342 },
	{ "chain-gap-scale", required_argument, 0, 343 }, { "junc-bed", required_argument, 0, 340 }, { "junc-bonus", required_argument, 0, 341 }, { "junc-pen", required_argument, 0, 358 }, { "spsc", required_argument, 0, 357 }, { "jump-min-match", required_argument, 0, 360 }, { "write-junc", no_argument, 0, 361 }, { "pass1", required_argument, 0, 362 }, { "spsc-scale", required_argument, 0, 363 }, { "spsc0", required_argument, 0, 364 }, { "alt", required_argument, 0, 344 }, { "alt-drop", required_argument, 0, 345 }, { "mask-len", required_argument, 0, 346 },
	{ "rmq", optional_argument, 0, 347 }, { "q-occ-frac", required_argument, 0, 350 }, { "chain-skip-scale", required_argument, 0, 351 },
	{ "no-hash-name", no_argument, 0, 353 }, { "secondary-seq", no_argument, 0, 354 }, { "ds", no_argument, 0, 355 },
	{ "rmq-inner", required_argument, 0, 356 }, { "help", no_argument, 0, 'h' }, { "version", no_argument, 0, 'V' },
	{ "min-count", required_argument, 0, 'n' }, { "min-chain-score", required_argument, 0, 'm' }, { "mask-level", required_argument, 0, 'M' },
	{ "min-dp-score", required_argument, 0, 's' }, { "sam", no_argument, 0, 'a' }, { 0, 0, 0, 0 }
};

extern "C" int mm_write_sam_hdr(const mm_idx_t *mi, const char *rg, const char *ver, int argc, char *argv[]); // mmpriv.h:104

int main(int argc, char *argv[])
{
	const char *opt_str = "2aSDw:k:K:t:r:f:Vv:g:G:I:d:XT:s:x:Hcp:M:n:z:A:B:b:O:E:m:N:Qu:R:hF:LC:yYPo:e:U:J:j:";
	mm_mapopt_t opt;
	mm_idxopt_t ipt;
	int c, n_threads = 3, old_best_n = -1, li = 0;
	char *fnw = 0, *s, *alt_list = 0, *fn_bed_junc = 0, *fn_bed_jump = 0, *fn_bed_pass1 = 0, *fn_spsc = 0, *rg = 0;
	float spsc_scale = 0.7f;
	mm_verbose = 3;
	mm_realtime0 = realtime();
	mm_set_opt(0, &ipt, &opt);
	opterr = 0;
	while ((c = getopt_long(argc, argv, opt_str, long_options, &li)) >= 0) { // presets first (main.c:150-163)
		if (c == 'x') {
			if (mm_set_opt(optarg, &ipt, &opt) < 0) { fprintf(stderr, "[ERROR] unknown preset '%s'\n", optarg); return 1; }
		} else if (c == '?') { fprintf(stderr, "[ERROR] unknown option in \"%s\"\n", argv[optind - 1]); return 1; }
	}
	optind = 1;
	while ((c = getopt_long(argc, argv, opt_str, long_options, &li)) >= 0) {
		if (c == 'w') ipt.w = atoi(optarg);
		else if (c == 'k') ipt.k = atoi(optarg);
		else if (c == 'H') ipt.flag |= MM_I_HPC;
		else if (c == 'd') fnw = optarg;
		else if (c == 't') n_threads = atoi(optarg);
		else if (c == 'v') mm_verbose = atoi(optarg);
		else if (c == 'g') opt.max_gap = (int)parse_num(optarg);
		else if (c == 'G') mm_mapopt_max_intron_len(&opt, (int)parse_num(optarg));
		else if (c == 'F') opt.max_frag_len = (int)parse_num(optarg);
		else if (c == 'N') old_best_n = opt.best_n, opt.best_n = atoi(optarg);
		else if (c == 'p') opt.pri_ratio = atof(optarg);
		else if (c == 'M') opt.mask_level = atof(optarg);
		else if (c == 'c') opt.flag |= MM_F_OUT_CG | MM_F_CIGAR;
		else if (c == 'D') opt.flag |= MM_F_NO_DIAG;
		else if (c == 'P') opt.flag |= MM_F_ALL_CHAINS;
		else if (c == 'X') opt.flag |= MM_F_ALL_CHAINS | MM_F_NO_DIAG | MM_F_NO_DUAL | MM_F_NO_LJOIN;
		else if (c == 'a') opt.flag |= MM_F_OUT_SAM | MM_F_CIGAR;
		else if (c == 'Q') opt.flag |= MM_F_NO_QUAL;
		else if (c == 'Y') opt.flag |= MM_F_SOFTCLIP;
		else if (c == 'L') opt.flag |= MM_F_LONG_CIGAR;
		else if (c == 'y') opt.flag |= MM_F_COPY_COMMENT;
		else if (c == 'T') opt.sdust_thres = atoi(optarg);
		else if (c == 'n') opt.min_cnt = atoi(optarg);
		else if (c == 'm') opt.min_chain_score = atoi(optarg);
		else if (c == 'A') opt.a = atoi(optarg);
		else if (c == 'B') opt.b = atoi(optarg);
		else if (c == 'b') opt.transition = atoi(optarg);
		else if (c == 's') opt.min_dp_max = atoi(optarg);
		else if (c == 'C') opt.noncan = atoi(optarg);
		else if (c == 'u') { // transcript strand (main.c:332-341)
			if (*optarg == 'b') opt.flag |= MM_F_SPLICE_FOR | MM_F_SPLICE_REV;
			else if (*optarg == 'f') opt.flag |= MM_F_SPLICE_FOR, opt.flag &= ~MM_F_SPLICE_REV;
			else if (*optarg == 'r') opt.flag |= MM_F_SPLICE_REV, opt.flag &= ~MM_F_SPLICE_FOR;
			else if (*optarg == 'n') opt.flag &= ~(MM_F_SPLICE_FOR | MM_F_SPLICE_REV);
			else { fprintf(stderr, "[ERROR] unrecognized cDNA direction\n"); return 1; }
		}
		else if (c == 'J') { // splice model (main.c:203-208)
			const int t = atoi(optarg);
			if (t == 0) opt.flag |= MM_F_SPLICE_OLD;
			else if (t == 1) opt.flag &= ~MM_F_SPLICE_OLD;
		}
		else if (c == 'R') rg = optarg; // SAM read group line (main.c:199; written by mm_write_sam_hdr, repeated as RG:Z: on every record)
		else if (c == 'j') fn_bed_jump = optarg; // annotated junctions to jump across (main.c:202)
		else if (c == 'I') ipt.batch_size = parse_num(optarg);
		else if (c == 'K') opt.mini_batch_size = parse_num(optarg);
		else if (c == 'e') opt.occ_dist = (int)parse_num(optarg);
		else if (c == '2') opt.flag |= MM_F_2_IO_THREADS;
		else if (c == 'o') {
			if (strcmp(optarg, "-") != 0 && freopen(optarg, "wb", stdout) == NULL) {
				fprintf(stderr, "[ERROR]\033[1;31m failed to write the output to file '%s'\033[0m: %s\n", optarg, strerror(errno));
				exit(1);
			}
		}
		else if (c == 300) ipt.bucket_bits = atoi(optarg);
		else if (c == 302) opt.seed = atoi(optarg);
		else if (c == 307) opt.max_chain_skip = atoi(optarg);
		else if (c == 339) opt.max_chain_iter = atoi(optarg);
		else if (c == 308) opt.min_ksw_len = atoi(optarg);
		else if (c == 310) opt.flag |= MM_F_SPLICE;
		else if (c == 312) opt.flag |= MM_F_NO_LJOIN;
		else if (c == 317) opt.end_bonus = atoi(optarg);
		else if (c == 319) yes_or_no(&opt, MM_F_SPLICE_FLANK, "splice-flank", optarg, 1);
		else if (c == 321) opt.anchor_ext_shift = atoi(optarg);
		else if (c == 330) fprintf(stderr, "[WARNING] \033[1;31m --lj-min-ratio has been deprecated.\033[0m\n");
		else if (c == 349) opt.cap_kalloc = (int64_t)parse_num(optarg); // no kalloc pool here: accepted, without effect
		else if (c == 303) { /* --no-kalloc: nothing to switch off */ }
		else if (c == 322) opt.flag |= MM_F_FOR_ONLY;
		else if (c == 348) opt.flag |= MM_F_QSTRAND | MM_F_NO_INV; // main.c:252
		else if (c == 323) opt.flag |= MM_F_REV_ONLY;
		else if (c == 327) opt.max_clip_ratio = atof(optarg);
		else if (c == 328) opt.min_mid_occ = atoi(optarg);
		else if (c == 329) opt.flag |= MM_F_OUT_MD;
		else if (c == 331) opt.sc_ambi = atoi(optarg);
		else if (c == 332) opt.flag |= MM_F_EQX;
		else if (c == 333) opt.flag |= MM_F_PAF_NO_HIT;
		else if (c == 335) opt.flag |= MM_F_NO_END_FLT;
		else if (c == 336) opt.flag |= MM_F_HARD_MLEVEL;
		else if (c == 337) opt.max_sw_mat = parse_num(optarg);
		else if (c == 338) opt.max_qlen = (int)parse_num(optarg);
		else if (c == 342) opt.flag |= MM_F_SAM_HIT_ONLY;
		else if (c == 343) opt.chain_gap_scale = atof(optarg);
		else if (c == 351) opt.chain_skip_scale = atof(optarg);
		else if (c == 340) fn_bed_junc = optarg;
		else if (c == 341) opt.junc_bonus = atoi(optarg);
		else if (c == 358 || c == 364) opt.junc_pen = atoi(optarg);
		else if (c == 357) fn_spsc = optarg;
		else if (c == 363) spsc_scale = (float)atof(optarg);
		else if (c == 360) opt.jump_min_match = (int)parse_num(optarg); // main.c:261-263
		else if (c == 361) opt.flag |= MM_F_OUT_JUNC | MM_F_CIGAR;
		else if (c == 362) fn_bed_pass1 = optarg;
		else if (c == 344) alt_list = optarg;
		else if (c == 345) opt.alt_drop = atof(optarg);
		else if (c == 346) opt.mask_len = (int)parse_num(optarg);
		else if (c == 350) opt.q_occ_frac = atof(optarg);
		else if (c == 353) opt.flag |= MM_F_NO_HASH_NAME;
		else if (c == 354) opt.flag |= MM_F_SECONDARY_SEQ;
		else if (c == 355) opt.flag |= MM_F_OUT_DS;
		else if (c == 356) opt.rmq_inner_dist = (int)parse_num(optarg);
		else if (c == 315) yes_or_no(&opt, MM_F_NO_PRINT_2ND, "secondary", optarg, 0);
		else if (c == 326) yes_or_no(&opt, MM_F_NO_DUAL, "dual", optarg, 0);
		else if (c == 324) yes_or_no(&opt, MM_F_HEAP_SORT, "heap-sort", optarg, 1);
		else if (c == 316) {
			opt.flag |= MM_F_OUT_CS | MM_F_CIGAR;
			if (optarg == 0 || strcmp(optarg, "short") == 0) opt.flag &= ~MM_F_OUT_CS_LONG;
			else if (strcmp(optarg, "long") == 0) opt.flag |= MM_F_OUT_CS_LONG;
			else if (strcmp(optarg, "none") == 0) opt.flag &= ~MM_F_OUT_CS;
		} else if (c == 347) {
			if (optarg) yes_or_no(&opt, MM_F_RMQ, "rmq", optarg, 1); else opt.flag |= MM_F_RMQ;
		} else if (c == 'S') opt.flag |= MM_F_OUT_CS | MM_F_CIGAR | MM_F_OUT_CS_LONG;
		else if (c == 'V') { puts(MM_VERSION); return 0; }
		else if (c == 'r') {
			opt.bw = (int)parse_num2(optarg, &s);
			if (*s == ',') opt.bw_long = (int)parse_num2(s + 1, &s);
		} else if (c == 'U') {
			opt.min_mid_occ = strtol(optarg, &s, 10);
			if (*s == ',') opt.max_mid_occ = strtol(s + 1, &s, 10);
		} else if (c == 'f') {
			char *p;
			double x = strtod(optarg, &p);
			if (x < 1.0) opt.mid_occ_frac = x, opt.mid_occ = 0;
			else opt.mid_occ = (int)(x + .499);
			if (*p == ',') opt.max_occ = (int)(strtod(p + 1, &p) + .499);
		} else if (c == 'z') {
			opt.zdrop = opt.zdrop_inv = strtol(optarg, &s, 10);
			if (*s == ',') opt.zdrop_inv = strtol(s + 1, &s, 10);
		} else if (c == 'O') {
			opt.q = opt.q2 = strtol(optarg, &s, 10);
			if (*s == ',') opt.q2 = strtol(s + 1, &s, 10);
		} else if (c == 'E') {
			opt.e = opt.e2 = strtol(optarg, &s, 10);
			if (*s == ',') opt.e2 = strtol(s + 1, &s, 10);
		} else if (c == 'h') {
			printf("Usage: minimap2-b200 [options] <target.fa>|<target.idx> [query.fa] [...]\n"
				   "  H100-native minimap2-compatible mapper; options follow minimap2 (-x -k -w -c -a -t -d --cs --MD --eqx ...)\n");
			return 0;
		}
	}
	if (mm_check_opt(&ipt, &opt) < 0) return 1;
	if (opt.best_n == 0) {
		fprintf(stderr, "[WARNING]\033[1;31m changed '-N 0' to '-N %d --secondary=no'.\033[0m\n", old_best_n);
		opt.best_n = old_best_n, opt.flag |= MM_F_NO_PRINT_2ND;
	}
	if (argc == optind) { fprintf(stderr, "Usage: minimap2-b200 [options] <target.fa>|<target.idx> [query.fa] [...]\n"); return 1; }
	mm_idx_reader_t *idx_rdr = mm_idx_reader_open(argv[optind], &ipt, fnw);
	if (idx_rdr == 0) { fprintf(stderr, "[ERROR] failed to open file '%s': %s\n", argv[optind], strerror(errno)); return 1; }
	if (!idx_rdr->is_idx && fnw == 0 && argc - optind < 2) {
		fprintf(stderr, "[ERROR] missing input: please specify a query file to map or option -d to keep the index\n");
		mm_idx_reader_close(idx_rdr);
		return 1;
	}
	mm_idx_t *mi;
	while ((mi = mm_idx_reader_read(idx_rdr, n_threads)) != 0) {
		int ret = 0;
		if ((opt.flag & MM_F_CIGAR) && (mi->flag & MM_I_NO_SEQ)) { // main.c:439-443
			fprintf(stderr, "[ERROR] the prebuilt index doesn't contain sequences.\n");
			mm_idx_destroy(mi);
			mm_idx_reader_close(idx_rdr);
			return 1;
		}
		if (fn_bed_junc) { // main.c:467-471
			mm_idx_bed_read(mi, fn_bed_junc, 1);
			if (mi->I == 0 && mm_verbose >= 2) fprintf(stderr, "[WARNING] failed to load the junction BED file\n");
		}
		if (fn_bed_jump) { // main.c:472-481: annotated junctions, then pass-1 junctions scoring at least 5, merged into one table
			mm_idx_jjump_read(mi, fn_bed_jump, MM_JUNC_ANNO, -1);
			if (mi->J == 0 && mm_verbose >= 2) fprintf(stderr, "[WARNING] failed to load the jump BED file\n");
		}
		if (fn_bed_pass1) {
			mm_idx_jjump_read(mi, fn_bed_pass1, MM_JUNC_MISC, 5);
			if (mi->J == 0 && mm_verbose >= 2) fprintf(stderr, "[WARNING] failed to load the pass-1 jump BED file\n");
		}
		if (fn_spsc) { // main.c:482-486
			mm_idx_spsc_read2(mi, fn_spsc, mm_max_spsc_bonus(&opt), spsc_scale);
			if (mi->spsc == 0 && mm_verbose >= 2) fprintf(stderr, "[WARNING] failed to load the splice score file\n");
		}
		if (alt_list) mm_idx_alt_read(mi, alt_list); // main.c:487
		if ((opt.flag & MM_F_OUT_SAM) && idx_rdr->n_parts == 1) { // SAM header (main.c:445-460, format.c:119-148)
			int hret;
			if (mm_idx_reader_eof(idx_rdr)) hret = mm_write_sam_hdr(mi, rg, MM_VERSION, argc, argv);
			else hret = mm_write_sam_hdr(0, rg, MM_VERSION, argc, argv);
			if (hret != 0) { mm_idx_destroy(mi); mm_idx_reader_close(idx_rdr); return 1; }
		}
		if (mm_verbose >= 3)
			fprintf(stderr, "[M::%s::%.3f*%.2f] loaded/built the index for %d target sequence(s)\n", __func__, realtime() - mm_realtime0, cputime() / (realtime() - mm_realtime0), mi->n_seq);
		if (argc != optind + 1) mm_mapopt_update(&opt, mi);
		if (mm_verbose >= 3) mm_idx_stat(mi);
		if (argc - (optind + 1) == 0) { mm_idx_destroy(mi); continue; }
		for (int i = optind + 1; i < argc; ++i) {
			ret = mm_map_file(mi, argv[i], &opt, n_threads);
			if (ret < 0) break;
		}
		mm_idx_destroy(mi);
		if (ret < 0) { fprintf(stderr, "ERROR: failed to map the query file\n"); exit(EXIT_FAILURE); }
	}
	mm_idx_reader_close(idx_rdr);
	if (fflush(stdout) == EOF) { perror("[ERROR] failed to write the results"); exit(EXIT_FAILURE); }
	if (mm_verbose >= 3) {
		fprintf(stderr, "[M::%s] Version: %s\n", __func__, MM_VERSION);
		fprintf(stderr, "[M::%s] CMD:", __func__);
		for (int i = 0; i < argc; ++i) fprintf(stderr, " %s", argv[i]);
		fprintf(stderr, "\n[M::%s] Real time: %.3f sec; CPU: %.3f sec\n", __func__, realtime() - mm_realtime0, cputime());
	}
	return 0;
}
