// minimap2_b200/csrc/hostlogic.h -- host orchestration pieces (hit post-processing, alignment driver, formatting).
#pragma once
#include <cstdint>
#include <cstdio>
#include <vector>
#include <string>
#include <unordered_map>
#include "minimap.h"
#include "mm_b200.h"
#include "mm_algo.cuh"

#define HL_PARENT_UNSET   (-1)   // mmpriv.h:9-10
#define HL_PARENT_TMP_PRI (-2)

// ---- hits.cc ----
void hl_reg_set_coor(mm_reg1_t *r, int32_t qlen, const m128 *a, int is_qstrand);
mm_reg1_t *hl_gen_regs(uint32_t hash, int qlen, int n_u, const uint64_t *u, const m128 *a, int is_qstrand);
void hl_split_reg(mm_reg1_t *r, mm_reg1_t *r2, int n, int qlen, m128 *a, int is_qstrand);
void hl_set_parent(float mask_level, int mask_len, int n, mm_reg1_t *r, int sub_diff, int hard_mask_level, float alt_diff_frac);
void hl_hit_sort(int *n_regs, mm_reg1_t *r, float alt_diff_frac);
void hl_sdust(const uint8_t *seq, int l_seq, int T, int W, std::vector<uint64_t> &res); // sdust_core (sdust.c:135-170): masked intervals start<<32|finish of an ASCII sequence
int hl_set_sam_pri(int n, mm_reg1_t *r);
void hl_sync_regs(int n_regs, mm_reg1_t *regs);
void hl_select_sub(float pri_ratio, int min_diff, int best_n, int check_strand, int min_strand_sc, int *n_, mm_reg1_t *r);
int hl_filter_strand_retained(int n_regs, mm_reg1_t *r);
void hl_filter_regs(const mm_mapopt_t *opt, int qlen, int *n_regs, mm_reg1_t *regs);
int hl_squeeze_a(int n_regs, mm_reg1_t *regs, m128 *a);
void hl_set_mapq(int n_regs, mm_reg1_t *regs, int min_chain_sc, int match_sc, int rep_len, int is_sr, int is_splice);
void hl_est_err(const mm_idx_t *mi, int qlen, int n_regs, mm_reg1_t *regs, const m128 *a, int32_t n, const uint64_t *mini_pos);
double hl_event_identity(const mm_reg1_t *r);
void hl_update_dp_max(int qlen, int n_regs, mm_reg1_t *regs, float frac, int a, int b);

// ---- align.cc: the alignment driver (mm_align_skeleton / mm_align1, align.c:645-1120) as a replayable routine ----
void hl_gen_mat(int8_t *mat, const mm_mapopt_t *opt); // the 5x5 score matrix of the options (align.c:11-38): the driver's and the kernels'
struct KswKey {
	int64_t q_start, t_start;
	int32_t q_step, t_step, qlen, tlen, w, zdrop, end_bonus, flag;
	bool operator==(const KswKey &o) const {
		return q_start == o.q_start && t_start == o.t_start && q_step == o.q_step && t_step == o.t_step && qlen == o.qlen &&
			   tlen == o.tlen && w == o.w && zdrop == o.zdrop && end_bonus == o.end_bonus && flag == o.flag;
	}
};
struct KswKeyHash {
	size_t operator()(const KswKey &k) const {
		uint64_t h = mmx_hash64_full((uint64_t)k.q_start * 0x9E3779B97F4A7C15ULL ^ (uint64_t)k.t_start);
		h = mmx_hash64_full(h ^ ((uint64_t)(uint32_t)k.qlen << 32 | (uint32_t)k.tlen));
		h = mmx_hash64_full(h ^ ((uint64_t)(uint32_t)k.flag << 32 | (uint32_t)k.w) ^ ((uint64_t)(uint32_t)k.zdrop << 20) ^ (uint32_t)k.end_bonus ^ ((uint64_t)(k.q_step + 2) << 60) ^ ((uint64_t)(k.t_step + 2) << 56));
		return (size_t)h;
	}
};

struct KswDone {            // a finished job: ksw_extz_t fields + its CIGAR (points into the wave's pinned result buffer)
	mmb_ksw_res_t r;
	const uint32_t *cig;
	const uint32_t *dcig = nullptr; // the same CIGAR in the device arena of its wave (kept until the batch ends; input of K4)
};
struct HlFinJob { const uint32_t *dcig; uint32_t n; };   // one piece of a hit's CIGAR (device address, operations)
struct HlFinHit {            // a hit whose CIGAR assembly / mm_fix_cigar / mm_update_extra is left to the device tail (finalize.cu)
	mm_extra_t *p;           // identifies the hit in the read's mm_reg1_t array (allocated once in this mode: header only)
	int32_t rev, qs, rid, rs, qspan, tspan; // strand the query piece is read on, its start there, target sequence and start, bases consumed
	int32_t job_first, n_jobs;
	uint32_t n_cig_max;      // sum of the pieces' operation counts (upper bound of the final count)
};
// What mm_align1 decides from the anchors alone (align.c:693-813: end filters, seed filters, the DP window, which anchor pairs get a
// gap fill), kept per hit across the replays of a read: a later replay goes straight to consuming results. slot = the job's index in
// the read's job cache once it has been requested (-1: not yet).
struct HlFill { int32_t i, qs, qe, rs, re, bw1, slot; };
struct HlHitPlan {
	int32_t as, cnt; int64_t splice_flag;                       // identity of the hit (anchor range after mm_squeeze_a) and the transcript-strand round
	int32_t as1, cnt1, rs, qs, re, qe, rs0, qs0, re0, qe0;
	int32_t slot_left = -1, slot_right = -1;
	std::vector<HlFill> fills;
	std::vector<std::pair<int32_t, uint64_t>> marks; // IGNORE / LONG_JOIN bits the seed filters put on the hit's anchors: put back when the plan is
	                                                  // reused, because a hit split off this one later is planned from the marked anchors (align.c:454-525)
};
struct HlFinOut { int32_t n_cigar, blen, mlen, n_ambi, dp_max, qshift, tshift, status, is_spliced, pad[3]; }; // = FinOut (pipeline.h)

struct ReadAlign {          // per-read alignment working set (lives across waves; pooled across batches, so the vectors keep their capacity)
	int qlen = 0;
	int64_t q_dev_off = 0;  // offset of this read's first base in the device query array
	const uint8_t *qseq[2] = {nullptr, nullptr}; // nt4 forward / reverse complement (align.c:1056-1061), slices of a pooled buffer
	// The two copies are made on first use: with the device tail on, only rare host paths read query bases (z-drop scan of a job the
	// packed kernel did not take, inversion probes, HPC seed adjustment), so most reads never pay for them.
	const char *raw_seq = nullptr; uint8_t *qbuf = nullptr; mutable bool qseq_ready = false;
	void ensure_qseq() const {
		if (qseq_ready || !qbuf) return;
		uint8_t *q0 = qbuf, *q1 = qbuf + qlen;
		for (int i = 0; i < qlen; ++i) { const uint8_t c = mmx_nt4((uint8_t)raw_seq[i]); q0[i] = c, q1[qlen - 1 - i] = c < 4? 3 - c : 4; }
		qseq_ready = true;
	}
	std::vector<KswKey> keys;      // job cache: keys[i] -> done_idx[i] (-1: requested, not delivered yet); ~50-100 entries, linear probe
	std::vector<int> done_idx;
	std::vector<KswDone> done;
	std::vector<mmb_ksw_job_t> want; // jobs requested by the current replay
	std::vector<int> want_slot;      // their slots in keys[]
	bool incomplete = false;
	bool defer = false;              // in: finished hits go to the device tail instead of the host's append / fix_cigar / update_extra
	bool defer_abort = false;        // out: the replay reached a step that needs a hit's final coordinates (inversion probe): redo it with defer off
	std::vector<HlFinHit> fin_hits;  // out (defer): the hits to finalize, in driver order, and their pieces
	std::vector<HlFinJob> fin_jobs;
	std::vector<HlHitPlan> plans;    // per-hit plans of this read (see HlHitPlan); cleared with the job cache
	mutable size_t hint = 0;         // a replay asks for its jobs in the order the previous one did: search from the last hit on
	void reset() { keys.clear(); done_idx.clear(); done.clear(); want.clear(); want_slot.clear(); fin_hits.clear(); fin_jobs.clear(); plans.clear(); incomplete = defer = defer_abort = false; hint = 0; }
	int find(const KswKey &k) const { // keys are unique (a key is added only after a miss)
		const size_t n = keys.size();
		for (size_t c = 0, i = hint < n? hint : 0; c < n; ++c, i = i + 1 == n? 0 : i + 1)
			if (keys[i] == k) { hint = i + 1; return (int)i; }
		return -1;
	}
};

// Runs the whole per-read alignment (mm_align_skeleton semantics) using cached ksw results; missing results are appended
// to ra.want and ra.incomplete is set. When complete, *n_regs_/regs hold the aligned hits (regs may be realloc'd).
// a[] must have its IGNORE/LONG_JOIN marks cleared by the caller before every replay.
mm_reg1_t *hl_align_skeleton(const mm_mapopt_t *opt, const mm_idx_t *mi, ReadAlign &ra, int *n_regs_, mm_reg1_t *regs, int n_a, m128 *a);
// With ra.defer set, a complete replay that produced ra.fin_hits stops before the hit-level tail of mm_align_skeleton (align.c:1103-1118);
// once the device has finalized the hits, hl_align_apply_fin() stores the results (fin[i] / CIGAR at out + off[i] for ra.fin_hits[i]; returns
// false if a hit must be redone on the host) and hl_align_finish() runs that tail.
bool hl_align_apply_fin(ReadAlign &ra, int n_regs, mm_reg1_t *regs, const HlFinOut *fin, const uint32_t *const *cig);
void hl_align_finish(const mm_mapopt_t *opt, ReadAlign &ra, int *n_regs_, mm_reg1_t *regs);
inline bool hl_defer_supported(const mm_mapopt_t *opt) { return !(opt->flag & (MM_F_SPLICE | MM_F_EQX | MM_F_QSTRAND | MM_F_SR | MM_F_SR_RNA)); }

// ---- host section profiler (MM_B200_TIMING only): cycles per section, summed over threads ----
enum { HP_SKEL, HP_TSEQ, HP_ZDROP, HP_EXTRA, HP_FETCH, HP_APPEND, HP_PRE, HP_POST, HP_HITS, HP_N };
extern uint64_t g_hp[HP_N];
extern bool g_hp_on;
extern thread_local uint64_t tl_hp[HP_N];
struct HpScope { // accumulates in thread-local counters; hl_hp_flush() adds them to the global sums (once per read)
	int k; uint64_t t0;
	explicit HpScope(int k_) : k(k_), t0(g_hp_on? __builtin_ia32_rdtsc() : 0) {}
	~HpScope() { if (g_hp_on) tl_hp[k] += __builtin_ia32_rdtsc() - t0; }
};
void hl_hp_flush();
void hl_hp_dump(const char *tag);

// ---- format.cc ----
struct hl_str { std::string s; };
void hl_set_seq_for_tags(const char *seq);
void hl_write_paf(std::string &s, const mm_idx_t *mi, const char *qname, int qlen, const mm_reg1_t *r, int64_t opt_flag, int rep_len);
void hl_write_junc(std::string &s, const mm_idx_t *mi, const char *qname, const mm_reg1_t *r);
void hl_write_sam(std::string &s, const mm_idx_t *mi, const char *qname, const char *seq, const char *qual, int qlen, int reg_idx,
				  int n_regs, const mm_reg1_t *regs, int64_t opt_flag, int rep_len);
int hl_write_sam_hdr(std::string &s, const mm_idx_t *mi, const char *rg, const char *ver, int argc, char *argv[]);
