// minimap2_b200/csrc/map.cu -- the GPU batch scheduler behind mm_map / mm_map_frag / mm_map_file (minimap.h).
//
// Replaces the reference's thread pipeline (map.c:403-691: worker_pipeline / kt_for(worker_for)) and the per-read
// orchestration mm_map_frag_core (map.c:227-378). A batch of reads goes through
//   stage 1 (device, whole batch per launch): encode -> K1 sketch -> K2a lookup/select -> K2b expand+sort -> K2c chain
//   stage 2 (host threads): chains -> hits (hits.cc), primary/secondary selection, divergence estimate
//   stage 3 (waves): host threads replay the alignment driver (align.cc) per read, the ksw2 jobs they request are run as
//            one K3 launch set per wave, results are scattered back into per-read caches; typically 2-3 waves
//   stage 4 (host threads): final hit selection and MAPQ
//   stage 5 (index with a jump table only): K5 junction jumps on the device, applied to the hits on the host threads
// Results are returned in input order with the reference's ownership rules (libc malloc, caller frees).
#include "pipeline.h"
#include "jump.cuh"
#include "hostlogic.h"
#include "scan.cuh"
#include "ksw_plan.h"
#include "fastx.h"
#include <thread>
#include <unistd.h>
#include <malloc.h>
#include <climits>
#include <atomic>
#include <functional>
#include <cstring>
#include <algorithm>
#include <mutex>
#include <condition_variable>
#include <deque>
#include <memory>

extern "C" double realtime(void);
extern "C" double cputime(void);
int mmb_resident_reads(void);

namespace {

// A persistent host worker pool shared by every group: a group's host phase is one Task (an index range consumed in
// grains); workers swarm the oldest unfinished task, and the submitting thread works on its own task too. This replaces
// kt_for (kthread.c:54-70) -- persistent threads keep their malloc arenas and avoid spawning ~100 threads per phase.
struct Task {
	const std::function<void(int64_t, int)> *fn;
	int64_t n, grain;
	std::atomic<int64_t> next{0}, done{0};
};
class HostPool {
public:
	explicit HostPool(int n_workers) {
		for (int t = 0; t < n_workers; ++t) th_.emplace_back([this, t]() { worker(t + 1); });
	}
	void run(int64_t n, const std::function<void(int64_t, int)> &fn) {
		if (n <= 0) return;
		auto task = std::make_shared<Task>();
		task->fn = &fn, task->n = n, task->grain = std::max<int64_t>(1, n / ((int64_t)(th_.size() + 1) * 8));
		{ std::lock_guard<std::mutex> lk(mu_); q_.push_back(task); }
		cv_.notify_all();
		work_on(*task, 0);
		if (task->done.load(std::memory_order_acquire) < n) { // wait for grains still running on workers
			std::unique_lock<std::mutex> lk(mu_);
			done_cv_.wait(lk, [&]() { return task->done.load(std::memory_order_acquire) >= n; });
		}
		std::lock_guard<std::mutex> lk(mu_);
		for (size_t i = 0; i < q_.size(); ++i) if (q_[i] == task) { q_.erase(q_.begin() + i); break; }
	}
private:
	void work_on(Task &t, int tid) {
		for (;;) {
			const int64_t b = t.next.fetch_add(t.grain);
			if (b >= t.n) break;
			const int64_t e = std::min(t.n, b + t.grain);
			for (int64_t i = b; i < e; ++i) (*t.fn)(i, tid);
			if (t.done.fetch_add(e - b, std::memory_order_acq_rel) + (e - b) >= t.n) { std::lock_guard<std::mutex> lk(mu_); done_cv_.notify_all(); }
		}
	}
	void worker(int tid) {
		for (;;) {
			std::shared_ptr<Task> t;
			{
				std::unique_lock<std::mutex> lk(mu_);
				cv_.wait(lk, [&]() {
					for (auto &x : q_) if (x->next.load(std::memory_order_relaxed) < x->n) { t = x; return true; }
					return false;
				});
			}
			work_on(*t, tid);
		}
	}
	std::mutex mu_;
	std::condition_variable cv_, done_cv_;
	std::deque<std::shared_ptr<Task>> q_;
	std::vector<std::thread> th_;
};
HostPool *g_pool = nullptr;
std::once_flag g_pool_once;

void parallel_for(int64_t n, int n_threads, const std::function<void(int64_t, int)> &fn)
{
	if (n <= 0) return;
	if (n_threads <= 1 || n == 1) { for (int64_t i = 0; i < n; ++i) fn(i, 0); return; }
	std::call_once(g_pool_once, [&]() { // sized by the first caller; never torn down
		// The group threads that feed the GPU must never wait for a core: with one worker per logical CPU the launches of
		// the next kernels queue behind replay work and the GPU idles (measured: 128 workers 1.42 s/step, 64 workers 1.05 s on
		// a 128-thread host). Default cap: half of the online CPUs; MM_B200_HOST_THREADS overrides.
		int cap = (int)sysconf(_SC_NPROCESSORS_ONLN) / 2;
		if (getenv("MM_B200_HOST_THREADS")) cap = atoi(getenv("MM_B200_HOST_THREADS"));
		if (cap < 2) cap = 2;
		g_pool = new HostPool(std::min(n_threads, cap) - 1);
	});
	g_pool->run(n, fn);
}

const int g_gpu_slots_env = getenv("MM_B200_GPU_SLOTS")? std::max(1, atoi(getenv("MM_B200_GPU_SLOTS"))) : 0;
int g_gpu_slots = g_gpu_slots_env; // 0: two thirds of the groups of the batch
int g_batch_groups = 1;
// FIFO gate bounding how many groups are in a device phase at once: with more groups than slots, the groups fall out of
// lock-step and one group's host phase overlaps the others' kernels. By default two thirds of the groups may hold a slot (8 of
// 12). A group in a device phase spends most of it waiting for its stream (mmb_stream_sync, which leaves the CPU to the host
// phases), a map-ont group about twice as long as in its host phases; so with a third of the groups on the host the device is
// rarely without work. Fewer slots keep groups waiting to enter stage 1 while the groups that got through run host phases
// with the device idle; with one slot per group they all move through the pipeline in lock-step (DESIGN §6).
class GpuGate {
public:
	// Two request classes: 0 = stage 1 of a group (sketch..chain), 1 = an alignment wave. Each class is FIFO. While both have
	// requests waiting, waves get all slots but one: finishing groups early spreads the host replay work over the batch,
	// and the reserved slot keeps new groups entering so that the end of the batch is not a single group's serial chain.
	void acquire(int cls) {
		std::unique_lock<std::mutex> lk(mu_);
		const uint64_t my = tail_[cls]++;
		cv_.wait(lk, [&]() {
			if (my != head_[cls] || in_[0] + in_[1] >= slots()) return false;
			const bool other_waiting = head_[1 - cls] != tail_[1 - cls];
			if (!other_waiting) return true;
			return cls == 1? in_[1] < std::max(1, slots() - 1) : in_[0] < 1;
		});
		++head_[cls], ++in_[cls];
		cv_.notify_all();
	}
	void release(int cls) { std::lock_guard<std::mutex> lk(mu_); --in_[cls]; cv_.notify_all(); }
	static int slots() { return g_gpu_slots > 0? g_gpu_slots : std::max(1, (2 * g_batch_groups + 2) / 3); }
private:
	std::mutex mu_;
	std::condition_variable cv_;
	uint64_t head_[2] = {0, 0}, tail_[2] = {0, 0};
	int in_[2] = {0, 0};
};
GpuGate g_gate;
struct GateHold {
	mmb_ctx_t *ctx; bool use, on = false; int cls;
	GateHold(mmb_ctx_t *c, bool use_, int cls_, bool now = true) : ctx(c), use(use_), cls(cls_) { if (now) take(); }
	void take() {
		if (!use || on) return;
		mmb_tl(ctx, MMB_TL_GATE_REQ, cls);
		g_gate.acquire(cls);
		mmb_tl(ctx, MMB_TL_GATE_GRANT, cls);
		on = true;
	}
	void drop() { if (on) g_gate.release(cls), mmb_tl(ctx, MMB_TL_GATE_REL, cls), on = false; }
	~GateHold() { drop(); }
};

// Host phases of a group's batch on the scheduler timeline (MMB_TL_HOST_BEGIN / _END arguments)
enum HostPhase { HPH_CONCAT, HPH_HITS, HPH_REPLAY, HPH_TAIL_PREP, HPH_TAIL_APPLY, HPH_JOBS, HPH_KSW_PLAN, HPH_SCATTER, HPH_FINALIZE };
struct HostSpan {
	mmb_ctx_t *ctx; int ph;
	HostSpan(mmb_ctx_t *c, int p) : ctx(c), ph(p) { mmb_tl(ctx, MMB_TL_HOST_BEGIN, ph); }
	~HostSpan() { mmb_tl(ctx, MMB_TL_HOST_END, ph); }
};

__global__ void encode_kernel(uint8_t *s, int64_t n)
{
	int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if (i + 3 < n) {
		uchar4 v = *reinterpret_cast<uchar4*>(s + i);
		v.x = mmx_nt4(v.x), v.y = mmx_nt4(v.y), v.z = mmx_nt4(v.z), v.w = mmx_nt4(v.w);
		*reinterpret_cast<uchar4*>(s + i) = v;
	} else for (; i < n; ++i) s[i] = mmx_nt4(s[i]);
}

__global__ void init_nmz_kernel(const int64_t *mz_off, int n, int32_t *n_mz)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) n_mz[i] = (int32_t)(mz_off[i + 1] - mz_off[i]);
}

// mm_dust_minier (map.c:33-57): minimizers of a read more than half covered by its masked (low-complexity) intervals are squeezed
// out, order kept. dreg: the read's intervals start<<32|finish in query order (host: hl_sdust). One thread per read -- the -T option
// is off by default and rarely used.
__global__ void dust_filter_kernel(m128 *mz, const int64_t *mz_off, int32_t *n_mz, const uint64_t *dreg, const int64_t *dreg_off, int n_reads)
{
	const int rd = blockIdx.x * blockDim.x + threadIdx.x;
	if (rd >= n_reads) return;
	const uint64_t *dr = dreg + dreg_off[rd];
	const int n_dreg = (int)(dreg_off[rd + 1] - dreg_off[rd]), n = n_mz[rd];
	if (n_dreg == 0) return;
	m128 *a = mz + mz_off[rd];
	int u = 0, k = 0;
	for (int j = 0; j < n; ++j) {
		const int32_t qpos = (int32_t)((uint32_t)a[j].y >> 1), span = (int32_t)(a[j].x & 0xff);
		const int32_t s = qpos - (span - 1), e = s + span;
		while (u < n_dreg && (int32_t)dr[u] <= s) ++u;
		if (u < n_dreg && (int32_t)(dr[u] >> 32) < e) {
			int l = 0;
			for (int v = u; v < n_dreg && (int32_t)(dr[v] >> 32) < e; ++v) { // intervals overlapping this minimizer
				const int ss = s > (int32_t)(dr[v] >> 32)? s : (int32_t)(dr[v] >> 32);
				const int ee = e < (int32_t)dr[v]? e : (int32_t)(uint32_t)dr[v];
				l += ee - ss;
			}
			if (l <= span >> 1) a[k++] = a[j];
		} else a[k++] = a[j];
	}
	n_mz[rd] = k;
}

__global__ void copy_i64_kernel(const int64_t *a, int n, int64_t *b)
{
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) b[i] = a[i];
}

// gather per-read slices (src at src_off[r], cnt[r] items) into a dense array at dst_off[r]; one warp per read
template<class T>
__global__ void gather_kernel(const T *src, const int64_t *src_off, const int32_t *cnt, const int64_t *dst_off, int n_reads, T *dst)
{
	const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (w >= n_reads) return;
	const T *s = src + src_off[w];
	T *d = dst + dst_off[w];
	for (int i = lane; i < cnt[w]; i += 32) d[i] = s[i];
}

inline uint32_t x31_hash_string(const char *s) // khash.h:383-388
{
	uint32_t h = (uint32_t)*s;
	if (h) for (++s; *s; ++s) h = (h << 5) - h + (uint32_t)*s;
	return h;
}
inline uint32_t wang_hash(uint32_t key) // khash.h:400-409
{
	key += ~(key << 15); key ^= (key >> 10); key += (key << 3); key ^= (key >> 6); key += ~(key << 11); key ^= (key >> 16);
	return key;
}

struct ReadState {
	int qlen = 0;
	const char *seq = nullptr, *name = nullptr;
	uint32_t hash = 0;
	int rep_len = 0, n_mini_pos = 0, n_u = 0, n_a = 0;
	const uint64_t *mini_pos = nullptr, *u = nullptr;
	const m128 *a_src = nullptr;
	int n_regs0 = 0;
	mm_reg1_t *regs0 = nullptr;            // after chain_post/est_err (pristine, no ->p)
	std::vector<m128> a;                   // working copy of the anchors for the alignment replay (capacity kept across batches)
	ReadAlign *ra = nullptr;               // points into the pooled ReadAlign array
	int n_regs = 0;
	mm_reg1_t *regs = nullptr;             // final
	bool done = false;
	bool fin_pending = false;              // the replay is complete; its hits wait for the device tail (K4)
};

struct BatchBufs { // device arenas reused across batches (per context)
	DevBuf a2, seq, off, mz, mz_off, n_mz, qlen, s_n, s_off, k_idx, k_aoff, flt, mini_pos, n_keep, rep_len, n_a, a_off, a, stk;
	DevBuf n_u, n_v, u, a_out, ch1, ch2, t1, t2, doff, dense_u, dense_a, dense_mp;
	DevBuf jobs, res, cig;
	std::vector<std::unique_ptr<DevBuf>> cig_keep; // one CIGAR arena per (wave, chunk), alive until the batch ends: K4 reads the pieces in place
	DevBuf fin_in, fin_out;                // K4: hit / piece descriptors; results + assembled CIGARs
	PinBuf h_fin_in, h_fin_out;
	DevBuf qlo, qhi, k_cnt;                // skip_seed inputs (ava / strand-restricted modes only)
	DevBuf dreg, dreg_off;                 // masked intervals of the reads (-T / SDUST only)
	DevBuf jump_io; PinBuf h_jump;         // K5 hit descriptors and decisions (jump table only)
	PinBuf h_seq, h_misc, h_jobs, h_res, h_used;
	std::vector<std::unique_ptr<PinBuf>> h_cig; // one CIGAR staging buffer per alignment wave (cached results point into them until the batch ends)
	std::vector<ReadState> rs_pool;        // persistent per-read objects: their vectors keep capacity => no allocation in steady state
	std::vector<ReadAlign> ra_pool;
	std::vector<uint8_t> qseq_pool;        // nt4 forward + reverse-complement copies of the batch (2 x total bases)
};
struct GroupCtx { mmb_ctx_t *ctx = nullptr; BatchBufs bb; bool gated = false; int64_t res_n = -1, res_bases = -1; const char *res_first = nullptr; };
const int MAX_GROUPS = 16;
GroupCtx *g_groups[MAX_GROUPS] = {nullptr};
std::mutex g_group_mu;


// false (after a message) for modes this build does not implement: the API calls then return an error / no hits instead of mapping
// with different semantics -- there is no CPU fallback, and a library must not take the caller's process down for an option
bool supported_mode(const mm_idx_t *mi, const mm_mapopt_t *opt)
{
	const char *what = nullptr;
	if (opt->flag & (MM_F_SR | MM_F_SR_RNA)) what = "short-read mode (-x sr / splice:sr)";
	else if (mi->J && (opt->flag & MM_F_SPLICE) && (opt->flag & MM_F_EQX)) what = "junction jumps (-j / --pass1) with =/X CIGARs (--eqx)"; // jump.c:198 asserts
	else if ((opt->flag & MM_F_QSTRAND) && (!(opt->flag & MM_F_NO_INV) || (opt->flag & (MM_F_SPLICE | MM_F_OUT_SAM)) || (mi->flag & MM_I_HPC)))
		what = "query-strand mode without MM_F_NO_INV (main.c:252 sets both), or combined with splice / SAM / HPC (mm_check_opt rejects those)";
	if (what) fprintf(stderr, "[ERROR] minimap2_b200: %s is not implemented in this build; refusing to map (no CPU fallback)\n", what);
	return what == nullptr;
}

} // namespace

// pass: first mapping pass, or the re-chaining pass of map.c:293-316 over the reads the first pass left without a chain
struct MapPass {
	int occ_cut;        // max_occ argument of mm_collect_matches (map.c:174): mid_occ, or opt->max_occ when re-chaining
	bool rescue;        // long-join re-chaining (map.c:283-292) only exists in the first pass
	uint8_t *no_chain;  // out (optional): 1 for reads that went through chaining and came out with no chain at all
};

namespace {

// One batch of a group on its way through the stages: what every stage reads, and what one stage hands to the next
struct Batch {
	mmb_ctx_t *ctx;
	BatchBufs &bb;
	bool gated;                        // device phases take a slot of g_gate
	const mm_idx_t *mi;
	const mm_mapopt_t *opt;
	int n_threads;
	std::vector<int> live;             // input indices of the reads that go through the pipeline (non-empty, within max_qlen)
	std::vector<int64_t> off;          // n+1 offsets of the live reads back to back
	int n = 0;
	int64_t total_bases = 0;
	uint8_t *d_seq = nullptr;          // the live reads on the device (nt4), their offsets and lengths
	int64_t *d_off = nullptr;
	int32_t *d_qlen = nullptr;
	SeedArgs S;                        // stage 1 device arrays, up to the sorted anchors
	int64_t total_mz = 0, total_a = 0;
	// stage 1 results on the host (in bb.h_misc): per-read offsets into the dense chains (u), their anchors (a) and the kept
	// seed positions (mini_pos), the three dense arrays, and rep_len
	int64_t *h_uo = nullptr, *h_vo = nullptr, *h_mo = nullptr;
	m128 *h_da = nullptr;
	uint64_t *h_du = nullptr, *h_dm = nullptr;
	int32_t *h_rep = nullptr;
	size_t keep_used = 0;              // device CIGAR arenas (bb.cig_keep) handed out so far, counted across the waves of the batch
	int wave = 0;
	Batch(mmb_ctx_t *c, BatchBufs &b, bool g, const mm_idx_t *m, const mm_mapopt_t *o, int nt)
		: ctx(c), bb(b), gated(g), mi(m), opt(o), n_threads(nt) {}
};

} // namespace

// Resets the per-read state and the outputs of every read, and lists the reads that are mapped. false: there are none.
static bool take_reads(Batch &b, int n_reads, const int *qlens, const char **seqs, const char **names, int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out)
{
	BatchBufs &bb = b.bb;
	if ((int)bb.rs_pool.size() < n_reads) bb.rs_pool.resize(n_reads), bb.ra_pool.resize(n_reads);
	std::vector<ReadState> &rs = bb.rs_pool;
	for (int i = 0; i < n_reads; ++i) {
		rs[i].qlen = qlens[i], rs[i].seq = seqs[i], rs[i].name = names? names[i] : nullptr;
		rs[i].ra = nullptr, rs[i].regs0 = nullptr, rs[i].regs = nullptr, rs[i].n_regs = rs[i].n_regs0 = 0, rs[i].done = false, rs[i].fin_pending = false;
		n_regs_out[i] = 0, regs_out[i] = nullptr;
		if (rep_len_out) rep_len_out[i] = 0;
		bool ok = qlens[i] > 0 && !(b.opt->max_qlen > 0 && qlens[i] > b.opt->max_qlen); // map.c:243-244
		if (ok) b.live.push_back(i);
	}
	const int n = b.n = (int)b.live.size();
	if (n == 0) return false;
	b.off.assign((size_t)n + 1, 0);
	for (int j = 0; j < n; ++j) b.off[j + 1] = b.off[j] + rs[b.live[j]].qlen;
	b.total_bases = b.off[n];
	return true;
}

// The reads to the device: host concat, H2D and nt4 encoding, all three skipped when the reads are resident (the group's previous
// batch was the same reads) and nothing on the host needs them back to back. Returns the concatenated reads on the host (ASCII), or
// null when they were not concatenated.
static const uint8_t *upload_reads(GroupCtx &G, Batch &b)
{
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	const std::vector<ReadState> &rs = bb.rs_pool;
	const std::vector<int> &live = b.live;
	const std::vector<int64_t> &off = b.off;
	const int n = b.n;
	const int64_t total_bases = b.total_bases;
	const bool resident_hit = mmb_resident_reads() && G.res_n == n && G.res_bases == total_bases && G.res_first == rs[live[0]].seq;
	// in seeding only SDUST reads the host copy (seed_batch); 300 MB of memcpy per step is otherwise spent on the shared host pool
	// while every group waits for it
	uint8_t *h_seq = nullptr;
	if (!resident_hit || b.opt->sdust_thres > 0) {
		HostSpan hs_(ctx, HPH_CONCAT);
		h_seq = bb.h_seq.as<uint8_t>((size_t)total_bases + 16);
		parallel_for(n, b.n_threads, [&](int64_t j, int) { memcpy(h_seq + off[j], rs[live[j]].seq, rs[live[j]].qlen); });
	}
	uint8_t *d_seq = b.d_seq = bb.seq.as<uint8_t>((size_t)total_bases + 16);
	int64_t *d_off = b.d_off = bb.off.as<int64_t>((size_t)n + 1);
	int32_t *d_qlen = b.d_qlen = bb.qlen.as<int32_t>((size_t)n);
	std::vector<int32_t> h_qlen(n);
	for (int j = 0; j < n; ++j) h_qlen[j] = rs[live[j]].qlen;
	ctx->last_d2h_bytes = 0, ctx->last_h2d_bytes = 0;
	if (!resident_hit) {
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_seq, h_seq, total_bases, cudaMemcpyHostToDevice, ctx->stream));
		ctx->last_h2d_bytes += (uint64_t)total_bases;
	}
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_qlen, h_qlen.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	if (!resident_hit) {
		encode_kernel<<<(unsigned)((total_bases / 4 + 256) / 256), 256, 0, ctx->stream>>>(d_seq, total_bases);
		++ctx->n_launch;
	}
	G.res_n = n, G.res_bases = total_bases, G.res_first = rs[live[0]].seq;
	return h_seq;
}

// Stage 1 from the reads on the device to the sorted anchors: K1 sketch -> query-side filter -> index lookup -> streak selection ->
// anchor expansion -> anchor sort (collect_minimizers + mm_collect_matches + collect_seed_hits, map.c:59-100,168-204), on the
// context's stream. Fills b.S, b.total_mz and b.total_a. occ_cut: the max_occ of mm_collect_matches. The optional host work runs
// between the sketch and the seed selection: SDUST intervals (b.opt->sdust_thres > 0) from h_seq, the reads on the host (ASCII);
// and skip_seed's query-name bounds when names (by input index) is not null.
static void seed_batch(Batch &b, const uint8_t *h_seq, const char **names, int occ_cut)
{
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	const mm_idx_t *mi = b.mi;
	const mm_mapopt_t *opt = b.opt;
	mm_idx_bucket_s *B = mi->B;
	const int n = b.n;
	int64_t *d_mz_off = bb.mz_off.as<int64_t>((size_t)n + 1);
	const int64_t total_mz = b.total_mz = mmb_sketch_device(ctx, b.d_seq, nullptr, b.d_off, n, nullptr, 0, mi->w, mi->k, mi->flag & MM_I_HPC, b.total_bases,
															bb.mz, d_mz_off, bb.t1, bb.t2, 1 /* rid = segment index 0 for every read (map.c:65) */);
	SeedArgs &S = b.S;
	S.ix = B->view(mi), S.n_reads = n, S.mz = (m128*)bb.mz.p, S.mz_off = d_mz_off, S.qlen = b.d_qlen;
	S.n_mz = bb.n_mz.as<int32_t>((size_t)n);
	S.q_occ_max = opt->mid_occ, S.q_occ_frac = opt->q_occ_frac;
	S.max_occ = occ_cut, S.max_max_occ = opt->max_max_occ, S.occ_dist = opt->occ_dist, S.flag = opt->flag;
	const size_t nm = (size_t)total_mz + 4;
	S.s_n = bb.s_n.as<uint32_t>(nm), S.s_off = bb.s_off.as<uint64_t>(nm), S.k_idx = bb.k_idx.as<uint32_t>(nm), S.k_aoff = bb.k_aoff.as<uint32_t>(nm);
	S.flt = bb.flt.as<uint8_t>(nm), S.mini_pos = bb.mini_pos.as<uint64_t>(nm);
	S.n_keep = bb.n_keep.as<int32_t>((size_t)n), S.rep_len = bb.rep_len.as<int32_t>((size_t)n), S.n_a = bb.n_a.as<int64_t>((size_t)n + 1);
	init_nmz_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_mz_off, n, S.n_mz);
	++ctx->n_launch;
	if (opt->sdust_thres > 0) { // map.c:68-69: low-complexity masking of the query minimizers; the intervals come from the host
		const std::vector<int64_t> &off = b.off;
		std::vector<std::vector<uint64_t>> regs((size_t)n);
		parallel_for(n, b.n_threads, [&](int64_t j, int) { hl_sdust(h_seq + off[j], (int)(off[j + 1] - off[j]), opt->sdust_thres, 64, regs[j]); });
		std::vector<int64_t> doff((size_t)n + 1, 0);
		for (int j = 0; j < n; ++j) doff[j + 1] = doff[j] + (int64_t)regs[j].size();
		std::vector<uint64_t> flat((size_t)doff[n] + 1);
		for (int j = 0; j < n; ++j) std::copy(regs[j].begin(), regs[j].end(), flat.begin() + doff[j]);
		uint64_t *d_dreg = bb.dreg.as<uint64_t>(flat.size());
		int64_t *d_doff = bb.dreg_off.as<int64_t>((size_t)n + 1);
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_dreg, flat.data(), sizeof(uint64_t) * flat.size(), cudaMemcpyHostToDevice, ctx->stream));
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_doff, doff.data(), sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, ctx->stream));
		dust_filter_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(S.mz, d_mz_off, S.n_mz, d_dreg, d_doff, n);
		mmb_stream_sync(ctx); // the pageable staging vectors go out of scope here
		++ctx->n_launch;
	}
	if (opt->flag & (MM_F_NO_DIAG | MM_F_NO_DUAL | MM_F_FOR_ONLY | MM_F_REV_ONLY)) { // skip_seed (map.c:78-100) runs on the device
		S.k_cnt = bb.k_cnt.as<uint32_t>(nm);
		if (names && (opt->flag & (MM_F_NO_DIAG | MM_F_NO_DUAL))) {
			{ // rank of every reference name in sorted order, built once per index
				std::lock_guard<std::mutex> lk(B->mu);
				if (!B->d_name_rank) {
					B->name_order.resize(mi->n_seq);
					for (uint32_t i = 0; i < mi->n_seq; ++i) B->name_order[i] = i;
					std::stable_sort(B->name_order.begin(), B->name_order.end(), [&](uint32_t x, uint32_t y) { return strcmp(mi->seq[x].name, mi->seq[y].name) < 0; });
					std::vector<uint32_t> rank(mi->n_seq);
					for (uint32_t i = 0; i < mi->n_seq; ++i) rank[B->name_order[i]] = i;
					MMB_CUDA_CHECK(cudaMalloc(&B->d_name_rank, sizeof(uint32_t) * (mi->n_seq + 1)));
					MMB_CUDA_CHECK(cudaMemcpy(B->d_name_rank, rank.data(), sizeof(uint32_t) * mi->n_seq, cudaMemcpyHostToDevice));
				}
			}
			std::vector<uint32_t> qlo(n), qhi(n);
			const std::vector<uint32_t> &ord = B->name_order;
			parallel_for(n, b.n_threads, [&](int64_t j, int) {
				const char *qn = names[b.live[j]];
				if (!qn) { qlo[j] = qhi[j] = 0; return; } // no name: no name test (map.c:81)
				qlo[j] = (uint32_t)(std::lower_bound(ord.begin(), ord.end(), qn, [&](uint32_t id, const char *q) { return strcmp(mi->seq[id].name, q) < 0; }) - ord.begin());
				qhi[j] = (uint32_t)(std::upper_bound(ord.begin(), ord.end(), qn, [&](const char *q, uint32_t id) { return strcmp(q, mi->seq[id].name) < 0; }) - ord.begin());
			});
			uint32_t *d_qlo = bb.qlo.as<uint32_t>((size_t)n), *d_qhi = bb.qhi.as<uint32_t>((size_t)n);
			MMB_CUDA_CHECK(cudaMemcpyAsync(d_qlo, qlo.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
			MMB_CUDA_CHECK(cudaMemcpyAsync(d_qhi, qhi.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
			mmb_stream_sync(ctx); // the host vectors go out of scope
			S.name_rank = B->d_name_rank, S.q_name_lo = d_qlo, S.q_name_hi = d_qhi;
		}
	}
	mmb_seed_select_device(ctx, S, total_mz);
	int64_t *d_a_off = bb.a_off.as<int64_t>((size_t)n + 1);
	copy_i64_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(S.n_a, n, d_a_off);
	++ctx->n_launch;
	const int64_t total_a = b.total_a = mmb_exclusive_scan_i64(ctx, d_a_off, n, true);
	S.a = bb.a.as<m128>((size_t)total_a + 4), S.a_off = d_a_off;
	S.a_sorted = bb.a2.as<m128>((size_t)total_a + 4);
	mmb_seed_expand_sort_device(ctx, S, total_mz, total_a, bb.stk);
}

// Stage 1 from the sorted anchors to the host: chaining (map.c:262-281), the long-join rescue (map.c:283-292), dense per-read copies
// of the chains, their anchors and the kept seed positions, and their D2H copy. Drops gate1, the group's device slot, as soon as the
// copies are in.
static void chain_batch(Batch &b, const MapPass &pass, GateHold &gate1)
{
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	const mm_mapopt_t *opt = b.opt;
	const SeedArgs &S = b.S;
	const int n = b.n;
	const int64_t total_a = b.total_a;
	const int64_t *d_a_off = S.a_off;
	// chaining parameters (map.c:262-281)
	mmb_chain_par_t cp;
	memset(&cp, 0, sizeof(cp));
	int max_chain_gap_qry = opt->max_gap, max_chain_gap_ref;
	if (opt->max_gap_ref > 0) max_chain_gap_ref = opt->max_gap_ref;
	else if (opt->max_frag_len > 0) { // qlen-dependent (map.c:266-268); only meaningful for paired short reads
		fprintf(stderr, "[ERROR] minimap2_b200: max_frag_len > 0 (short-read pairing) is not implemented\n");
		abort();
	} else max_chain_gap_ref = opt->max_gap;
	cp.max_dist_x = max_chain_gap_ref, cp.max_dist_y = max_chain_gap_qry, cp.bw = opt->bw, cp.max_skip = opt->max_chain_skip;
	cp.max_iter = opt->max_chain_iter, cp.min_cnt = opt->min_cnt, cp.min_sc = opt->min_chain_score;
	cp.chn_pen_gap = (float)(opt->chain_gap_scale * 0.01 * b.mi->k), cp.chn_pen_skip = (float)(opt->chain_skip_scale * 0.01 * b.mi->k);
	cp.is_cdna = (opt->flag & MM_F_SPLICE) != 0, cp.n_seg = 1; // map.c:277 (is_splice selects the cDNA gap model of comput_sc)
	int32_t *d_n_u = bb.n_u.as<int32_t>((size_t)n), *d_n_v = bb.n_v.as<int32_t>((size_t)n);
	uint64_t *d_u = bb.u.as<uint64_t>((size_t)total_a + 4);
	m128 *d_a_out = bb.a_out.as<m128>((size_t)total_a + 4);
	if (opt->flag & MM_F_RMQ) // map.c:275-276
		cp.use_rmq = 1, cp.max_dist_x = opt->max_gap, cp.max_dist_inner = opt->rmq_inner_dist, cp.rmq_size_cap = opt->rmq_size_cap;
	// long-join rescue (map.c:283-292): re-chain on the device with mg_lchain_rmq at bw_long
	RescuePar rp;
	memset(&rp, 0, sizeof(rp));
	const bool rescue = pass.rescue && opt->bw_long > opt->bw && (opt->flag & (MM_F_SPLICE | MM_F_SR | MM_F_NO_LJOIN)) == 0;
	if (rescue) {
		rp.qlen = b.d_qlen, rp.rescue_size = opt->rmq_rescue_size, rp.rescue_ratio = opt->rmq_rescue_ratio;
		rp.max_dist = opt->max_gap, rp.max_dist_inner = opt->rmq_inner_dist, rp.bw = opt->bw_long, rp.max_skip = opt->max_chain_skip;
		rp.rmq_size_cap = opt->rmq_size_cap, rp.min_cnt = opt->min_cnt, rp.min_sc = opt->min_chain_score;
		rp.pen_gap = cp.chn_pen_gap, rp.pen_skip = cp.chn_pen_skip;
	}
	// dense copies for the host: offsets for u, a and mini_pos
	int64_t *d_doff = bb.doff.as<int64_t>((size_t)(n + 1) * 3);
	int64_t *d_uo = d_doff, *d_vo = d_doff + (n + 1), *d_mo = d_doff + 2 * (n + 1);
	mmb_chain_stage(ctx, &cp, rescue? &rp : nullptr, n, S.a_sorted, d_a_off, total_a, d_n_u, d_n_v, d_u, d_a_out, d_vo, bb.ch1, bb.ch2, bb.t1);
	mmb_widen_i32_async(ctx, d_n_u, n, d_uo);
	mmb_widen_i32_async(ctx, d_n_v, n, d_vo);
	mmb_widen_i32_async(ctx, S.n_keep, n, d_mo);
	const int64_t tot_u = mmb_exclusive_scan_i64(ctx, d_uo, n, true);
	const int64_t tot_v = mmb_exclusive_scan_i64(ctx, d_vo, n, true);
	const int64_t tot_m = mmb_exclusive_scan_i64(ctx, d_mo, n, true);
	uint64_t *d_du = bb.dense_u.as<uint64_t>((size_t)tot_u + 1);
	m128 *d_da = bb.dense_a.as<m128>((size_t)tot_v + 1);
	uint64_t *d_dm = bb.dense_mp.as<uint64_t>((size_t)tot_m + 1);
	const unsigned gw = (unsigned)(((int64_t)n * 32 + 255) / 256);
	gather_kernel<uint64_t><<<gw, 256, 0, ctx->stream>>>(d_u, d_a_off, d_n_u, d_uo, n, d_du);
	gather_kernel<m128><<<gw, 256, 0, ctx->stream>>>(d_a_out, d_a_off, d_n_v, d_vo, n, d_da);
	gather_kernel<uint64_t><<<gw, 256, 0, ctx->stream>>>(S.mini_pos, S.mz_off, S.n_keep, d_mo, n, d_dm);
	ctx->n_launch += 3;
	// host copies
	const size_t misc_bytes = sizeof(int64_t) * (size_t)(n + 1) * 3 + sizeof(int32_t) * (size_t)n + sizeof(uint64_t) * (size_t)(tot_u + tot_m) + sizeof(m128) * (size_t)tot_v + 64;
	uint8_t *hm = bb.h_misc.as<uint8_t>(misc_bytes);
	int64_t *h_uo = b.h_uo = (int64_t*)hm;
	b.h_vo = h_uo + (n + 1), b.h_mo = b.h_vo + (n + 1);
	m128 *h_da = b.h_da = (m128*)(b.h_mo + (n + 1));
	uint64_t *h_du = b.h_du = (uint64_t*)(h_da + tot_v), *h_dm = b.h_dm = h_du + tot_u;
	int32_t *h_rep = b.h_rep = (int32_t*)(h_dm + tot_m);
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_uo, d_doff, sizeof(int64_t) * (size_t)(n + 1) * 3, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_da, d_da, sizeof(m128) * (size_t)tot_v, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_du, d_du, sizeof(uint64_t) * (size_t)tot_u, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_dm, d_dm, sizeof(uint64_t) * (size_t)tot_m, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_rep, S.rep_len, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
	mmb_tl(ctx, MMB_TL_ENQUEUED, 0);
	mmb_stream_sync(ctx);
	gate1.drop();
	ctx->last_d2h_bytes += misc_bytes;
	if (ctx->profiling) {
		const int64_t total_mz = b.total_mz;
		ctx->prof_bytes[MMB_PROF_SKETCH] += (uint64_t)(b.total_bases / 4) + 16ull * (uint64_t)total_mz;
		ctx->prof_bytes[MMB_PROF_SEED] += 32ull * (uint64_t)total_mz + 24ull * (uint64_t)total_a;
		ctx->prof_bytes[MMB_PROF_SORT] += 32ull * (uint64_t)total_a;
		ctx->prof_bytes[MMB_PROF_CHAIN] += 16ull * (uint64_t)total_a + 16ull * (uint64_t)tot_v + 8ull * (uint64_t)tot_u;
	}
}

// Stage 2 (map.c:317-336): chains -> hits on the host threads. Reads with hits to align (MM_F_CIGAR) get their alignment state;
// the others are done.
static void chains_to_hits(Batch &b, const MapPass &pass)
{
	BatchBufs &bb = b.bb;
	std::vector<ReadState> &rs = bb.rs_pool;
	const std::vector<int> &live = b.live;
	const std::vector<int64_t> &off = b.off;
	const mm_idx_t *mi = b.mi;
	const mm_mapopt_t *opt = b.opt;
	const int n = b.n;
	const bool with_cigar = (opt->flag & MM_F_CIGAR) != 0;
	HostSpan hs_(b.ctx, HPH_HITS);
	if (with_cigar && bb.qseq_pool.size() < (size_t)b.total_bases * 2 + 16) bb.qseq_pool.resize((size_t)b.total_bases * 2 + 16);
	parallel_for(n, b.n_threads, [&](int64_t j, int) {
		HpScope hp_(HP_HITS);
		ReadState &r = rs[live[j]];
		r.rep_len = b.h_rep[j];
		r.n_u = (int)(b.h_uo[j + 1] - b.h_uo[j]), r.u = b.h_du + b.h_uo[j];
		if (pass.no_chain) pass.no_chain[live[j]] = r.n_u == 0;
		r.n_a = (int)(b.h_vo[j + 1] - b.h_vo[j]), r.a_src = b.h_da + b.h_vo[j];
		r.n_mini_pos = (int)(b.h_mo[j + 1] - b.h_mo[j]), r.mini_pos = b.h_dm + b.h_mo[j];
		uint32_t hash = r.name && !(opt->flag & MM_F_NO_HASH_NAME)? x31_hash_string(r.name) : 0; // map.c:246-248
		hash ^= wang_hash((uint32_t)r.qlen) + wang_hash((uint32_t)opt->seed);
		r.hash = wang_hash(hash);
		r.a.assign(r.a_src, r.a_src + r.n_a);
		int n_regs0 = r.n_u;
		mm_reg1_t *regs0 = hl_gen_regs(r.hash, r.qlen, r.n_u, r.u, r.a.data(), !!(opt->flag & MM_F_QSTRAND)); // map.c:320
		if (mi->n_alt) { // map.c:321-324 (mm_mark_alt, hit.c:91-97)
			for (int k = 0; k < n_regs0; ++k) if (mi->seq[regs0[k].rid].is_alt) regs0[k].is_alt = 1;
			hl_hit_sort(&n_regs0, regs0, opt->alt_drop);
		}
		if (!(opt->flag & MM_F_ALL_CHAINS)) { // chain_post (map.c:206-213)
			hl_set_parent(opt->mask_level, opt->mask_len, n_regs0, regs0, opt->a * 2 + opt->b, opt->flag & MM_F_HARD_MLEVEL, opt->alt_drop);
			hl_select_sub(opt->pri_ratio, mi->k * 2, opt->best_n, 1, (int)(opt->max_gap * 0.8), &n_regs0, regs0);
		}
		if (!(opt->flag & MM_F_QSTRAND)) { // map.c:333-336
			hl_est_err(mi, r.qlen, n_regs0, regs0, r.a.data(), r.n_mini_pos, r.mini_pos);
			n_regs0 = hl_filter_strand_retained(n_regs0, regs0);
		}
		r.n_regs0 = n_regs0, r.regs0 = regs0;
		if (with_cigar && n_regs0 > 0) {
			ReadAlign *ra = &bb.ra_pool[live[j]];
			ra->reset();
			ra->qlen = r.qlen, ra->q_dev_off = off[j];
			r.ra = ra;
		} else r.done = true, r.n_regs = n_regs0, r.regs = regs0, r.regs0 = nullptr;
	});
	if (with_cigar) { // nt4 forward / reverse-complement copies of the reads (align.c:1056-1061): room is set aside, the copies are made on first use
		for (int j = 0; j < n; ++j) {
			ReadState &r = rs[live[j]];
			if (!r.ra) continue;
			uint8_t *q0 = bb.qseq_pool.data() + 2 * off[j];
			r.ra->raw_seq = r.seq, r.ra->qbuf = q0, r.ra->qseq_ready = false;
			r.ra->qseq[0] = q0, r.ra->qseq[1] = q0 + r.qlen;
		}
	}
}

// the ksw2 scoring of the options, with the alignment driver's matrix
static mmb_ksw_score_t ksw_score(const mm_mapopt_t *opt)
{
	mmb_ksw_score_t sc;
	hl_gen_mat(sc.mat, opt);
	sc.q = (int8_t)opt->q, sc.e = (int8_t)opt->e, sc.q2 = (int8_t)opt->q2, sc.e2 = (int8_t)opt->e2;
	sc.noncan = (int8_t)opt->noncan, sc.junc_bonus = (int8_t)opt->junc_bonus, sc.junc_pen = (int8_t)opt->junc_pen;
	// mm_test_zdrop only compares the largest drop with zdrop and (unless the inversion probe is off, align.c:92) zdrop_inv: a
	// path whose total penalty stays below both needs no scan
	const bool inv_off = (opt->flag & (MM_F_SPLICE | MM_F_SR | MM_F_FOR_ONLY | MM_F_REV_ONLY)) != 0;
	const int th = inv_off? opt->zdrop : std::min(opt->zdrop, opt->zdrop_inv);
	sc.zd_skip = (int16_t)std::max(0, std::min(th, 30000));
	return sc;
}

// align_regs (map.c:215-225): the read's aligned hits get their parents and secondaries; the read is done
static void post_align(const Batch &b, ReadState &r, int n_regs, mm_reg1_t *regs)
{
	HpScope hp_(HP_POST);
	const mm_mapopt_t *opt = b.opt;
	if (!(opt->flag & MM_F_ALL_CHAINS)) {
		hl_set_parent(opt->mask_level, opt->mask_len, n_regs, regs, opt->a * 2 + opt->b, opt->flag & MM_F_HARD_MLEVEL, opt->alt_drop);
		hl_select_sub(opt->pri_ratio, b.mi->k * 2, opt->best_n, 0, (int)(opt->max_gap * 0.8), &n_regs, regs);
		hl_set_sam_pri(n_regs, regs);
	}
	r.n_regs = n_regs, r.regs = regs, r.done = true, r.fin_pending = false;
}

// one pass of the alignment driver over the read's pristine chains
static mm_reg1_t *replay_read(const Batch &b, ReadState &r, bool defer, int *n_regs_out)
{
	ReadAlign &ra = *r.ra;
	int n_regs = r.n_regs0;
	mm_reg1_t *regs;
	{
		HpScope hp_(HP_PRE);
		r.a.assign(r.a_src, r.a_src + r.n_a); // pristine anchors (IGNORE/LONG_JOIN marks cleared)
		regs = (mm_reg1_t*)malloc(sizeof(mm_reg1_t) * (n_regs > 0? n_regs : 1));
		memcpy(regs, r.regs0, sizeof(mm_reg1_t) * n_regs);
	}
	ra.defer = defer;
	regs = hl_align_skeleton(b.opt, b.mi, ra, &n_regs, regs, r.n_a, r.a.data());
	*n_regs_out = n_regs;
	return regs;
}

static void drop_regs(int n_regs, mm_reg1_t *regs) { for (int i = 0; i < n_regs; ++i) free(regs[i].p); free(regs); }

// K4: the device tail (CIGAR assembly, mm_fix_cigar, mm_update_extra) for the reads of the wave whose replay is complete
static void device_tail(Batch &b, const std::vector<int> &active, const FinPar &fpar)
{
	std::vector<ReadState> &rs = b.bb.rs_pool;
	std::vector<int> fr;
	for (size_t t = 0; t < active.size(); ++t) if (rs[active[t]].fin_pending) fr.push_back(active[t]);
	if (fr.empty()) return;
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	const mm_idx_t *mi = b.mi;
	const size_t nf = fr.size();
	mmb_tl(ctx, MMB_TL_HOST_BEGIN, HPH_TAIL_PREP);
	std::vector<int64_t> hoff(nf + 1, 0), joff2(nf + 1, 0);
	for (size_t t = 0; t < nf; ++t) {
		const ReadAlign &ra = *rs[fr[t]].ra;
		hoff[t + 1] = hoff[t] + (int64_t)ra.fin_hits.size(), joff2[t + 1] = joff2[t] + (int64_t)ra.fin_jobs.size();
	}
	const int64_t n_hits = hoff[nf], n_pieces = joff2[nf];
	std::vector<int64_t> coff((size_t)n_hits + 1, 0); // output CIGAR offsets (room for the sum of the pieces)
	for (size_t t = 0; t < nf; ++t) {
		const ReadAlign &ra = *rs[fr[t]].ra;
		for (size_t k = 0; k < ra.fin_hits.size(); ++k) coff[hoff[t] + k + 1] = ra.fin_hits[k].n_cig_max;
	}
	for (int64_t i = 0; i < n_hits; ++i) coff[i + 1] += coff[i];
	const int64_t tot_cig = coff[n_hits];
	const size_t in_bytes = sizeof(FinReg) * (size_t)n_hits + sizeof(FinJobRef) * (size_t)n_pieces;
	uint8_t *h_in = bb.h_fin_in.as<uint8_t>(in_bytes + 64);
	FinReg *h_regs = (FinReg*)h_in;
	FinJobRef *h_pieces = (FinJobRef*)(h_regs + n_hits);
	parallel_for((int64_t)nf, b.n_threads, [&](int64_t t, int) {
		const ReadState &r = rs[fr[t]];
		const ReadAlign &ra = *r.ra;
		for (size_t k = 0; k < ra.fin_jobs.size(); ++k) { FinJobRef &j = h_pieces[joff2[t] + k]; j.cig = ra.fin_jobs[k].dcig, j.n = ra.fin_jobs[k].n, j.pad = 0; }
		for (size_t k = 0; k < ra.fin_hits.size(); ++k) {
			const HlFinHit &h = ra.fin_hits[k];
			FinReg &f = h_regs[hoff[t] + k];
			f.q0 = ra.q_dev_off, f.t0 = (int64_t)mi->seq[h.rid].offset + h.rs, f.out_off = coff[hoff[t] + k];
			f.qlen = r.qlen, f.qs = h.qs, f.rev = h.rev, f.qspan = h.qspan, f.tspan = h.tspan;
			f.job_first = (int32_t)(joff2[t] + h.job_first), f.n_jobs = h.n_jobs, f.pad = 0;
		}
	});
	uint8_t *d_in = bb.fin_in.as<uint8_t>(in_bytes + 64);
	const size_t out_bytes = sizeof(FinOut) * (size_t)n_hits + 4 * (size_t)tot_cig;
	uint8_t *d_out = bb.fin_out.as<uint8_t>(out_bytes + 64);
	uint8_t *h_out = bb.h_fin_out.as<uint8_t>(out_bytes + 64);
	mmb_tl(ctx, MMB_TL_HOST_END, HPH_TAIL_PREP);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_in, h_in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
	mmb_finalize_device(ctx, (const FinReg*)d_in, (const FinJobRef*)(d_in + sizeof(FinReg) * (size_t)n_hits), (int)n_hits, b.d_seq, (const uint32_t*)mi->B->d_S,
						(uint32_t*)(d_out + sizeof(FinOut) * (size_t)n_hits), (FinOut*)d_out, fpar);
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_out, d_out, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
	mmb_tl(ctx, MMB_TL_ENQUEUED, 2);
	mmb_stream_sync(ctx);
	ctx->last_h2d_bytes += in_bytes, ctx->last_d2h_bytes += out_bytes;
	HostSpan hs2_(ctx, HPH_TAIL_APPLY);
	const HlFinOut *h_fin = (const HlFinOut*)h_out;
	const uint32_t *h_fcig = (const uint32_t*)(h_out + sizeof(FinOut) * (size_t)n_hits);
	parallel_for((int64_t)nf, b.n_threads, [&](int64_t t, int) {
		hl_hp_flush();
		ReadState &r = rs[fr[t]];
		ReadAlign &ra = *r.ra;
		std::vector<const uint32_t*> cp(ra.fin_hits.size());
		for (size_t k = 0; k < cp.size(); ++k) cp[k] = h_fcig + coff[hoff[t] + k];
		int n_regs = r.n_regs;
		mm_reg1_t *regs = r.regs;
		bool ok;
		{ HpScope hp_(HP_EXTRA); ok = hl_align_apply_fin(ra, n_regs, regs, h_fin + hoff[t], cp.data()); }
		if (ok) hl_align_finish(b.opt, ra, &n_regs, regs);
		else { // a hit's CIGAR did not consume its query / target span (the reference asserts this): the host driver redoes the read
			drop_regs(n_regs, regs);
			regs = replay_read(b, r, false, &n_regs);
			if (ra.incomplete) { fprintf(stderr, "[ERROR] minimap2_b200: host redo of a finished read is incomplete\n"); abort(); }
		}
		post_align(b, r, n_regs, regs);
	});
}

// One K3 wave: the ksw2 jobs the unfinished reads of the wave asked for run in chunks on the device, and the results are handed to
// the per-read caches. Returns the number of jobs.
static int64_t ksw_wave(Batch &b, const std::vector<int> &active, const mmb_ksw_score_t &sc)
{
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	std::vector<ReadState> &rs = bb.rs_pool;
	// gather jobs
	std::vector<int64_t> joff(active.size() + 1, 0);
	for (size_t t = 0; t < active.size(); ++t) {
		ReadState &r = rs[active[t]];
		joff[t + 1] = joff[t] + (r.done? 0 : (int64_t)r.ra->want.size());
	}
	const int64_t n_jobs = joff[active.size()];
	if (n_jobs == 0) return 0;
	mmb_tl(ctx, MMB_TL_HOST_BEGIN, HPH_JOBS);
	// every wave executes all jobs the replays asked for, so each read advances by at least one ksw call per wave and the
	// loop ends; reads that keep splitting under a very small z-drop (-z 30) legitimately need dozens of waves. The
	// bound only guards against a logic error.
	if (b.wave >= 100000) { fprintf(stderr, "[ERROR] minimap2_b200: too many alignment waves\n"); abort(); }
	mmb_ksw_job_t *jobs = bb.h_jobs.as<mmb_ksw_job_t>((size_t)n_jobs);
	parallel_for((int64_t)active.size(), b.n_threads, [&](int64_t t, int) {
		ReadState &r = rs[active[t]];
		if (!r.done && !r.ra->want.empty()) memcpy(&jobs[joff[t]], r.ra->want.data(), sizeof(mmb_ksw_job_t) * r.ra->want.size());
	});
	// run in chunks to bound the device result buffers; results land in pinned host memory that stays alive until
	// the end of the batch, so per-read caches just point into it
	static const int64_t CH = getenv("MM_B200_JOB_CHUNK")? std::max(1, atoi(getenv("MM_B200_JOB_CHUNK"))) : 1 << 20; // test hook: tiny chunks exercise the multi-chunk bookkeeping
	mmb_ksw_res_t *res = bb.h_res.as<mmb_ksw_res_t>((size_t)n_jobs);
	// CIGAR arena estimate per job: (qlen+tlen)/2 + 8 operations covers every realistic alignment, the true bound is qlen+tlen
	// (alternating 1I1D); an overflow is recovered below by rerunning the chunk with the exact size the kernels reported
	// and growing the host staging buffer. MM_B200_CIG_SHIFT (test hook) shrinks the estimate to force that path.
	static const int cig_shift = getenv("MM_B200_CIG_SHIFT")? atoi(getenv("MM_B200_CIG_SHIFT")) : 0;
	// (a spliced job's target spans its introns, each a single N operation: only a query-sized part of the target can turn into operations)
	auto cig_est = [&](const mmb_ksw_job_t &jb) -> int64_t {
		if (jb.flag & MMB_JOB_LL) return 0;
		const int64_t t_eff = (jb.flag & MMB_JOB_SPLICE)? std::min<int64_t>(jb.tlen, 2 * (int64_t)jb.qlen + 64) : jb.tlen;
		return (((int64_t)jb.qlen + t_eff) / 2 + 8 >> cig_shift) + 1;
	};
	// with the device tail on, every (wave, chunk) keeps its arena until the batch ends (K4 reads the pieces in place);
	// otherwise one arena is reused, as the host has its copy (spliced jobs reserve room for intron-sized CIGAR estimates)
	const bool keep_arenas = hl_defer_supported(b.opt);
	int64_t cap_tot = 0;
	for (int64_t i = 0; i < n_jobs; ++i) cap_tot += cig_est(jobs[i]);
	while (bb.h_cig.size() <= (size_t)b.wave) bb.h_cig.emplace_back(new PinBuf);
	uint32_t *h_cig = bb.h_cig[b.wave]->as<uint32_t>((size_t)cap_tot + 64);
	mmb_tl(ctx, MMB_TL_HOST_END, HPH_JOBS);
	// the slot is taken per chunk once its launch is planned: the host planning overlaps the other groups' kernels
	GateHold gatew(ctx, b.gated, 1, false);
	std::vector<int64_t> chunk_base; // offset of each chunk's CIGAR block inside h_cig
	std::vector<const uint32_t*> chunk_dev; // and the block's address in its device arena
	int64_t cig_fill = 0;
	for (int64_t c0 = 0; c0 < n_jobs; c0 += CH) {
		const int64_t m = std::min(CH, n_jobs - c0);
		int64_t cap = 0;
		for (int64_t i = 0; i < m; ++i) cap += cig_est(jobs[c0 + i]);
		for (;;) {
			mmb_ksw_job_t *d_jobs = bb.jobs.as<mmb_ksw_job_t>((size_t)m);
			mmb_ksw_res_t *d_res = bb.res.as<mmb_ksw_res_t>((size_t)m);
			const size_t ki = keep_arenas? b.keep_used : 0;
			while (bb.cig_keep.size() <= ki) bb.cig_keep.emplace_back(new DevBuf);
			uint32_t *d_cig = bb.cig_keep[ki]->as<uint32_t>((size_t)cap + 4);
			unsigned long long *d_used = (unsigned long long*)d_cig;
			KswLaunch K;
			{
				HostSpan hs_(ctx, HPH_KSW_PLAN);
				mmb_ksw_plan(ctx, &sc, (int)m, &jobs[c0], d_jobs, b.d_seq, b.mi->B->d_S, 1, d_res, d_cig + 2, cap, d_used, K);
			}
			gatew.take();
			MMB_CUDA_CHECK(cudaMemcpyAsync(d_jobs, &jobs[c0], sizeof(mmb_ksw_job_t) * m, cudaMemcpyHostToDevice, ctx->stream));
			MMB_CUDA_CHECK(cudaMemsetAsync(d_used, 0, 8, ctx->stream));
			mmb_ksw_enqueue(ctx, K);
			// (pinned: a copy to pageable memory would wait for the stream in a spin loop)
			unsigned long long *h_used = bb.h_used.as<unsigned long long>(1);
			MMB_CUDA_CHECK(cudaMemcpyAsync(&res[c0], d_res, sizeof(mmb_ksw_res_t) * m, cudaMemcpyDeviceToHost, ctx->stream));
			MMB_CUDA_CHECK(cudaMemcpyAsync(h_used, d_used, 8, cudaMemcpyDeviceToHost, ctx->stream));
			mmb_tl(ctx, MMB_TL_ENQUEUED, 1);
			mmb_stream_sync(ctx);
			const unsigned long long used = *h_used;
			if ((int64_t)used > cap) { cap = (int64_t)used + 16; gatew.drop(); continue; } // rare: rerun the chunk with a larger CIGAR arena
			if (cig_fill + (int64_t)used > cap_tot) { // grow the wave's host staging buffer, keeping the chunks already staged
				int64_t rest = 0;
				for (int64_t i = c0 + m; i < n_jobs; ++i) rest += cig_est(jobs[i]);
				const int64_t new_tot = cig_fill + (int64_t)used + rest + 64;
				std::unique_ptr<PinBuf> nb(new PinBuf);
				uint32_t *np_ = nb->as<uint32_t>((size_t)new_tot + 64);
				if (cig_fill) memcpy(np_, h_cig, (size_t)cig_fill * 4);
				bb.h_cig[b.wave]->release();
				bb.h_cig[b.wave] = std::move(nb);
				h_cig = np_, cap_tot = new_tot;
			}
			ctx->last_d2h_bytes += sizeof(mmb_ksw_res_t) * (uint64_t)m + 4ull * used;
			ctx->last_h2d_bytes += sizeof(mmb_ksw_job_t) * (uint64_t)m;
			if (ctx->profiling) ctx->prof_bytes[MMB_PROF_KSW] += 4ull * used;
			chunk_base.push_back(cig_fill);
			chunk_dev.push_back(d_cig + 2);
			++b.keep_used;
			if (used) MMB_CUDA_CHECK(cudaMemcpyAsync(h_cig + cig_fill, d_cig + 2, used * 4, cudaMemcpyDeviceToHost, ctx->stream));
			cig_fill += (int64_t)used;
			mmb_stream_sync(ctx);
			gatew.drop();
			break;
		}
	}
	// hand the results to the per-read caches (pointers only)
	HostSpan hs_(ctx, HPH_SCATTER);
	parallel_for((int64_t)active.size(), b.n_threads, [&](int64_t t, int) {
		ReadState &r = rs[active[t]];
		if (r.done) return;
		ReadAlign &ra = *r.ra;
		for (size_t i = 0; i < ra.want.size(); ++i) {
			const int64_t jid = joff[t] + (int64_t)i;
			KswDone d; d.r = res[jid], d.cig = h_cig + chunk_base[jid / CH] + res[jid].cigar_off, d.dcig = chunk_dev[jid / CH] + res[jid].cigar_off;
			ra.done_idx[ra.want_slot[i]] = (int)ra.done.size();
			ra.done.push_back(d);
		}
	});
	return n_jobs;
}

// Stage 3: alignment waves. Every wave replays the driver for each unfinished read, runs the device tail for the reads whose replay
// is complete, and runs the ksw2 jobs the others asked for.
static void align_waves(Batch &b)
{
	std::vector<ReadState> &rs = b.bb.rs_pool;
	const mmb_ksw_score_t sc = ksw_score(b.opt);
	std::vector<int> active;
	for (int j = 0; j < b.n; ++j) if (!rs[b.live[j]].done) active.push_back(b.live[j]);
	// The hit-level tail of the driver (CIGAR assembly, mm_fix_cigar, mm_update_extra) runs on the device for finished reads (K4,
	// finalize.cu) unless the mode needs it on the host (spliced / =X CIGARs / query-strand).
	const bool use_fin = hl_defer_supported(b.opt);
	FinPar fpar;
	for (int i = 0; i < 25; ++i) fpar.mat[i] = sc.mat[i];
	fpar.q = (int8_t)b.opt->q, fpar.e = (int8_t)b.opt->e, fpar.log_gap = 1;
	while (!active.empty()) {
		// replay every active read; collect the jobs they miss
		mmb_tl(b.ctx, MMB_TL_HOST_BEGIN, HPH_REPLAY);
		parallel_for((int64_t)active.size(), b.n_threads, [&](int64_t t, int) {
			hl_hp_flush();
			ReadState &r = rs[active[t]];
			ReadAlign &ra = *r.ra;
			ra.want.clear(); ra.want_slot.clear();
			int n_regs;
			mm_reg1_t *regs = replay_read(b, r, use_fin, &n_regs);
			if (ra.defer_abort) { // an inversion probe needs final hit coordinates: this read keeps the whole driver on the host
				drop_regs(n_regs, regs);
				regs = replay_read(b, r, false, &n_regs); // jobs the aborted pass asked for stay queued (the full pass asks for a superset)
			}
			if (ra.incomplete) drop_regs(n_regs, regs);
			else if (ra.defer && !ra.fin_hits.empty()) r.n_regs = n_regs, r.regs = regs, r.fin_pending = true;
			else post_align(b, r, n_regs, regs);
		});
		mmb_tl(b.ctx, MMB_TL_HOST_END, HPH_REPLAY);
		device_tail(b, active, fpar);
		const int64_t n_jobs = ksw_wave(b, active, sc);
		std::vector<int> still;
		for (size_t t = 0; t < active.size(); ++t) if (!rs[active[t]].done) still.push_back(active[t]);
		if (!still.empty() && n_jobs == 0) { fprintf(stderr, "[ERROR] minimap2_b200: alignment scheduler made no progress\n"); abort(); }
		active.swap(still);
		++b.wave;
	}
}

// Stage 4 (map.c:338-343): MAPQ, and the results to the caller's arrays
static void finalize_batch(Batch &b, int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out)
{
	std::vector<ReadState> &rs = b.bb.rs_pool;
	const std::vector<int> &live = b.live;
	const mm_mapopt_t *opt = b.opt;
	HostSpan hs_(b.ctx, HPH_FINALIZE);
	parallel_for(b.n, b.n_threads, [&](int64_t j, int) {
		hl_hp_flush();
		ReadState &r = rs[live[j]];
		if (r.regs0) free(r.regs0);
		r.regs0 = nullptr, r.ra = nullptr;
		r.regs = (mm_reg1_t*)realloc(r.regs, sizeof(mm_reg1_t) * (r.n_regs > 0? r.n_regs : 1));
		hl_set_mapq(r.n_regs, r.regs, opt->min_chain_score, opt->a, r.rep_len, 0, (opt->flag & MM_F_SPLICE) != 0); // map.c:342
		if (r.n_regs == 0) { free(r.regs); r.regs = nullptr; }
		n_regs_out[live[j]] = r.n_regs, regs_out[live[j]] = r.regs;
		if (rep_len_out) rep_len_out[live[j]] = r.rep_len;
	});
}

// K5 launch (the kernel is in jump.cuh)
void mmb_jump_device(mmb_ctx_t *ctx, const mm_idx_t *mi, const mm_mapopt_t *opt, int n_hits, const mmb_jump_hit_t *d_hits, const uint8_t *d_seq, mmb_jump_dec_t *d_out)
{
	if (n_hits <= 0) return;
	const mm_idx_bucket_s *B = mi->B;
	JumpArgs A;
	A.hits = d_hits, A.n_hits = n_hits, A.seq = d_seq;
	A.S = B->d_S, A.seq_off = B->d_seq_off, A.seq_len = B->d_seq_len;
	A.jump_off = B->d_jump_off, A.jump = B->d_jump;
	A.ext = 1 + (opt->b + opt->a - 1) / opt->a + 1, A.jump_min_match = opt->jump_min_match; // jump.c:55
	A.out = d_out;
	ProfScope ps_(ctx, MMB_PROF_OTHER, (uint64_t)n_hits);
	jump_kernel<<<(unsigned)((n_hits + 7) / 8), 256, 0, ctx->stream>>>(A);
	MMB_CUDA_CHECK(cudaGetLastError());
	++ctx->n_launch;
}

// Stage 5 (map.c:362-364): junction jumps of every hit, secondaries included, after MAPQ (which they do not change). The hits whose
// ends K5 may move go to the device as descriptors; the decisions come back and are applied here, to the hits and their CIGARs.
static void jump_batch(Batch &b, const int *n_regs_out, mm_reg1_t *const *regs_out)
{
	mmb_ctx_t *ctx = b.ctx;
	BatchBufs &bb = b.bb;
	const std::vector<int> &live = b.live;
	const std::vector<ReadState> &rs = bb.rs_pool;
	std::vector<std::vector<int>> sel((size_t)b.n);
	parallel_for(b.n, b.n_threads, [&](int64_t j, int) {
		const int i = live[j];
		for (int k = 0; k < n_regs_out[i]; ++k)
			if (mmb_jump_wanted(b.mi, b.opt, rs[i].qlen, &regs_out[i][k])) sel[j].push_back(k);
	});
	std::vector<int64_t> hoff((size_t)b.n + 1, 0);
	for (int j = 0; j < b.n; ++j) hoff[j + 1] = hoff[j] + (int64_t)sel[j].size();
	const int64_t n_hits = hoff[b.n];
	if (n_hits == 0) return;
	const size_t in_bytes = sizeof(mmb_jump_hit_t) * (size_t)n_hits, out_bytes = sizeof(mmb_jump_dec_t) * (size_t)n_hits;
	uint8_t *h_io = bb.h_jump.as<uint8_t>(in_bytes + out_bytes);
	mmb_jump_hit_t *h_hits = (mmb_jump_hit_t*)h_io;
	mmb_jump_dec_t *h_dec = (mmb_jump_dec_t*)(h_io + in_bytes);
	parallel_for(b.n, b.n_threads, [&](int64_t j, int) {
		const int i = live[j];
		for (size_t t = 0; t < sel[j].size(); ++t) {
			const mm_reg1_t *r = &regs_out[i][sel[j][t]];
			mmb_jump_hit_t &h = h_hits[hoff[j] + (int64_t)t];
			h.rid = r->rid, h.rs = r->rs, h.re = r->re, h.qs = r->qs, h.qe = r->qe, h.rev = r->rev;
			h.qlen = rs[i].qlen, h.n_cigar = (int32_t)r->p->n_cigar, h.q_off = b.off[j];
			h.cig_first = r->p->cigar[0], h.cig_last = r->p->cigar[r->p->n_cigar - 1];
		}
	});
	uint8_t *d_io = bb.jump_io.as<uint8_t>(in_bytes + out_bytes);
	{
		GateHold gate(ctx, b.gated, 1);
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_io, h_io, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
		mmb_jump_device(ctx, b.mi, b.opt, (int)n_hits, (const mmb_jump_hit_t*)d_io, b.d_seq, (mmb_jump_dec_t*)(d_io + in_bytes));
		MMB_CUDA_CHECK(cudaMemcpyAsync(h_dec, d_io + in_bytes, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
		mmb_stream_sync(ctx);
	}
	ctx->last_h2d_bytes += in_bytes, ctx->last_d2h_bytes += out_bytes;
	parallel_for(b.n, b.n_threads, [&](int64_t j, int) {
		const int i = live[j];
		for (size_t t = 0; t < sel[j].size(); ++t) mmb_jump_apply(b.opt, rs[i].qlen, &regs_out[i][sel[j][t]], &h_dec[hoff[j] + (int64_t)t]);
	});
}

static int map_group(GroupCtx &G, const mm_idx_t *mi, int n_reads, const int *qlens, const char **seqs, const char **names,
					 int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out, const mm_mapopt_t *opt, int n_threads, const MapPass &pass)
{
	if (n_reads <= 0) return 0;
	mmb_ctx_t *ctx = G.ctx;
	Batch b(ctx, G.bb, G.gated, mi, opt, n_threads < 1? 1 : n_threads);
	mm_idx_bucket_s *B = mi->B;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	// annotated introns of the index (mm_idx_bed_read) for the spliced kernel: what mm_get_junc / mm_idx_bed_junc feed ksw_exts2 (align.c:638-643)
	ctx->n_junc = B->n_junc, ctx->junc_st = B->d_junc, ctx->junc_en = B->d_junc? B->d_junc + B->n_junc : nullptr;
	ctx->junc_strand = B->d_junc? (const int8_t*)(B->d_junc + 2 * B->n_junc) : nullptr;
	for (int t = 0; t < 2; ++t) // splice scores (mm_idx_spsc_read): what mm_idx_spsc_get feeds ksw_exts2 (align.c:640)
		ctx->n_spsc[t] = B->n_spsc[t], ctx->spsc_pos[t] = (const int64_t*)B->d_spsc[t], ctx->spsc_val[t] = B->d_spsc[t]? B->d_spsc[t] + B->n_spsc[t] * 8 : nullptr;
	if (!take_reads(b, n_reads, qlens, seqs, names, n_regs_out, regs_out, rep_len_out)) return 0;
	const uint8_t *h_seq = upload_reads(G, b);
	// the reads are on their way before the group queues for a device slot: every group's upload starts when the batch starts and
	// overlaps the kernels of the groups ahead of it
	GateHold gate1(ctx, b.gated, 0);
	seed_batch(b, h_seq, names, pass.occ_cut);
	chain_batch(b, pass, gate1);
	chains_to_hits(b, pass);
	if (opt->flag & MM_F_CIGAR) align_waves(b);
	finalize_batch(b, n_regs_out, regs_out, rep_len_out);
	if (mi->J && (opt->flag & MM_F_SPLICE) && (opt->flag & MM_F_CIGAR)) jump_batch(b, n_regs_out, regs_out);
	if (g_hp_on) hl_hp_dump("group");
	return 0;
}

// Kernel-level entry for tests: the seeding stage alone (seed_batch) on the context's stream. seqs: the reads back to back (ASCII),
// off: n_reads+1 offsets. Outputs (host): a_off_out[n_reads+1], rep_len_out, n_mini_out; anchors_xy / mini_pos (if non-null) receive
// the sorted anchors (16 B each, a_cap entries) and the kept seeds' span<<32|qpos words (mp_cap entries) read after read. Returns the
// total number of anchors (or -1 if a buffer is too small).
extern "C" int64_t mmb_seed_batch_host(mmb_ctx_t *ctx, const mm_idx_t *mi, int n_reads, const char *seqs, const int64_t *off, int64_t flag, int mid_occ,
										float q_occ_frac, int max_max_occ, int occ_dist, int64_t *a_off_out, int32_t *rep_len_out, int32_t *n_mini_out,
										uint64_t *anchors_xy, int64_t a_cap, uint64_t *mini_pos, int64_t mp_cap)
{
	if (n_reads <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	static BatchBufs bb; // test entry: one caller at a time
	mm_mapopt_t opt; // what seed_batch reads; sdust_thres = 0: no low-complexity masking
	memset(&opt, 0, sizeof(opt));
	opt.flag = flag, opt.mid_occ = mid_occ, opt.q_occ_frac = q_occ_frac, opt.max_max_occ = max_max_occ, opt.occ_dist = occ_dist;
	Batch b(ctx, bb, false, mi, &opt, 1);
	const int n = b.n = n_reads;
	b.live.resize(n);
	for (int j = 0; j < n; ++j) b.live[j] = j;
	b.off.assign(off, off + n + 1);
	const int64_t total_bases = b.total_bases = off[n];
	uint8_t *d_seq = b.d_seq = bb.seq.as<uint8_t>((size_t)total_bases + 16);
	int64_t *d_off = b.d_off = bb.off.as<int64_t>((size_t)n + 1);
	int32_t *d_qlen = b.d_qlen = bb.qlen.as<int32_t>((size_t)n);
	std::vector<int32_t> h_qlen(n);
	for (int j = 0; j < n; ++j) h_qlen[j] = (int32_t)(off[j + 1] - off[j]);
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_seq, seqs, total_bases, cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_off, off, sizeof(int64_t) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_qlen, h_qlen.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	if (total_bases > 0) encode_kernel<<<(unsigned)((total_bases / 4 + 256) / 256), 256, 0, ctx->stream>>>(d_seq, total_bases);
	seed_batch(b, (const uint8_t*)seqs, nullptr, mid_occ);
	const SeedArgs &S = b.S;
	const int64_t total_a = b.total_a;
	std::vector<int64_t> h_mz_off((size_t)n + 1);
	MMB_CUDA_CHECK(cudaMemcpyAsync(a_off_out, S.a_off, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(rep_len_out, S.rep_len, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(n_mini_out, S.n_keep, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaMemcpyAsync(h_mz_off.data(), S.mz_off, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	if (anchors_xy) {
		if (total_a > a_cap) return -1;
		if (total_a) MMB_CUDA_CHECK(cudaMemcpyAsync(anchors_xy, S.a_sorted, sizeof(m128) * (size_t)total_a, cudaMemcpyDeviceToHost, ctx->stream));
	}
	if (mini_pos) {
		int64_t o = 0;
		for (int j = 0; j < n; ++j) {
			if (o + n_mini_out[j] > mp_cap) return -1;
			if (n_mini_out[j]) MMB_CUDA_CHECK(cudaMemcpyAsync(mini_pos + o, S.mini_pos + h_mz_off[j], sizeof(uint64_t) * (size_t)n_mini_out[j], cudaMemcpyDeviceToHost, ctx->stream));
			o += n_mini_out[j];
		}
	}
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return total_a;
}

extern "C" int mmb_jump_batch_host(mmb_ctx_t *ctx, const mm_idx_t *mi, const mm_mapopt_t *opt, int n_reads, const char *seqs, const int64_t *off,
								   int n_hits, const mmb_jump_hit_t *hits, mmb_jump_dec_t *out)
{
	if (!mi->J || !mi->B->d_jump_off) return -1;
	if (n_hits <= 0) return 0;
	MMB_CUDA_CHECK(cudaSetDevice(ctx->device));
	const int64_t total_bases = n_reads > 0? off[n_reads] : 0;
	const size_t in_bytes = sizeof(mmb_jump_hit_t) * (size_t)n_hits, out_bytes = sizeof(mmb_jump_dec_t) * (size_t)n_hits;
	uint8_t *d_seq = ctx->d_a.as<uint8_t>((size_t)total_bases + 16);
	uint8_t *d_io = ctx->d_b.as<uint8_t>(in_bytes + out_bytes);
	if (total_bases > 0) {
		MMB_CUDA_CHECK(cudaMemcpyAsync(d_seq, seqs, total_bases, cudaMemcpyHostToDevice, ctx->stream));
		encode_kernel<<<(unsigned)((total_bases / 4 + 256) / 256), 256, 0, ctx->stream>>>(d_seq, total_bases);
	}
	MMB_CUDA_CHECK(cudaMemcpyAsync(d_io, hits, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
	mmb_jump_device(ctx, mi, opt, n_hits, (const mmb_jump_hit_t*)d_io, d_seq, (mmb_jump_dec_t*)(d_io + in_bytes));
	MMB_CUDA_CHECK(cudaMemcpyAsync(out, d_io + in_bytes, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
	MMB_CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
	return 0;
}

mmb_ctx_t *mmb_default_ctx(void);
void mmb_register_ctx(mmb_ctx_t *c);

static int g_groups_override = 0;
extern "C" void mmb_set_gpu_slots(int n) { g_gpu_slots = n < 1? g_gpu_slots_env : n; } // 0 = default (MM_B200_GPU_SLOTS or two thirds of the groups)
extern "C" void mmb_set_groups(int n) { g_groups_override = n; } // 0 = default (MM_B200_GROUPS or 12); negative: that many groups, one after another

// The scheduler timeline of scheduler group `group` for the last mm_map_batch call (mmb_timeline_enable(1) first): copies up to cap
// (time, event, argument) triples to out (3 doubles each) and returns how many there are; -1 for a group that does not exist.
extern "C" int64_t mmb_timeline_get(int group, double *out, int64_t cap)
{
	std::lock_guard<std::mutex> lk(g_group_mu);
	if (group < 0 || group >= MAX_GROUPS || !g_groups[group]) return -1;
	const std::vector<double> &tl = g_groups[group]->ctx->tl;
	const int64_t n = (int64_t)tl.size() / 3;
	if (out) std::copy(tl.begin(), tl.begin() + 3 * std::min(n, std::max<int64_t>(cap, 0)), out);
	return n;
}

static GroupCtx &get_group(int g, int device)
{
	std::lock_guard<std::mutex> lk(g_group_mu);
	if (!g_groups[g]) {
		g_groups[g] = new GroupCtx();
		g_groups[g]->ctx = mmb_ctx_create(device);
		if (!g_groups[g]->ctx) abort();
		g_groups[g]->ctx->group_id = g;
		g_groups[g]->ctx->profiling = mmb_default_ctx()->profiling;
		mmb_register_ctx(g_groups[g]->ctx);
	}
	return *g_groups[g];
}

// The batch is split into NG contiguous groups (balanced by bases) that run the whole pipeline concurrently, each on its
// own CUDA stream with its own arenas: while one group is in a host phase (hit logic, alignment replay) the others keep
// the GPU busy. This is the scheduler that replaces kt_pipeline/kt_for (map.c:541-691, kthread.c:54-159).
static int map_batch_pass(const mm_idx_t *mi, int n_reads, const int *qlens, const char **seqs, const char **names,
						  int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out, const mm_mapopt_t *opt, int n_threads, const MapPass &pass)
{
	static int ng_env = getenv("MM_B200_GROUPS")? atoi(getenv("MM_B200_GROUPS")) : 12;
	const bool sequential = g_groups_override < 0; // negative override: same groups, run one after another (clean per-kernel timing)
	const int ng_req = g_groups_override > 0? g_groups_override : g_groups_override < 0? -g_groups_override : ng_env;
	int NG = ng_req < 1? 1 : ng_req > MAX_GROUPS? MAX_GROUPS : ng_req;
	int64_t total = 0;
	for (int i = 0; i < n_reads; ++i) total += qlens[i] > 0? qlens[i] : 0;
	if (n_reads < 64 * NG || total < 4000000) NG = 1;
	const int device = mi->B->ctx->device;
	for (int g = 0; g < NG; ++g) { GroupCtx &gc = get_group(g, device); gc.ctx->profiling = mmb_default_ctx()->profiling; gc.gated = gc.ctx->sleepy_sync = NG > 1 && !sequential; }
	g_batch_groups = NG;
	if (NG == 1) return map_group(get_group(0, device), mi, n_reads, qlens, seqs, names, n_regs_out, regs_out, rep_len_out, opt, n_threads, pass);
	std::vector<int> cut(NG + 1, 0);
	{
		// equal shares, except that the last three groups shrink (3/4, 1/2, 1/4 of a share): the end of the batch is then
		// the short serial chain of a small group instead of a full-size one
		std::vector<double> wsum(NG + 1, 0.0);
		for (int g2 = 0; g2 < NG; ++g2) wsum[g2 + 1] = wsum[g2] + (NG >= 8 && g2 >= NG - 3? 0.25 * (NG - g2) : 1.0);
		int64_t acc = 0; int g = 1;
		for (int i = 0; i < n_reads && g < NG; ++i) {
			acc += qlens[i] > 0? qlens[i] : 0;
			if ((double)acc >= (double)total * wsum[g] / wsum[NG]) cut[g++] = i + 1;
		}
		for (; g < NG; ++g) cut[g] = n_reads;
		cut[NG] = n_reads;
	}
	auto run_group = [&](int g) {
		const int b = cut[g], m = cut[g + 1] - cut[g];
		MapPass p = pass; // the pass as a group starting at read b sees it
		if (p.no_chain) p.no_chain += b;
		if (m > 0) map_group(get_group(g, device), mi, m, qlens + b, seqs + b, names? names + b : nullptr, n_regs_out + b, regs_out + b,
							 rep_len_out? rep_len_out + b : nullptr, opt, n_threads, p);
	};
	if (sequential) {
		for (int g = 0; g < NG; ++g) run_group(g);
		return 0;
	}
	std::vector<std::thread> th;
	for (int g = 0; g < NG; ++g) th.emplace_back(run_group, g);
	for (auto &x : th) x.join();
	return 0;
}

extern "C" int mm_map_batch(const mm_idx_t *mi, int n_reads, const int *qlens, const char **seqs, const char **names,
							int *n_regs_out, mm_reg1_t **regs_out, int *rep_len_out, const mm_mapopt_t *opt, int n_threads)
{
	if (n_reads <= 0) return 0;
	static std::mutex batch_mu; // the scheduler groups (streams, arenas) are process-wide: concurrent callers take turns
	std::lock_guard<std::mutex> batch_lk(batch_mu);
	static std::once_flag heap_once;
	std::call_once(heap_once, []() {
		// Keep freed heap memory in the process. Every batch allocates and frees the same few GB on the host threads (hits,
		// CIGARs, job lists of up to a few MB); with glibc's defaults the large blocks are mmap'd and unmapped each time and the heap
		// top is trimmed, so the next batch takes its page faults again, serialised on the process's address-space lock, and
		// the host phases of all groups slow down together (map-ont on an H100 host with 16 CPUs: steps whose host phases took
		// 2-4 times as long as usual, 60-190 ms with the device idle; none with these settings).
		mallopt(M_MMAP_THRESHOLD, 32 << 20);
		mallopt(M_TRIM_THRESHOLD, INT_MAX);
		mallopt(M_TOP_PAD, 256 << 20);
	});
	if (g_mmb_tl_on) { // the timeline holds the current batch only
		std::lock_guard<std::mutex> lk(g_group_mu);
		for (GroupCtx *g : g_groups) if (g) g->ctx->tl.clear();
	}
	if (!supported_mode(mi, opt)) { // mm_map / mm_map_frag report no hits, mm_map_file returns the error (main.c:389 exits on it)
		for (int i = 0; i < n_reads; ++i) { n_regs_out[i] = 0, regs_out[i] = nullptr; if (rep_len_out) rep_len_out[i] = 0; }
		return -1;
	}
	const bool rechain = opt->max_occ > opt->mid_occ && !(opt->flag & MM_F_RMQ); // map.c:293
	if (!rechain) {
		const MapPass first = { opt->mid_occ, true, nullptr };
		return map_batch_pass(mi, n_reads, qlens, seqs, names, n_regs_out, regs_out, rep_len_out, opt, n_threads, first);
	}
	// Re-chaining with the higher occurrence cutoff (map.c:293-316). For single-segment queries the test "the best chain has all
	// the segments" always holds, so exactly the reads that came out of chaining with no chain and have rep_len > 0 collect their
	// seeds again with max_occ = opt->max_occ and are chained again (no long-join pass after it: the two are one if / else if).
	// Those reads have no hits from the first pass, so the second pass simply supplies their result.
	std::vector<uint8_t> no_chain((size_t)n_reads, 0);
	std::vector<int> rep_tmp;
	if (!rep_len_out) { rep_tmp.assign((size_t)n_reads, 0); rep_len_out = rep_tmp.data(); }
	const MapPass first = { opt->mid_occ, true, no_chain.data() };
	map_batch_pass(mi, n_reads, qlens, seqs, names, n_regs_out, regs_out, rep_len_out, opt, n_threads, first);
	std::vector<int> idx;
	for (int i = 0; i < n_reads; ++i) if (no_chain[i] && rep_len_out[i] > 0) idx.push_back(i);
	if (idx.empty()) return 0;
	const int m = (int)idx.size();
	std::vector<int> ql(m), nr(m, 0), rl(m, 0);
	std::vector<const char*> sq(m), nm(m);
	std::vector<mm_reg1_t*> rg(m, nullptr);
	for (int k = 0; k < m; ++k) ql[k] = qlens[idx[k]], sq[k] = seqs[idx[k]], nm[k] = names? names[idx[k]] : nullptr;
	const MapPass second = { opt->max_occ, false, nullptr };
	map_batch_pass(mi, m, ql.data(), sq.data(), names? nm.data() : nullptr, nr.data(), rg.data(), rl.data(), opt, n_threads, second);
	for (int k = 0; k < m; ++k) {
		const int i = idx[k];
		for (int j = 0; j < n_regs_out[i]; ++j) free(regs_out[i][j].p);
		free(regs_out[i]);
		n_regs_out[i] = nr[k], regs_out[i] = rg[k], rep_len_out[i] = rl[k];
	}
	return 0;
}

// ---- the classic single-read API (map.c:13-31, 380-397): a batch of one ----
extern "C" mm_tbuf_t *mm_tbuf_init(void) { return (mm_tbuf_t*)calloc(1, sizeof(mm_tbuf_t)); }
extern "C" void mm_tbuf_destroy(mm_tbuf_t *b) { free(b); }
extern "C" void *mm_tbuf_get_km(mm_tbuf_t *b) { return b? b->km : 0; }

// mm_map is re-entrant in the reference (one mm_tbuf_t per thread, the index shared read-only: minimap.h:341-348, map.c:380-397; mappy drops
// the GIL around it). Here every call is work for the one GPU scheduler, so concurrent callers are COALESCED instead of taking turns: a
// caller queues its read; whoever finds no batch in flight becomes the leader, takes every queued request that uses the same index and
// the same options, runs them as ONE mm_map_batch() and hands the results back. Requests that arrive meanwhile form the next batch.
namespace {
struct MapReq {
	const mm_idx_t *mi; const mm_mapopt_t *opt;
	int qlen; const char *seq, *name;
	int n_regs = 0, rep_len = 0; mm_reg1_t *regs = nullptr;
	bool done = false;
};
std::mutex g_req_mu;
std::condition_variable g_req_cv;
std::deque<MapReq*> g_req_q;
bool g_req_leader = false;
}

extern "C" void mm_map_frag(const mm_idx_t *mi, int n_segs, const int *qlens, const char **seqs, int *n_regs, mm_reg1_t **regs, mm_tbuf_t *b, const mm_mapopt_t *opt, const char *qname)
{
	if (n_segs != 1) {
		fprintf(stderr, "[ERROR] minimap2_b200: multi-segment (paired-end) mapping is not implemented\n");
		abort();
	}
	MapReq me;
	me.mi = mi, me.opt = opt, me.qlen = qlens[0], me.seq = seqs[0], me.name = qname;
	std::unique_lock<std::mutex> lk(g_req_mu);
	g_req_q.push_back(&me);
	while (!me.done) {
		if (g_req_leader) { g_req_cv.wait(lk); continue; }
		g_req_leader = true;
		// my request is still queued (only a leader removes requests, and it marks them done before it steps down)
		std::vector<MapReq*> batch;
		for (auto it = g_req_q.begin(); it != g_req_q.end();) {
			MapReq *r = *it;
			if (r->mi == mi && (r->opt == opt || memcmp(r->opt, opt, sizeof(mm_mapopt_t)) == 0)) { batch.push_back(r); it = g_req_q.erase(it); }
			else ++it;
		}
		lk.unlock();
		const int n = (int)batch.size();
		std::vector<int> ql(n), nr(n, 0), rl(n, 0);
		std::vector<const char*> sq(n), nm(n);
		std::vector<mm_reg1_t*> rg(n, nullptr);
		bool any_name = false;
		for (int i = 0; i < n; ++i) { ql[i] = batch[i]->qlen, sq[i] = batch[i]->seq, nm[i] = batch[i]->name; any_name |= batch[i]->name != nullptr; }
		// query names enter the result only through the hash that breaks ties (map.c:246-248) and skip_seed's name tests; a missing name is
		// passed as such (NULL entry), exactly like a lone call without a name
		mm_map_batch(mi, n, ql.data(), sq.data(), any_name? nm.data() : nullptr, nr.data(), rg.data(), rl.data(), opt, n > 1? 8 : 1);
		lk.lock();
		for (int i = 0; i < n; ++i) batch[i]->n_regs = nr[i], batch[i]->regs = rg[i], batch[i]->rep_len = rl[i], batch[i]->done = true;
		g_req_leader = false;
		g_req_cv.notify_all();
	}
	lk.unlock();
	*n_regs = me.n_regs, regs[0] = me.regs;
	if (b) {
		b->rep_len = me.rep_len;
		b->frag_gap = opt->max_gap_ref > 0? opt->max_gap_ref : opt->max_gap; // map.c:263-271,317
	}
}

extern "C" mm_reg1_t *mm_map(const mm_idx_t *mi, int qlen, const char *seq, int *n_regs, mm_tbuf_t *b, const mm_mapopt_t *opt, const char *qname)
{
	mm_reg1_t *regs = nullptr;
	mm_map_frag(mi, 1, &qlen, &seq, n_regs, &regs, b, opt, qname);
	return regs;
}

// ---- mm_map_file (map.c:541-691): three overlapped steps like the reference's worker_pipeline -- a reader thread parses the next
// mini-batch while the current one is on the GPU, and a writer thread formats (in parallel over reads) and prints the previous one.
// Output order is the input order. ----
namespace {

struct FileBatch {
	std::vector<FastxRecord> recs;
	std::vector<int> qlens, n_regs, rep_len;
	std::vector<const char*> seqs, names;
	std::vector<mm_reg1_t*> regs;
};

template<class T> class HandOff { // bounded FIFO between two pipeline steps
public:
	explicit HandOff(size_t cap) : cap_(cap) {}
	void push(T v) {
		std::unique_lock<std::mutex> lk(mu_);
		cv_.wait(lk, [&] { return q_.size() < cap_; });
		q_.push_back(std::move(v));
		cv_.notify_all();
	}
	void close() { std::lock_guard<std::mutex> lk(mu_); closed_ = true; cv_.notify_all(); }
	bool pop(T &v) { // false once closed and drained
		std::unique_lock<std::mutex> lk(mu_);
		cv_.wait(lk, [&] { return !q_.empty() || closed_; });
		if (q_.empty()) return false;
		v = std::move(q_.front());
		q_.pop_front();
		cv_.notify_all();
		return true;
	}
private:
	std::mutex mu_; std::condition_variable cv_; std::deque<T> q_; size_t cap_; bool closed_ = false;
};

// output step (map.c:578-641) for reads [lo,hi) of one batch, appended to `out`; frees the hits
void format_reads(std::string &out, FileBatch &fb, int lo, int hi, const mm_idx_t *idx, const mm_mapopt_t *opt, bool with_comment)
{
	for (int i = lo; i < hi; ++i) {
		const FastxRecord &rec = fb.recs[i];
		const char *qual = rec.qual.empty()? nullptr : rec.qual.c_str();
		const int n_regs = fb.n_regs[i];
		mm_reg1_t *regs = fb.regs[i];
		if (opt->flag & MM_F_OUT_JUNC) { // --write-junc (map.c:601-607): junctions of the primary hits of MAPQ >= 10 instead of PAF / SAM
			for (int j = 0; j < n_regs; ++j)
				if (regs[j].id == regs[j].parent && regs[j].mapq >= 10) hl_write_junc(out, idx, fb.names[i], &regs[j]);
		} else if (n_regs > 0) {
			for (int j = 0; j < n_regs; ++j) {
				const mm_reg1_t *rg = &regs[j];
				if ((opt->flag & MM_F_NO_PRINT_2ND) && rg->id != rg->parent) continue;
				if (opt->flag & MM_F_OUT_SAM) hl_write_sam(out, idx, fb.names[i], fb.seqs[i], qual, fb.qlens[i], j, n_regs, regs, opt->flag, fb.rep_len[i]);
				else { hl_set_seq_for_tags(fb.seqs[i]); hl_write_paf(out, idx, fb.names[i], fb.qlens[i], rg, opt->flag, fb.rep_len[i]); }
				if (with_comment && !rec.comment.empty()) out += '\t', out += rec.comment;
				out += '\n';
			}
		} else if ((opt->flag & MM_F_PAF_NO_HIT) || ((opt->flag & MM_F_OUT_SAM) && !(opt->flag & MM_F_SAM_HIT_ONLY))) {
			if (opt->flag & MM_F_OUT_SAM) hl_write_sam(out, idx, fb.names[i], fb.seqs[i], qual, fb.qlens[i], -1, 0, nullptr, opt->flag, fb.rep_len[i]);
			else hl_write_paf(out, idx, fb.names[i], fb.qlens[i], nullptr, opt->flag, fb.rep_len[i]);
			if (with_comment && !rec.comment.empty()) out += '\t', out += rec.comment;
			out += '\n';
		}
		for (int j = 0; j < n_regs; ++j) free(regs[j].p);
		free(regs);
		fb.regs[i] = nullptr;
	}
}

} // namespace

extern "C" int mm_map_file_frag(const mm_idx_t *idx, int n_segs, const char **fn, const mm_mapopt_t *opt, int n_threads)
{
	if (n_segs != 1) { fprintf(stderr, "[ERROR] minimap2_b200: multi-file (paired) input is not implemented\n"); return -1; }
	if (!supported_mode(idx, opt)) return -1;
	FastxReader rd(fn[0]);
	if (!rd.ok()) {
		if (mm_verbose >= 1) fprintf(stderr, "ERROR: failed to open file '%s'\n", fn[0]);
		return -1;
	}
	const bool with_qual = (opt->flag & MM_F_OUT_SAM) && !(opt->flag & MM_F_NO_QUAL);
	const bool with_comment = (opt->flag & MM_F_COPY_COMMENT) != 0;
	typedef std::unique_ptr<FileBatch> BatchPtr;
	HandOff<BatchPtr> parsed(1), mapped(1);
	std::thread reader([&]() { // step 0: mm_bseq_read3 (bseq.c:80-119)
		for (;;) {
			BatchPtr fb(new FileBatch);
			int64_t size = 0;
			FastxRecord r;
			int ret;
			while ((ret = rd.next(r, with_qual, with_comment)) > 0) {
				size += (int64_t)r.seq.size();
				fb->recs.push_back(std::move(r));
				if (size >= opt->mini_batch_size) break;
			}
			if (fb->recs.empty()) break;
			const int n = (int)fb->recs.size();
			fb->qlens.resize(n), fb->n_regs.resize(n), fb->rep_len.resize(n), fb->seqs.resize(n), fb->names.resize(n), fb->regs.resize(n);
			for (int i = 0; i < n; ++i) fb->qlens[i] = (int)fb->recs[i].seq.size(), fb->seqs[i] = fb->recs[i].seq.c_str(), fb->names[i] = fb->recs[i].name.c_str();
			parsed.push(std::move(fb));
			if (ret <= 0) break;
		}
		parsed.close();
	});
	std::thread writer([&]() { // step 2: format in parallel over blocks of reads, print in input order
		// formatting runs next to the following batch's host phases: keep it to an eighth of the CPUs (at most 16 threads), the
		// scheduler's own threads must not queue behind it (see the pool cap in HostPool)
		const int hw = (int)std::thread::hardware_concurrency();
		int n_fmt = hw >= 16? hw / 8 : 1;
		if (n_fmt > n_threads) n_fmt = n_threads;
		if (n_fmt > 16) n_fmt = 16;
		if (n_fmt < 1) n_fmt = 1;
		BatchPtr fb;
		while (mapped.pop(fb)) {
			const int n = (int)fb->recs.size(), blk = 128, n_blk = (n + blk - 1) / blk;
			std::vector<std::string> outs(n_blk);
			std::atomic<int> next(0);
			auto work = [&]() { for (int b; (b = next.fetch_add(1)) < n_blk;) format_reads(outs[b], *fb, b * blk, std::min(n, (b + 1) * blk), idx, opt, with_comment); };
			std::vector<std::thread> th;
			for (int t = 1; t < n_fmt && t < n_blk; ++t) th.emplace_back(work);
			work();
			for (auto &x : th) x.join();
			for (const std::string &o : outs) fwrite(o.data(), 1, o.size(), stdout);
			fb.reset();
		}
		fflush(stdout);
	});
	BatchPtr fb;
	while (parsed.pop(fb)) { // step 1: the GPU pipeline
		const int n = (int)fb->recs.size();
		mm_map_batch(idx, n, fb->qlens.data(), fb->seqs.data(), fb->names.data(), fb->n_regs.data(), fb->regs.data(), fb->rep_len.data(), opt, n_threads);
		if (mm_verbose >= 3)
			fprintf(stderr, "[M::%s::%.3f*%.2f] mapped %d sequences\n", __func__, realtime() - mm_realtime0, cputime() / (realtime() - mm_realtime0), n);
		mapped.push(std::move(fb));
	}
	mapped.close();
	reader.join();
	writer.join();
	return 0;
}

extern "C" int mm_map_file(const mm_idx_t *idx, const char *fn, const mm_mapopt_t *opt, int n_threads)
{
	return mm_map_file_frag(idx, 1, &fn, opt, n_threads);
}
