// minimap2_b200/csrc/index.h -- the device index object behind mm_idx_t::B.
//
// Layout in HBM (device-resident for the lifetime of the index; one replica per GPU):
//   tab[2^bits]   open-addressing hash table, 16 B slots {key = minimizer hash (x>>8), val = off<<28 | n};
//                 one 128-bit load per probe, linear probing, load factor <= 0.5
//   pos[n_pos]    occurrence words rid<<32|lastPos<<1|strand, grouped by key, ascending inside a key
//                 (what mm_idx_get returns; index.c:93-110, order per index.c:264-266)
//   S[]           4-bit packed reference, identical to mm_idx_t::S (mmpriv.h:34-35), + per-sequence offset/len
// Host copies (keys/val/pos sorted by key) are materialised lazily for the host API (mm_idx_get, stat, dump).
#pragma once
#include "mmb_internal.h"
#include "minimap.h"
#include "annot.h"
#include <string>
#include <unordered_map>
#include <mutex>

#define MMB_IDX_NBITS 28                      // low bits of val hold the occurrence count
#define MMB_IDX_EMPTY (~0ULL)

struct IdxSlot { uint64_t key, val; };

struct DevIndexView {     // passed by value to kernels
	const IdxSlot *tab;
	uint64_t tab_mask;
	int tab_bits;
	const uint64_t *pos;
	const uint32_t *S;
	const uint64_t *seq_off;
	const uint32_t *seq_len;
	uint32_t n_seq;
};

struct mm_idx_bucket_s {  // the opaque "B" of mm_idx_t
	mmb_ctx_t *ctx = nullptr;
	bool external = false;              // device arrays are owned by the caller (adopted after an NCCL broadcast)
	int64_t n_keys = 0, n_pos = 0;
	// device
	IdxSlot *d_tab = nullptr; int tab_bits = 0;
	uint64_t *d_pos = nullptr;
	uint32_t *d_S = nullptr;
	uint64_t *d_seq_off = nullptr;
	uint32_t *d_seq_len = nullptr;
	uint32_t *d_cnt_sorted = nullptr;   // ascending occurrence counts (for mm_idx_cal_max_occ)
	uint32_t *d_name_rank = nullptr;    // rank of every sequence name in the sorted name list (skip_seed, map.c:78-100); lazy
	std::vector<uint32_t> name_order;   // sequence ids in name order (host side of the same)
	uint64_t *d_ukeys = nullptr; uint32_t *d_ucnt = nullptr; int64_t *d_uoff = nullptr; // key list kept for the lazy host mirror
	uint8_t *d_spsc[2] = {nullptr, nullptr}; int64_t n_spsc[2] = {0, 0}; // splice scores per strand (mm_idx_spsc_read): n positions (int64, global S coordinates) | n bytes
	int64_t *d_junc = nullptr; int64_t n_junc = 0; // annotated introns (mm_idx_bed_read): n_junc starts | n_junc ends (global S coordinates, int64) | n_junc strands (int8)
	int64_t *d_jump_off = nullptr; mm_idx_jjump1_t *d_jump = nullptr; // jump table (mm_idx_jjump_read): n_seq+1 entry offsets | the entries of mi->J, contig after contig (one allocation)
	// host (lazy)
	std::mutex mu;
	bool host_ready = false;
	std::vector<uint64_t> h_keys, h_val, h_pos;
	std::unordered_map<uint64_t, uint32_t> *h_map = nullptr; // key -> rank (built on first host mm_idx_get)
	DevIndexView view(const mm_idx_t *mi) const {
		DevIndexView v;
		v.tab = d_tab, v.tab_mask = (1ULL << tab_bits) - 1, v.tab_bits = tab_bits, v.pos = d_pos, v.S = d_S;
		v.seq_off = d_seq_off, v.seq_len = d_seq_len, v.n_seq = mi->n_seq;
		return v;
	}
};

__device__ __forceinline__ uint64_t idx_slot_of(uint64_t key, int bits)
{
	return (key * 0x9E3779B97F4A7C15ULL) >> (64 - bits);
}

// device-side mm_idx_get: returns n (0 if absent) and the offset of the occurrence list in pos[]
__device__ __forceinline__ uint32_t idx_get_dev(const DevIndexView &ix, uint64_t key, uint64_t *off)
{
	uint64_t s = idx_slot_of(key, ix.tab_bits);
	for (;;) {
		const ulonglong2 e = *reinterpret_cast<const ulonglong2*>(&ix.tab[s]);
		if (e.x == key) { *off = e.y >> MMB_IDX_NBITS; return (uint32_t)(e.y & ((1ULL << MMB_IDX_NBITS) - 1)); }
		if (e.x == MMB_IDX_EMPTY) { *off = 0; return 0; }
		s = (s + 1) & ix.tab_mask;
	}
}

mmb_ctx_t *mmb_default_ctx(void);   // process-wide context (device from MM_B200_DEVICE / LOCAL_RANK / 0)
void mmb_idx_host_sync(const mm_idx_t *mi); // materialise host copies

// build the device side from mi->S / mi->seq (host) -- index.cu
void mmb_idx_build_device(mm_idx_t *mi);
// build the device side from explicit (key, occurrences) lists (used by mm_idx_load) -- keys need not be sorted
void mmb_idx_build_from_lists(mm_idx_t *mi, std::vector<uint64_t> &keys, std::vector<uint32_t> &cnt, std::vector<uint64_t> &pos);

// sketch.cu
int64_t mmb_sketch_device(mmb_ctx_t *ctx, const uint8_t *d_bytes, const uint32_t *d_packed, const int64_t *d_seq_off, int n_seq,
						  const uint32_t *d_rid, uint32_t rid0, int w, int k, int is_hpc, int64_t total_bases,
						  DevBuf &out, int64_t *d_mz_off, DevBuf &tmp_a, DevBuf &tmp_b, int same_rid = 0);
