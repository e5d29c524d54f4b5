// minimap2_b200/csrc/scan.cuh -- small device prefix-sum helpers (plumbing between the stage kernels).
#pragma once
#include "mmb_internal.h"

// In-place exclusive scan of d[0..n) (int64). If with_total, d[n] receives the total. Returns the total (this
// synchronises the stream: callers use the total to size the next stage's buffers).
int64_t mmb_exclusive_scan_i64(mmb_ctx_t *ctx, int64_t *d, int64_t n, bool with_total);
// Same without returning/synchronising (total written to d[n]).
void mmb_exclusive_scan_i64_async(mmb_ctx_t *ctx, int64_t *d, int64_t n);

// Stacks of mmx_rs_sort for every read of a batch with n_tot anchors in all (which reads will need one is not known in advance).
// Reserves head_bytes for the caller at the start of buf, then n_reads+1 per-read stack offsets, then the stacks; fills the offsets on
// the device (exclusive scan of mmx_rs_stack_len over a_off) and returns them. head_bytes must be a multiple of 8.
int64_t *mmb_sort_stacks_async(mmb_ctx_t *ctx, const int64_t *a_off, int n_reads, int64_t n_tot, DevBuf &buf, size_t head_bytes);
// The stacks, right after the offsets
inline int32_t *mmb_sort_stacks(int64_t *stk_off, int n_reads) { return (int32_t*)(stk_off + n_reads + 1); }
