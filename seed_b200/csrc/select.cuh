// select.cuh -- block-wide selection primitives of the 1024-thread generation kernels (sampler, logits processors,
// beam candidates, contrastive candidates), and the device side of the step-counter protocol (GenSlot in ops.h).
//
// Every fp32 reduction here runs in one fixed order, so that each kernel keeps its bits: the xor butterfly 16 -> 1
// within each warp, then warp 0 over the SEL_WARPS per-warp partials.
#pragma once

#include "common.cuh"
#include "ops.h"

namespace sb {

constexpr int SEL_THREADS = 1024;      // block size of every kernel that calls the block-wide helpers below
constexpr int SEL_WARPS = SEL_THREADS / 32;
static_assert(SEL_WARPS == 32, "warp 0 reduces one per-warp partial per lane");

// block-wide max (IS_MAX) or sum of v; red holds SEL_WARPS partials.  Every thread returns the result.
template <bool IS_MAX>
__device__ __forceinline__ float block_reduce(float v, float* red) {
  v = IS_MAX ? warp_max(v) : warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                     // red may still be read from the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    const float t = IS_MAX ? warp_max(red[lane]) : warp_sum(red[lane]);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_sum(float v, float* red) { return block_reduce<false>(v, red); }
__device__ __forceinline__ float block_max(float v, float* red) { return block_reduce<true>(v, red); }

// sum over the block of expf(row[i] - mx), this thread's elements [i0, i1) in index order
__device__ __forceinline__ float block_exp_sum(const __half* row, int i0, int i1, float mx, float* red) {
  float z = 0.0f;
  for (int i = i0; i < i1; ++i) z += expf(__half2float(row[i]) - mx);
  return block_sum(z, red);
}

// (key a, index ia) beats (b, ib): the larger key, ties to the lower index.  A NaN key never wins.
__device__ __forceinline__ bool key_better(float a, int ia, float b, int ib) { return a > b || (a == b && ia < ib); }

__device__ __forceinline__ void warp_best(float& key, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ok = __shfl_xor_sync(0xffffffffu, key, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (key_better(ok, oi, key, idx)) { key = ok; idx = oi; }
  }
}

// the block's best (key, idx) under key_better, stored to *best_key / *best_idx, which every thread may read on
// return.  red / redi hold SEL_WARPS partials.
__device__ __forceinline__ void block_best(float key, int idx, float* red, int* redi, float* best_key, int* best_idx) {
  warp_best(key, idx);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) { red[warp] = key; redi[warp] = idx; }
  __syncthreads();
  if (warp == 0) {
    key = red[lane]; idx = redi[lane];
    warp_best(key, idx);
    if (lane == 0) { *best_key = key; *best_idx = idx; }
  }
  __syncthreads();
}

// One thread's best N (key, index) pairs in registers, best first; empty entries hold (-inf, 0x7fffffff).
template <int N>
struct BestList {
  float key[N];
  int idx[N];
  __device__ __forceinline__ BestList() {
#pragma unroll
    for (int q = 0; q < N; ++q) { key[q] = -INFINITY; idx[q] = 0x7fffffff; }
  }
  __device__ __forceinline__ void insert(float k, int i) {
#pragma unroll
    for (int q = 0; q < N; ++q) {
      if (key_better(k, i, key[q], idx[q])) {
        const float tk = key[q]; const int ti = idx[q];
        key[q] = k; idx[q] = i; k = tk; i = ti;
      }
    }
  }
  // n block-wide rounds: round r stores the best head of all threads' lists to s_key[r] / s_idx[r] and pops it from
  // the list that held it.  red / redi hold SEL_WARPS partials.
  __device__ __forceinline__ void pop_rounds(int n, float* red, int* redi, float* s_key, int* s_idx) {
    for (int r = 0; r < n; ++r) {
      block_best(key[0], idx[0], red, redi, &s_key[r], &s_idx[r]);
      if (idx[0] == s_idx[r] && idx[0] != 0x7fffffff) {
#pragma unroll
        for (int q = 0; q + 1 < N; ++q) { key[q] = key[q + 1]; idx[q] = idx[q + 1]; }
        key[N - 1] = -INFINITY; idx[N - 1] = 0x7fffffff;
      }
    }
  }
};

// ---- step counters (GenSlot) ---------------------------------------------------------------------------------------
// Sequence b emits `tok` at `step` (one thread per sequence).  A sequence that already finished emits pad instead (HF:
// next * unfinished + pad * (1 - unfinished)) and eos finishes it; finished NULL: no sequence ever finishes.  Writes
// out[b, S + step] when out is given.  Returns the token emitted; *was_unfinished: b had not finished before.
__device__ __forceinline__ long long emit_token(long long tok, int b, long long step, const GenParams& gp,
                                                int* finished, long long* out, long long out_ld, bool* was_unfinished) {
  bool unfinished = true;
  if (finished != nullptr) {
    unfinished = finished[b] == 0;
    if (!unfinished) tok = gp.pad;
    else if (gp.eos >= 0 && tok == gp.eos) finished[b] = 1;
  }
  if (out != nullptr) out[(long long)b * out_ld + gp.proc.S + step] = tok;
  *was_unfinished = unfinished;
  return tok;
}

// Arrival of one of B sequences at the end of `step` (one thread each, after its writes).  The last to arrive calls
// on_last(), resets the arrival count, advances GS_STEP to step + 1 and, when a decode forward consumed this step's
// input, GS_CACHE_LEN by one.
template <typename OnLast>
__device__ __forceinline__ void step_arrive(int* state, int B, int step, bool advance_cache, OnLast on_last) {
  __threadfence();
  if (atomicAdd(&state[GS_ARRIVE], 1) == B - 1) {
    on_last();
    state[GS_ARRIVE] = 0;
    state[GS_STEP] = step + 1;
    if (advance_cache) state[GS_CACHE_LEN] += 1;
    __threadfence();
  }
}

// step_arrive of the sampler and contrastive loops: a sequence unfinished before this step raises GS_UNFINISHED, and
// the last arriver then records the step as one HF keeps (GS_VALID; HF stops once every sequence has finished)
__device__ __forceinline__ void seq_arrive(int* state, int B, int step, bool advance_cache, bool was_unfinished) {
  if (was_unfinished) atomicOr(&state[GS_UNFINISHED], 1);
  step_arrive(state, B, step, advance_cache, [&] {
    if (atomicOr(&state[GS_UNFINISHED], 0) != 0) state[GS_VALID] = step + 1;
    state[GS_UNFINISHED] = 0;
  });
}

// a run's reset: the cache holds the prompt's cache_len positions, every other slot is zero
__device__ __forceinline__ void gen_state_reset(int* state, int cache_len) {
  state[GS_CACHE_LEN] = cache_len;
#pragma unroll
  for (int s = GS_CACHE_LEN + 1; s < GS_SLOTS; ++s) state[s] = 0;
}

}  // namespace sb
