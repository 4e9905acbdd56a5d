// gemm_wgmma.cu -- out = epilogue(A[M,K] . W[N,K]^T), fp16 operands, fp32 accumulate.
//
// This is the kernel that carries >97% of the encode FLOPs (SURVEY.md 2.4 rows E1,E4,E6,E7,
// E10-E15) and all LLaMA linears (rows L4,L8,L9,L10).  It replaces the cuBLAS calls behind
// torch.nn.functional.linear in the reference (eva_vit.py:133-135,157,60-65;
// qformer_causual.py:176-181,251-255,320-337; llama_xformer.py:186,223-225,258,718).
//
// Design (H100 / sm_90a):
//   * persistent, warp-specialised, 3 warpgroups: warpgroup 0 = TMA producer (one thread),
//     warpgroups 1 and 2 = consumers, each owning 64 rows of the 128 x BN tile;
//   * A and W tiles are fetched by TMA (cp.async.bulk.tensor, 128-byte swizzle) into a
//     multi-stage shared-memory ring guarded by full/empty mbarriers;
//   * the consumers run wgmma.mma_async m64nBNk16 straight from shared memory, accumulators in
//     registers (setmaxnreg moves the producer's register budget to them);
//   * epilogue from registers: bias / activation / residual with the reference's fp16 rounding
//     points.  Its operands are fetched while the k-loop runs (column vectors staged in shared memory, LayerNorm
//     statistics in registers, residual rows prefetched into L2), and its kind is chosen once per tile, so the
//     per-column work is arithmetic and stores.  While it runs, the producer already streams the next tile's operands.  SiLU-gate
//     mode reads the gate and up halves of the same accumulator tile (llama_xformer.py:186).
#include <stdio.h>

#include "common.cuh"
#include "int8.cuh"
#include "ops.h"

namespace sb {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;
constexpr int GEMM_THREADS = 384;      // producer warpgroup + 2 consumer warpgroups

struct GemmParams {
  int M, N, K;
  int m_tiles, n_tiles;
  const __half* bias;
  const __half* residual;
  long long ldr;
  __half* out;
  long long ldo;
  int act;
  int row_group, row_stride, row_offset;
  int res_mod, res_offset;
  const float2* ln_stats;    // LayerNorm folded into this GEMM (see seedb200_gemm_desc.ln_stats): per-row (mean, rstd),
  const float* ln_c;         // per-column c[n] = sum_k W'[n,k] and b'[n] = sum_k W[n,k] beta[k] + bias[n]:
  const float* ln_b;         //   out = rstd * (acc - mean * c) + b'
  int sched;                 // 0: round robin.  1: balanced tail -- the tiles of the last column go last, to the units
                             // that got one full tile fewer
  float2* row_moments;       // (sum, sum of squares) per 64-column group of the stored output rows
};

// Persistent schedule: the tile (mt * n_tiles + nt) of unit `unit`'s round-th iteration, >= m_tiles * n_tiles when the
// unit is done.  sched 0: round robin rotated by tile_shift per round.  sched 1: balanced tail.
__host__ __device__ inline int sched_tile(int sched, int round, int unit, int units, int m_tiles, int n_tiles, int tile_shift) {
  const int total_tiles = m_tiles * n_tiles;
  if (sched == 0) {
    const int t = round * units + (unit + round * tile_shift) % units;
    return t < total_tiles ? t : total_tiles;
  }
  const int ncol_full = n_tiles - 1;
  const int F = m_tiles * ncol_full;               // full-width tiles; the m_tiles tiles of the last column come last
  const int q = F / units, r = F % units;
  const int nf = q + (unit < r ? 1 : 0);
  if (round < nf) {
    const int f = round * units + unit;
    return (f / ncol_full) * n_tiles + (f % ncol_full);
  }
  if (r != 0 && unit < r) return total_tiles;      // already has one full tile more than the others
  const int S = (r == 0) ? units : units - r;
  const int t = (unit - (r == 0 ? 0 : r)) + (round - nf) * S;
  return t < m_tiles ? t * n_tiles + ncol_full : total_tiles;
}

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  static constexpr int B_BYTES = BN * GEMM_BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES_RAW = (200 * 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAGES * STAGE_BYTES + 2 * STAGES * 8 + 2 * 2 * BN * 4;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(B_BYTES % 1024 == 0, "W stage must keep 1024-byte alignment for SWIZZLE_128B");
  static_assert(BN % 16 == 0 && BN <= 256, "invalid wgmma N");
  static_assert(STAGES >= 3, "pipeline too shallow");
};

__device__ __forceinline__ float rcp_approx(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float gelu_erf(float x) {
  // 0.5 x (1 + erf(x / sqrt 2)) = 0.5 (x + |x| erf(|x| / sqrt 2)); erf by Abramowitz-Stegun 7.1.26
  // (|err| < 1.5e-7, far below fp16 resolution); ~15 issue slots per element, 2 of them MUFU
  const float ax = fabsf(x);
  const float t = rcp_approx(fmaf(0.3275911f * 0.70710678118654752f, ax, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  const float e = ex2_approx(ax * ax * (-0.5f * 1.4426950408889634f));   // exp(-(|x|/sqrt2)^2)
  const float erf_abs = fmaf(-p, e, 1.0f);
  return 0.5f * fmaf(ax, erf_abs, x);
}

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case SEEDB200_ACT_GELU: return gelu_erf(x);
    case SEEDB200_ACT_TANH: return tanhf(x);
    case SEEDB200_ACT_RELU: return x < 0.0f ? 0.0f : x;   // NaN stays NaN, as torch.relu (fmaxf would give 0)
    default: return x;
  }
}

// ---- wgmma ------------------------------------------------------------------
// 64-bit shared-memory matrix descriptor (sm_90), K-major operand, 128-byte swizzle: rows are 128 B (64 halves),
// 8-row groups 1024 B apart (SBO); LBO is unused for swizzled K-major layouts.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);   // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                      // leading byte offset [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // stride byte offset [32,46)
  d |= static_cast<uint64_t>(1) << 62;                      // layout type: SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads above a wgmma.wait_group
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// mbar_wait / mbar_wait_relaxed without the printf call of mbar_timeout_trap: a function call anywhere in a kernel
// makes ptxas serialise its wgmma instructions
__device__ __forceinline__ void mbar_wait_nocall(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++polls & 4095u) == 0 && clock64() - t0 > SB_MBAR_TIMEOUT_CYCLES) __trap();
  }
}
__device__ __forceinline__ void mbar_wait_relaxed_nocall(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (!mbar_try_wait_hint(bar, parity, 2000u)) {
    if ((++polls & 255u) == 0 && clock64() - t0 > SB_MBAR_TIMEOUT_CYCLES) __trap();
  }
}

// D[64 x N] += A[64 x 16] . B[N x 16]^T, both operands K-major in shared memory; issued by a whole warpgroup
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t a, uint64_t b);
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<176>(float (&d)[88], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n176k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87}, %88, %89, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<192>(float (&d)[96], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16<256>(float (&d)[128], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
               : "l"(a), "l"(b));
}

// D[64 x N] += A[64 x 32] . B[N x 32]^T, int8 operands K-major in shared memory, int32 accumulators
template <int N>
__device__ __forceinline__ void wgmma_s8(int (&d)[N / 2], uint64_t a, uint64_t b);
template <> __device__ __forceinline__ void wgmma_s8<64>(int (&d)[32], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_s8<128>(int (&d)[64], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
               : "l"(a), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_s8<256>(int (&d)[128], uint64_t a, uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
               : "l"(a), "l"(b));
}

// Per-tile epilogue kinds of MODE 0 (one branch per tile, not per output pair)
enum EpiCols { EPI_NONE = 0, EPI_BIAS = 1, EPI_LN = 2 };

// Two adjacent columns of one output row, MODE 0: (LN fold | bias) -> fp16 -> act -> fp16 -> (+residual) -> fp16.
// c, b: the columns' ln_c / ln_b (EPI_LN) or bias (b, EPI_BIAS), staged in shared memory per tile.
template <int COLS>
__device__ __forceinline__ __half2 epilogue_pair(float v0, float v1, float2 c, float2 b, float2 ln_st, int act,
                                                 bool has_res, __half2 res) {
  if (COLS == EPI_LN) {
    // LayerNorm folded into the GEMM: acc = sum_k W'[n,k] x[m,k] with W' = W diag(gamma), so
    // W LN(x) + bias = rstd * (acc - mean * c[n]) + b'[n]   (fp32, one rounding to fp16 below)
    v0 = fmaf(ln_st.y, fmaf(-ln_st.x, c.x, v0), b.x);
    v1 = fmaf(ln_st.y, fmaf(-ln_st.x, c.y, v1), b.y);
  } else if (COLS == EPI_BIAS) {
    v0 += b.x;
    v1 += b.y;
  }
  __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
  if (act != SEEDB200_ACT_NONE) {
    h0 = __float2half_rn(apply_act(__half2float(h0), act));
    h1 = __float2half_rn(apply_act(__half2float(h1), act));
  }
  if (has_res) {
    h0 = __float2half_rn(__half2float(h0) + __half2float(__low2half(res)));
    h1 = __float2half_rn(__half2float(h1) + __half2float(__high2half(res)));
  }
  return __halves2half2(h0, h1);
}

__device__ __forceinline__ void store_pair(__half* op, __half2 h, bool pair_ok) {
  if (pair_ok && (reinterpret_cast<uintptr_t>(op) & 3) == 0) {
    *reinterpret_cast<__half2*>(op) = h;
  } else {
    op[0] = __low2half(h);
    if (pair_ok) op[1] = __high2half(h);
  }
}

__device__ __forceinline__ __half2 load_pair(const __half* ip, bool pair_ok) {
  if (pair_ok && (reinterpret_cast<uintptr_t>(ip) & 3) == 0) return *reinterpret_cast<const __half2*>(ip);
  return __halves2half2(ip[0], pair_ok ? ip[1] : __float2half_rn(0.0f));
}

// Output row of GEMM row m (row remap of the patch embed) and the residual row it adds
__device__ __forceinline__ long long out_row_of(const GemmParams& p, int m) {
  return p.row_group > 0 ? (long long)(m / p.row_group) * p.row_stride + (m % p.row_group) + p.row_offset : m;
}
__device__ __forceinline__ long long res_row_of(const GemmParams& p, int m) {
  return p.res_mod > 0 ? (long long)(m % p.res_mod) + p.res_offset : out_row_of(p, m);
}

// MODE 0 epilogue of one tile for one consumer thread: rows m0 and m0 + 8 (row_ok, out_row, res_row per row), per
// 8-column group j the columns n0 + 8 j + col_in_pair (+1).  One 64-column chunk per call, J0 = its first group;
// the chunks are unrolled by recursion so that acc stays in registers.  The chunk's residual is loaded for both rows
// before any of its results is stored (the output may be the residual, so the compiler cannot hoist these loads
// above the stores itself): one memory latency per chunk instead of one per column pair.
template <int BN, int COLS, int J0>
__device__ __forceinline__ void epilogue_chunks(const GemmParams& p, const float (&acc)[BN / 2], int m0, int n0,
                                                int col_in_pair, int lane, const float* col_c, const float* col_b,
                                                const float2 (&ln_st)[2], const bool (&row_ok)[2],
                                                __half* const (&out_row)[2], const __half* const (&res_row)[2]) {
  constexpr int NJ = BN / 8, CH = 8;
  if constexpr (J0 < NJ) {
    const bool has_res = p.residual != nullptr;
    __half2 rv[2][CH];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < CH; ++jj) {
        const int n = n0 + 8 * (J0 + jj) + col_in_pair;
        rv[h][jj] = __float2half2_rn(0.0f);
        if (has_res && J0 + jj < NJ && row_ok[h] && n < p.N) rv[h][jj] = load_pair(res_row[h] + n, n + 1 < p.N);
      }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mom_s = 0.0f, mom_q = 0.0f;
#pragma unroll
      for (int jj = 0; jj < CH && J0 + jj < NJ; ++jj) {
        const int j = J0 + jj;
        const int nl = 8 * j + col_in_pair, n = n0 + nl;
        const bool col_ok = row_ok[h] && n < p.N;
        __half2 o = __float2half2_rn(0.0f);
        if (col_ok) {
          float2 c = make_float2(0.0f, 0.0f), b = make_float2(0.0f, 0.0f);
          if (COLS == EPI_LN) c = *reinterpret_cast<const float2*>(col_c + nl);
          if (COLS != EPI_NONE) b = *reinterpret_cast<const float2*>(col_b + nl);
          o = epilogue_pair<COLS>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], c, b, ln_st[h], p.act, has_res,
                                  rv[h][jj]);
          store_pair(out_row[h] + n, o, n + 1 < p.N);
        }
        if (p.row_moments != nullptr) {
          const float2 f = __half22float2(o);
          mom_s += f.x + f.y;
          mom_q = fmaf(f.x, f.x, mom_q);
          mom_q = fmaf(f.y, f.y, mom_q);
          if ((j & 7) == 7) {          // a 64-column group is complete: reduce over the 4 threads of the row
            mom_s += __shfl_xor_sync(0xffffffffu, mom_s, 1);
            mom_q += __shfl_xor_sync(0xffffffffu, mom_q, 1);
            mom_s += __shfl_xor_sync(0xffffffffu, mom_s, 2);
            mom_q += __shfl_xor_sync(0xffffffffu, mom_q, 2);
            // a last tile that reaches past N (N % BN != 0) has groups beyond the row: they belong to no one
            const int groups = p.N >> 6, g = (n0 >> 6) + (j >> 3);
            if (row_ok[h] && (lane & 3) == 0 && g < groups)
              p.row_moments[(long long)(m0 + 8 * h) * groups + g] = make_float2(mom_s, mom_q);
            mom_s = 0.0f; mom_q = 0.0f;
          }
        }
      }
    }
    epilogue_chunks<BN, COLS, J0 + CH>(p, acc, m0, n0, col_in_pair, lane, col_c, col_b, ln_st, row_ok, out_row,
                                       res_row);
  }
}

template <int BN, int COLS>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float (&acc)[BN / 2], int m0, int n0,
                                              int col_in_pair, int lane, const float* col_c, const float* col_b,
                                              const float2 (&ln_st)[2]) {
  bool row_ok[2];
  __half* out_row[2];
  const __half* res_row[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + 8 * h;
    row_ok[h] = m < p.M;
    out_row[h] = p.out + out_row_of(p, m) * p.ldo;
    res_row[h] = (p.residual != nullptr && row_ok[h]) ? p.residual + res_row_of(p, m) * p.ldr : nullptr;
  }
  epilogue_chunks<BN, COLS, 0>(p, acc, m0, n0, col_in_pair, lane, col_c, col_b, ln_st, row_ok, out_row, res_row);
}

template <int BN, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B stages need 1024-byte alignment
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_base + STAGES * Cfg::A_BYTES;
  const uint32_t full_bar = smem_base + STAGES * Cfg::STAGE_BYTES;   // [STAGES]
  const uint32_t empty_bar = full_bar + STAGES * 8;                  // [STAGES]
  const uint32_t col_vecs = empty_bar + STAGES * 8;                // epilogue column vectors, 2 x 2 x BN floats

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);    // the producer's arrive.expect_tx
      mbar_init(empty_bar + 8 * s, 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int total_tiles = p.m_tiles * p.n_tiles;
  auto tile_of = [&](int round) -> int {
    return sched_tile(p.sched, round, blockIdx.x, gridDim.x, p.m_tiles, p.n_tiles, 0);
  };

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int round = 0;; ++round) {
        const int tile = tile_of(round);
        if (tile >= total_tiles) break;
        const int m_idx = (tile / p.n_tiles) * GEMM_BLOCK_M, n_idx = (tile % p.n_tiles) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_relaxed_nocall(empty_bar + 8 * stage, phase ^ 1);
          mbar_arrive_expect_tx(full_bar + 8 * stage, (uint32_t)Cfg::STAGE_BYTES);
          tma_load_2d(smem_a + stage * Cfg::A_BYTES, &tmap_a, full_bar + 8 * stage, kb * GEMM_BLOCK_K, m_idx);
          tma_load_2d(smem_b + stage * Cfg::B_BYTES, &tmap_b, full_bar + 8 * stage, kb * GEMM_BLOCK_K, n_idx);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: 64 rows each =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = (threadIdx.x >> 5) & 3;          // warp within the warpgroup: rows 16 cw .. 16 cw + 15
  const int row_in_tile = (wg - 1) * 64 + cw * 16 + (lane >> 2);
  const int col_in_pair = (lane & 3) * 2;
  const uint32_t a_off = (uint32_t)(wg - 1) * 64 * 128;   // this warpgroup's 64 rows of the A stage
  const int ct = threadIdx.x - 128;               // 0 .. 255 over both consumer warpgroups
  const int cols = p.ln_stats != nullptr ? EPI_LN : p.bias != nullptr ? EPI_BIAS : EPI_NONE;
  float* col_smem = reinterpret_cast<float*>(smem_raw + (col_vecs - smem_u32(smem_raw)));   // [2][c | b][BN]
  int stage = 0; uint32_t phase = 0;
  float acc[BN / 2];
  for (int round = 0;; ++round) {
    const int tile = tile_of(round);
    if (tile >= total_tiles) break;
    const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
    const int n0 = nt * BN;
    // MODE 0: fetch what the epilogue reads besides the accumulators while the k-loop runs -- this thread's column of
    // ln_c / ln_b or bias (staged in shared memory after the k-loop), its rows' LayerNorm statistics, and the tile's
    // residual rows into L2
    float col_c = 0.0f, col_b = 0.0f;
    float2 ln_st[2] = {make_float2(0.0f, 1.0f), make_float2(0.0f, 1.0f)};
    if constexpr (MODE == 0) {
      if (ct < BN && n0 + ct < p.N) {
        if (cols == EPI_LN) { col_c = p.ln_c[n0 + ct]; col_b = p.ln_b[n0 + ct]; }
        else if (cols == EPI_BIAS) col_b = __half2float(p.bias[n0 + ct]);
      }
      if (cols == EPI_LN) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = mt * GEMM_BLOCK_M + row_in_tile + 8 * h;
          if (m < p.M) ln_st[h] = p.ln_stats[m];
        }
      }
      const int m = mt * GEMM_BLOCK_M + (ct >> 1);
      if (p.residual != nullptr && m < p.M) {
        const uintptr_t lo = reinterpret_cast<uintptr_t>(p.residual + res_row_of(p, m) * p.ldr + n0);
        const uintptr_t hi = lo + 2 * (uintptr_t)min(BN, p.N - n0);
        for (uintptr_t a = (lo & ~(uintptr_t)127) + (ct & 1) * 128; a < hi; a += 256)
          prefetch_l2(reinterpret_cast<const void*>(a));
      }
    }
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_nocall(full_bar + 8 * stage, phase);
      wgmma_fence();
      const uint64_t adesc = wgmma_desc_sw128(smem_a + stage * Cfg::A_BYTES + a_off);
      const uint64_t bdesc = wgmma_desc_sw128(smem_b + stage * Cfg::B_BYTES);
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)
        wgmma_f16<BN>(acc, adesc + 2 * k, bdesc + 2 * k);   // +32 bytes inside the 128-byte swizzle atom
      wgmma_commit();
      wgmma_wait<1>();                     // the previous k-block's MMAs are done: its stage can be refilled
      if (prev_stage >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      }
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (prev_stage >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
    }

    // ---- epilogue: thread holds rows r, r + 8 and, per 8-column group j, columns 8 j + col_in_pair (+1) ----
    const int m0 = mt * GEMM_BLOCK_M + row_in_tile;
    if constexpr (MODE == 1) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + 8 * h;
        const bool row_ok = m < p.M;
        __half* out_row = p.out + out_row_of(p, m) * p.ldo;
        // SiLU-gate: columns [0,128) of the tile are gates, [128,256) the matching ups.
        // silu(fp16(gate)) rounded to fp16, times fp16(up), rounded (llama_xformer.py:186)
        const int n_limit = p.N / 2;
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          __half o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float g = __half2float(__float2half_rn(acc[4 * j + 2 * h + e]));
            const float u = __half2float(__float2half_rn(acc[4 * (j + BN / 16) + 2 * h + e]));
            const float s = __half2float(__float2half_rn(g * rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * g))));
            o[e] = __float2half_rn(s * u);
          }
          const int n = nt * (BN / 2) + 8 * j + col_in_pair;
          if (row_ok && n < n_limit) store_pair(out_row + n, __halves2half2(o[0], o[1]), n + 1 < n_limit);
        }
      }
    } else {
      // this tile's column vectors: visible to both consumer warpgroups once all 256 threads have stored theirs.
      // Double-buffered by round: a thread writes buffer (round & 1) only after the previous round's barrier, which
      // every reader of that buffer two rounds ago passed after its epilogue.
      float* colv = col_smem + (round & 1) * 2 * BN;
      if (cols != EPI_NONE) {
        if (ct < BN) { colv[ct] = col_c; colv[BN + ct] = col_b; }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      if (cols == EPI_LN) epilogue_tile<BN, EPI_LN>(p, acc, m0, n0, col_in_pair, lane, colv, colv + BN, ln_st);
      else if (cols == EPI_BIAS) epilogue_tile<BN, EPI_BIAS>(p, acc, m0, n0, col_in_pair, lane, colv, colv + BN, ln_st);
      else epilogue_tile<BN, EPI_NONE>(p, acc, m0, n0, col_in_pair, lane, colv, colv + BN, ln_st);
    }
  }
}

// ---- int8 operands (LLM.int8(), seedb200_gemm_int8) ----------------------------------------------------------------
// The same warp-specialised TMA / mbarrier pipeline over int8 rows: a 128-byte swizzled row holds 128 int8 values,
// so a stage is BK = 128 deep with the byte layout of the fp16 kernel's 64-deep stage, and its four 32-byte k-steps
// are wgmma m64nBNk32 s8 x s8 -> s32.  The epilogue dequantises, adds the outlier correction and then applies the
// residual (mode 0) or SiLU-gate (mode 1), with the rounding points of int8.cuh.  The outlier correction is computed
// before it by int8_correction (a dense product over the gathered outlier columns) and read from `corr`.
struct GemmI8Params {
  int M, N, K;
  int m_tiles, n_tiles;
  const float* sca;                    // [M] activation row scales
  const float* scb;                    // [N] weight row scales
  const __half* corr; long long ldc;   // [M,N] outlier corrections (int8_correction), read when there are outliers
  const int* n_outliers;
  const __half* residual; long long ldr;
  __half* out; long long ldo;
};

template <int R>
__device__ __forceinline__ void acc_fence_i(int (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

template <int BN, int MODE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_i8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmI8Params p) {
  using Cfg = GemmCfg<BN>;             // 128 x 128 int8 = 128 x 64 fp16 bytes: the fp16 kernel's stage sizes
  constexpr int STAGES = Cfg::STAGES;
  constexpr int BK = 128;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_a = smem_base;
  const uint32_t smem_b = smem_base + STAGES * Cfg::A_BYTES;
  const uint32_t full_bar = smem_base + STAGES * Cfg::STAGE_BYTES;
  const uint32_t empty_bar = full_bar + STAGES * 8;

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_kb = (p.K + BK - 1) / BK;
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int round = 0;; ++round) {
        const int tile = sched_tile(0, round, blockIdx.x, gridDim.x, p.m_tiles, p.n_tiles, 0);
        if (tile >= total_tiles) break;
        const int m_idx = (tile / p.n_tiles) * GEMM_BLOCK_M, n_idx = (tile % p.n_tiles) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_relaxed_nocall(empty_bar + 8 * stage, phase ^ 1);
          mbar_arrive_expect_tx(full_bar + 8 * stage, (uint32_t)Cfg::STAGE_BYTES);
          tma_load_2d(smem_a + stage * Cfg::A_BYTES, &tmap_a, full_bar + 8 * stage, kb * BK, m_idx);
          tma_load_2d(smem_b + stage * Cfg::B_BYTES, &tmap_b, full_bar + 8 * stage, kb * BK, n_idx);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = (threadIdx.x >> 5) & 3;
  const int row_in_tile = (wg - 1) * 64 + cw * 16 + (lane >> 2);
  const int col_in_pair = (lane & 3) * 2;
  const uint32_t a_off = (uint32_t)(wg - 1) * 64 * 128;
  const int cnt = *p.n_outliers;
  int stage = 0; uint32_t phase = 0;
  int acc[BN / 2];
  for (int round = 0;; ++round) {
    const int tile = sched_tile(0, round, blockIdx.x, gridDim.x, p.m_tiles, p.n_tiles, 0);
    if (tile >= total_tiles) break;
    const int mt = tile / p.n_tiles, nt = tile % p.n_tiles;
    const int n0 = nt * BN;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0;
    int prev_stage = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_nocall(full_bar + 8 * stage, phase);
      wgmma_fence();
      const uint64_t adesc = wgmma_desc_sw128(smem_a + stage * Cfg::A_BYTES + a_off);
      const uint64_t bdesc = wgmma_desc_sw128(smem_b + stage * Cfg::B_BYTES);
#pragma unroll
      for (int k = 0; k < BK / 32; ++k) wgmma_s8<BN>(acc, adesc + 2 * k, bdesc + 2 * k);   // +32 bytes per k-step
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
      }
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence_i(acc);
    if (prev_stage >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar + 8 * prev_stage);
    }

    // ---- epilogue: rows m0, m0 + 8; per 8-column group j the columns 8 j + col_in_pair (+1) of the tile ----
    const int m0 = mt * GEMM_BLOCK_M + row_in_tile;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = m0 + 8 * h;
      if (m >= p.M) continue;
      const float sa = p.sca[m];
      const __half* crow = p.corr + (long long)m * p.ldc;
      __half* orow = p.out + (long long)m * p.ldo;
      if constexpr (MODE == 1) {
        // columns [0,128) of the tile are gates, [128,256) the matching ups
#pragma unroll
        for (int j = 0; j < BN / 16; ++j) {
          __half o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ng = n0 + 8 * j + col_in_pair + e, nu = ng + 128;
            const float sg = p.scb[ng], su = p.scb[nu];
            float g = int8_base(acc[4 * j + 2 * h + e], sa, sg), u = int8_base(acc[4 * (j + BN / 16) + 2 * h + e], sa, su);
            const __half gh = cnt ? int8_add_corr(g, crow[ng]) : __float2half_rn(g);
            const __half uh = cnt ? int8_add_corr(u, crow[nu]) : __float2half_rn(u);
            o[e] = int8_silu_mul(gh, uh);
          }
          const int n = nt * (BN / 2) + 8 * j + col_in_pair;
          store_pair(orow + n, __halves2half2(o[0], o[1]), true);
        }
      } else {
        const __half* rrow = p.residual != nullptr ? p.residual + (long long)m * p.ldr : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int n = n0 + 8 * j + col_in_pair;
          if (n >= p.N) continue;
          __half o[2] = {__float2half_rn(0.0f), __float2half_rn(0.0f)};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (n + e < p.N) {
              const float sb = p.scb[n + e];
              const float b = int8_base(acc[4 * j + 2 * h + e], sa, sb);
              __half y = cnt ? int8_add_corr(b, crow[n + e]) : __float2half_rn(b);
              if (rrow != nullptr) y = __float2half_rn(__half2float(y) + __half2float(rrow[n + e]));
              o[e] = y;
            }
          }
          store_pair(orow + n, __halves2half2(o[0], o[1]), n + 1 < p.N);
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------
int get_option(const char* key);

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// [rows, cols] row-major with leading dimension ld (elements of esize bytes: fp16 by default, int8 for the int8 GEMM);
// box = box_rows x one 128-byte row (64 fp16 or 128 int8 columns), 128B swizzle
static int make_tmap(CUtensorMap* tm, const void* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                     CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16, int esize = 2) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
    return SEEDB200_ERR_CUDA;
  }
  SB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "gemm: operand pointer %p not 16-byte aligned", ptr);
  SB_REQUIRE((ld * esize) % 16 == 0, "gemm: leading dimension %lld (elements) is not a multiple of %d", (long long)ld,
             16 / esize);
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, dtype, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld box_rows=%d)", (int)r,
              (long long)rows, (long long)cols, (long long)ld, box_rows);
    return SEEDB200_ERR_CUDA;
  }
  return 0;
}

// Host side of the persistent schedule: tile grid and units.
struct TileSchedule { int m_tiles, n_tiles, units, sched; };

static TileSchedule make_schedule(int M, int N, int bn, int sched, int sms) {
  TileSchedule t;
  t.m_tiles = (M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
  t.n_tiles = (N + bn - 1) / bn;
  const int tiles = t.m_tiles * t.n_tiles;
  t.units = sms;
  if (t.units > tiles) t.units = tiles;
  if (t.units < 1) t.units = 1;
  t.sched = (sched == 1 && t.n_tiles >= 2) ? 1 : 0;
  return t;
}

template <int BN, int MODE>
static int launch_gemm(const seedb200_gemm_desc& d, cudaStream_t stream, int sched) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set_dev[SB_MAX_DEVICES] = {};   // cudaFuncSetAttribute is per device
  bool& attr_set = attr_set_dev[cur_device()];
  auto kern = gemm_wgmma_kernel<BN, MODE>;
  if (!attr_set) {
    SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  CUtensorMap ta, tb;
  SB_PROPAGATE(make_tmap(&ta, d.A, d.M, d.K, d.lda, GEMM_BLOCK_M));
  SB_PROPAGATE(make_tmap(&tb, d.W, d.N, d.K, d.ldw, BN));
  const TileSchedule ts = make_schedule(d.M, d.N, BN, sched, num_sms());

  GemmParams p;
  p.M = d.M; p.N = d.N; p.K = d.K;
  p.m_tiles = ts.m_tiles;
  p.n_tiles = ts.n_tiles;
  p.bias = static_cast<const __half*>(d.bias);
  p.residual = static_cast<const __half*>(d.residual);
  p.ldr = d.ldr;
  p.out = static_cast<__half*>(d.out);
  p.ldo = d.ldo;
  p.act = d.act;
  p.row_group = d.row_group; p.row_stride = d.row_stride; p.row_offset = d.row_offset;
  p.res_mod = d.res_mod; p.res_offset = d.res_offset;
  p.row_moments = static_cast<float2*>(d.row_moments);
  p.sched = ts.sched;
  p.ln_stats = static_cast<const float2*>(d.ln_stats);
  p.ln_c = static_cast<const float*>(d.ln_c);
  p.ln_b = static_cast<const float*>(d.ln_b);

  profile_mark_begin(0, stream);
  kern<<<ts.units, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, p);
  profile_mark_end(0, stream, 2.0 * (double)d.M * (double)d.N * (double)d.K);
  SB_LAUNCH_CHECK();
  return 0;
}

// Tile width: one that divides N exactly (no half-empty last column), the widest first.
static int pick_bn(int N, int mode) {
  if (mode == 1) return 256;
  if (N % 256 == 0) return 256;
  if (N % 192 == 0) return 192;
  if (N % 176 == 0) return 176;
  if (N % 128 == 0) return 128;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  return 256;
}

// Largest number of output columns any unit of the persistent schedule works through.
static int plan_max_cols(int M, int N, int bn, int sms) {
  const TileSchedule t = make_schedule(M, N, bn, 0, sms);
  const int tiles = t.m_tiles * t.n_tiles;
  int worst = 0;
  for (int u = 0; u < t.units; ++u) {
    int cols = 0;
    for (int round = 0;; ++round) {
      if (sched_tile(0, round, u, t.units, t.m_tiles, t.n_tiles, 0) >= tiles) break;
      cols += bn;
    }
    if (cols > worst) worst = cols;
  }
  return worst;
}

// Short prompts (M <= 256: at most two rows of tiles): with 256-wide tiles N = 5120 gives 40 tiles for 132 SMs;
// 128-wide tiles double the busy SMs at a lower per-tile efficiency.  The score weighs the busiest unit's columns
// against the share of busy SMs (the shapes are half HBM-bound: every W byte is read once).
static int plan_short_prompt(const seedb200_gemm_desc& d, int sms) {
  struct Cand { int bn; double eff; };
  static const Cand cands[] = {{256, 1.00}, {128, 0.80}};
  double best = 1e30;
  int bn = 256;
  for (const Cand& c : cands) {
    const double cost = plan_max_cols(d.M, d.N, c.bn, sms) / c.eff;
    const int tiles = ((d.M + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M) * ((d.N + c.bn - 1) / c.bn);
    const double busy = tiles >= sms ? 1.0 : (double)tiles / sms;
    const double score = cost / (0.5 + 0.5 * busy);
    if (score < best) { best = score; bn = c.bn; }
  }
  return bn;
}

// A leading dimension of 0 means packed rows (K for A and W, the output width for out and the residual), as
// seedb200_gemv's ldo <= 0: a zero-initialised descriptor describes contiguous operands.
static seedb200_gemm_desc with_packed_defaults(seedb200_gemm_desc d) {
  const int n_out = d.mode == 1 ? d.N / 2 : d.N;
  if (d.lda == 0) d.lda = d.K;
  if (d.ldw == 0) d.ldw = d.K;
  if (d.ldo == 0) d.ldo = n_out;
  if (d.ldr == 0) d.ldr = n_out;
  return d;
}

struct GemmPlan { int bn, sched; };
static int choose_plan(const seedb200_gemm_desc& d, int sms, GemmPlan& plan) {
  SB_REQUIRE(d.M > 0 && d.N > 0 && d.K > 0, "gemm: non-positive shape M=%d N=%d K=%d", d.M, d.N, d.K);
  SB_REQUIRE(d.mode == 0 || d.mode == 1, "gemm: unknown mode %d", d.mode);
  SB_REQUIRE(d.K % 8 == 0, "gemm: K=%d must be a multiple of 8 (16-byte TMA rows)", d.K);
  if (d.ln_stats != nullptr) {
    SB_REQUIRE(d.mode == 0 && d.ln_c != nullptr && d.ln_b != nullptr && d.bias == nullptr && d.row_group == 0,
               "gemm: LayerNorm-folded mode takes ln_stats + ln_c + ln_b, no bias (it is inside ln_b), mode 0, no row remap");
  }
  if (d.mode == 1) {
    SB_REQUIRE(d.N % 256 == 0, "gemm: SiLU-gate mode needs N %% 256 == 0 (got %d)", d.N);
    SB_REQUIRE(d.bias == nullptr && d.act == 0 && d.residual == nullptr,
               "gemm: SiLU-gate mode takes no bias/activation/residual");
  }
  // the operand rows are read K wide and the output rows written n_out wide: a shorter leading dimension would make
  // rows overlap
  const int n_out = d.mode == 1 ? d.N / 2 : d.N;
  SB_REQUIRE(d.lda >= d.K && d.ldw >= d.K, "gemm: lda=%lld / ldw=%lld below K=%d", (long long)d.lda,
             (long long)d.ldw, d.K);
  SB_REQUIRE(d.ldo >= n_out, "gemm: ldo=%lld below the %d output columns", (long long)d.ldo, n_out);
  SB_REQUIRE(d.residual == nullptr || d.ldr >= n_out, "gemm: ldr=%lld below the %d output columns",
             (long long)d.ldr, n_out);
  SB_REQUIRE(d.ctas >= 0 && d.ctas <= 2, "gemm: ctas must be 0, 1 or 2 (got %d)", d.ctas);
  if (d.row_moments != nullptr) {
    SB_REQUIRE(d.mode == 0 && d.N % 64 == 0, "gemm: row_moments needs mode 0 and N %% 64 == 0 (N=%d)", d.N);
    if (d.bn != 0 && d.bn % 64 != 0) {
      set_error("gemm: row_moments needs a tile width that is a multiple of 64 (bn=%d)", d.bn);
      return SEEDB200_ERR_UNSUPPORTED;
    }
  }
  int bn = d.bn > 0 ? d.bn : pick_bn(d.N, d.mode);
  // the epilogue moments need whole 64-column groups per tile
  if (d.row_moments != nullptr && d.bn == 0 && bn % 64 != 0) bn = d.N % 128 == 0 ? 128 : 256;
  int sched = 0;
  if (d.bn == 0 && d.mode == 0 && d.N >= 1024 && d.N % 128 == 0 && d.M <= 2 * GEMM_BLOCK_M &&
      get_option("gemm_sched") != 0 && d.ln_stats == nullptr && d.row_moments == nullptr && d.row_group == 0 &&
      d.res_mod == 0) {
    bn = plan_short_prompt(d, sms);
  } else if (d.bn != 0 && get_option("gemm_sched") == 2) {
    sched = 1;                                           // A/B runs with an explicit tile width
  }
  plan.bn = bn; plan.sched = sched;
  return 0;
}

int gemm(const seedb200_gemm_desc& desc, cudaStream_t stream) {
  const seedb200_gemm_desc d = with_packed_defaults(desc);
  GemmPlan plan;
  SB_PROPAGATE(choose_plan(d, num_sms(), plan));
  SB_REQUIRE(d.A && d.W && d.out, "gemm: null operand");
  const int bn = plan.bn, sched = plan.sched;
#define SB_GEMM_CASE(BN_, MD_) \
  if (bn == BN_ && d.mode == MD_) return launch_gemm<BN_, MD_>(d, stream, sched);
  SB_GEMM_CASE(256, 0) SB_GEMM_CASE(192, 0) SB_GEMM_CASE(176, 0) SB_GEMM_CASE(128, 0) SB_GEMM_CASE(64, 0)
  SB_GEMM_CASE(32, 0) SB_GEMM_CASE(256, 1)
#undef SB_GEMM_CASE
  set_error("gemm: unsupported tile configuration bn=%d mode=%d", bn, d.mode);
  return SEEDB200_ERR_UNSUPPORTED;
}

// ---- int8 GEMM host side ----
template <int BN, int MODE>
static int launch_gemm_i8(const seedb200_gemm_int8_desc& d, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set_dev[SB_MAX_DEVICES] = {};
  bool& attr_set = attr_set_dev[cur_device()];
  auto kern = gemm_i8_kernel<BN, MODE>;
  if (!attr_set) {
    SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  CUtensorMap ta, tb;
  SB_PROPAGATE(make_tmap(&ta, d.A, d.M, d.K, d.lda, GEMM_BLOCK_M, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1));
  SB_PROPAGATE(make_tmap(&tb, d.W, d.N, d.K, d.ldw, BN, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1));
  const TileSchedule ts = make_schedule(d.M, d.N, BN, 0, num_sms());
  GemmI8Params p;
  p.M = d.M; p.N = d.N; p.K = d.K;
  p.m_tiles = ts.m_tiles; p.n_tiles = ts.n_tiles;
  p.sca = static_cast<const float*>(d.SCA);
  p.scb = static_cast<const float*>(d.SCB);
  p.corr = static_cast<const __half*>(d.workspace); p.ldc = d.N;
  p.n_outliers = d.n_outliers;
  p.residual = static_cast<const __half*>(d.residual); p.ldr = d.ldr;
  p.out = static_cast<__half*>(d.out); p.ldo = d.ldo;
  kern<<<ts.units, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, p);
  SB_LAUNCH_CHECK();
  return 0;
}

int gemm_int8(const seedb200_gemm_int8_desc& desc, cudaStream_t stream) {
  seedb200_gemm_int8_desc d = desc;
  SB_REQUIRE(d.M > 0 && d.N > 0 && d.K > 0, "gemm_int8: non-positive shape M=%d N=%d K=%d", d.M, d.N, d.K);
  SB_REQUIRE(d.mode == 0 || d.mode == 1, "gemm_int8: unknown mode %d", d.mode);
  SB_REQUIRE(d.K % 16 == 0, "gemm_int8: K=%d must be a multiple of 16 (16-byte TMA rows)", d.K);
  SB_REQUIRE(d.mode == 0 || (d.N % 256 == 0 && d.residual == nullptr),
             "gemm_int8: SiLU-gate mode needs N %% 256 == 0 and no residual");
  const int n_out = d.mode == 1 ? d.N / 2 : d.N;
  if (d.lda == 0) d.lda = d.K;
  if (d.ldw == 0) d.ldw = d.K;
  if (d.lda16 == 0) d.lda16 = d.K;
  if (d.ldo == 0) d.ldo = n_out;
  if (d.ldr == 0) d.ldr = n_out;
  SB_REQUIRE(d.lda >= d.K && d.ldw >= d.K && d.lda16 >= d.K, "gemm_int8: a leading dimension is below K=%d", d.K);
  SB_REQUIRE(d.ldo >= n_out && (d.residual == nullptr || d.ldr >= n_out),
             "gemm_int8: ldo / ldr below the %d output columns", n_out);
  SB_REQUIRE(d.A && d.SCA && d.A16 && d.outliers && d.n_outliers && d.W && d.SCB && d.out && d.workspace,
             "gemm_int8: null operand");
  int bn = d.bn;
  if (bn == 0) bn = d.mode == 1 ? 256 : d.N % 256 == 0 ? 256 : d.N <= 64 ? 64 : 128;
  SB_REQUIRE(d.mode == 0 || bn == 256, "gemm_int8: SiLU-gate mode needs bn 256");
  SB_REQUIRE(bn == 256 || bn == 128 || bn == 64, "gemm_int8: unsupported tile width bn=%d (64, 128 or 256)", bn);
  SB_PROPAGATE(int8_correction(d.A16, d.lda16, d.W, d.ldw, d.SCB, d.outliers, d.n_outliers, d.M, d.N, d.workspace,
                               stream));
  if (bn == 256 && d.mode == 1) return launch_gemm_i8<256, 1>(d, stream);
  if (bn == 256) return launch_gemm_i8<256, 0>(d, stream);
  if (bn == 128) return launch_gemm_i8<128, 0>(d, stream);
  if (bn == 64) return launch_gemm_i8<64, 0>(d, stream);
  set_error("gemm_int8: unsupported tile width bn=%d (64, 128 or 256)", bn);
  return SEEDB200_ERR_UNSUPPORTED;
}

}  // namespace sb

extern "C" int seedb200_gemm_int8(const seedb200_gemm_int8_desc* d, void* stream) {
  if (d == nullptr) {
    sb::set_error("seedb200_gemm_int8: null descriptor");
    return SEEDB200_ERR_INVALID;
  }
  return sb::gemm_int8(*d, static_cast<cudaStream_t>(stream));
}

extern "C" int seedb200_gemm_plan(const seedb200_gemm_desc* d, int sms, int32_t* out9) {
  if (d == nullptr || out9 == nullptr || sms <= 0) {
    sb::set_error("seedb200_gemm_plan: null argument or sms <= 0");
    return SEEDB200_ERR_INVALID;
  }
  sb::GemmPlan plan;
  SB_PROPAGATE(sb::choose_plan(sb::with_packed_defaults(*d), sms, plan));
  const sb::TileSchedule t = sb::make_schedule(d->M, d->N, plan.bn, plan.sched, sms);
  const int32_t v[9] = {plan.bn, 1, t.sched, 1, t.m_tiles, t.n_tiles, t.units, 0, 0};
  for (int i = 0; i < 9; ++i) out9[i] = v[i];
  return 0;
}

extern "C" int seedb200_gemm_schedule_tile(int sched, int round, int unit, int units, int m_tiles, int n_tiles,
                                           int tile_shift) {
  return sb::sched_tile(sched, round, unit, units, m_tiles, n_tiles, tile_shift);
}

extern "C" int seedb200_gemm(const seedb200_gemm_desc* d, void* stream) {
  if (d == nullptr) {
    sb::set_error("seedb200_gemm: null descriptor");
    return SEEDB200_ERR_INVALID;
  }
  return sb::gemm(*d, static_cast<cudaStream_t>(stream));
}
