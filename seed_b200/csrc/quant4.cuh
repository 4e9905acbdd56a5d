// quant4.cuh -- the bitsandbytes 4-bit weight formats (FP4 / NF4, blocks of 64, include/seedb200.h) shared by the
// quantiser / dequantiser (quant4.cu) and the 4-bit GEMV (misc.cu).
#pragma once

#include "common.cuh"

namespace sb {

constexpr int Q4_BLOCK = 64;

// dequantisation value of code c (0..15) per quant type (SEEDB200_Q4_FP4, SEEDB200_Q4_NF4): bitsandbytes'
// dDequantizeFP4Tree (bit 8 = sign) and dDequantizeNF4, as fp32 constants
static __constant__ float kQ4Value[2][16] = {
    {0.0f, 0.005208333333f, 0.66666667f, 1.0f, 0.33333333f, 0.5f, 0.16666667f, 0.25f,
     -0.0f, -0.005208333333f, -0.66666667f, -1.0f, -0.33333333f, -0.5f, -0.16666667f, -0.25f},
    {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,
     -0.18477343022823334f, -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f,
     0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f,
     1.0f}};

// W' of one packed group of 8 weights (4 bytes, the even-index element in the high nibble): fp16_rn(value * absmax)
// per element, in element order, as 8 halves in a uint4 (the fp16 GEMV's 16-byte vector).  tab: kQ4Value[type] in
// shared memory (a code-indexed local array would live in local memory).
__device__ __forceinline__ uint4 q4_deq8(uint32_t p, float absmax, const float* tab) {
  uint4 o;
  uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const uint32_t byte = (p >> (8 * b)) & 0xffu;
    const __half e0 = __float2half_rn(__fmul_rn(tab[byte >> 4], absmax));     // element 2b
    const __half e1 = __float2half_rn(__fmul_rn(tab[byte & 15u], absmax));    // element 2b + 1
    ow[b] = (uint32_t)__half_as_ushort(e0) | ((uint32_t)__half_as_ushort(e1) << 16);
  }
  return o;
}

}  // namespace sb
