// bin_b200 -- epilogue of the x-stacked 3x3 convs (conv_igemm.cu SX path, rdb_tail.cu).
// The three kx taps of such a conv are GEMM columns: a 64 x 3NT wgmma accumulator block holds D_kx[r][c] in column
// kx NT + c, and the conv output of pixel (GEMM row) r is  out[r] = (D0[r] + D1[r+1]) + D2[r+2].
// Fragment: acc[4 i + 2 h + e] = row 16 wq + lane/4 + 8 h, column 8 i + 2 k4 + e (wq = warp in the warpgroup, k4 = lane & 3).
// Rows r+1 and r+2 are in the same warp (lane + 4, lane + 8, or the other h half) except rows 16 and 17 of each 32-row
// group, which the odd warp of the pair (wq = 1, 3) holds; only those go through shared memory.  Rows r with r % 32 >= 30
// are the tile's junk columns and come out with unspecified values; no valid row reads past its 32-row group.
#pragma once
#include "common.cuh"

namespace binb {

template <int NT>
constexpr int kXsFloats = 3 * NT;   // exchange buffer of one warp pair: D1 row 16, D2 rows 16 and 17

// Overwrites the D0 group acc[0, NT/2) with out.  Both warps of the pair call it with the same `xs` and `bar_id`
// (a named barrier over their 64 threads).  A caller that reuses `xs` for the next exchange must order it after the
// even warp's reads: another barrier the pair both passes in between, or a second buffer.
template <int NT>
__device__ __forceinline__ void xstack_sum(float (&acc)[3 * NT / 2], float* xs, int bar_id) {
  const int lane = threadIdx.x & 31, g = lane >> 2, k4 = lane & 3;
  constexpr int I1 = NT / 8, I2 = 2 * NT / 8;     // first fragment column block of D1, D2
  if (((threadIdx.x >> 5) & 1) && g < 2) {        // odd warp, rows 0 and 1 (= rows 16, 17 of the 32-row group)
#pragma unroll
    for (int i = 0; i < NT / 8; ++i) {
      const int col = 8 * i + 2 * k4;
      if (g == 0) *reinterpret_cast<float2*>(xs + col) = make_float2(acc[4 * (I1 + i)], acc[4 * (I1 + i) + 1]);
      *reinterpret_cast<float2*>(xs + NT * (1 + g) + col) = make_float2(acc[4 * (I2 + i)], acc[4 * (I2 + i) + 1]);
    }
  }
  asm volatile("bar.sync %0, 64;" ::"r"(bar_id) : "memory");
  const int src1 = (lane + 4) & 31, src2 = (lane + 8) & 31;
#pragma unroll
  for (int i = 0; i < NT / 8; ++i)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = 8 * i + 2 * k4 + e;
      const float a1 = __shfl_sync(0xffffffffu, acc[4 * (I1 + i) + e], src1);       // D1 of lane + 4, h = 0
      const float b1 = __shfl_sync(0xffffffffu, acc[4 * (I1 + i) + 2 + e], src1);   // D1 of lane + 4, h = 1
      const float a2 = __shfl_sync(0xffffffffu, acc[4 * (I2 + i) + e], src2);       // D2 of lane + 8, h = 0
      const float b2 = __shfl_sync(0xffffffffu, acc[4 * (I2 + i) + 2 + e], src2);   // D2 of lane + 8, h = 1
      // lane + 4 wraps from row 7 to row 8 (h = 1 of lane - 28), lane + 8 from rows 6, 7 to rows 8, 9
      const float x1h0 = g < 7 ? a1 : b1, x1h1 = g < 7 ? b1 : xs[col];
      const float x2h0 = g < 6 ? a2 : b2, x2h1 = g < 6 ? b2 : xs[NT * (g - 5) + col];
      acc[4 * i + e] = (acc[4 * i + e] + x1h0) + x2h0;
      acc[4 * i + 2 + e] = (acc[4 * i + 2 + e] + x1h1) + x2h1;
    }
}

}  // namespace binb
