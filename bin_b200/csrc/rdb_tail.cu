// bin_b200 -- fused tail of a residual dense block of width G0 (64 or 96) for sm_90a:
//   g3 = ReLU(conv3x3(cat(x, g0, g1, g2)))        RDN.py:141-147 (RDB_Conv, the 4th of RDN.py:156-160)
//   x' = LFF(cat(x, g0, g1, g2, g3)) + x          RDN.py:162-165 (1x1 conv G0+128 -> G0, local residual)
// in ONE kernel.  Layer by layer these two move 448 + 832 bytes per position through HBM at G0 = 96; fused, the G0+96
// input channels are fetched once (the 1x1 LFF reads the centre of the very halo tile the 3x3 conv already has in shared
// memory), g3 never leaves the SM, and only x' is written: 768 bytes per position at G0 = 96.
//
// GEMM view per 128-pixel tile (4 rows x 32-pixel smem pitch, 30 valid columns) and 32-channel chunk c (G0/32 chunks of
// x, then the three of g0..g2):
//   conv accumulator  (128 x 96, the three kx taps stacked in N as in conv_igemm.cu)  += A(ky) * Wc[c][ky],  ky = 0..2
//   LFF accumulator   (128 x G0)                                                      += A(centre) * Wl[c]
// then the conv accumulator's kx column groups are added (xstack_sum), bias + ReLU applied, g3 written as a
// K-major fp16 operand into shared memory, and ONE more K = 32 step  LFF accumulator += g3 * Wl[last]  finishes x'.
// The accumulation order per accumulator is that of conv_igemm_kernel (chunk, ky, k16 step), so the fused and the
// layer-by-layer results are bit-identical.  All weights (150 KB at G0 = 96, 114 KB at 64) stay resident in shared
// memory; the activation ring takes what they leave (5 stages at G0 = 96, 8 at 64).
//
// Roles (384 threads, 1 CTA/SM, persistent):
//   warp 0 lane 0 : TMA producer (weights once, then one activation chunk per ring slot)
//   warpgroup 1+m : tile rows [64 m, 64 m + 64): both accumulators in registers, the g3 rows, the x' stores
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"
#include "xstack.cuh"

namespace binb {

constexpr int kRtTH = 4;                               // output rows per tile (128 GEMM rows)
constexpr int kRtRows = kRtTH + 2;                     // + 3x3 halo
constexpr int kRtTW = kTWH - 2;                        // valid output columns per tile
constexpr int kRtAPlane = kRtRows * kTWH * 16;         // bytes of one 8-channel plane of a stage
constexpr int kRtABytes = kKPL * kRtAPlane;            // 12 288
constexpr int kRtN = 96;                               // N of the conv's wgmmas (3 kx x 32 conv channels)
constexpr int kRtSlab = kKPL * kRtN * 16;              // conv slab [4 planes][96 rows][16 B] = 6 144
constexpr int kRtHPlane = 128 * 16;
constexpr int kRtHBytes = kKPL * kRtHPlane;            // g3 tile: [4 planes][128 pixels][16 B]
constexpr int kRtXsBytes = 4 * kXsFloats<32> * 4;      // xstack_sum buffers of the 4 consumer warp pairs
constexpr int kRtCtrl = 1024;                          // barriers (512 B) and the two bias vectors (512 B)
static_assert(kRtABytes % 128 == 0, "TMA destinations must be 128-byte aligned");

// Geometry of the tail of a G0-wide block.  The LFF's wgmmas have N = G0.
template <int G0>
struct RtCfg {
  static_assert(G0 == 64 || G0 == 96, "rdb_tail: G0 is 64 or 96");
  static constexpr int XChunks = G0 / 32;                        // 32-channel chunks of x
  static constexpr int Chunks = XChunks + 3;                     // input chunks of the conv: x, g0, g1, g2
  static constexpr int LSlab = kKPL * G0 * 16;                   // LFF slab [4 planes][G0 rows][16 B]
  static constexpr int WChunk = 3 * kRtSlab + LSlab;             // conv ky = 0,1,2 + LFF slab of the chunk
  static constexpr int WBytes = Chunks * WChunk + LSlab;         // + the LFF slab of the g3 channels
  // the activation ring takes all shared memory the resident weights, the g3 tile and the exchange buffers leave
  static constexpr int Stages = (kSmemMax - kRtCtrl - WBytes - kRtHBytes - kRtXsBytes) / kRtABytes;
  static constexpr int Smem = kRtCtrl + WBytes + kRtHBytes + Stages * kRtABytes + kRtXsBytes;
  static_assert(Stages >= 2 && Smem <= kSmemMax, "rdb_tail shared memory");
  static_assert((kRtCtrl + WBytes + kRtHBytes) % 128 == 0, "TMA destinations must be 128-byte aligned");
  static_assert(32 + G0 <= 128, "the two bias vectors share 512 bytes");
};

struct alignas(64) RdbTailParams {
  CUtensorMap tmap0, tmap1;             // x planes, growth planes
  int plane0_0, plane0_1;
  const uint8_t* w_conv;                // conv_igemm SX pack: [chunk][ky][4][kx*32+co][8]
  const uint8_t* w_lff;                 // conv_igemm 1x1 pack: [chunk][4][co][8]
  const float* b_conv;
  const float* b_lff;
  int H, W;
  int b0, y0, ny;
  int tiles_x, tiles_y, ntiles;
  __half* out; int out_planes, out_plane0;
};

template <int G0>
struct RtCtrl {
  uint64_t full[RtCfg<G0>::Stages], empty[RtCfg<G0>::Stages];
  uint64_t wfull[RtCfg<G0>::Chunks + 1];
};
static_assert(sizeof(RtCtrl<96>) <= 512 && sizeof(RtCtrl<64>) <= 512, "ctrl block");

template <int G0>
__global__ void __launch_bounds__(384, 1) rdb_tail_kernel(const __grid_constant__ RdbTailParams p) {
  using Cf = RtCfg<G0>;
  constexpr int kRtChunks = Cf::Chunks, kRtStages = Cf::Stages, kRtWChunk = Cf::WChunk, kRtWBytes = Cf::WBytes;
  constexpr int kLSlab = Cf::LSlab;
  extern __shared__ __align__(1024) uint8_t smem[];
  RtCtrl<G0>* ctrl = reinterpret_cast<RtCtrl<G0>*>(smem);
  float* sb_conv = reinterpret_cast<float*>(smem + 512);           // 32 floats
  float* sb_lff = sb_conv + 32;                                    // G0 floats
  uint8_t* res_w = smem + kRtCtrl;
  uint8_t* htile = res_w + kRtWBytes;
  uint8_t* stage0 = htile + kRtHBytes;                            // TMA destinations: 128-byte aligned
  float* xs0 = reinterpret_cast<float*>(stage0 + kRtStages * kRtABytes);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  auto tile_of = [&](int tq, int& txi, int& tyi, int& b) {
    int t = tq;
    txi = t % p.tiles_x; t /= p.tiles_x;
    tyi = t % p.tiles_y;
    b = p.b0 + t / p.tiles_y;
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmap0);
    tma_prefetch_desc(&p.tmap1);
    for (int i = 0; i < kRtStages; ++i) { mbar_init(&ctrl->full[i], 1); mbar_init(&ctrl->empty[i], 8); }
    for (int i = 0; i <= kRtChunks; ++i) mbar_init(&ctrl->wfull[i], 1);
    fence_barrier_init();
  }
  if (threadIdx.x < 32) sb_conv[threadIdx.x] = p.b_conv[threadIdx.x];
  else if (threadIdx.x < 32 + G0) sb_lff[threadIdx.x - 32] = p.b_lff[threadIdx.x - 32];
  __syncthreads();

  if (warp == 0) {
    if (lane != 0) return;
    // ========================================================== TMA producer
    for (int c = 0; c < kRtChunks; ++c) {
      mbar_expect_tx(&ctrl->wfull[c], kRtWChunk);
      bulk_load_1d(res_w + c * kRtWChunk, p.w_conv + (size_t)c * 3 * kRtSlab, 3 * kRtSlab, &ctrl->wfull[c]);
      bulk_load_1d(res_w + c * kRtWChunk + 3 * kRtSlab, p.w_lff + (size_t)c * kLSlab, kLSlab, &ctrl->wfull[c]);
    }
    mbar_expect_tx(&ctrl->wfull[kRtChunks], kLSlab);
    bulk_load_1d(res_w + kRtChunks * kRtWChunk, p.w_lff + (size_t)kRtChunks * kLSlab, kLSlab, &ctrl->wfull[kRtChunks]);
    uint32_t s = 0, ph = 0;
    for (int tq = blockIdx.x; tq < p.ntiles; tq += gridDim.x) {
      int txi, tyi, b;
      tile_of(tq, txi, tyi, b);
      const int x0 = txi * kRtTW - 1, y0 = p.y0 + tyi * kRtTH - 1;
      for (int c = 0; c < kRtChunks; ++c) {
        mbar_wait(&ctrl->empty[s], ph ^ 1);
        mbar_expect_tx(&ctrl->full[s], kRtABytes);
        const bool seg1 = c >= Cf::XChunks;
        tma_load_4d(stage0 + (size_t)s * kRtABytes, seg1 ? (const void*)&p.tmap1 : (const void*)&p.tmap0, &ctrl->full[s],
                    x0 * 8, y0, seg1 ? p.plane0_1 + (c - Cf::XChunks) * kKPL : p.plane0_0 + c * kKPL, b);
        if (++s == kRtStages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  if (warp < 4) return;

  // ============================================================ consumer warpgroups
  const int m = (warp - 4) >> 2;                 // tile rows [64 m, 64 m + 64)
  const int wq = warp & 3;
  const int k4 = lane & 3;
  float* xs = xs0 + (2 * m + (wq >> 1)) * kXsFloats<32>;
  const int xs_bar = 3 + 2 * m + (wq >> 1);      // named barrier of the warp pair (1, 2: wg_sync)
  float acc_c[kRtN / 2], acc_l[G0 / 2];          // fragment: [4 i + 2 h + e] = row 16 wq + lane/4 + 8 h, column 8 i + 2 k4 + e
  // residual x of this thread's pixels (rows 16 wq + lane/4 + 8 h), channels 8 i + 2 k4, +1: the centre of x chunks
  // 0..2, read from their ring slots while the LFF consumes them (the bytes the TMA copied from x, so x' is unchanged)
  uint32_t res[2][G0 / 8];
  const uint32_t res_off = (uint32_t)(m * 64 + wq * 16 + (lane >> 2) + kTWH + 1) * 16 + 4 * k4;
  uint32_t s = 0, ph = 0;
  for (int tq = blockIdx.x; tq < p.ntiles; tq += gridDim.x) {
    int prev = -1;
#pragma unroll
    for (int c = 0; c < kRtChunks; ++c) {
      mbar_wait(&ctrl->full[s], ph);
      if (tq == (int)blockIdx.x) mbar_wait(&ctrl->wfull[c], 0);
      const uint32_t a_base = smem_u32(stage0 + (size_t)s * kRtABytes) + m * 64 * 16;
      const uint32_t b_base = smem_u32(res_w + c * kRtWChunk);
      const uint32_t first = c == 0 ? 0u : 1u;
      wgmma_fence();
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {                               // conv: A shifted by ky rows, B = slab ky
#pragma unroll
        for (int jj = 0; jj < kKC / 16; ++jj)
          Wgmma<kRtN>::mma(acc_c, gmma_desc(a_base + ky * kTWH * 16 + jj * 2 * kRtAPlane, kRtAPlane, 128),
                           gmma_desc(b_base + ky * kRtSlab + jj * 2 * kRtN * 16, kRtN * 16, 128),
                           (jj == 0 && ky == 0) ? first : 1u);
      }
#pragma unroll
      for (int jj = 0; jj < kKC / 16; ++jj)                          // LFF: centre row, +1 pixel, B = slab 3
        Wgmma<G0>::mma(acc_l, gmma_desc(a_base + (kTWH + 1) * 16 + jj * 2 * kRtAPlane, kRtAPlane, 128),
                       gmma_desc(b_base + 3 * kRtSlab + jj * 2 * G0 * 16, G0 * 16, 128), jj == 0 ? first : 1u);
      if (c < Cf::XChunks) {                                           // x chunk: keep this thread's residual values
        const uint8_t* st = stage0 + (size_t)s * kRtABytes + res_off;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int q = 0; q < kKPL; ++q)
            res[h][kKPL * c + q] = *reinterpret_cast<const uint32_t*>(st + h * 8 * 16 + q * kRtAPlane);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&ctrl->empty[prev]);
      prev = (int)s;
      if (++s == kRtStages) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc_c);
    acc_fence(acc_l);
    if (lane == 0) mbar_arrive(&ctrl->empty[prev]);

    // ---------------------------------------------------------- this thread's pixels
    int txi, tyi, b;
    tile_of(tq, txi, tyi, b);
    bool valid[2];
    int y[2], x[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int L = m * 64 + wq * 16 + (lane >> 2) + 8 * h;
      y[h] = p.y0 + tyi * kRtTH + (L >> 5);
      x[h] = txi * kRtTW + (L & 31);
      valid[h] = (L & 31) < kRtTW && y[h] < p.y0 + p.ny && x[h] < p.W;
    }

    // ---------------------------------------------------------- g3 = ReLU(D0[p] + D1[p+1] + D2[p+2] + b) -> smem
    xstack_sum<32>(acc_c, xs, xs_bar);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wq * 16 + (lane >> 2) + 8 * h;
      uint8_t* hrow = htile + (m * 64 + r) * 16 + 4 * k4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float f[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) f[e] = fmaxf(acc_c[4 * i + 2 * h + e] + sb_conv[8 * i + 2 * k4 + e], 0.f);
        *reinterpret_cast<uint32_t*>(hrow + i * kRtHPlane) = pack_h2(f[0], f[1]);
      }
    }
    fence_proxy_async();                                             // generic-proxy stores -> visible to wgmma
    wg_sync(1 + m);

    // ---------------------------------------------------------- LFF += g3 * Wl[6]
    if (tq == (int)blockIdx.x) mbar_wait(&ctrl->wfull[kRtChunks], 0);
    wgmma_fence();
    {
      const uint32_t h_base = smem_u32(htile) + m * 64 * 16;
      const uint32_t b_base = smem_u32(res_w + kRtChunks * kRtWChunk);
#pragma unroll
      for (int jj = 0; jj < kKC / 16; ++jj)
        Wgmma<G0>::mma(acc_l, gmma_desc(h_base + jj * 2 * kRtHPlane, kRtHPlane, 128),
                       gmma_desc(b_base + jj * 2 * G0 * 16, G0 * 16, 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence(acc_l);

    // ---------------------------------------------------------- x' = LFF + b + x
    const size_t plane = (size_t)p.H * p.W * 8;                     // halves per P8 plane
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (valid[h]) {
        // the pixel's offset once, then one plane stride per plane
        __half* dst = p.out + ((((size_t)b * p.out_planes + p.out_plane0) * p.H + y[h]) * p.W + x[h]) * 8 + 2 * k4;
#pragma unroll
        for (int i = 0; i < G0 / 8; ++i) {
          const int n = 8 * i + 2 * k4;
          const float2 g = unpack_h2(res[h][i]);
          *reinterpret_cast<uint32_t*>(dst + (size_t)i * plane) =
              pack_h2((acc_l[4 * i + 2 * h] + sb_lff[n]) + g.x, (acc_l[4 * i + 2 * h + 1] + sb_lff[n + 1]) + g.y);
        }
      }
    }
    wg_sync(1 + m);                                                  // htile / xs are rewritten by the next tile
  }
}

// ------------------------------------------------------------------ host side
template <int G0>
static int launch_rdb_tail_g(RdbTailParams& p, const bin_act_t& x, const bin_act_t& g, cudaStream_t s) {
  BIN_TRY(make_p8_tmap(&p.tmap0, x, kTWH, kRtRows, kKPL));    // every argument is checked before the first tensor map
  BIN_TRY(make_p8_tmap(&p.tmap1, g, kTWH, kRtRows, kKPL));
  static std::atomic<unsigned long long> opted{0};   // per instantiation, per device
  BIN_TRY(ensure_dynamic_smem(rdb_tail_kernel<G0>, RtCfg<G0>::Smem, opted));
  const int sms = num_sms();
  const int grid = p.ntiles < sms ? p.ntiles : sms;
  rdb_tail_kernel<G0><<<grid, 384, RtCfg<G0>::Smem, s>>>(p);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

int launch_rdb_tail(int g0, const bin_act_t& x, int x_plane0, const bin_act_t& g, int g_plane0, const void* w_conv,
                    const float* b_conv, const void* w_lff, const float* b_lff, const bin_act_t& out, int out_plane0,
                    int b_begin, int b_count, int y_begin, int y_count, cudaStream_t s) {
  if (g0 != 64 && g0 != 96) return fail(BIN_ERR_ARG, "rdb_tail: G0 must be 64 or 96");
  const int H = x.H, W = x.W, B = x.B, P = g0 / 8;
  if (g.H != H || g.W != W || g.B != B || out.H != H || out.W != W || out.B != B)
    return fail(BIN_ERR_ARG, "rdb_tail: tensor geometry mismatch");
  if (x_plane0 < 0 || g_plane0 < 0 || out_plane0 < 0 || x_plane0 + P > x.planes || g_plane0 + 12 > g.planes ||
      out_plane0 + P > out.planes)
    return fail(BIN_ERR_ARG, "rdb_tail: plane range exceeds tensor");
  RdbTailParams p;
  memset(&p, 0, sizeof(p));
  p.plane0_0 = x_plane0; p.plane0_1 = g_plane0;
  p.w_conv = reinterpret_cast<const uint8_t*>(w_conv); p.w_lff = reinterpret_cast<const uint8_t*>(w_lff);
  p.b_conv = b_conv; p.b_lff = b_lff;
  p.H = H; p.W = W;
  p.b0 = b_begin; p.y0 = y_begin;
  const int nb = b_count > 0 ? b_count : B - b_begin;
  p.ny = y_count > 0 ? y_count : H - y_begin;
  if (p.b0 < 0 || p.y0 < 0 || nb < 1 || p.ny < 1 || p.b0 + nb > B || p.y0 + p.ny > H)
    return fail(BIN_ERR_ARG, "rdb_tail: batch/row sub-range outside the tensor");
  if (!x.ptr || !g.ptr || !out.ptr || !w_conv || !b_conv || !w_lff || !b_lff) return fail(BIN_ERR_ARG, "rdb_tail_fwd: null argument");
  p.tiles_x = (W + kRtTW - 1) / kRtTW;
  p.tiles_y = (p.ny + kRtTH - 1) / kRtTH;
  p.ntiles = nb * p.tiles_x * p.tiles_y;
  p.out = reinterpret_cast<__half*>(out.ptr); p.out_planes = out.planes; p.out_plane0 = out_plane0;
  return g0 == 96 ? launch_rdb_tail_g<96>(p, x, g, s) : launch_rdb_tail_g<64>(p, x, g, s);
}

}  // namespace binb
