// bin_b200 -- weight-gradient GEMM for sm_90a (wgmma with MN-major operands).
//
// dW[co][ci][ky][kx] += (1/scale) * sum_{b,y,x} dY[b,co,y,x] * X[b,ci,y+ky-pad,x+kx-pad]
// (the wgrad of every nn.Conv2d of RDN.py; autograd of bin_model.optimize_parameters, bin_model.py:130-141).
//
// GEMM view: D_tap[ci][co] = sum_pixels X_tap[pixel][ci] * dY[pixel][co], i.e. M = Cin tile (128),
// N = Cout, K = pixels.  P8 tiles in shared memory ([plane][row][px][8 ch]) are exactly the canonical
// MN-major / no-swizzle wgmma layout with K = pixel index: 8 channels contiguous (16 B), 8 consecutive
// pixels 16 B apart (one 128-byte core matrix), next 8-pixel group +128 B (LBO), next 8-channel plane
// +plane stride (SBO).  A tap is again a 16-byte start-address shift of the X halo tile.
// One wgmma = 64(ci) x N(co) x 16 pixels (one 16-pixel tile row); each of the two consumer warpgroups keeps one
// register accumulator per tap for its 64 input channels (taps x N <= 256 columns; wider layers run several tap
// groups), walks a slice of the pixel tiles, and finally writes its partial sums into a per-CTA slab.
// SX mode (the Cout=32 RDB convs): dW[ky][kx] = sum_p' dY[p'-(kx-1)] X[p'+(ky-1)*row], so the three kx taps
// share the SAME X operand when dY is shifted instead: the dY tile is loaded three times at x offsets
// +1, 0, -1 into consecutive plane groups and becomes one N = 96 operand (8 rows x 3 ky = 24 wgmma per tile
// instead of 72 with N = 32).
#include <stdio.h>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"

namespace binb {

constexpr int kWgTW = 16, kWgTH = 8;      // pixel tile: 8 rows x 16 px (K = 16 px per MMA)

struct alignas(64) WgradParams {
  CUtensorMap xmap0, xmap1, ymap;
  int x0_plane0, x0_planes, x1_plane0, x1_planes;   // Cin segments (planes of 8 channels)
  int ci_tile_plane0;                               // first logical input plane of this launch's 128-channel tile
  int dy_plane0, n;                                 // N = cout padded to 16
  int ks, pad, pw, rows;                            // X tile pitch (px) and rows incl. halo
  int tap0, ntaps;                                  // tap group handled by this launch
  int sx;                                           // 3x3 / Cout=32: the 3 kx taps stacked into N (see below)
  int cout, cin;                                    // real sizes (flush bounds)
  int B, H, W, tiles_x, tiles_y, ntiles;
  int nstages;
  const float* scale;
  float* dw;
  float* partial;                                   // [gridDim.x][ntaps][128][n] fp32 per-CTA partial sums
};

struct WgCtrl {
  uint64_t full[4], empty[4];
};

template <int N>
struct WgCfg {
  static constexpr int TAPS = 256 / N;               // accumulators per thread: TAPS x N / 2 <= 128 registers
};

// Roles (384 threads, 1 CTA/SM): warp 0 lane 0 = TMA producer; warpgroup 1+m = input channels [64 m, 64 m + 64).
template <int N>
__global__ void __launch_bounds__(384, 1) wgrad_kernel(const __grid_constant__ WgradParams p) {
  constexpr int TAPS = WgCfg<N>::TAPS;
  extern __shared__ __align__(1024) uint8_t smem[];
  WgCtrl* ctrl = reinterpret_cast<WgCtrl*>(smem);
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int x_plane_bytes = p.rows * p.pw * 16;
  const int x_bytes = 16 * x_plane_bytes;                       // 16 planes = 128 input channels
  const int y_planes = N / 8;                                   // SX: 3 shifted copies of the 4 dY planes
  const int y_plane_bytes = kWgTH * kWgTW * 16;
  const int y_bytes = y_planes * y_plane_bytes;
  const int stage_bytes = x_bytes + y_bytes;
  uint8_t* stage0 = smem + 1024;
  const uint32_t S = p.nstages;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.xmap0);
    if (p.x1_planes > 0) tma_prefetch_desc(&p.xmap1);
    tma_prefetch_desc(&p.ymap);
    for (int i = 0; i < 4; ++i) { mbar_init(&ctrl->full[i], 1); mbar_init(&ctrl->empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane != 0) return;
    // ------------------------------------------------ TMA producer
    uint32_t s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      int t = tile;
      const int txi = t % p.tiles_x; t /= p.tiles_x;
      const int tyi = t % p.tiles_y;
      const int b = t / p.tiles_y;
      mbar_wait(&ctrl->empty[s], ph ^ 1);
      uint8_t* dst = stage0 + (size_t)s * stage_bytes;
      // the X tile is assembled from 4-plane boxes; planes past the conv's Cin are zero-filled by hand-off
      // to TMA's out-of-bounds fill (coordinates beyond the tensor) or skipped (rows ignored at the flush)
      int nbox = 0;
      for (int q = 0; q < 4; ++q) {
        const int lp = p.ci_tile_plane0 + 4 * q;               // logical input plane
        if (lp < p.x0_planes + p.x1_planes) ++nbox;
      }
      mbar_expect_tx(&ctrl->full[s], (uint32_t)(nbox * 4 * x_plane_bytes + y_bytes));
      for (int q = 0; q < 4; ++q) {
        const int lp = p.ci_tile_plane0 + 4 * q;
        if (lp >= p.x0_planes + p.x1_planes) continue;
        const bool seg1 = lp >= p.x0_planes;
        const void* tmap = seg1 ? (const void*)&p.xmap1 : (const void*)&p.xmap0;
        const int plane = seg1 ? p.x1_plane0 + (lp - p.x0_planes) : p.x0_plane0 + lp;
        tma_load_4d(dst + (size_t)q * 4 * x_plane_bytes, tmap, &ctrl->full[s], (txi * kWgTW - (p.sx ? 0 : p.pad)) * 8,
                    tyi * kWgTH - p.pad, plane, b);
      }
      if (p.sx) {
        for (int kx = 0; kx < 3; ++kx)
          tma_load_4d(dst + x_bytes + kx * 4 * y_plane_bytes, &p.ymap, &ctrl->full[s], (txi * kWgTW + 1 - kx) * 8,
                      tyi * kWgTH, p.dy_plane0, b);
      } else {
        tma_load_4d(dst + x_bytes, &p.ymap, &ctrl->full[s], txi * kWgTW * 8, tyi * kWgTH, p.dy_plane0, b);
      }
      if (++s == S) { s = 0; ph ^= 1; }
    }
    return;
  }
  if (warp < 4) return;
  // ------------------------------------------------ consumers: D_tap[ci][co] += X_tap^T * dY
  const int m = (warp - 4) >> 2, wq = warp & 3, k4 = lane & 3;
  float acc[TAPS][N / 2];
  uint32_t s = 0, ph = 0;
  int prev = -1;
  bool first = true;
  for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
    mbar_wait(&ctrl->full[s], ph);
    const uint32_t xb = smem_u32(stage0 + (size_t)s * stage_bytes) + m * 8 * x_plane_bytes;
    const uint32_t yb = smem_u32(stage0 + (size_t)s * stage_bytes) + x_bytes;
    wgmma_fence();
#pragma unroll
    for (int tp = 0; tp < TAPS; ++tp) {
      if (tp >= p.ntaps) break;
      const int tap = p.tap0 + tp, ky = p.sx ? tap : tap / p.ks, kx = p.sx ? 0 : tap % p.ks;   // SX: tap = ky
#pragma unroll
      for (int r = 0; r < kWgTH; ++r) {
        const uint64_t ad = gmma_desc(xb + (uint32_t)((r + ky) * p.pw + kx) * 16, 128, x_plane_bytes);
        const uint64_t bd = gmma_desc(yb + (uint32_t)(r * kWgTW) * 16, 128, y_plane_bytes);
        Wgmma<N, 1, 1>::mma(acc[tp], ad, bd, (first && r == 0) ? 0u : 1u);
      }
    }
    wgmma_commit();
    if (S > 1) {                         // release the previous stage: this tile's wgmmas overlap the next load
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&ctrl->empty[prev]);
      prev = (int)s;
    } else {                             // a one-stage ring (wide Cout x 5x5): the only stage is freed at once, or the
      wgmma_wait<0>();                   // producer would wait for it while this warpgroup waits for the next load
      if (lane == 0) mbar_arrive(&ctrl->empty[s]);
    }
    first = false;
    if (++s == S) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int tp = 0; tp < TAPS; ++tp) acc_fence(acc[tp]);
  // ------------------------------------------------ flush: this CTA's slab of the partial-sum workspace
  // (plain stores; wgrad_reduce_kernel sums the slabs afterwards in a fixed order)
  float* slab = p.partial + (size_t)blockIdx.x * p.ntaps * 128 * N;
#pragma unroll
  for (int tp = 0; tp < TAPS; ++tp) {
    if (tp >= p.ntaps) break;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m * 64 + wq * 16 + (lane >> 2) + 8 * h;   // accumulator row = input channel within the tile
#pragma unroll
      for (int i = 0; i < N / 8; ++i)
        *reinterpret_cast<float2*>(slab + ((size_t)tp * 128 + row) * N + 8 * i + 2 * k4) =
            first ? make_float2(0.f, 0.f) : make_float2(acc[tp][4 * i + 2 * h], acc[tp][4 * i + 2 * h + 1]);
    }
  }
}

// dW[co][ci][tap] += (1/scale) * sum over CTAs of partial[cta][tp][ci - ci0][col]   (col = co, or kx*32+co in SX mode)
// 256 threads = 64 elements x 4 slab groups: thread (e, grp) sums slabs grp, grp+4, ... with 8 independent partial sums
// (the ~148 slab reads of an element are independent loads; a single dependent chain kept a handful in flight and made
// this kernel as slow as the GEMM: 34 us per launch for 22 MB of slabs).  The four group sums are combined in a fixed
// order through shared memory, so dW stays bit-reproducible.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partial, int nctas, int ntaps, int n, int sx,
                                                           int tap0, int ci0, int cout, int cin, int kk,
                                                           const float* __restrict__ scale, float* __restrict__ dw) {
  __shared__ float part[4][64];
  const int total = ntaps * 128 * n;
  const int e = threadIdx.x & 63, grp = threadIdx.x >> 6;
  const int i = blockIdx.x * 64 + e;
  float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (i < total) {
    const float* src = partial + i;
    int c = grp;
    for (; c + 28 < nctas; c += 32) {
#pragma unroll
      for (int u = 0; u < 8; ++u) a[u] += __ldg(src + (size_t)(c + 4 * u) * total);
    }
    for (int u = 0; c < nctas; c += 4, ++u) a[u] += __ldg(src + (size_t)c * total);
  }
  part[grp][e] = ((a[0] + a[1]) + (a[2] + a[3])) + ((a[4] + a[5]) + (a[6] + a[7]));
  __syncthreads();
  if (grp == 0 && i < total) {
    const float acc = (part[0][e] + part[1][e]) + (part[2][e] + part[3][e]);
    const int col = i % n, row = (i / n) % 128, tp = i / (n * 128);
    const int ci = ci0 + row;
    const int co = sx ? (col & 31) : col;
    const int tap = sx ? (tap0 + tp) * 3 + (col >> 5) : tap0 + tp;
    if (ci < cin && co < cout) dw[((size_t)co * cin + ci) * kk + tap] += acc / scale[0];
  }
}

template <int N>
static int run_wgrad(WgradParams p, int smem_bytes, int ci_planes, int kk, int ks, cudaStream_t s, bool det) {
  static std::atomic<unsigned long long> smem_opted{0};   // per instantiation, per device
  BIN_TRY(ensure_dynamic_smem(wgrad_kernel<N>, kSmemMax, smem_opted));
  const int taps_per_group = WgCfg<N>::TAPS < kk ? WgCfg<N>::TAPS : kk;   // SX: kk = 3, one accumulator per ky
  // CTA c sums tiles c, c + grid, ... into its slab, so the grid fixes the bits of dW.  Deterministic mode uses a constant
  // grid (the SM count of an H100 SXM) so that dW does not depend on the card; on fewer SMs it runs as a second wave.
  const int sms = det ? kDetCtas : num_sms();
  const int grid = p.ntiles < sms ? p.ntiles : sms;
  if (grid < 1) return BIN_OK;
  for (int cp = 0; cp < ci_planes; cp += 16) {
    for (int t0 = 0; t0 < kk; t0 += taps_per_group) {
      p.ci_tile_plane0 = cp;
      p.tap0 = t0;
      p.ntaps = kk - t0 < taps_per_group ? kk - t0 : taps_per_group;
      wgrad_kernel<N><<<grid, 384, smem_bytes, s>>>(p);
      BIN_CUDA_OK(cudaGetLastError());
      const int total = p.ntaps * 128 * N;
      wgrad_reduce_kernel<<<(total + 63) / 64, 256, 0, s>>>(p.partial, grid, p.ntaps, N, p.sx, t0, cp * 8, p.cout, p.cin,
                                                           ks * ks, p.scale, p.dw);
      BIN_CUDA_OK(cudaGetLastError());
    }
  }
  return BIN_OK;
}

int launch_wgrad(const bin_act_t& x0, int x0_plane0, int x0_planes, const bin_act_t& x1, int x1_plane0, int x1_planes,
                 const bin_act_t& dy, int dy_plane0, int cout, int cin, int ks, const float* scale, float* dw,
                 float* partial_ws, cudaStream_t s, bool det) {
  if (ks != 1 && ks != 3 && ks != 5) return fail(BIN_ERR_ARG, "wgrad: ksize must be 1, 3 or 5");
  if (!partial_ws) return fail(BIN_ERR_ARG, "wgrad: partial-sum workspace missing");
  // TMA zero-fills a box that runs past its tensor, so a bad plane range or geometry would silently give wrong
  // gradients: reject it here, before any tensor map is built
  if (x0_planes <= 0 || x0_planes % kKPL || x1_planes < 0 || x1_planes % kKPL)
    return fail(BIN_ERR_ARG, "wgrad: segment plane counts must be multiples of 4 (x0 non-empty)");
  if (x0_plane0 < 0 || x0_plane0 + x0_planes > x0.planes ||
      (x1_planes > 0 && (x1_plane0 < 0 || x1_plane0 + x1_planes > x1.planes)))
    return fail(BIN_ERR_ARG, "wgrad: input plane range exceeds tensor");
  if ((x1_planes > 0 && (x1.B != x0.B || x1.H != x0.H || x1.W != x0.W)) || dy.B != x0.B || dy.H != x0.H || dy.W != x0.W)
    return fail(BIN_ERR_ARG, "wgrad: x1 / dY geometry differs from x0");
  if (cin <= 0 || cout <= 0 || cin > 8 * (x0_planes + x1_planes))
    return fail(BIN_ERR_ARG, "wgrad: Cin exceeds the input planes provided");
  int n = (cout + 15) / 16 * 16;
  if (n > 256) return fail(BIN_ERR_UNSUPPORTED, "wgrad: Cout > 256");
  if (dy_plane0 < 0 || dy_plane0 + n / 8 > dy.planes) return fail(BIN_ERR_ARG, "wgrad: dY plane range exceeds tensor");   // (before SX widening)
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.pad = ks / 2; p.ks = ks;
  p.sx = (ks == 3 && cout == 32) ? 1 : 0;
  if (p.sx) n = 96;                                   // MMA N = 3 shifted copies of the 32 dY channels
  // wgmma N of the kernel: the next of 16, 32, 48, 64, 96, 128, 256 (dY planes past Cout are zero-filled by TMA or read
  // and then dropped by the reduction's co < cout test)
  n = n <= 64 ? n : n <= 96 ? 96 : n <= 128 ? 128 : 256;
  p.pw = kWgTW + (p.sx ? 0 : 2 * p.pad); p.rows = kWgTH + 2 * p.pad;
  BIN_TRY(make_p8_tmap(&p.xmap0, x0, p.pw, p.rows, 4));
  if (x1_planes > 0) BIN_TRY(make_p8_tmap(&p.xmap1, x1, p.pw, p.rows, 4));
  BIN_TRY(make_p8_tmap(&p.ymap, dy, kWgTW, kWgTH, p.sx ? 4 : n / 8));
  p.x0_plane0 = x0_plane0; p.x0_planes = x0_planes; p.x1_plane0 = x1_plane0; p.x1_planes = x1_planes;
  p.dy_plane0 = dy_plane0; p.n = n; p.cout = cout; p.cin = cin;
  p.B = x0.B; p.H = x0.H; p.W = x0.W;
  p.tiles_x = (p.W + kWgTW - 1) / kWgTW; p.tiles_y = (p.H + kWgTH - 1) / kWgTH;
  p.ntiles = p.B * p.tiles_x * p.tiles_y;
  p.scale = scale; p.dw = dw; p.partial = partial_ws;
  const int x_bytes = 16 * p.rows * p.pw * 16, y_bytes = (n / 8) * kWgTH * kWgTW * 16;
  int S = (kSmemMax - 1024) / (x_bytes + y_bytes);
  if (S > 3) S = 3;
  if (S < 1) return fail(BIN_ERR_UNSUPPORTED, "wgrad: tile does not fit in shared memory");
  p.nstages = S;
  const int smem_bytes = 1024 + S * (x_bytes + y_bytes);
  switch (n) {
#define BIN_WGRAD_N(NN) \
    case NN: return run_wgrad<NN>(p, smem_bytes, x0_planes + x1_planes, p.sx ? 3 : ks * ks, ks, s, det);
    BIN_WGRAD_N(16) BIN_WGRAD_N(32) BIN_WGRAD_N(48) BIN_WGRAD_N(64) BIN_WGRAD_N(96) BIN_WGRAD_N(128) BIN_WGRAD_N(256)
#undef BIN_WGRAD_N
  }
  return fail(BIN_ERR_UNSUPPORTED, "wgrad: no kernel for this Cout");
}

}  // namespace binb
