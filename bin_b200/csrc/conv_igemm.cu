// bin_b200 -- implicit-GEMM convolution for sm_90a (wgmma + TMA + mbarrier).
//
// Replaces every nn.Conv2d on the BIN hot path (reference models/archs/RDN.py:141,162,187-188,
// 199-200,205,207 and the 36/60-channel twins): stride 1, zero padding k/2, bias, optional ReLU
// (RDN.py:142), optional residual (RDN.py:165,219), PixelShuffle(2) folded into the store
// (RDN.py:206) or the final "+ mean(input frames)" fp32 NCHW store (RDN.py:221,279,333).
//
// GEMM view: M = pixels, N = Cout, K = taps x Cin.  Activations are P8 fp16
// [B][C/8][H][W][8]: one pixel of one 8-channel plane is exactly one 16-byte row of a wgmma
// K-major / no-swizzle core matrix, and pixels are contiguous, so the A operand of tap (ky,kx)
// is the SAME shared-memory tile addressed through a descriptor whose start is shifted by
// (ky*32+kx)*16 bytes -- no im2col, the halo tile is fetched once per 32-channel chunk by one
// 4-D TMA box load whose out-of-bounds zero fill implements the conv's zero padding.
// Tile: 8 rows x 32-pixel smem pitch = 256 GEMM rows = four 64-row wgmma blocks, fp32 accumulators in
// registers; the 2*PAD right-most columns of each row are junk rows that are never stored.
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "internal.h"
#include "wgmma.cuh"
#include "xstack.cuh"

namespace binb {

// SX ("stack x"): the KS horizontal taps are folded into the GEMM N dimension -- B rows are
// (kx, cout), the A operand is NOT shifted in x, and the epilogue adds the kx-th column group of
// the accumulator row of pixel p+kx.  One wgmma then does 64 x (KS*NT) x 16 instead of 64 x NT x 16
// for the same A read: the Cout=32 RDB convs would otherwise issue N=32 instructions, whose operand
// traffic per FLOP is three times as high.
template <int NT, int KS, bool SX>
struct ConvCfg {
  static constexpr int PAD = KS / 2;
  static constexpr int TW = kTWH - 2 * PAD;              // valid output columns per tile
  static constexpr bool ROWSPLIT = (KS == 5);            // 5x5: one stage per (chunk, ky)
  static constexpr int ROWS = ROWSPLIT ? kTH : kTH + 2 * PAD;
  static constexpr int A_PLANE = ROWS * kTWH * 16;       // bytes of one plane of a stage
  static constexpr int A_BYTES = kKPL * A_PLANE;
  static constexpr int NMMA = SX ? NT * KS : NT;         // N of one wgmma
  static constexpr int TAPS_C = SX ? KS : KS * KS;       // B slabs ("taps") per chunk
  static constexpr int TAPS_S = (SX || ROWSPLIT) ? KS : KS * KS;  // taps per stage
  static constexpr int NSUB = ROWSPLIT ? KS : 1;         // stages per chunk
  static constexpr int W_TAP = kKPL * NMMA * 16;         // bytes per tap per chunk
  static constexpr int W_STAGE = TAPS_S * W_TAP;
  static constexpr int W_CHUNK = TAPS_C * W_TAP;
  // SX: xstack_sum exchange buffers, one per warp pair (2 per warpgroup) and 64-row block (2 per accumulator), so the
  // second block's exchange needs no barrier against the first block's reads
  static constexpr int XS_BYTES = SX ? kMT * 2 * 2 * kXsFloats<NT> * 4 : 0;
  // fp16 SX P8 epilogue (tma_store below): a consumer warpgroup's staging buffer [NT/8 planes][4 rows][TW px][16 B]
  static constexpr int ST_PLANE = (kTH / kMT) * TW * 16;
  static constexpr int ST_BYTES = NT / 8 * ST_PLANE;
  static_assert(XS_BYTES % 128 == 0 && ST_BYTES % 128 == 0, "TMA store sources must be 128-byte aligned");
  static_assert(!(SX && ROWSPLIT), "SX is only used for 3x3");
  static_assert(NMMA % 16 == 0 && NMMA <= 256, "invalid wgmma N");
};

struct Ctrl {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
  uint64_t wfull[kMaxResidentChunks];
};
static_assert(sizeof(Ctrl) <= 1024, "ctrl block");

constexpr int kThreads = 384;   // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: wgmma + epilogue

// PixelShuffle epilogue staging buffer of one consumer warp: one accumulator row set (8 low-res pixels x 128 channels)
// as [plane q][pixel r][sub-pixel s][8 channels] fp16, each pixel's 4 sub-pixels padded by 16 bytes so that the
// 2-byte writes of a warp spread over the banks (2-way conflicts instead of 4-way); X3 adds a second part for lo.
constexpr int kPsRowBytes = 4 * 16 + 16;
constexpr int kPsPartBytes = 4 * 8 * kPsRowBytes;
template <bool X3>
constexpr int kPsWarpBytes = (X3 ? 2 : 1) * kPsPartBytes;

// X3 ("fp32-accurate" mode, 1e-5 parity bar): every value is carried as an fp16 pair hi = fp16(x), lo = fp16(x - hi).
// The pair is within 2^-22 |x| of x while lo is a normal fp16 number; below |x| ~ 2^-3 lo is subnormal and the pair
// carries an absolute 2^-25 instead (the fp16 subnormal half-spacing), which is what tests/test_gpu_forward_fuzz.py bars.
// Tensors hold, per 32-channel chunk, 4 planes of hi followed by 4 planes of lo; a logical K chunk becomes three
// physical chunks  x_hi*W_hi + x_lo*W_hi + x_hi*W_lo  (the lo*lo term is below 2^-22 |x w|), the weights are packed
// pre-scaled by 2^8 so that W_lo stays a normal fp16 number, and the epilogue un-scales the fp32 accumulator and
// splits its result into (hi, lo) again.  Same kernel, same descriptors: 3x the MMAs, 2x the activation bytes.
__device__ __forceinline__ int x3_plane(int logical_plane) { return 2 * (logical_plane & ~3) + (logical_plane & 3); }
// stores 2 consecutive channels (4 bytes) of one pixel, or their (hi, lo) split
template <bool X3>
__device__ __forceinline__ void store_pair(__half* p, size_t lo_off, float a, float b) {
  if constexpr (X3) {
    const __half h0 = __float2half_rn(a), h1 = __float2half_rn(b);
    const __half2 hh = __halves2half2(h0, h1);
    *reinterpret_cast<__half2*>(p) = hh;
    *reinterpret_cast<__half2*>(p + lo_off) = __floats2half2_rn(a - __half2float(h0), b - __half2float(h1));
  } else {
    *reinterpret_cast<uint32_t*>(p) = pack_h2(a, b);
  }
}

// Roles (384 threads, 1 CTA/SM, persistent over tiles):
//   warp 0 lane 0 : TMA producer (activation box + weight slab per stage, mbarrier ring)
//   warpgroup 1+m : accumulator m = tile rows [128 m, 128 m + 128) as two 64-row wgmma blocks held in registers; it
//                   waits for each stage, issues its wgmmas, releases the stage one stage later (wait_group 1), and
//                   runs the epilogue of its rows straight from the accumulator fragments.
// Weight sets that fit (RDB convs, LFF, SFENet2, GFF.1, UPNet.2) stay resident in shared memory.
// A pipeline stage holds up to p.cps "units" (unit = one 32-channel chunk, or one (chunk, ky) for 5x5).
template <int NT, int KS, int EPI, bool SX, bool X3>
__global__ void __launch_bounds__(kThreads, 1) conv_igemm_kernel(const __grid_constant__ ConvParams p) {
  using C = ConvCfg<NT, KS, SX>;
  static_assert(EPI != BIN_EPI_PIXSHUF || NT == 128, "the PixelShuffle staging buffer holds 4 output planes");
  // The fp16 x-stacked P8 epilogue (the RDB growth convs) stages each warpgroup's 4 output rows of the tile in shared
  // memory and writes them with one TMA tensor store over p.tmap_out, whose out-of-bounds clipping stands in for every
  // pixel validity test but the junk columns.
  constexpr bool TSTORE = SX && EPI == BIN_EPI_P8 && !X3;
  constexpr int NA = C::NMMA / 2;                              // accumulator registers per thread and 64-row block
  extern __shared__ __align__(1024) uint8_t smem[];
  Ctrl* ctrl = reinterpret_cast<Ctrl*>(smem);
  float* sbias = reinterpret_cast<float*>(smem + 1024);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);   // provably warp-uniform for the compiler
  const int lane = threadIdx.x & 31;
  const uint32_t S = p.nstages;
  const int nchunks = p.nch0 + p.nch1;
  const int nunits = nchunks * C::NSUB;
  const int cps = p.cps;
  const int spt = (nunits + cps - 1) / cps;                   // stages per tile
  const int unit_bytes = C::A_BYTES + (p.resident ? 0 : C::W_STAGE);
  const int stage_bytes = cps * unit_bytes;
  uint8_t* res_w = smem + kCtrlBytes;
  uint8_t* stage0 = res_w + (p.resident ? nchunks * C::W_CHUNK : 0);

  // ------------------------------------------------------------ one-time setup
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmap0);
    if (p.nch1 > 0) tma_prefetch_desc(&p.tmap1);
    if (TSTORE) tma_prefetch_desc(&p.tmap_out);
    for (int i = 0; i < kMaxStages; ++i) {
      mbar_init(&ctrl->full[i], 1);
      mbar_init(&ctrl->empty[i], 8);                           // one arrival per consumer warp
    }
    for (int i = 0; i < kMaxResidentChunks; ++i) mbar_init(&ctrl->wfull[i], 1);
    fence_barrier_init();
  }
  const bool bias_in_smem = NT * p.nh <= 256;                  // else (wide data-gradient launches) read it from global
  if (bias_in_smem)
    for (int i = threadIdx.x; i < NT * p.nh; i += blockDim.x) sbias[i] = p.bias[i];
  const float* bsrc = bias_in_smem ? sbias : p.bias;
  __syncthreads();

  if (warp == 0) {
    if (lane != 0) return;
    // ========================================================== TMA producer
    if (p.resident) {
      for (int c = 0; c < nchunks; ++c) {
        mbar_expect_tx(&ctrl->wfull[c], C::W_CHUNK);
        bulk_load_1d(res_w + c * C::W_CHUNK, reinterpret_cast<const uint8_t*>(p.w) + (size_t)c * C::W_CHUNK, C::W_CHUNK,
                     &ctrl->wfull[c]);
      }
    }
    uint32_t s = 0, ph = 0;
    for (int tq = blockIdx.x; tq < p.ntiles; tq += gridDim.x) {
      const int t1 = p.div_nh.div(tq), t2 = p.div_tx.div(t1), t3 = p.div_ty.div(t2);
      const int nh = tq - t1 * p.nh;
      const int txi = t1 - t2 * p.tiles_x;
      const int tyi = t2 - t3 * p.tiles_y;
      const int b = p.b0 + t3;
      const int x0 = txi * C::TW - C::PAD, y0 = p.y0 + tyi * kTH - C::PAD;
      int unit = 0;
      for (int j = 0; j < spt; ++j) {
        const int nu = (nunits - unit < cps) ? nunits - unit : cps;
        mbar_wait(&ctrl->empty[s], ph ^ 1);
        uint8_t* dst = stage0 + (size_t)s * stage_bytes;
        mbar_expect_tx(&ctrl->full[s], (uint32_t)(nu * unit_bytes));
        for (int u = 0; u < nu; ++u) {
          const int c = (unit + u) / C::NSUB, sub = (unit + u) % C::NSUB;
          const int lc = X3 ? c / 3 : c;                     // logical 32-channel chunk
          const bool seg1 = lc >= p.nch0l;
          const void* tmap = seg1 ? (const void*)&p.tmap1 : (const void*)&p.tmap0;
          const int lplane = seg1 ? p.plane0_1 + (lc - p.nch0l) * kKPL : p.plane0_0 + lc * kKPL;
          const int plane = X3 ? 2 * lplane + ((c % 3) == 1 ? 4 : 0) : lplane;   // X3: hi, lo, hi again
          tma_load_4d(dst + (size_t)u * unit_bytes, tmap, &ctrl->full[s], x0 * 8, y0 + (C::ROWSPLIT ? sub : 0), plane, b);
          if (!p.resident) {
            const size_t woff = ((size_t)(nh * nchunks + c) * C::TAPS_C + (C::ROWSPLIT ? sub * KS : 0)) * C::W_TAP;
            bulk_load_1d(dst + (size_t)u * unit_bytes + C::A_BYTES, reinterpret_cast<const uint8_t*>(p.w) + woff,
                         C::W_STAGE, &ctrl->full[s]);
          }
        }
        unit += nu;
        if (++s == S) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  if (warp < 4) return;

  // ============================================================ consumer warpgroups
  const int m = (warp - 4) >> 2;                               // accumulator: tile rows [128 m, 128 m + 128)
  const int wq = warp & 3;                                     // warp within the warpgroup: 16 rows of each 64-row block
  const int k4 = lane & 3;                                     // fragment column pair: columns 8 i + 2 k4, +1
  float* xs = reinterpret_cast<float*>(stage0 + (size_t)S * stage_bytes) + (2 * m + (wq >> 1)) * 2 * kXsFloats<NT>;
  uint8_t* psbuf = stage0 + (size_t)S * stage_bytes + (warp - 4) * kPsWarpBytes<X3>;   // PIXSHUF staging buffer
  uint8_t* stbuf = stage0 + (size_t)S * stage_bytes + C::XS_BYTES + m * C::ST_BYTES;   // TSTORE staging buffer
  const bool st_leader = (threadIdx.x & 127) == 0;            // TSTORE: the thread that issues the warpgroup's stores
  float acc[2][NA];
  constexpr float kAcc = X3 ? (1.f / 256.f) : 1.f;            // X3 weights are packed scaled by 2^8
  uint32_t s = 0, ph = 0;
  // tile tq -> (cout block nh, tile column txi, tile row tyi, image b)
  auto tile_coords = [&](int tq, int& nh, int& txi, int& tyi, int& b) {
    const int t1 = p.div_nh.div(tq), t2 = p.div_tx.div(t1), t3 = p.div_ty.div(t2);
    nh = tq - t1 * p.nh;
    txi = t1 - t2 * p.tiles_x;
    tyi = t2 - t3 * p.tiles_y;
    b = p.b0 + t3;
  };
  // fragment of a 64-row block: acc[mb][4 i + 2 h + e] = row 16 wq + lane/4 + 8 h, column 8 i + 2 k4 + e
  auto pixel = [&](int txi, int tyi, int mb, int h, int& y, int& x) {
    const int L = m * 128 + mb * 64 + wq * 16 + (lane >> 2) + 8 * h;
    const int ty = L >> 5, tx = L & 31;
    y = p.y0 + tyi * kTH + ty; x = txi * C::TW + tx;
    return (tx < C::TW) && (y < p.y0 + p.ny) && (x < p.W);
  };
  // BIN_EPI_P8 residual: load_res reads accumulator row set (mb, h)'s residual words into r, r[i] = output channels
  // 8 i + 2 k4, +1 of the tile's cout block (X3: hi, lo).  fp16 loads one row set ahead (RES_AHEAD): row set (0, 0)
  // during the tile's last K stage, under its wgmmas, and row set k + 1 before the stores of row set k, so one memory
  // round trip is in flight under each row's epilogue instead of four exposed after the MMAs.  X3 holds twice the words
  // and has no registers to spare under the 168-register cap: it loads each row set just before its own stores.
  constexpr bool RES = EPI == BIN_EPI_P8 && !SX;
  constexpr bool RES_AHEAD = RES && !X3;
  constexpr int NR = RES ? NT / 8 : 1;
  // Offset of channel pair 2 k4 of pixel (y, x) in the first plane a tile of cout block nh touches; plane i of the
  // block is x3_plane(i) (fp16: i) planes further on.  X3 plane offsets and each block's first plane are
  // multiples of 4 (launch_conv_t checks the offsets), so x3_plane(plane0 + i) = x3_plane(plane0) + x3_plane(i) there.
  // Computing the offset once per pixel instead of once per plane takes about a third of the epilogue's instructions.
  static_assert(EPI != BIN_EPI_P8 || NT % 32 == 0, "a cout block starts at a multiple of 4 planes");
  const size_t plane = (size_t)p.H * p.W * 8;                   // halves per P8 plane
  auto plane_off = [&](int planes, int plane0, int nh, int b, int y, int x) {
    const int lp = plane0 + (nh * NT) / 8;
    return ((((size_t)b * planes + (X3 ? x3_plane(lp) : lp)) * p.H + y) * p.W + x) * 8 + 2 * k4;
  };
  auto load_res = [&](uint32_t (&r)[NR][X3 ? 2 : 1], int nh, int txi, int tyi, int b, int mb, int h) {
    int y, x;
    if (!pixel(txi, tyi, mb, h, y, x)) return;
    const __half* src = p.res + plane_off(p.res_planes, p.res_plane0, nh, b, y, x);
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      if ((nh * NT) / 8 + i >= p.store_planes) continue;
      const __half* q = src + (size_t)(X3 ? x3_plane(i) : i) * plane;
      r[i][0] = *reinterpret_cast<const uint32_t*>(q);
      if constexpr (X3) r[i][X3 ? 1 : 0] = *reinterpret_cast<const uint32_t*>(q + 4 * plane);
    }
  };
  for (int tq = blockIdx.x; tq < p.ntiles; tq += gridDim.x) {
    uint32_t rcur[NR][X3 ? 2 : 1], rnxt[NR][X3 ? 2 : 1];      // this row set's residual words, the next one's
    // BIN_EPI_FINAL: the input frames this thread's outputs add are loaded here, so their latency hides behind the
    // main loop; the epilogue sums them.
    constexpr int NFR = EPI == BIN_EPI_FINAL ? BIN_MAX_FRAMES : 1;
    float fpre[2][2][2][NFR];                                   // [mb][h][e][frame]
    if constexpr (EPI == BIN_EPI_FINAL) {
      int nh, txi, tyi, b;
      tile_coords(tq, nh, txi, tyi, b);
      const int call = b / p.fr.Bc, bb = b % p.fr.Bc;
      const size_t hw = (size_t)p.H * p.W;
#pragma unroll
      for (int mb = 0; mb < 2; ++mb)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int y, x;
          const bool valid = pixel(txi, tyi, mb, h, y, x);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 2 * k4 + e;
            const size_t off = ((size_t)bb * 3 + c) * hw + (size_t)y * p.W + x;
#pragma unroll
            for (int fi = 0; fi < NFR; ++fi)
              fpre[mb][h][e][fi] = (valid && c < 3 && fi < p.fr.nframes) ? __ldg(p.fr.frame[call][fi] + off) : 0.f;
          }
        }
    }
    // ---------------------------------------------------------- main loop: K = chunks x taps
    int unit = 0, prev = -1;
    for (int j = 0; j < spt; ++j) {
      const int nu = (nunits - unit < cps) ? nunits - unit : cps;
      mbar_wait(&ctrl->full[s], ph);
      if (p.resident && tq == (int)blockIdx.x) {
        for (int u = 0; u < nu; ++u)
          if ((unit + u) % C::NSUB == 0) mbar_wait(&ctrl->wfull[(unit + u) / C::NSUB], 0);
      }
      if constexpr (RES_AHEAD) {
        if (j == spt - 1 && p.res != nullptr) {
          int nh, txi, tyi, b;
          tile_coords(tq, nh, txi, tyi, b);
          load_res(rcur, nh, txi, tyi, b, 0, 0);
        }
      }
      const uint32_t st_base = smem_u32(stage0 + (size_t)s * stage_bytes);
      wgmma_fence();
      for (int u = 0; u < nu; ++u) {
        const int c = (unit + u) / C::NSUB, sub = (unit + u) % C::NSUB;
        const uint32_t a_base = st_base + u * unit_bytes;
        const uint32_t w_base = p.resident ? smem_u32(res_w + c * C::W_CHUNK) + (C::ROWSPLIT ? sub * KS * C::W_TAP : 0)
                                           : a_base + C::A_BYTES;
        const uint32_t not_first = (unit + u) != 0 ? 1u : 0u;
#pragma unroll
        for (int tp = 0; tp < C::TAPS_S; ++tp) {
          const int ky = SX ? tp : (C::ROWSPLIT ? 0 : tp / KS);
          const int kx = SX ? 0 : (C::ROWSPLIT ? tp : tp % KS);
#pragma unroll
          for (int jj = 0; jj < kKC / 16; ++jj) {
            const uint64_t bd = gmma_desc(w_base + tp * C::W_TAP + jj * 2 * C::NMMA * 16, C::NMMA * 16, 128);
#pragma unroll
            for (int mb = 0; mb < 2; ++mb) {
              const uint32_t a_row = (uint32_t)(m * 128 + mb * 64 + ky * kTWH + kx);   // 16-byte rows
              const uint64_t ad = gmma_desc(a_base + a_row * 16 + jj * 2 * C::A_PLANE, C::A_PLANE, 128);
              Wgmma<C::NMMA>::mma(acc[mb], ad, bd, (tp == 0 && jj == 0) ? not_first : 1u);
            }
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                                         // the previous stage's wgmmas have retired
      if (prev >= 0 && lane == 0) mbar_arrive(&ctrl->empty[prev]);
      prev = (int)s;
      unit += nu;
      if (++s == S) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    if (lane == 0) mbar_arrive(&ctrl->empty[prev]);

    // ---------------------------------------------------------- epilogue from the accumulator fragments
    int nh, txi, tyi, b;
    tile_coords(tq, nh, txi, tyi, b);
    if constexpr (TSTORE) {
      // The previous tile's store has had this tile's main loop to read the buffer, so this wait should not stall.
      if (st_leader) bulk_wait_read_all();
      wg_sync(1 + m);
#pragma unroll
      for (int mb = 0; mb < 2; ++mb) {
        xstack_sum<NT>(acc[mb], xs + mb * kXsFloats<NT>, 3 + 2 * m + (wq >> 1));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int tx = (wq & 1) * 16 + (lane >> 2) + 8 * h;     // pixel of row 2 mb + wq / 2 of the warpgroup's 4
          if (tx >= C::TW) continue;                               // junk column
          uint8_t* dst = stbuf + ((2 * mb + (wq >> 1)) * C::TW + tx) * 16 + 4 * k4;
#pragma unroll
          for (int i = 0; i < NT / 8; ++i) {                       // planes past store_planes lie outside the box
            const int n = nh * NT + 8 * i + 2 * k4;                // NT * nh <= 256: the bias is in shared memory
            float f0 = acc[mb][4 * i + 2 * h] + sbias[n], f1 = acc[mb][4 * i + 2 * h + 1] + sbias[n + 1];
            if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
            *reinterpret_cast<uint32_t*>(dst + i * C::ST_PLANE) = pack_h2(f0, f1);
          }
        }
      }
      fence_proxy_async();                                         // generic-proxy writes -> visible to the TMA
      wg_sync(1 + m);
      if (st_leader) {
        tma_store_4d(&p.tmap_out, stbuf, txi * C::TW * 8, tyi * kTH + (kTH / kMT) * m, p.out_plane0 + (nh * NT) / 8,
                     b - p.b0);
        bulk_commit();
      }
      continue;
    }
#pragma unroll
    for (int mb = 0; mb < 2; ++mb) {
      if constexpr (SX) xstack_sum<NT>(acc[mb], xs + mb * kXsFloats<NT>, 3 + 2 * m + (wq >> 1));   // barrier per warp pair
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int y, x;
        const bool valid = pixel(txi, tyi, mb, h, y, x);
        // value of output channel column 8 i + 2 k4 + e of this pixel (SX: xstack_sum has added the kx = 1, 2 groups)
        auto val = [&](int i, int e) { return acc[mb][4 * i + 2 * h + e] * kAcc; };
        if constexpr (EPI == BIN_EPI_P8) {
          // Residual loads come before the row's stores: a store to p.out may alias p.res, so the compiler keeps every
          // load behind the stores that precede it in program order.  fp16 loads row set (mb, h) + 1 before the stores
          // of row set (mb, h).  That order is exact even in place (out and res the same planes): row sets are disjoint
          // pixels, each thread reads and writes only its own fragment's pixels, so the early loads read nothing that
          // the stores between them and their use write.
          if constexpr (RES) {
            if (p.res != nullptr) {
              if constexpr (RES_AHEAD) {
                if (2 * mb + h < 3) load_res(rnxt, nh, txi, tyi, b, (2 * mb + h + 1) >> 1, (2 * mb + h + 1) & 1);
              } else {
                load_res(rcur, nh, txi, tyi, b, mb, h);
              }
            }
          }
          if (valid) {
            __half* dst = p.out + plane_off(p.out_planes, p.out_plane0, nh, b, y, x);
#pragma unroll
            for (int i = 0; i < NT / 8; ++i) {
              const int rel = (nh * NT) / 8 + i;                // channel plane relative to out_plane0
              if (rel >= p.store_planes) continue;
              const int n = nh * NT + 8 * i + 2 * k4;
              float f0 = val(i, 0) + bsrc[n], f1 = val(i, 1) + bsrc[n + 1];
              if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
              if (RES && p.res != nullptr) {
                const float2 g = unpack_h2(rcur[RES ? i : 0][0]);
                f0 += g.x; f1 += g.y;
                if constexpr (X3) {
                  const float2 g2 = unpack_h2(rcur[RES ? i : 0][X3 ? 1 : 0]);
                  f0 += g2.x; f1 += g2.y;
                }
              }
              if constexpr (SX) {                                // X3 x-stacked kernel: its own addressing
                const int op = p.out_plane0 + rel;
                const size_t off = ((((size_t)b * p.out_planes + (X3 ? x3_plane(op) : op)) * p.H + y) * p.W + x) * 8 + 2 * k4;
                store_pair<X3>(p.out + off, (size_t)4 * p.H * p.W * 8, f0, f1);
              } else {
                store_pair<X3>(dst + (size_t)(X3 ? x3_plane(i) : i) * plane, 4 * plane, f0, f1);
              }
            }
          }
          if constexpr (RES_AHEAD) {
#pragma unroll
            for (int i = 0; i < NR; ++i) rcur[i][0] = rnxt[i][0];
          }
        } else if constexpr (EPI == BIN_EPI_PIXSHUF) {
          // out[c, 2y+i, 2x+j] = conv[4c+2i+j, y, x]   (nn.PixelShuffle(2), RDN.py:206).  Column 8 (4 q + m) + 2 k4 + e
          // of this row is channel 2 m + k4/2 of output plane nh NT/32 + q at full-res pixel (2y + (k4 & 1), 2x + e).
          // The warp writes the fp16 values into its staging buffer in P8 order, then each lane reads back whole
          // 16-byte pixels (lane = row r, sub-pixel s = 2 dy + dx; its row is its own fragment row) and stores them:
          // a warp store covers two full-res rows of 256 contiguous bytes instead of 4 bytes in each of 16 sectors.
          const int r = lane >> 2;
#pragma unroll
          for (int i = 0; i < NT / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int n = nh * NT + 8 * i + 2 * k4 + e;
              const float a = val(i, e) + sbias[n];
              const __half hi = __float2half_rn(a);
              __half* dst = reinterpret_cast<__half*>(psbuf + ((i >> 2) * 8 + r) * kPsRowBytes + (2 * (k4 & 1) + e) * 16) +
                            2 * (i & 3) + (k4 >> 1);
              dst[0] = hi;
              if constexpr (X3) dst[kPsPartBytes / 2] = __float2half_rn(a - __half2float(hi));
            }
          }
          __syncwarp();
          if (valid) {
            const int H2 = 2 * p.H, W2 = 2 * p.W;
            const int yy = 2 * y + (k4 >> 1), xx = 2 * x + (k4 & 1);
#pragma unroll
            for (int q = 0; q < NT / 32; ++q) {
              const int op = p.out_plane0 + nh * (NT / 32) + q;
              const size_t off = ((((size_t)b * p.out_planes + (X3 ? x3_plane(op) : op)) * H2 + yy) * W2 + xx) * 8;
#pragma unroll
              for (int part = 0; part < (X3 ? 2 : 1); ++part)
                *reinterpret_cast<uint4*>(p.out + off + (size_t)part * 4 * H2 * W2 * 8) =
                    *reinterpret_cast<const uint4*>(psbuf + part * kPsPartBytes + (q * 8 + r) * kPsRowBytes + k4 * 16);
            }
          }
          __syncwarp();                                        // the buffer is rewritten by the next row
        } else {  // BIN_EPI_FINAL: fp32 NCHW = conv + bias + mean(frames) (RDN.py:221/279/333); channels 0..2
          if (valid && k4 < 2) {
            const int call = b / p.fr.Bc, bb = b % p.fr.Bc;
            const size_t hw = (size_t)p.H * p.W;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 2 * k4 + e;
              if (c >= 3) continue;
              const size_t off = ((size_t)bb * 3 + c) * hw + (size_t)y * p.W + x;
              float fm = fpre[mb][h][e][0];
#pragma unroll
              for (int fi = 1; fi < NFR; ++fi)
                if (fi < p.fr.nframes) fm += fpre[mb][h][e][fi];   // left to right
              p.fr.out[call][off] = (val(0, e) + sbias[c]) + fm / (float)p.fr.nframes;
            }
          }
        }
      }
    }
  }
  if constexpr (TSTORE) {
    if (st_leader) bulk_wait_all();                              // the staging buffers outlive no store
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(ptr);
  }();
  return fn;
}

int make_p8_tmap(CUtensorMap* m, const bin_act_t& t, int box_px, int box_rows, int box_planes, int b0, int nb, int y0,
                 int ny) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(BIN_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  if ((reinterpret_cast<uintptr_t>(t.ptr) & 15) != 0) return fail(BIN_ERR_ARG, "P8 tensor not 16-byte aligned");
  if (box_px * 8 > 256 || box_rows > 256 || box_planes > 256) return fail(BIN_ERR_ARG, "TMA box dimension exceeds 256");
  // The (8 channels, W) dims of a P8 plane row are contiguous in memory, so they are described as ONE
  // dimension of W*8 elements: a conv box row is then 32 px * 16 B = 512 contiguous bytes (a 16-byte
  // inner box made the TMA unit the bottleneck).  OOB zero fill works per element, i.e. per pixel.
  const size_t row = (size_t)t.W * 16, plane = (size_t)t.H * row, image = (size_t)t.planes * plane;
  void* base = static_cast<uint8_t*>(t.ptr) + (size_t)b0 * image + (size_t)y0 * row;   // stays 16-byte aligned
  cuuint64_t dims[4] = {(cuuint64_t)t.W * 8, (cuuint64_t)(ny > 0 ? ny : t.H), (cuuint64_t)t.planes,
                        (cuuint64_t)(nb > 0 ? nb : t.B)};
  cuuint64_t strides[3] = {row, plane, image};
  cuuint32_t box[4] = {(cuuint32_t)box_px * 8, (cuuint32_t)box_rows, (cuuint32_t)box_planes, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(BIN_ERR_CUDA, "cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return BIN_OK;
}

// Every argument check of a conv launch runs before the first tensor map is encoded (launch_conv_t, then the
// shared-memory fit here), so a rejected call has touched neither the driver nor the device.
template <int NT, int KS, int EPI, bool SX, bool X3>
static int launch_inst(const bin_conv_args_t& a, cudaStream_t s) {
  using C = ConvCfg<NT, KS, SX>;
  ConvParams p;
  memset(&p, 0, sizeof(p));
  const int H = a.in0.H, W = a.in0.W, B = a.in0.B;
  // X3: plane indices are LOGICAL (the tensors hold 2x the planes: hi/lo groups of 4), K has 3 chunks per logical chunk
  p.plane0_0 = a.in0_plane0; p.nch0l = a.in0_planes / kKPL; p.nch0 = (X3 ? 3 : 1) * p.nch0l;
  p.plane0_1 = a.in1_plane0; p.nch1 = (X3 ? 3 : 1) * (a.in1_planes / kKPL);
  p.w = reinterpret_cast<const __half*>(a.w_packed);
  p.bias = a.bias;
  p.H = H; p.W = W; p.Btot = B;
  p.b0 = a.b_begin; p.y0 = a.y_begin;
  const int nb = a.b_count > 0 ? a.b_count : B - a.b_begin;
  p.ny = a.y_count > 0 ? a.y_count : H - a.y_begin;   // launch_conv_t has checked the sub-range
  p.tiles_x = (W + C::TW - 1) / C::TW;
  p.tiles_y = (p.ny + kTH - 1) / kTH;
  p.nh = a.cout_pad / NT;
  p.ntiles = nb * p.tiles_x * p.tiles_y * p.nh;
  p.div_nh = fast_div(p.nh); p.div_tx = fast_div(p.tiles_x); p.div_ty = fast_div(p.tiles_y);
  p.relu = a.relu;
  const int nchunks = p.nch0 + p.nch1;
  constexpr bool tma_store = SX && EPI == BIN_EPI_P8 && !X3;   // see conv_igemm_kernel
  const int xbytes = C::XS_BYTES + (EPI == BIN_EPI_PIXSHUF ? 8 * kPsWarpBytes<X3> : 0) +   // + the consumer warps' staging
                     (tma_store ? kMT * C::ST_BYTES : 0);
  // keep the whole weight set resident in smem when it leaves room for >= 3 activation stages
  p.resident = (p.nh == 1 && nchunks <= kMaxResidentChunks &&
                kCtrlBytes + nchunks * C::W_CHUNK + xbytes + 3 * C::A_BYTES + 256 <= kSmemMax) ? 1 : 0;
  const int res_bytes = p.resident ? nchunks * C::W_CHUNK : 0;
  const int unit_bytes = C::A_BYTES + (p.resident ? 0 : C::W_STAGE);
  const int nunits = nchunks * C::NSUB;
  // units per pipeline stage: enough for kStageMmas wgmma instructions per warpgroup
  const int mma_per_unit = kMT * C::TAPS_S * (kKC / 16);
  int cps = (kStageMmas + mma_per_unit - 1) / mma_per_unit;
  if (cps > nunits) cps = nunits;
  const int avail = kSmemMax - kCtrlBytes - res_bytes - xbytes - 256;
  while (cps > 1 && avail / (cps * unit_bytes) < 2) --cps;
  int S = avail / (cps * unit_bytes);
  if (S > kMaxStages) S = kMaxStages;
  if (S < 2) return fail(BIN_ERR_UNSUPPORTED, "conv configuration does not fit in shared memory");
  p.nstages = S;
  p.cps = cps;
  const int smem_bytes = kCtrlBytes + res_bytes + S * cps * unit_bytes + xbytes + 256;
  p.out = reinterpret_cast<__half*>(a.out.ptr); p.out_planes = a.out.planes; p.out_plane0 = a.out_plane0;
  p.store_planes = a.store_planes > 0 ? a.store_planes : a.cout_pad / 8;
  p.res = reinterpret_cast<const __half*>(a.res.ptr); p.res_planes = a.res.planes; p.res_plane0 = a.res_plane0;
  p.fr = a.fr;
  BIN_TRY(make_p8_tmap(&p.tmap0, a.in0, kTWH, C::ROWS, kKPL));
  if (a.in1_planes > 0) BIN_TRY(make_p8_tmap(&p.tmap1, a.in1, kTWH, C::ROWS, kKPL));
  if (tma_store) BIN_TRY(make_p8_tmap(&p.tmap_out, a.out, C::TW, kTH / kMT, p.store_planes, p.b0, nb, p.y0, p.ny));
  auto kern = conv_igemm_kernel<NT, KS, EPI, SX, X3>;
  static std::atomic<unsigned long long> smem_opted{0};   // per instantiation, per device
  BIN_TRY(ensure_dynamic_smem(kern, kSmemMax, smem_opted));
  int grid = p.ntiles < num_sms() ? p.ntiles : num_sms();
  if (grid < 1) return BIN_OK;
  kern<<<grid, kThreads, smem_bytes, s>>>(p);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

template <bool X3>
static int launch_conv_t(const bin_conv_args_t& a, cudaStream_t s) {
  constexpr int f = X3 ? 2 : 1;      // X3 tensors hold hi+lo: twice the planes of their logical channel count
  // one past the last PHYSICAL plane that logical planes [plane0, plane0 + n) occupy (X3: the lo plane of the last one)
  auto plane_end = [](int plane0, int n) { return X3 ? 2 * ((plane0 + n - 1) & ~3) + ((plane0 + n - 1) & 3) + 5 : plane0 + n; };
  auto misaligned = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) != 0; };
  const bool has_in1 = a.in1_planes > 0;
  const int H = a.in0.H, W = a.in0.W, B = a.in0.B;
  // ---- geometry: plane counts, offsets and ranges, shapes, sub-range, epilogue options
  if (a.in0_planes % kKPL || a.in1_planes % kKPL || a.in0_planes <= 0 || a.in1_planes < 0)
    return fail(BIN_ERR_ARG, "conv: input plane counts must be positive multiples of 4 (32 channels)");
  if (a.in0_plane0 < 0 || (has_in1 && a.in1_plane0 < 0) || a.out_plane0 < 0 || (a.res.ptr && a.res_plane0 < 0) ||
      a.store_planes < 0)
    return fail(BIN_ERR_ARG, "conv: negative plane offset or store_planes");
  if (X3 && ((a.in0_plane0 | a.in1_plane0 | a.out_plane0 | a.res_plane0) & 3))
    return fail(BIN_ERR_ARG, "conv: x3 mode: plane offsets must be multiples of 4");
  if (f * (a.in0_plane0 + a.in0_planes) > a.in0.planes || (has_in1 && f * (a.in1_plane0 + a.in1_planes) > a.in1.planes))
    return fail(BIN_ERR_ARG, "conv: input plane range exceeds tensor");
  if (has_in1 && (a.in1.H != H || a.in1.W != W || a.in1.B != B)) return fail(BIN_ERR_ARG, "conv: in1 geometry differs from in0");
  const int nb = a.b_count > 0 ? a.b_count : B - a.b_begin;
  const int ny = a.y_count > 0 ? a.y_count : H - a.y_begin;
  if (a.b_begin < 0 || a.y_begin < 0 || a.b_count < 0 || a.y_count < 0 || nb < 1 || ny < 1 || a.b_begin + nb > B ||
      a.y_begin + ny > H)
    return fail(BIN_ERR_ARG, "conv: batch/row sub-range outside the tensor");
  if (a.epilogue != BIN_EPI_P8 && (a.relu || a.res.ptr))
    return fail(BIN_ERR_ARG, "conv: the pixel-shuffle and final epilogues take no ReLU and no residual");
  const bool sx = a.ksize == 3 && a.cout_pad == 32 && a.variant == BIN_CONV_DEFAULT;
  if (a.epilogue == BIN_EPI_P8) {
    const int nstore = a.store_planes > 0 ? a.store_planes : a.cout_pad / 8;
    if (a.out.H != H || a.out.W != W || a.out.B != B || nstore > a.cout_pad / 8 || plane_end(a.out_plane0, nstore) > a.out.planes)
      return fail(BIN_ERR_ARG, "conv: output tensor geometry mismatch");
    if (a.res.ptr && (a.res.H != H || a.res.W != W || a.res.B != B || plane_end(a.res_plane0, nstore) > a.res.planes))
      return fail(BIN_ERR_ARG, "conv: residual tensor geometry mismatch");
    if (sx && a.res.ptr) return fail(BIN_ERR_ARG, "conv: the x-stacked 3x3 / Cout 32 kernel takes no residual");
  } else if (a.epilogue == BIN_EPI_PIXSHUF) {
    if (a.out.H != 2 * H || a.out.W != 2 * W || a.out.B != B || plane_end(a.out_plane0, a.cout_pad / 32) > a.out.planes)
      return fail(BIN_ERR_ARG, "conv: pixel-shuffle output geometry mismatch");
    if (misaligned(a.out.ptr)) return fail(BIN_ERR_ARG, "conv: P8 tensor not 16-byte aligned");   // 16-byte pixel stores
  } else if (a.epilogue == BIN_EPI_FINAL) {
    if (a.fr.ncalls < 1 || a.fr.ncalls > BIN_MAX_CALLS || a.fr.nframes < 1 || a.fr.nframes > BIN_MAX_FRAMES ||
        a.fr.Bc < 1 || a.fr.ncalls * a.fr.Bc != B)
      return fail(BIN_ERR_ARG, "conv: frame table does not match the batch");
  }
  // ---- pointers
  if (!a.in0.ptr || (has_in1 && !a.in1.ptr)) return fail(BIN_ERR_ARG, "conv: null input tensor");
  if (misaligned(a.in0.ptr) || (has_in1 && misaligned(a.in1.ptr))) return fail(BIN_ERR_ARG, "conv: P8 tensor not 16-byte aligned");
  if (!a.w_packed || !a.bias) return fail(BIN_ERR_ARG, "conv: null weights or bias");
  if (a.epilogue != BIN_EPI_FINAL && !a.out.ptr) return fail(BIN_ERR_ARG, "conv: null output tensor");
  if (a.epilogue == BIN_EPI_FINAL)
    for (int k = 0; k < a.fr.ncalls; ++k) {
      bool ok = a.fr.out[k] != nullptr;
      for (int fi = 0; fi < a.fr.nframes; ++fi) ok = ok && a.fr.frame[k][fi] != nullptr;
      if (!ok) return fail(BIN_ERR_ARG, "conv: null frame or output pointer in the frame table");
    }
  // ---- the instantiation
  if (a.epilogue == BIN_EPI_P8) {
    if (sx) return launch_inst<32, 3, BIN_EPI_P8, true, X3>(a, s);
    if (a.ksize == 3 && a.cout_pad == 32 && a.variant == BIN_CONV_PLAIN && !X3) return launch_inst<32, 3, BIN_EPI_P8, false, false>(a, s);
    if (a.ksize == 3 && a.cout_pad % 96 == 0) return launch_inst<96, 3, BIN_EPI_P8, false, X3>(a, s);
    if (a.ksize == 5 && a.cout_pad == 96) return launch_inst<96, 5, BIN_EPI_P8, false, X3>(a, s);
    if (a.ksize == 1 && a.cout_pad % 96 == 0) return launch_inst<96, 1, BIN_EPI_P8, false, X3>(a, s);
    // G0 = 64 backbones: SFENet1 (5x5), SFENet2 and GFF.1 (3x3), GFF.0 and the LFF (1x1)
    if (a.ksize == 3 && a.cout_pad == 64) return launch_inst<64, 3, BIN_EPI_P8, false, X3>(a, s);
    if (a.ksize == 5 && a.cout_pad == 64) return launch_inst<64, 5, BIN_EPI_P8, false, X3>(a, s);
    if (a.ksize == 1 && a.cout_pad == 64) return launch_inst<64, 1, BIN_EPI_P8, false, X3>(a, s);
  } else if (a.epilogue == BIN_EPI_PIXSHUF) {
    if (a.ksize == 3 && a.cout_pad == 256) return launch_inst<128, 3, BIN_EPI_PIXSHUF, false, X3>(a, s);
  } else if (a.epilogue == BIN_EPI_FINAL) {
    if (a.ksize == 3 && a.cout_pad == 16 && a.variant == BIN_CONV_DEFAULT) return launch_inst<16, 3, BIN_EPI_FINAL, true, X3>(a, s);
    if (a.ksize == 3 && a.cout_pad == 16 && a.variant == BIN_CONV_PLAIN && !X3) return launch_inst<16, 3, BIN_EPI_FINAL, false, false>(a, s);
  }
  return fail(BIN_ERR_UNSUPPORTED, "conv: no kernel instantiation for this conv (ksize/cout_pad/epilogue/precision)");
}

int launch_conv(const bin_conv_args_t& a, cudaStream_t s) {
  return a.x3 ? launch_conv_t<true>(a, s) : launch_conv_t<false>(a, s);
}

}  // namespace binb
