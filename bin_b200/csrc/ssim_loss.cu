// Fused SSIM loss of the training step (pixel_criterion 'cb+ssim', DESIGN §4r): for npairs fp32 pairs (a_k, b_k) of one
// shape (planes = B * C image planes of h x w), the sum over every plane and valid position p of the SSIM map
//   S = (2 mu_a mu_b + C1)(2 s_ab + C2) / ((mu_a^2 + mu_b^2 + C1)(s_aa + s_bb + C2)),
// mu = G * x, s_xy = G * (x y) - mu_x mu_y, with G the 11 x 11 window outer(g, g) of utils/util.py:211-231 (valid
// correlation: (h - 10)(w - 10) positions per plane), C1 = 0.01^2, C2 = 0.03^2 (data range 1).
//
// ssim_fwd_kernel: one CTA per 32 x 32 block of valid positions of one plane of one pair.  It stages the 42 x 42 pixels
// the block reads (the block plus a 10-pixel halo) of both images in shared memory, runs the horizontal 11-tap pass of
// the five moments a, b, a^2, b^2, ab into shared memory, then the vertical pass and the map per position.  Each CTA adds
// its positions in a fixed tree and writes one partial (BIN_DETERMINISTIC: ssim_reduce_kernel adds a pair's partials in
// index order) or adds it to the pair's sum with a float atomic.  With `maps`, it also keeps the derivatives of S with
// respect to the raw filtered moments,
//   alpha_a = dS/d(G*a), alpha_b = dS/d(G*b), beta = dS/d(G*a^2) = dS/d(G*b^2), gamma = dS/d(G*ab),
// so the backward does not recompute the moments.
//
// ssim_bwd_kernel: one CTA per 32 x 32 block of pixels of one plane of one pair.  With F = G (*) map, the full
// correlation of a map with the window (zero outside the valid positions):
//   dS/da = F(alpha_a) + 2 a F(beta) + b F(gamma),   dS/db = F(alpha_b) + 2 b F(beta) + a F(gamma),
// each times the pair's upstream weight, ADDED to da_k / db_k (which bin_pixel_loss_bwd writes first).  Every pixel has
// one writer, so the backward is deterministic in either mode.
#include <stdint.h>
#include <string.h>

#include "gauss11.cuh"
#include "internal.h"

namespace binb {

constexpr int kSTile = 32;                    // positions (forward) / pixels (backward) per CTA side
constexpr int kSRows = kSTile + 10;           // staged rows and columns: the block and the window's 10-pixel reach
constexpr int kSThreads = 256;
constexpr int kSRedThreads = 256;
constexpr int kSMaps = 4;                     // alpha_a, alpha_b, beta, gamma
constexpr float kSC1 = 0.01f * 0.01f, kSC2 = 0.03f * 0.03f;

struct SsimPairs {
  const float* a[BIN_MAX_LOSS_PAIRS];
  const float* b[BIN_MAX_LOSS_PAIRS];
  float* da[BIN_MAX_LOSS_PAIRS];
  float* db[BIN_MAX_LOSS_PAIRS];
};

struct SsimFwdSmem {
  float a[kSRows][kSRows], b[kSRows][kSRows];
  float h[5][kSRows][kSTile];   // horizontal sums of a, b, a^2, b^2, ab
};
struct SsimBwdSmem {
  float m[kSMaps][kSRows][kSRows];
  float h[kSMaps][kSRows][kSTile];
};

__device__ __forceinline__ void gauss11_f32(float (&g)[11]) {
#pragma unroll
  for (int t = 0; t < 11; ++t) g[t] = (float)kGauss11[t];
}

// grid (tiles, planes, npairs); tile = ty * tiles_x + tx over the (h - 10) x (w - 10) valid positions
__global__ void __launch_bounds__(kSThreads) ssim_fwd_kernel(const __grid_constant__ SsimPairs P, int planes, int h, int w,
                                                             int tiles_x, float* __restrict__ sums,
                                                             float* __restrict__ partial, float* __restrict__ maps) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SsimFwdSmem& S = *reinterpret_cast<SsimFwdSmem*>(smem_raw);
  const int tid = threadIdx.x, plane = blockIdx.y, k = blockIdx.z;
  const int y0 = (blockIdx.x / tiles_x) * kSTile, x0 = (blockIdx.x % tiles_x) * kSTile;
  const int hv = h - 10, wv = w - 10;
  const size_t hw = (size_t)h * w;
  const float* A = P.a[k] + plane * hw;
  const float* B = P.b[k] + plane * hw;
  float g[11];
  gauss11_f32(g);

  for (int i = tid; i < kSRows * kSRows; i += kSThreads) {   // pixels past the image feed no valid position
    const int r = i / kSRows, c = i - r * kSRows;
    const int gy = y0 + r, gx = x0 + c;
    const bool in = gy < h && gx < w;
    S.a[r][c] = in ? A[(size_t)gy * w + gx] : 0.f;
    S.b[r][c] = in ? B[(size_t)gy * w + gx] : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < kSRows * kSTile; i += kSThreads) {
    const int r = i / kSTile, j = i - r * kSTile;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, s4 = 0.f;
#pragma unroll
    for (int t = 0; t < 11; ++t) {
      const float xa = S.a[r][j + t], xb = S.b[r][j + t];
      s0 = fmaf(g[t], xa, s0);
      s1 = fmaf(g[t], xb, s1);
      s2 = fmaf(g[t], xa * xa, s2);
      s3 = fmaf(g[t], xb * xb, s3);
      s4 = fmaf(g[t], xa * xb, s4);
    }
    S.h[0][r][j] = s0; S.h[1][r][j] = s1; S.h[2][r][j] = s2; S.h[3][r][j] = s3; S.h[4][r][j] = s4;
  }
  __syncthreads();

  float acc = 0.f;
  const size_t nv = (size_t)hv * wv;
  for (int i = tid; i < kSTile * kSTile; i += kSThreads) {
    const int r = i / kSTile, j = i - r * kSTile;
    const int py = y0 + r, px = x0 + j;
    if (py >= hv || px >= wv) continue;
    float ma = 0.f, mb = 0.f, saa = 0.f, sbb = 0.f, sab = 0.f;
#pragma unroll
    for (int t = 0; t < 11; ++t) {
      ma = fmaf(g[t], S.h[0][r + t][j], ma);
      mb = fmaf(g[t], S.h[1][r + t][j], mb);
      saa = fmaf(g[t], S.h[2][r + t][j], saa);
      sbb = fmaf(g[t], S.h[3][r + t][j], sbb);
      sab = fmaf(g[t], S.h[4][r + t][j], sab);
    }
    const float mab = ma * mb, maa = ma * ma, mbb = mb * mb;
    const float A1 = 2.f * mab + kSC1, A2 = 2.f * (sab - mab) + kSC2;
    const float B1 = maa + mbb + kSC1, B2 = (saa - maa) + (sbb - mbb) + kSC2;
    const float D = B1 * B2;
    const float s = (A1 * A2) / D;
    acc += s;
    if (maps) {
      // dS/dmu_a = 2 mu_b (A2 - A1) / D + 2 mu_a S (B1 - B2) / D (through A1, A2, B1, B2); dS/ds_aa = -S / B2
      const float inv = 1.f / D;
      const float u = (A2 - A1) * inv, v = s * (B1 - B2) * inv;
      const size_t off = ((size_t)k * kSMaps * planes + plane) * nv + (size_t)py * wv + px, mstride = (size_t)planes * nv;
      maps[off] = 2.f * (mb * u + ma * v);
      maps[off + mstride] = 2.f * (ma * u + mb * v);
      maps[off + 2 * mstride] = -s / B2;
      maps[off + 3 * mstride] = 2.f * A1 * inv;
    }
  }
  // fixed tree over the CTA: lanes by xor shuffle, then the warps in index order
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float red[kSThreads / 32];
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int wv2 = 0; wv2 < kSThreads / 32; ++wv2) t += red[wv2];
    if (partial) partial[((size_t)k * planes + plane) * gridDim.x + blockIdx.x] = t;
    else atomicAdd(sums + k, t);
  }
}

// one CTA per pair: its planes * tiles partials in index order, then a fixed tree
__global__ void __launch_bounds__(kSRedThreads) ssim_reduce_kernel(const float* __restrict__ partial, int nparts,
                                                                   float* __restrict__ sums) {
  const float* p = partial + (size_t)blockIdx.x * nparts;
  float v = 0.f;
  for (int i = threadIdx.x; i < nparts; i += kSRedThreads) v += p[i];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ float red[kSRedThreads / 32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < kSRedThreads / 32; ++i) t += red[i];
    sums[blockIdx.x] = t;
  }
}

// grid (tiles, planes, npairs); tile = ty * tiles_x + tx over the h x w pixels
__global__ void __launch_bounds__(kSThreads) ssim_bwd_kernel(const __grid_constant__ SsimPairs P, int planes, int h, int w,
                                                             int tiles_x, const float* __restrict__ maps,
                                                             const float* __restrict__ upstream) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SsimBwdSmem& S = *reinterpret_cast<SsimBwdSmem*>(smem_raw);
  const int tid = threadIdx.x, plane = blockIdx.y, k = blockIdx.z;
  const int y0 = (blockIdx.x / tiles_x) * kSTile, x0 = (blockIdx.x % tiles_x) * kSTile;
  const int hv = h - 10, wv = w - 10;
  const size_t nv = (size_t)hv * wv, mstride = (size_t)planes * nv;
  const float* M = maps + ((size_t)k * kSMaps * planes + plane) * nv;
  float g[11];
  gauss11_f32(g);

  // positions y0-10 .. y0+31, x0-10 .. x0+31 reach the block's pixels; the ones outside the valid region are 0
  for (int i = tid; i < kSRows * kSRows; i += kSThreads) {
    const int r = i / kSRows, c = i - r * kSRows;
    const int py = y0 - 10 + r, px = x0 - 10 + c;
    const bool in = py >= 0 && py < hv && px >= 0 && px < wv;
    const size_t off = in ? (size_t)py * wv + px : 0;
#pragma unroll
    for (int m = 0; m < kSMaps; ++m) S.m[m][r][c] = in ? M[m * mstride + off] : 0.f;
  }
  __syncthreads();
  // pixel column x0+j is reached by positions x0+j-10 .. x0+j, staged columns j .. j+10 (g is symmetric)
  for (int i = tid; i < kSRows * kSTile; i += kSThreads) {
    const int r = i / kSTile, j = i - r * kSTile;
    float s[kSMaps] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 11; ++t) {
#pragma unroll
      for (int m = 0; m < kSMaps; ++m) s[m] = fmaf(g[t], S.m[m][r][j + t], s[m]);
    }
#pragma unroll
    for (int m = 0; m < kSMaps; ++m) S.h[m][r][j] = s[m];
  }
  __syncthreads();

  const float u = upstream[k];
  const size_t hw = (size_t)h * w;
  const float* A = P.a[k] + plane * hw;
  const float* B = P.b[k] + plane * hw;
  float* dA = P.da[k] ? P.da[k] + plane * hw : nullptr;
  float* dB = P.db[k] ? P.db[k] + plane * hw : nullptr;
  for (int i = tid; i < kSTile * kSTile; i += kSThreads) {
    const int r = i / kSTile, j = i - r * kSTile;
    const int y = y0 + r, x = x0 + j;
    if (y >= h || x >= w) continue;
    float f[kSMaps] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 11; ++t) {
#pragma unroll
      for (int m = 0; m < kSMaps; ++m) f[m] = fmaf(g[t], S.h[m][r + t][j], f[m]);
    }
    const size_t o = (size_t)y * w + x;
    const float va = A[o], vb = B[o];
    if (dA) dA[o] += u * (f[0] + 2.f * va * f[2] + vb * f[3]);
    if (dB) dB[o] += u * (f[1] + 2.f * vb * f[2] + va * f[3]);
  }
}

static inline int ssim_tiles(int n) { return (n + kSTile - 1) / kSTile; }

static bool ssim_shape_ok(int npairs, int planes, int h, int w) {
  return npairs >= 1 && npairs <= BIN_MAX_LOSS_PAIRS && planes >= 1 && planes <= 65535 && h >= 11 && w >= 11 &&
         h <= 65535 && w <= 65535;
}

size_t ssim_loss_scratch_bytes(int npairs, int planes, int h, int w) {
  if (!ssim_shape_ok(npairs, planes, h, w)) return 0;
  return (size_t)npairs * planes * ssim_tiles(h - 10) * ssim_tiles(w - 10) * sizeof(float);
}

size_t ssim_loss_maps_bytes(int npairs, int planes, int h, int w) {
  if (!ssim_shape_ok(npairs, planes, h, w)) return 0;
  return (size_t)npairs * kSMaps * planes * (h - 10) * (w - 10) * sizeof(float);
}

static int ssim_check(const char* fn, const float* const* a, const float* const* b, int npairs, int planes, int h, int w) {
  const std::string f = fn;
  if (!a || !b) return fail(BIN_ERR_ARG, f + ": null pointer table");
  if (npairs < 1 || npairs > BIN_MAX_LOSS_PAIRS) return fail(BIN_ERR_ARG, f + ": npairs must be 1..BIN_MAX_LOSS_PAIRS");
  if (h < 11 || w < 11) return fail(BIN_ERR_ARG, f + ": h and w must be at least 11 (the 11x11 SSIM window)");
  if (planes < 1 || planes > 65535 || h > 65535 || w > 65535)
    return fail(BIN_ERR_ARG, f + ": planes, h and w must be at most 65535");
  for (int k = 0; k < npairs; ++k)
    if (!a[k] || !b[k]) return fail(BIN_ERR_ARG, f + ": null image pointer");
  return BIN_OK;
}

int launch_ssim_loss_fwd(const float* const* a, const float* const* b, int npairs, int planes, int h, int w, float* sums,
                         float* maps, int flags, void* scratch, size_t scratch_bytes, cudaStream_t s) {
  BIN_TRY(ssim_check("ssim_loss_fwd", a, b, npairs, planes, h, w));
  if (!sums) return fail(BIN_ERR_ARG, "ssim_loss_fwd: null output");
  if (flags & ~BIN_DETERMINISTIC) return fail(BIN_ERR_ARG, "ssim_loss_fwd: unknown flags");
  const bool det = flags & BIN_DETERMINISTIC;
  if (det && !scratch) return fail(BIN_ERR_ARG, "ssim_loss_fwd: BIN_DETERMINISTIC needs a scratch buffer");
  if (det && scratch_bytes < ssim_loss_scratch_bytes(npairs, planes, h, w))
    return fail(BIN_ERR_WORKSPACE, "ssim_loss_fwd: scratch too small (see bin_ssim_loss_scratch_bytes)");
  SsimPairs P;
  memset(&P, 0, sizeof(P));
  for (int k = 0; k < npairs; ++k) { P.a[k] = a[k]; P.b[k] = b[k]; }
  static std::atomic<unsigned long long> smem_mask{0};
  BIN_TRY(ensure_dynamic_smem(ssim_fwd_kernel, (int)sizeof(SsimFwdSmem), smem_mask));
  const int tx = ssim_tiles(w - 10), ntiles = tx * ssim_tiles(h - 10);
  const dim3 grid(ntiles, planes, npairs);
  if (det) {                                   // every sums[k] has one writer: no memset, no atomics
    ssim_fwd_kernel<<<grid, kSThreads, sizeof(SsimFwdSmem), s>>>(P, planes, h, w, tx, sums, (float*)scratch, maps);
    BIN_CUDA_OK(cudaGetLastError());
    ssim_reduce_kernel<<<npairs, kSRedThreads, 0, s>>>((const float*)scratch, planes * ntiles, sums);
    BIN_CUDA_OK(cudaGetLastError());
    return BIN_OK;
  }
  BIN_CUDA_OK(cudaMemsetAsync(sums, 0, npairs * sizeof(float), s));
  ssim_fwd_kernel<<<grid, kSThreads, sizeof(SsimFwdSmem), s>>>(P, planes, h, w, tx, sums, nullptr, maps);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

int launch_ssim_loss_bwd(const float* const* a, const float* const* b, const float* maps, float* const* da,
                         float* const* db, int npairs, int planes, int h, int w, const float* upstream, cudaStream_t s) {
  BIN_TRY(ssim_check("ssim_loss_bwd", a, b, npairs, planes, h, w));
  if (!maps || !upstream || !da) return fail(BIN_ERR_ARG, "ssim_loss_bwd: null argument");
  SsimPairs P;
  memset(&P, 0, sizeof(P));
  for (int k = 0; k < npairs; ++k) { P.a[k] = a[k]; P.b[k] = b[k]; P.da[k] = da[k]; P.db[k] = db ? db[k] : nullptr; }
  static std::atomic<unsigned long long> smem_mask{0};
  BIN_TRY(ensure_dynamic_smem(ssim_bwd_kernel, (int)sizeof(SsimBwdSmem), smem_mask));
  const int tx = ssim_tiles(w);
  const dim3 grid(tx * ssim_tiles(h), planes, npairs);
  ssim_bwd_kernel<<<grid, kSThreads, sizeof(SsimBwdSmem), s>>>(P, planes, h, w, tx, maps, upstream);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

}  // namespace binb
