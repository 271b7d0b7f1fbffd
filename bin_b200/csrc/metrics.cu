// Image-quality metrics of the evaluation loop (test.py:404-458) for one pair of uint8 HWC images:
//   sum |a-b| and sum (a-b)^2 (exact, integers), the mean Gaussian-11 SSIM of utils/util.py:211-231 and the mean
//   box-7 SSIM of skimage <= 0.17 compare_ssim with its defaults.
//
// metrics_tile_batch_kernel: one CTA per kTile x kTile block of the image and pair.  It stages the block plus a 5-pixel
// halo of both images in shared memory, then per channel runs the horizontal passes of both windows (Gaussian in fp64,
// box in int32: exact) into shared memory and the vertical passes over the valid outputs of the block.  Each CTA writes
// its four partial sums to the workspace; metrics_reduce_batch_kernel adds each pair's in tile order.  A single pair is a
// batch of one, so each pair of a batch gets the single call's bits.  The grid depends only on (n, h, w), every sum has a
// fixed order, so the result is bit-reproducible and independent of the SM count.
#include <stdint.h>

#include "gauss11.cuh"
#include "internal.h"

namespace binb {

constexpr int kTile = 32;                 // output pixels per CTA side
constexpr int kHalo = 5;                  // Gaussian radius (the box radius, 3, fits inside)
constexpr int kRows = kTile + 2 * kHalo;  // staged rows / columns
constexpr int kMetThreads = 256;
constexpr int kRedThreads = 512;

struct MetricsPartial {
  unsigned long long abs_sum, sq_sum;
  double gauss_sum, box_sum;
};

struct MetricsSmem {
  uint8_t a[3][kRows][kRows], b[3][kRows][kRows];  // channel-planar copy of the staged block
  double hg[5][kRows][kTile];                      // horizontal Gaussian sums of a, b, a^2, b^2, ab
  int hb[5][kRows][kTile];                         // horizontal 7-tap box sums of the same
};

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* red) {   // fixed tree: deterministic for a fixed blockDim
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[warp] = v;
  __syncthreads();
  T t = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < nw; ++i) t += red[i];
  return t;   // valid in thread 0
}

// One tile of one pair; bgr stages source channel 2-ch as channel ch (c = 3), so the per-thread channel loop sums in RGB
// order over a BGR image.
__device__ __forceinline__ void metrics_tile(const uint8_t* __restrict__ A, const uint8_t* __restrict__ B, int h, int w,
                                             int c, bool bgr, MetricsPartial* __restrict__ part) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  MetricsSmem& S = *reinterpret_cast<MetricsSmem*>(smem_raw);
  const int tid = threadIdx.x;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;

  // stage rows y0-5 .. y0+36 and columns x0-5 .. x0+36 (pixels outside the image are 0 and feed no valid output)
  const int rowbytes = kRows * c;
  for (int i = tid; i < kRows * rowbytes; i += kMetThreads) {
    const int r = i / rowbytes, k = i - r * rowbytes;
    const int px = k / c, ch = k - px * c;
    const int gy = y0 - kHalo + r, gx = x0 - kHalo + px;
    uint8_t va = 0, vb = 0;
    if (gy >= 0 && gy < h && gx >= 0 && gx < w) {
      const size_t off = ((size_t)gy * w + gx) * c + ch;
      va = A[off];
      vb = B[off];
    }
    const int sc = bgr ? 2 - ch : ch;
    S.a[sc][r][px] = va;
    S.b[sc][r][px] = vb;
  }
  __syncthreads();

  unsigned long long abs_acc = 0, sq_acc = 0;
  double g_acc = 0.0, b_acc = 0.0;
  constexpr double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  for (int ch = 0; ch < c; ++ch) {
    // horizontal passes: output column j of the block is staged column j+5
    for (int i = tid; i < kRows * kTile; i += kMetThreads) {
      const int r = i / kTile, j = i - r * kTile;
      double g0 = 0, g1 = 0, g2 = 0, g3 = 0, g4 = 0;
      int b0 = 0, b1 = 0, b2 = 0, b3 = 0, b4 = 0;
#pragma unroll
      for (int t = 0; t < 11; ++t) {
        const int xa = S.a[ch][r][j + t], xb = S.b[ch][r][j + t];
        const double wt = kGauss11[t];
        g0 = fma(wt, (double)xa, g0);
        g1 = fma(wt, (double)xb, g1);
        g2 = fma(wt, (double)(xa * xa), g2);
        g3 = fma(wt, (double)(xb * xb), g3);
        g4 = fma(wt, (double)(xa * xb), g4);
        if (t >= 2 && t <= 8) { b0 += xa; b1 += xb; b2 += xa * xa; b3 += xb * xb; b4 += xa * xb; }
      }
      S.hg[0][r][j] = g0; S.hg[1][r][j] = g1; S.hg[2][r][j] = g2; S.hg[3][r][j] = g3; S.hg[4][r][j] = g4;
      S.hb[0][r][j] = b0; S.hb[1][r][j] = b1; S.hb[2][r][j] = b2; S.hb[3][r][j] = b3; S.hb[4][r][j] = b4;
    }
    __syncthreads();
    // vertical passes + per-pixel terms over the kTile x kTile outputs of the block
    for (int i = tid; i < kTile * kTile; i += kMetThreads) {
      const int r = i / kTile, j = i - r * kTile;
      const int gy = y0 + r, gx = x0 + j;
      if (gy >= h || gx >= w) continue;
      const int d = (int)S.a[ch][r + kHalo][j + kHalo] - (int)S.b[ch][r + kHalo][j + kHalo];
      abs_acc += (unsigned)(d < 0 ? -d : d);
      sq_acc += (unsigned)(d * d);
      if (gy >= 5 && gy < h - 5 && gx >= 5 && gx < w - 5) {   // utils/util.py:220 [5:-5, 5:-5]
        double m1 = 0, m2 = 0, s11 = 0, s22 = 0, s12 = 0;
#pragma unroll
        for (int t = 0; t < 11; ++t) {
          const double wt = kGauss11[t];
          m1 = fma(wt, S.hg[0][r + t][j], m1);
          m2 = fma(wt, S.hg[1][r + t][j], m2);
          s11 = fma(wt, S.hg[2][r + t][j], s11);
          s22 = fma(wt, S.hg[3][r + t][j], s22);
          s12 = fma(wt, S.hg[4][r + t][j], s12);
        }
        const double mu1_sq = m1 * m1, mu2_sq = m2 * m2, mu1_mu2 = m1 * m2;
        const double sigma1_sq = s11 - mu1_sq, sigma2_sq = s22 - mu2_sq, sigma12 = s12 - mu1_mu2;
        g_acc += ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2));
      }
      if (gy >= 3 && gy < h - 3 && gx >= 3 && gx < w - 3) {   // skimage crop(S, (7-1)//2)
        int sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
        for (int t = 2; t <= 8; ++t) {
          sx += S.hb[0][r + t][j]; sy += S.hb[1][r + t][j];
          sxx += S.hb[2][r + t][j]; syy += S.hb[3][r + t][j]; sxy += S.hb[4][r + t][j];
        }
        // u = S/49, v = 49/48 (Sxx/49 - (Sx/49)^2) = (49 Sxx - Sx^2) / (49*48): every numerator is an exact integer
        const double ux_uy = (double)(sx * sy) / 2401.0, ux2_uy2 = (double)(sx * sx + sy * sy) / 2401.0;
        const double vx_vy = (double)(49 * (sxx + syy) - sx * sx - sy * sy) / 2352.0;
        const double vxy = (double)(49 * sxy - sx * sy) / 2352.0;
        b_acc += ((2 * ux_uy + C1) * (2 * vxy + C2)) / ((ux2_uy2 + C1) * (vx_vy + C2));
      }
    }
    __syncthreads();
  }

  __shared__ unsigned long long red_u[kMetThreads / 32];
  __shared__ double red_d[kMetThreads / 32];
  MetricsPartial p;
  p.abs_sum = block_sum(abs_acc, red_u);
  p.sq_sum = block_sum(sq_acc, red_u);
  p.gauss_sum = block_sum(g_acc, red_d);
  p.box_sum = block_sum(b_acc, red_d);
  if (tid == 0) part[blockIdx.y * gridDim.x + blockIdx.x] = p;
}

struct MetricsPairs {
  const uint8_t* a[BIN_METRICS_MAX_BATCH];
  const uint8_t* b[BIN_METRICS_MAX_BATCH];
};

// blockIdx.z = pair; pair z's tiles occupy part[z * ntiles, (z + 1) * ntiles) in row-major tile order.
__global__ void __launch_bounds__(kMetThreads) metrics_tile_batch_kernel(const MetricsPairs pairs, int h, int w, int c, int bgr,
                                                                         MetricsPartial* __restrict__ part) {
  const int z = blockIdx.z;
  metrics_tile(pairs.a[z], pairs.b[z], h, w, c, bgr != 0, part + (size_t)z * gridDim.x * gridDim.y);
}

__device__ __forceinline__ void metrics_reduce(const MetricsPartial* __restrict__ part, int ntiles, double n_gauss,
                                               double n_box, double* __restrict__ out4) {
  unsigned long long a = 0, q = 0;
  double g = 0.0, bx = 0.0;
  for (int i = threadIdx.x; i < ntiles; i += kRedThreads) {
    const MetricsPartial p = part[i];
    a += p.abs_sum; q += p.sq_sum; g += p.gauss_sum; bx += p.box_sum;
  }
  __shared__ unsigned long long red_u[kRedThreads / 32];
  __shared__ double red_d[kRedThreads / 32];
  a = block_sum(a, red_u);
  q = block_sum(q, red_u);
  g = block_sum(g, red_d);
  bx = block_sum(bx, red_d);
  if (threadIdx.x == 0) {
    out4[0] = (double)a;   // < 2^31 * 255: exact
    out4[1] = (double)q;   // < 2^31 * 65025 < 2^53: exact
    out4[2] = n_gauss > 0 ? g / n_gauss : __longlong_as_double(0x7ff8000000000000ll);   // numpy's empty-slice mean
    out4[3] = bx / n_box;
  }
}

// One CTA per pair: a tile-order sum over that pair's slice.
__global__ void __launch_bounds__(kRedThreads) metrics_reduce_batch_kernel(const MetricsPartial* __restrict__ part, int ntiles,
                                                                           double n_gauss, double n_box,
                                                                           double* __restrict__ out) {
  metrics_reduce(part + (size_t)blockIdx.x * ntiles, ntiles, n_gauss, n_box, out + 4 * blockIdx.x);
}

static inline int metrics_ntiles(int h, int w) { return ((h + kTile - 1) / kTile) * ((w + kTile - 1) / kTile); }

size_t metrics_workspace_bytes(int h, int w) {
  if (h < 7 || w < 7 || h > 65535 || w > 65535) return 0;
  return (size_t)metrics_ntiles(h, w) * sizeof(MetricsPartial);
}

size_t metrics_batch_workspace_bytes(int n, int h, int w) {
  if (n < 1 || n > BIN_METRICS_MAX_BATCH) return 0;
  return (size_t)n * metrics_workspace_bytes(h, w);
}

// bin_image_metrics_u8: a batch of one pair.  Its NULL a or b is reported before the one-entry tables exist.
int launch_image_metrics_u8(const uint8_t* a, const uint8_t* b, int h, int w, int c, double* out4, void* workspace,
                            size_t workspace_bytes, cudaStream_t s) {
  if (!a || !b) return fail(BIN_ERR_ARG, "image_metrics: null argument");
  return launch_image_metrics_batch_u8("image_metrics", &a, &b, 1, h, w, c, 0, out4, workspace, workspace_bytes, s);
}

int launch_image_metrics_batch_u8(const char* who, const uint8_t* const* a_host, const uint8_t* const* b_host, int n, int h,
                                  int w, int c, int flags, double* out, void* workspace, size_t workspace_bytes,
                                  cudaStream_t s) {
  // every check precedes the first CUDA call
  const std::string fn = who;
  if (!a_host || !b_host) return fail(BIN_ERR_ARG, fn + ": null pointer table");
  if (n < 1 || n > BIN_METRICS_MAX_BATCH) return fail(BIN_ERR_ARG, fn + ": n must be 1..BIN_METRICS_MAX_BATCH");
  if (flags & ~BIN_METRICS_BGR) return fail(BIN_ERR_ARG, fn + ": unknown flag");
  if ((flags & BIN_METRICS_BGR) && c != 3) return fail(BIN_ERR_ARG, fn + ": BIN_METRICS_BGR needs c = 3");
  if (!out || !workspace) return fail(BIN_ERR_ARG, fn + ": null argument");
  if (c != 1 && c != 3) return fail(BIN_ERR_ARG, fn + ": c must be 1 or 3");
  if (h < 7 || w < 7) return fail(BIN_ERR_ARG, fn + ": h and w must be at least 7 (the 7x7 SSIM window)");
  if (h > 65535 || w > 65535 || (long long)h * w * c >= (1ll << 31))
    return fail(BIN_ERR_ARG, fn + ": image too large (h, w <= 65535 and h*w*c < 2^31)");
  if ((reinterpret_cast<uintptr_t>(workspace) & 7) || (reinterpret_cast<uintptr_t>(out) & 7))
    return fail(BIN_ERR_ARG, fn + ": workspace and the output must be 8-byte aligned");
  if (workspace_bytes < metrics_batch_workspace_bytes(n, h, w))
    return fail(BIN_ERR_ARG, fn + ": workspace too small (see bin_" + fn + "_workspace_bytes)");
  MetricsPairs pairs = {};
  for (int i = 0; i < n; ++i) {
    if (!a_host[i] || !b_host[i]) return fail(BIN_ERR_ARG, fn + ": null image pointer");
    pairs.a[i] = a_host[i];
    pairs.b[i] = b_host[i];
  }

  static std::atomic<unsigned long long> smem_mask{0};
  BIN_TRY(ensure_dynamic_smem(metrics_tile_batch_kernel, (int)sizeof(MetricsSmem), smem_mask));
  MetricsPartial* part = static_cast<MetricsPartial*>(workspace);
  const dim3 grid((w + kTile - 1) / kTile, (h + kTile - 1) / kTile, n);
  metrics_tile_batch_kernel<<<grid, kMetThreads, sizeof(MetricsSmem), s>>>(pairs, h, w, c, flags & BIN_METRICS_BGR, part);
  BIN_CUDA_OK(cudaGetLastError());
  const double n_gauss = (h >= 11 && w >= 11) ? (double)c * (h - 10) * (w - 10) : 0.0;
  const double n_box = (double)c * (h - 6) * (w - 6);
  metrics_reduce_batch_kernel<<<n, kRedThreads, 0, s>>>(part, metrics_ntiles(h, w), n_gauss, n_box, out);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}

}  // namespace binb
