// bin_b200 -- memory-bound helper kernels: layout conversion, input packer (space-to-depth),
// weight packer, ConvLSTM cell.
#include <climits>

#include "common.cuh"
#include "internal.h"

namespace binb {

// ------------------------------------------------------------------ fp32 NCHW <-> P8 fp16
__global__ void nchw_to_p8_kernel(const float* __restrict__ x, int C, __half* __restrict__ dst, int planes,
                                  int plane0, int nplanes, int B, int H, int W) {
  const size_t total = (size_t)B * nplanes * H * W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int xw = i % W;
    const int y = (i / W) % H;
    const int pl = (i / ((size_t)W * H)) % nplanes;
    const int b = i / ((size_t)W * H * nplanes);
    __align__(16) __half v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = pl * 8 + e;
      v[e] = __float2half_rn(c < C ? x[(((size_t)b * C + c) * H + y) * W + xw] : 0.f);
    }
    const size_t off = ((((size_t)b * planes + plane0 + pl) * H + y) * W + xw) * 8;
    *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(v);
  }
}

__global__ void p8_to_nchw_kernel(const __half* __restrict__ src, int planes, int plane0, int C,
                                  float* __restrict__ y_out, int B, int H, int W) {
  const size_t total = (size_t)B * C * H * W;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int xw = i % W;
    const int y = (i / W) % H;
    const int c = (i / ((size_t)W * H)) % C;
    const int b = i / ((size_t)W * H * C);
    const size_t off = ((((size_t)b * planes + plane0 + (c >> 3)) * H + y) * W + xw) * 8 + (c & 7);
    y_out[i] = __half2float(src[off]);
  }
}

// ------------------------------------------------------------------ K3: frame concat + space-to-depth + cast
// Reference: RDN.py:211/269/323 torch.cat(frames,1) then pixel_reshuffle(.,2) (RDN.py:107-132):
// packed channel = (f*3+rgb)*4 + dy*2 + dx for pixel (2y+dy, 2x+dx); zero-padded to dst.planes*8.
// grid = (pixel groups, logical planes, batch); every thread packs kPkU output pixels of ONE 8-channel plane: all of its
// 2 x 2 x kPkU 8-byte loads are issued before the first store (bytes in flight), index math is 32-bit, and consecutive
// threads touch consecutive pixels (256-byte warp rows in, 512-byte warp rows out).
constexpr int kPkU = 4;
__global__ void __launch_bounds__(256) pack_frames_kernel(const __grid_constant__ bin_frames_t fr, int H, int W,
                                                          __half* __restrict__ dst, int planes, int x3) {
  // planes = LOGICAL planes; x3: dst holds hi/lo groups of 4
  const int h = H >> 1, w = W >> 1;
  const int hw = h * w;
  const int pl = blockIdx.y, b = blockIdx.z;
  const int call = b / fr.Bc, bb = b % fr.Bc;
  const int cin = 12 * fr.nframes;
  const float* src[2];
#pragma unroll
  for (int half8 = 0; half8 < 2; ++half8) {              // 4 packed channels = one (frame, rgb) 2x2 patch
    const int c4 = pl * 2 + half8;                       // index of the (f,rgb) pair
    src[half8] = (c4 * 4 < cin) ? fr.frame[call][c4 / 3] + ((size_t)bb * 3 + (c4 % 3)) * H * W : nullptr;
  }
  float2 r[kPkU][2][2];
  int pos[kPkU];
#pragma unroll
  for (int u = 0; u < kPkU; ++u) {
    pos[u] = (blockIdx.x * kPkU + u) * 256 + threadIdx.x;
    const int y = pos[u] / w, x = pos[u] - y * w;
#pragma unroll
    for (int half8 = 0; half8 < 2; ++half8) {
      if (src[half8] != nullptr && pos[u] < hw) {
        const float* q = src[half8] + (size_t)(2 * y) * W + 2 * x;
        r[u][half8][0] = __ldg(reinterpret_cast<const float2*>(q));
        r[u][half8][1] = __ldg(reinterpret_cast<const float2*>(q + W));
      } else {
        r[u][half8][0] = r[u][half8][1] = make_float2(0.f, 0.f);
      }
    }
  }
  const int pplanes = x3 ? 2 * planes : planes;
  const int pp = x3 ? 2 * (pl & ~3) + (pl & 3) : pl;
  __half* base = dst + ((size_t)b * pplanes + pp) * hw * 8;
#pragma unroll
  for (int u = 0; u < kPkU; ++u) {
    if (pos[u] >= hw) continue;
    const float fv[8] = {r[u][0][0].x, r[u][0][0].y, r[u][0][1].x, r[u][0][1].y, r[u][1][0].x, r[u][1][0].y, r[u][1][1].x, r[u][1][1].y};
    __align__(16) __half v[8];
    __align__(16) __half vl[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] = __float2half_rn(fv[e]);
      vl[e] = __float2half_rn(fv[e] - __half2float(v[e]));
    }
    *reinterpret_cast<uint4*>(base + (size_t)pos[u] * 8) = *reinterpret_cast<const uint4*>(v);
    if (x3) *reinterpret_cast<uint4*>(base + (size_t)pos[u] * 8 + (size_t)4 * hw * 8) = *reinterpret_cast<const uint4*>(vl);
  }
}

// ------------------------------------------------------------------ weight packer
// OIHW fp32 -> [nh][chunk][ky][kx][4][NT][8] fp16, or (stackx) [chunk][ky][4][kx*cout_pad+co][8].
// transpose != 0 packs the data-gradient weights instead: V[co'][ci'][ky][kx] = W[ci'][row0+co'][k-1-ky][k-1-kx]
// (a conv with V over dY gives dX for stride-1 / pad k/2 convs), co' < nrows, ci' < cout.
// x3 != 0 (BIN_PREC_F32X3): three slabs per logical chunk -- hi, hi, lo of (w * 2^8) -- matching the kernel's
// x_hi*W_hi + x_lo*W_hi + x_hi*W_lo chunk order.
__device__ __forceinline__ void pack_weight_range(const float* __restrict__ w, int cout, int cin, int ks, int cout_pad, int cin_pad,
                                                  int nt, int stackx, int transpose, int row0, int nrows, int x3,
                                                  __half* __restrict__ dst, size_t first, size_t stride) {
  const int rep = x3 ? 3 : 1;
  const size_t total = (size_t)cout_pad * cin_pad * ks * ks * rep;
  const int nchunks = (cin_pad / kKC) * rep;
  for (size_t i = first; i < total; i += stride) {
    size_t t = i;
    int e, kp, kx, ky, ch, co;
    e = t % 8; t /= 8;
    if (stackx) {
      const int n = t % (ks * cout_pad); t /= (ks * cout_pad);
      kx = n / cout_pad; co = n % cout_pad;
      kp = t % kKPL; t /= kKPL;
      ky = t % ks; t /= ks;
      ch = (int)t;
    } else {
      const int n = t % nt; t /= nt;
      kp = t % kKPL; t /= kKPL;
      kx = t % ks; t /= ks;
      ky = t % ks; t /= ks;
      ch = t % nchunks; t /= nchunks;
      co = (int)t * nt + n;
    }
    const int ci = (ch / rep) * kKC + kp * 8 + e;
    float v = 0.f;
    if (!transpose) {
      if (co < cout && ci < cin) v = w[(((size_t)co * cin + ci) * ks + ky) * ks + kx];
    } else {
      if (co < nrows && ci < cout) v = w[(((size_t)ci * cin + row0 + co) * ks + (ks - 1 - ky)) * ks + (ks - 1 - kx)];
    }
    if (x3) {
      v *= 256.f;
      const __half hi = __float2half_rn(v);
      dst[i] = (ch % 3) < 2 ? hi : __float2half_rn(v - __half2float(hi));
    } else {
      dst[i] = __float2half_rn(v);
    }
  }
}
// All conv weights + biases of one backbone in ONE launch (a training step re-packs 4 backbones x 2 layouts after every
// optimizer step: 720 launches of a per-tensor kernel).  The per-tensor entry points run one-job batches.  Block -> job
// by binary search in the parameter table.
__global__ void __launch_bounds__(256) pack_batch_kernel(const __grid_constant__ PackBatch P) {
  int lo = 0, hi = P.njobs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.job[mid].block0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const PackJob& j = P.job[lo];
  const size_t first = (size_t)((int)blockIdx.x - j.block0) * 256 + threadIdx.x, stride = (size_t)j.nblocks * 256;
  if (j.is_bias) {
    float* d = reinterpret_cast<float*>(j.dst);
    for (size_t i = first; i < (size_t)j.cout_pad; i += stride) d[i] = (int)i < j.cout ? j.src[i] : 0.f;
  } else {
    pack_weight_range(j.src, j.cout, j.cin, j.ks, j.cout_pad, j.cin_pad, j.nt, j.stackx, j.transpose, j.row0, j.nrows, j.x3,
                      reinterpret_cast<__half*>(j.dst), first, stride);
  }
}

// ------------------------------------------------------------------ element-wise helpers of the backward pass
// dst += src on P8 plane ranges (fp16).
// grid = (pixel groups, planes, batch): no 64-bit div/mod per element, two 16-byte pixels in flight per thread
__global__ void __launch_bounds__(256) p8_add_kernel(__half* __restrict__ dst, int dplanes, int dplane0,
                                                     const __half* __restrict__ src, int splanes, int splane0, int hw) {
  const int pl = blockIdx.y, b = blockIdx.z;
  uint4* d = reinterpret_cast<uint4*>(dst + ((size_t)b * dplanes + dplane0 + pl) * (size_t)hw * 8);
  const uint4* sp = reinterpret_cast<const uint4*>(src + ((size_t)b * splanes + splane0 + pl) * (size_t)hw * 8);
  const int p0 = blockIdx.x * 512 + threadIdx.x, p1 = p0 + 256;
  uint4 sv[2], dv[2];
  if (p0 < hw) { sv[0] = __ldg(sp + p0); dv[0] = d[p0]; }
  if (p1 < hw) { sv[1] = __ldg(sp + p1); dv[1] = d[p1]; }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int px = u ? p1 : p0;
    if (px >= hw) continue;
    __half2* dh = reinterpret_cast<__half2*>(&dv[u]);
    const __half2* sh = reinterpret_cast<const __half2*>(&sv[u]);
#pragma unroll
    for (int k = 0; k < 4; ++k) dh[k] = __hadd2(dh[k], sh[k]);
    d[px] = dv[u];
  }
}
// ReLU backward: dg *= (g > 0), both P8 plane ranges.
__global__ void __launch_bounds__(256) p8_relu_mask_kernel(__half* __restrict__ dg, int dplanes, int dplane0,
                                                           const __half* __restrict__ g, int gplanes, int gplane0, int hw) {
  const int pl = blockIdx.y, b = blockIdx.z;
  uint4* d = reinterpret_cast<uint4*>(dg + ((size_t)b * dplanes + dplane0 + pl) * (size_t)hw * 8);
  const uint4* gp = reinterpret_cast<const uint4*>(g + ((size_t)b * gplanes + gplane0 + pl) * (size_t)hw * 8);
  const int p0 = blockIdx.x * 512 + threadIdx.x, p1 = p0 + 256;
  uint4 gv[2], dv[2];
  if (p0 < hw) { gv[0] = __ldg(gp + p0); dv[0] = d[p0]; }
  if (p1 < hw) { gv[1] = __ldg(gp + p1); dv[1] = d[p1]; }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int px = u ? p1 : p0;
    if (px >= hw) continue;
    __half* dh = reinterpret_cast<__half*>(&dv[u]);
    const __half* gh = reinterpret_cast<const __half*>(&gv[u]);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (!(__half2float(gh[k]) > 0.f)) dh[k] = __float2half_rn(0.f);
    d[px] = dv[u];
  }
}
// PixelShuffle(2) backward: dU P8 (B, 8 planes, 2h, 2w) -> d(conv out) P8 (B, 32 planes, h, w), n = 4c+2i+j.
__global__ void pixel_unshuffle_kernel(const __half* __restrict__ du, __half* __restrict__ dst, int B, int h, int w) {
  const size_t total = (size_t)B * 32 * h * w;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = i % w;
    const int y = (i / w) % h;
    const int pl = (i / ((size_t)w * h)) % 32;      // output plane: channels n = pl*8 .. pl*8+7
    const int b = i / ((size_t)w * h * 32);
    __align__(16) __half v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int n = pl * 8 + e, c = n >> 2, ii = (n >> 1) & 1, jj = n & 1;
      v[e] = du[((((size_t)b * 8 + (c >> 3)) * (2 * h) + 2 * y + ii) * (2 * w) + 2 * x + jj) * 8 + (c & 7)];
    }
    *reinterpret_cast<uint4*>(dst + ((((size_t)b * 32 + pl) * h + y) * w + x) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}
// Backward of pack_frames + of the final "+ mean(frames)": for call k, frame f (fp32 NCHW):
//   dframe = inv_scale * depth_to_space(dX0 channels of frame f) + dOut / nframes
// A NULL dfr.frame[call][f] is a frame whose gradient nobody asked for: nothing is written for it.
__global__ void unpack_frames_grad_kernel(const __half* __restrict__ dx0, int planes, const __grid_constant__ bin_frames_t dout,
                                          const __grid_constant__ bin_frames_t dfr, int H, int W, const float* __restrict__ scale) {
  const int h = H / 2, w = W / 2;
  const int Btot = dfr.ncalls * dfr.Bc;
  const size_t total = (size_t)Btot * dfr.nframes * 3 * h * w;
  const float inv = 1.f / scale[0];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = i % w;
    const int y = (i / w) % h;
    const int rgb = (i / ((size_t)w * h)) % 3;
    const int f = (i / ((size_t)w * h * 3)) % dfr.nframes;
    const int b = i / ((size_t)w * h * 3 * dfr.nframes);
    const int call = b / dfr.Bc, bb = b % dfr.Bc;
    if (dfr.frame[call][f] == nullptr) continue;
    const int c4 = (f * 3 + rgb) * 4;                 // packed channels c4..c4+3 = (dy,dx) of this (frame,rgb)
    const __half* src = dx0 + ((((size_t)b * planes + (c4 >> 3)) * h + y) * w + x) * 8 + (c4 & 7);
    const float* go = dout.out[call] + (((size_t)bb * 3 + rgb) * H + 2 * y) * W + 2 * x;
    float* dst = const_cast<float*>(dfr.frame[call][f]) + (((size_t)bb * 3 + rgb) * H + 2 * y) * W + 2 * x;
    const float rn = 1.f / (float)dfr.nframes;
    dst[0] = __half2float(src[0]) * inv + go[0] * rn;
    dst[1] = __half2float(src[1]) * inv + go[1] * rn;
    dst[W] = __half2float(src[2]) * inv + go[W] * rn;
    dst[W + 1] = __half2float(src[3]) * inv + go[W + 1] * rn;
  }
}
// dOut (fp32 NCHW, per call) * scale -> P8 (Btot, 4 planes, H, W), channels 3..31 zero.
__global__ void grad_out_to_p8_kernel(const __grid_constant__ bin_frames_t dout, int H, int W, __half* __restrict__ dst,
                                      const float* __restrict__ scale) {
  const int Btot = dout.ncalls * dout.Bc;
  const size_t hw = (size_t)H * W;
  const size_t total = (size_t)Btot * 4 * hw;
  const float sc = scale[0];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t px = i % hw;
    const int pl = (i / hw) % 4;
    const int b = i / (hw * 4);
    const int call = b / dout.Bc, bb = b % dout.Bc;
    __align__(16) __half v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __float2half_rn(0.f);
    if (pl == 0) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = __float2half_rn(dout.out[call][((size_t)bb * 3 + c) * hw + px] * sc);
    }
    *reinterpret_cast<uint4*>(dst + (((size_t)b * 4 + pl) * hw + px) * 8) = *reinterpret_cast<const uint4*>(v);
  }
}
// ---- deterministic reductions (BIN_DETERMINISTIC): a kernel writes one partial per block, a second launch sums them.
// Warp w of block b owns output 8b + w: lane l adds partials l, l+32, ... in index order, then a fixed xor-shuffle tree
// adds the 32 lane sums.  Partial i of the output is partial[i * istride].  The order depends only on nparts, which
// depends only on the shape, never on which block finished first.
__device__ __forceinline__ float ordered_warp_sum(const float* __restrict__ partial, int nparts, size_t istride) {
  const int lane = threadIdx.x & 31;
  float v = 0.f;
  for (int i = lane; i < nparts; i += 32) v += partial[(size_t)i * istride];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// db[c] += inv_scale * sum over (B, H, W) of dY[c] for P8 planes [plane0, plane0+ceil(C/8)).
// grid = (pixel groups, planes, batch): no 64-bit div/mod per element, 4 independent 16-byte loads in flight per thread.
// partial == NULL: each block adds its sums with atomicAdd; otherwise it writes them to partial [B][blocks_x][C].
__global__ void __launch_bounds__(256) p8_bias_grad_kernel(const __half* __restrict__ dy, int planes, int plane0, int C, int hw,
                                                           const float* __restrict__ scale, float* __restrict__ db,
                                                           float* __restrict__ partial) {
  __shared__ float part[8][8];
  const int pl = blockIdx.y, b = blockIdx.z;
  const __half* base = dy + ((size_t)b * planes + plane0 + pl) * (size_t)hw * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  uint4 v[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int px = (blockIdx.x * 4 + u) * 256 + threadIdx.x;
    v[u] = px < hw ? __ldg(reinterpret_cast<const uint4*>(base + (size_t)px * 8)) : make_uint4(0, 0, 0, 0);
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const __half* h8 = reinterpret_cast<const __half*>(&v[u]);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] += __half2float(h8[k]);
  }
#pragma unroll
  for (int k = 0; k < 8; ++k)
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0)
    for (int k = 0; k < 8; ++k) part[warp][k] = acc[k];
  __syncthreads();
  if (threadIdx.x < 8) {
    float sum = 0.f;
    for (int wv = 0; wv < 8; ++wv) sum += part[wv][threadIdx.x];
    const int c = pl * 8 + threadIdx.x;
    if (c < C) {
      if (partial) partial[((size_t)b * gridDim.x + blockIdx.x) * C + c] = sum;        // [B][blocks_x][C]
      else atomicAdd(db + c, sum / scale[0]);
    }
  }
}
// Deterministic bias gradient: db[c] += (sum of the nparts = B * blocks_x partials of channel c, in index order) / scale.
__global__ void __launch_bounds__(256) bias_grad_reduce_kernel(const float* __restrict__ partial, int nparts, int C,
                                                               const float* __restrict__ scale, float* __restrict__ db) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= C) return;
  const float s = ordered_warp_sum(partial + c, nparts, (size_t)C);
  if ((threadIdx.x & 31) == 0) db[c] += s / scale[0];
}

// ---- loss scale of a backbone's backward (autograd.py): scale = 2^floor(log2(target / max|dOut|)), kept on the device
struct GradPtrs { const float* p[BIN_MAX_CALLS]; int n; };
__global__ void __launch_bounds__(256) grad_absmax_kernel(const __grid_constant__ GradPtrs G, size_t numel, unsigned* __restrict__ bits) {
  const float* g = G.p[blockIdx.y];
  float m = 0.f;
  const size_t n4 = numel / 4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  if (blockIdx.x == 0 && threadIdx.x < (int)(numel & 3)) m = fmaxf(m, fabsf(g[n4 * 4 + threadIdx.x]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(bits, __float_as_uint(m));     // non-negative floats order like their bit patterns
}
// The exponent comes from ilogbf, not from log2f(target / gmax): that quotient rounds to a power of two when gmax is a
// few ulps above one, and the scale came out twice too large.  s = 2^(ilogb(target) - ilogb(gmax)) has s * gmax <= target
// iff gmax's significand is at most target's; halving once otherwise gives s * gmax <= target < 2 s gmax.  Both
// products are exact (s is a power of two, the results are normal).  An all-zero gradient is clamped to 1e-30 (a finite
// scale); an infinite one gives scale 0, so every gradient of that backward is NaN and the optimizer's guard skips it.
__global__ void grad_scale_finalize_kernel(const unsigned* __restrict__ bits, float target, float* __restrict__ scale) {
  const float gmax = fmaxf(__uint_as_float(*bits), 1e-30f);
  if (isinf(gmax)) { *scale = 0.f; return; }
  float s = ldexpf(1.f, ilogbf(target) - ilogbf(gmax));
  if (s * gmax > target) s *= 0.5f;
  *scale = s;
}

// ------------------------------------------------------------------ K5: ConvLSTMCell (RDN.py:50-95)
// g = Conv3x3(cat(x, h)) 6 -> 12 ; i,j,f,o = chunk(g,4) ; c' = c*sigmoid(f+1) + sigmoid(i)*tanh(j) ; h' = tanh(c')*sigmoid(o).
// 648 FMA (324 when prev_state is None: h = 0 contributes nothing, RDN.py:57-68) and 15 transcendentals per pixel against
// 36-60 bytes: arithmetic intensity 36 FLOP/B, above the fp32 CUDA-core ridge (~75 TFLOP/s / 6.5 TB/s = 11.5 FLOP/B) --
// the kernel is FP32-FMA bound, so the design minimises instructions per FMA:
//   * 64 x 16 pixel tile per 256-thread block; the (16+2) x (64+2) halo tile of every input channel is staged once in
//     shared memory (zero fill = the conv's zero padding), so each input value is fetched from DRAM/L2 once;
//   * each thread owns 4 consecutive pixels x 12 gate channels = 48 register accumulators; per (channel, ky) it reads its
//     6 inputs with one 128-bit + one 64-bit shared load and per tap its 12 weights with three 128-bit broadcast loads:
//     48 FMAs per 3 weight loads;
//   * gates use ex2.approx-based sigmoid / tanh (|error| < 3e-7, two decades under the 1e-5 fp32 bar);
//   * up to 3 independent cells (the cells of one recurrent hand-off, RDN.py:451-456) ride one launch in grid.z.
constexpr int kLsTW = 64, kLsTH = 16, kLsPitch = 72;      // smem row: [x0-1 .. x0+64] at index 3..68 -> pixel x0+k at index 4+k
__device__ __forceinline__ float fast_sigmoid(float v) { return __frcp_rn(1.f + __expf(-v)); }
__device__ __forceinline__ float fast_tanh(float v) { return 2.f * __frcp_rn(1.f + __expf(-2.f * v)) - 1.f; }

template <bool STATE>
__global__ void __launch_bounds__(256, STATE ? 2 : 3) convlstm_kernel(const __grid_constant__ LstmCells P, int B, int H, int W, int tiles_x,
                                                       int tiles_y) {
  constexpr int C = STATE ? 6 : 3;
  __shared__ __align__(16) float sin_[C][kLsTH + 2][kLsPitch];
  __shared__ __align__(16) float sw[C * 9 * 12];                 // [c][ky][kx][gate channel]
  __shared__ float sb[12];
  const int cell = blockIdx.z;
  const float* __restrict__ w = P.w[cell];
  for (int i = threadIdx.x; i < C * 9 * 12; i += 256) {
    const int k = i % 12, t = (i / 12) % 9, c = i / 108;
    sw[i] = w[(k * 6 + c) * 9 + t];                              // (12,6,3,3) OIHW
  }
  if (threadIdx.x < 12) sb[threadIdx.x] = P.b[cell][threadIdx.x];
  int t = blockIdx.x;
  const int txi = t % tiles_x; t /= tiles_x;
  const int tyi = t % tiles_y;
  const int b = t / tiles_y;
  const int x0 = txi * kLsTW, y0 = tyi * kLsTH;
  const size_t hw = (size_t)H * W;
  // stage the halo tile: rows y0-1 .. y0+16, columns x0-1 .. x0+64 (index 3 .. 68 of the padded row).  The trip count is a
  // compile-time constant and all loads of a batch are issued before the first shared-memory store, so a thread has up
  // to 14 global loads in flight (a dependent load->store loop ran at one DRAM round trip per element).
  constexpr int kElems = C * (kLsTH + 2) * (kLsTW + 2), kIt = (kElems + 255) / 256, kBatch = 14;
  static_assert(kIt % kBatch == 0, "staging batches");
#pragma unroll 1
  for (int it0 = 0; it0 < kIt; it0 += kBatch) {
    float v[kBatch];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int i = (it0 + u) * 256 + threadIdx.x;
      const int cx = i % (kLsTW + 2), r = (i / (kLsTW + 2)) % (kLsTH + 2), c = i / ((kLsTW + 2) * (kLsTH + 2));
      const int yy = y0 + r - 1, xx = x0 + cx - 1;
      v[u] = 0.f;
      if (i < kElems && yy >= 0 && yy < H && xx >= 0 && xx < W) {
        const float* src = c < 3 ? P.x[cell] + ((size_t)b * 3 + c) * hw : P.h_prev[cell] + ((size_t)b * 3 + (c - 3)) * hw;
        v[u] = __ldg(src + (size_t)yy * W + xx);
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int i = (it0 + u) * 256 + threadIdx.x;
      const int cx = i % (kLsTW + 2), r = (i / (kLsTW + 2)) % (kLsTH + 2), c = i / ((kLsTW + 2) * (kLsTH + 2));
      if (i < kElems) sin_[c][r][3 + cx] = v[u];
    }
  }
  __syncthreads();
  const int tx4 = (threadIdx.x & 15) * 4, ty = threadIdx.x >> 4;
  float acc[4][12];
#pragma unroll
  for (int px = 0; px < 4; ++px)
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[px][k] = sb[k];
#pragma unroll 1
  for (int c = 0; c < C; ++c) {
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const float4* row = reinterpret_cast<const float4*>(&sin_[c][ty + ky][tx4]);   // [3] = pixel tx4-1, [4..7] = the 4 pixels, [8] = +1
      const float4 lo = row[0], a = row[1], hi = row[2];         // three conflict-free 128-bit loads (scalar loads at a
      const float v[6] = {lo.w, a.x, a.y, a.z, a.w, hi.x};       // 4-word thread stride were 2-way bank conflicts)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4* wp = reinterpret_cast<const float4*>(&sw[((c * 3 + ky) * 3 + kx) * 12]);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2];
        const float wk[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
#pragma unroll
        for (int px = 0; px < 4; ++px)
#pragma unroll
          for (int k = 0; k < 12; ++k) acc[px][k] = fmaf(wk[k], v[px + kx], acc[px][k]);
      }
    }
  }
  const int y = y0 + ty, x = x0 + tx4;
  if (y >= H || x >= W) return;
  const bool vec = ((W & 3) == 0) && (x + 3 < W);
#pragma unroll
  for (int c = 0; c < 3; ++c) {                                  // i,j,f,o = chunk(4) (RDN.py:79)
    const size_t off = ((size_t)b * 3 + c) * hw + (size_t)y * W + x;
    float cp[4] = {0.f, 0.f, 0.f, 0.f};
    if (STATE) {
      if (vec) { const float4 q = *reinterpret_cast<const float4*>(P.c_prev[cell] + off); cp[0] = q.x; cp[1] = q.y; cp[2] = q.z; cp[3] = q.w; }
      else {
#pragma unroll
        for (int px = 0; px < 4; ++px) if (x + px < W) cp[px] = P.c_prev[cell][off + px];
      }
    }
    float hn[4], cn[4];
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const float si = fast_sigmoid(acc[px][c]), sf = fast_sigmoid(acc[px][6 + c] + 1.0f);   // forget_bias = 1.0 (RDN.py:16,81)
      const float so = fast_sigmoid(acc[px][9 + c]);
      cn[px] = cp[px] * sf + si * fast_tanh(acc[px][3 + c]);
      hn[px] = fast_tanh(cn[px]) * so;
    }
    if (vec) {
      *reinterpret_cast<float4*>(P.h_out[cell] + off) = make_float4(hn[0], hn[1], hn[2], hn[3]);
      if (P.c_out[cell]) *reinterpret_cast<float4*>(P.c_out[cell] + off) = make_float4(cn[0], cn[1], cn[2], cn[3]);
    } else {
#pragma unroll
      for (int px = 0; px < 4; ++px)
        if (x + px < W) {
          P.h_out[cell][off + px] = hn[px];
          if (P.c_out[cell]) P.c_out[cell][off + px] = cn[px];
        }
    }
  }
}

// ------------------------------------------------------------------ image boundary kernels (SURVEY 8f rank 2)
// utils/util.py:113-137 tensor2img on one (3,Hs,Ws) fp32 RGB image + the crop of test.py:394-402:
// clamp to [0,1], *255, round half to even (numpy .round()), uint8, HWC, BGR.
__global__ void tensor2img_u8_kernel(const float* __restrict__ src, int Hs, int Ws, int top, int left, int h, int w,
                                     uint8_t* __restrict__ dst) {
  const size_t total = (size_t)h * w;
  const size_t hws = (size_t)Hs * Ws;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = i % w, y = i / w;
    const size_t so = (size_t)(y + top) * Ws + (x + left);
#pragma unroll
    for (int c = 0; c < 3; ++c) {                       // dst channel c = BGR -> source channel 2-c
      const float v = fminf(fmaxf(src[(size_t)(2 - c) * hws + so], 0.f), 1.f);
      dst[i * 3 + c] = (uint8_t)rintf(v * 255.0f);
    }
  }
}
// test.py:44-56 read_image (uint8 HWC BGR -> fp32 CHW RGB / 255) fused with the ReplicationPad2d of test.py:366-371.
__global__ void u8_to_frame_kernel(const uint8_t* __restrict__ src, int h, int w, int pl, int pt, int Hp, int Wp,
                                   float* __restrict__ dst) {
  const size_t total = (size_t)Hp * Wp;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int X = i % Wp, Y = i / Wp;
    int x = X - pl, y = Y - pt;
    x = x < 0 ? 0 : (x >= w ? w - 1 : x);
    y = y < 0 ? 0 : (y >= h ? h - 1 : y);
    const uint8_t* px = src + ((size_t)y * w + x) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[(size_t)c * total + i] = (float)px[2 - c] / 255.f;
  }
}

// ------------------------------------------------------------------ fused pixel loss (SURVEY 8f rank 3)
// bin_model.get_loss (bin_model.py:395-425): loss = mean over pairs of cri_pix(a_k, b_k) with cri_pix = L1 sum
// (bin_model.py:55), MSE sum (:57) or Charbonnier mean sqrt(d^2+eps) (loss.py:130-140).  One launch reduces all
// pairs (up to 17: 14 outputs vs GT + 3 cycle terms), one launch writes all gradients.
struct LossPairs {
  const float* a[BIN_MAX_LOSS_PAIRS];
  const float* b[BIN_MAX_LOSS_PAIRS];
  float* da[BIN_MAX_LOSS_PAIRS];
  float* db[BIN_MAX_LOSS_PAIRS];
  int npairs;
};
__device__ __forceinline__ float loss_term(float d, int kind, float eps) {
  return kind == 0 ? fabsf(d) : (kind == 1 ? d * d : sqrtf(d * d + eps));
}
// DET = false: every block adds its sum to pair_loss[k] with atomicAdd (last bits depend on block order).
// DET = true: block x of pair k writes its sum to partial[k][x]; pixel_loss_reduce_kernel adds them in index order.
template <bool DET>
__global__ void pixel_loss_fwd_kernel(const __grid_constant__ LossPairs P, size_t n, int kind, float eps,
                                      float* __restrict__ pair_loss, float* __restrict__ partial) {
  const int k = blockIdx.y;
  const float* a = P.a[k];
  const float* b = P.b[k];
  float acc = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    acc += loss_term(a[i] - b[i], kind, eps);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) s += part[wv];
    if (DET) partial[(size_t)k * gridDim.x + blockIdx.x] = s;
    else atomicAdd(pair_loss + k, kind == 2 ? s / (float)n : s);
  }
}
__global__ void __launch_bounds__(256) pixel_loss_reduce_kernel(const float* __restrict__ partial, int nparts, int npairs,
                                                                int kind, size_t n, float* __restrict__ pair_loss) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (k >= npairs) return;
  const float s = ordered_warp_sum(partial + (size_t)k * nparts, nparts, 1);
  if ((threadIdx.x & 31) == 0) pair_loss[k] = kind == 2 ? s / (float)n : s;          // the Charbonnier mean: one divide
}
// da_k = g * dterm/dd, db_k = -da_k, with g = upstream / npairs (and / n for the Charbonnier mean)
__global__ void pixel_loss_bwd_kernel(const __grid_constant__ LossPairs P, size_t n, int kind, float eps,
                                      const float* __restrict__ upstream) {
  const int k = blockIdx.y;
  const float* a = P.a[k];
  const float* b = P.b[k];
  float* da = P.da[k];
  float* db = P.db[k];
  const float g = upstream[0] / (float)P.npairs * (kind == 2 ? 1.f / (float)n : 1.f);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float d = a[i] - b[i];
    const float t = kind == 0 ? (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) : (kind == 1 ? 2.f * d : d / sqrtf(d * d + eps));
    if (da) da[i] = g * t;
    if (db) db[i] = -g * t;
  }
}

// ------------------------------------------------------------------ ConvLSTMCell backward (fp32)
// Pass 1 (per pixel): recompute the gates (RDN.py:74-82), write d(gate pre-activations) [B,12,H,W] and dc_prev.
__global__ void convlstm_bwd_gates_kernel(const float* __restrict__ x, const float* __restrict__ c_prev,
                                          const float* __restrict__ h_prev, const float* __restrict__ w,
                                          const float* __restrict__ bias, const float* __restrict__ dh,
                                          const float* __restrict__ dc, float* __restrict__ dgates,
                                          float* __restrict__ dc_prev, int B, int H, int W) {
  __shared__ float sw[12 * 6 * 9];
  __shared__ float sb[12];
  for (int i = threadIdx.x; i < 12 * 6 * 9; i += blockDim.x) sw[i] = w[i];
  if (threadIdx.x < 12) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const size_t hw = (size_t)H * W;
  const size_t total = (size_t)B * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int xw = i % W;
    const int y = (i / W) % H;
    const int b = i / hw;
    float g[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) g[k] = sb[k];
    const int nin = h_prev ? 6 : 3;
    for (int c = 0; c < nin; ++c) {
      const float* src = (c < 3 ? x + ((size_t)b * 3 + c) * hw : h_prev + ((size_t)b * 3 + (c - 3)) * hw);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int yy = y + ky - 1;
        if (yy < 0 || yy >= H) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int xx = xw + kx - 1;
          if (xx < 0 || xx >= W) continue;
          const float v = src[(size_t)yy * W + xx];
#pragma unroll
          for (int k = 0; k < 12; ++k) g[k] = fmaf(sw[(k * 6 + c) * 9 + ky * 3 + kx], v, g[k]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const size_t off = ((size_t)b * 3 + c) * hw + (size_t)y * W + xw;
      const float cp = c_prev ? c_prev[off] : 0.f;
      const float si = 1.f / (1.f + expf(-g[c]));
      const float tj = tanhf(g[3 + c]);
      const float sf = 1.f / (1.f + expf(-(g[6 + c] + 1.0f)));
      const float so = 1.f / (1.f + expf(-g[9 + c]));
      const float cn = cp * sf + si * tj;
      const float tc = tanhf(cn);
      const float dhv = dh ? dh[off] : 0.f;
      const float dct = (dc ? dc[off] : 0.f) + dhv * so * (1.f - tc * tc);
      const size_t gb = ((size_t)b * 12) * hw + (size_t)y * W + xw;
      dgates[gb + (size_t)(0 + c) * hw] = dct * tj * si * (1.f - si);          // d i
      dgates[gb + (size_t)(3 + c) * hw] = dct * si * (1.f - tj * tj);          // d j
      dgates[gb + (size_t)(6 + c) * hw] = dct * cp * sf * (1.f - sf);          // d f
      dgates[gb + (size_t)(9 + c) * hw] = dhv * tc * so * (1.f - so);          // d o
      if (dc_prev) dc_prev[off] = dct * sf;
    }
  }
}
// Pass 2: dW[k][c][tap] += sum_p dgates[k][p] * in[c][p+off], db[k] += sum_p dgates[k][p]  (660 outputs).
// 9 warps per block, warp v owns tap v: 72 register accumulators acc[k][c] (all indices compile-time), lanes
// stride over pixels; one warp-shuffle reduction + 72 atomics per warp at the end (warp 0 also sums the biases).
// partial != NULL (deterministic): block x writes its 660 sums to partial[x][660] instead (dw order, then the 12 biases),
// and convlstm_wgrad_reduce_kernel adds the blocks in index order.
constexpr int kLstmGradN = 12 * 6 * 9 + 12;
__global__ void __launch_bounds__(288) convlstm_bwd_weights_kernel(const float* __restrict__ x, const float* __restrict__ h_prev,
                                                                    const float* __restrict__ dgates, float* __restrict__ dw,
                                                                    float* __restrict__ db, int B, int H, int W,
                                                                    float* __restrict__ partial) {
  const size_t hw = (size_t)H * W;
  const size_t total = (size_t)B * hw;
  const int tap = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int dy = tap / 3 - 1, dx = tap % 3 - 1;
  float acc[12][6];
  float accb[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) {
    accb[k] = 0.f;
#pragma unroll
    for (int c = 0; c < 6; ++c) acc[k][c] = 0.f;
  }
  for (size_t p = (size_t)blockIdx.x * 32 + lane; p < total; p += (size_t)gridDim.x * 32) {
    const int xw = p % W, y = (p / W) % H, b = p / hw;
    const int yy = y + dy, xx = xw + dx;
    const bool inb = yy >= 0 && yy < H && xx >= 0 && xx < W;
    float in[6];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      in[c] = inb ? x[((size_t)b * 3 + c) * hw + (size_t)yy * W + xx] : 0.f;
      in[3 + c] = (inb && h_prev) ? h_prev[((size_t)b * 3 + c) * hw + (size_t)yy * W + xx] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      const float d = dgates[((size_t)b * 12 + k) * hw + (size_t)y * W + xw];
      accb[k] += d;
#pragma unroll
      for (int c = 0; c < 6; ++c) acc[k][c] = fmaf(d, in[c], acc[k][c]);
    }
  }
#pragma unroll
  for (int k = 0; k < 12; ++k) {
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      float v = acc[k][c];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) {
        if (partial) partial[(size_t)blockIdx.x * kLstmGradN + (k * 6 + c) * 9 + tap] = v;
        else if (dw) atomicAdd(dw + (k * 6 + c) * 9 + tap, v);
      }
    }
    if (tap == 0) {
      float v = accb[k];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) {
        if (partial) partial[(size_t)blockIdx.x * kLstmGradN + 648 + k] = v;
        else if (db) atomicAdd(db + k, v);
      }
    }
  }
}
__global__ void __launch_bounds__(256) convlstm_wgrad_reduce_kernel(const float* __restrict__ partial, int nparts,
                                                                    float* __restrict__ dw, float* __restrict__ db) {
  const int o = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= kLstmGradN) return;
  const float s = ordered_warp_sum(partial + o, nparts, (size_t)kLstmGradN);
  if ((threadIdx.x & 31) == 0) {
    if (o < 648) { if (dw) dw[o] += s; }
    else if (db) db[o - 648] += s;
  }
}
// Pass 3: dx[c][q] = sum_{k,tap} W[k][c][tap] * dgates[k][q - off(tap)]  (and dh_prev for c = 3..5).
__global__ void convlstm_bwd_input_kernel(const float* __restrict__ dgates, const float* __restrict__ w,
                                          float* __restrict__ dx, float* __restrict__ dh_prev, int B, int H, int W) {
  __shared__ float sw[12 * 6 * 9];
  for (int i = threadIdx.x; i < 12 * 6 * 9; i += blockDim.x) sw[i] = w[i];
  __syncthreads();
  const size_t hw = (size_t)H * W;
  const size_t total = (size_t)B * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int xw = i % W;
    const int y = (i / W) % H;
    const int b = i / hw;
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int yy = y - (ky - 1);                       // output pixel that read this input through tap (ky,kx)
      if (yy < 0 || yy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int xx = xw - (kx - 1);
        if (xx < 0 || xx >= W) continue;
        for (int k = 0; k < 12; ++k) {
          const float d = dgates[((size_t)b * 12 + k) * hw + (size_t)yy * W + xx];
#pragma unroll
          for (int c = 0; c < 6; ++c) acc[c] = fmaf(sw[(k * 6 + c) * 9 + ky * 3 + kx], d, acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const size_t off = ((size_t)b * 3 + c) * hw + (size_t)y * W + xw;
      if (dx) dx[off] = acc[c];
      if (dh_prev) dh_prev[off] = acc[3 + c];
    }
  }
}

// ------------------------------------------------------------------ launch wrappers
// ---------------------------------------------------------------------------------------------------------
// Multi-tensor Adam (SURVEY 8f rank 3): torch.optim.Adam.step as bin_model.py:97-100,141 drives it
// (L2 weight decay folded into the gradient, no amsgrad), one launch over all 540 parameter tensors.
// Block b owns kAdamChunk consecutive elements of tensor t, t = the last entry with chunk_prefix[t] <= b.
// HBM-bound: 16 B read + 12 B written per parameter.
constexpr int kAdamChunk = 4096;
__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float lr_bc1, float b1, float b2,
                                         float eps, float wd, float inv_sqrt_bc2, float gscale) {
  g = g * gscale;
  if (wd != 0.f) g = g + wd * p;                       // grad.add(param, alpha=weight_decay)
  m = m + (g - m) * (1.f - b1);                        // exp_avg.lerp_(grad, 1 - beta1)
  v = v * b2 + (1.f - b2) * g * g;                     // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
  const float denom = sqrtf(v) * inv_sqrt_bc2 + eps;   // (exp_avg_sq.sqrt() / sqrt(bias_correction2)).add_(eps)
  p = p - lr_bc1 * (m / denom);                        // param.addcdiv_(exp_avg, denom, value=-lr / bias_correction1)
}
// kAdamGuarded: the step obeys the record grad_audit_reduce_kernel left in `audit` (DESIGN 4i).  A block of a skipped step
// returns before it loads anything else; an applied one scales the gradient by grad_scale * coef, which is grad_scale
// itself when coef == 1, so an unclipped guarded step writes the plain step's bits.
// adam_one with every rounding spelled out: the fused multiply-adds nvcc forms from adam_one in the plain and guarded
// kernels.  The device-scalar kernel reads lr_bc1 and inv_sqrt_bc2 from memory, and nvcc contracts adam_one differently
// there; this form gives it the plain kernel's bits whatever the compiler does.
__device__ __forceinline__ void adam_one_rn(float& p, float g, float& m, float& v, float lr_bc1, float b1, float b2,
                                            float eps, float wd, float inv_sqrt_bc2, float gscale) {
  g = __fmul_rn(g, gscale);
  if (wd != 0.f) g = __fmaf_rn(wd, p, g);
  m = __fmaf_rn(__fsub_rn(g, m), __fsub_rn(1.f, b1), m);
  v = __fmaf_rn(v, b2, __fmul_rn(__fmul_rn(__fsub_rn(1.f, b2), g), g));
  const float denom = __fmaf_rn(__fsqrt_rn(v), inv_sqrt_bc2, eps);
  p = __fmaf_rn(-lr_bc1, __fdiv_rn(m, denom), p);
}
// kMode: kAdamPlain, kAdamGuarded (the record `audit`), or kAdamDevice (bin_adam_scalars_t: lr_bc1 and inv_sqrt_bc2
// from adam_scalars_kernel, the guard from the record sc->audit names -- for an unguarded step one that never skips,
// coef 1).  All three give the same bits (the device form through adam_one_rn).
enum AdamMode { kAdamPlain = 0, kAdamGuarded = 1, kAdamDevice = 2 };
template <int kMode>
__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, float lr_bc1, float b1, float b2,
                                            float eps, float wd, float inv_sqrt_bc2, float gscale) {
  if (kMode == kAdamDevice) adam_one_rn(p, g, m, v, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
  else adam_one(p, g, m, v, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
}
template <int kMode>
__global__ void adam_step_kernel(const bin_adam_tensor_t* __restrict__ table, const int* __restrict__ chunk_prefix,
                                 int ntensors, float lr_bc1, float b1, float b2, float eps, float wd,
                                 float inv_sqrt_bc2, float gscale, const bin_grad_audit_t* __restrict__ audit,
                                 const bin_adam_scalars_t* __restrict__ sc) {
  if (kMode == kAdamDevice) {
    audit = sc->audit;
    lr_bc1 = sc->lr_bc1;
    inv_sqrt_bc2 = sc->inv_sqrt_bc2;
  }
  if (kMode != kAdamPlain) {
    if (audit->skip) return;
    gscale = gscale * audit->coef;
  }
  __shared__ int s_t;
  if (threadIdx.x == 0) {
    int lo = 0, hi = ntensors - 1;                     // chunk_prefix[0] == 0 <= blockIdx.x
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (chunk_prefix[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    s_t = lo;
  }
  __syncthreads();
  const int t = s_t;
  const bin_adam_tensor_t T = table[t];
  const size_t base = (size_t)((int)blockIdx.x - chunk_prefix[t]) * kAdamChunk;
  const size_t end = (base + kAdamChunk < T.n) ? base + kAdamChunk : (size_t)T.n;
  float* __restrict__ P = T.p;
  const float* __restrict__ G = T.g;
  float* __restrict__ M = T.m;
  float* __restrict__ V = T.v;
  const bool vec = ((((uintptr_t)P) | ((uintptr_t)G) | ((uintptr_t)M) | ((uintptr_t)V)) & 15u) == 0;
  if (vec) {                                           // base is a multiple of 4 elements
    const size_t end4 = base + ((end - base) & ~(size_t)3);
    for (size_t i = base + threadIdx.x * 4; i < end4; i += blockDim.x * 4) {
      float4 p = *reinterpret_cast<float4*>(P + i), m = *reinterpret_cast<float4*>(M + i),
             v = *reinterpret_cast<float4*>(V + i);
      const float4 g = *reinterpret_cast<const float4*>(G + i);
      adam_update<kMode>(p.x, g.x, m.x, v.x, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      adam_update<kMode>(p.y, g.y, m.y, v.y, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      adam_update<kMode>(p.z, g.z, m.z, v.z, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      adam_update<kMode>(p.w, g.w, m.w, v.w, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      *reinterpret_cast<float4*>(P + i) = p;
      *reinterpret_cast<float4*>(M + i) = m;
      *reinterpret_cast<float4*>(V + i) = v;
    }
    for (size_t i = end4 + threadIdx.x; i < end; i += blockDim.x) {
      float p = P[i], m = M[i], v = V[i];
      adam_update<kMode>(p, G[i], m, v, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      P[i] = p; M[i] = m; V[i] = v;
    }
  } else {
    for (size_t i = base + threadIdx.x; i < end; i += blockDim.x) {
      float p = P[i], m = M[i], v = V[i];
      adam_update<kMode>(p, G[i], m, v, lr_bc1, b1, b2, eps, wd, inv_sqrt_bc2, gscale);
      P[i] = p; M[i] = m; V[i] = v;
    }
  }
}

// One-thread prologue of the device-scalar step (bin_adam_scalars_t): the scalars the host would pass by value for
// step + 1, formed the way the host forms them -- 1 - beta^step in fp64, rounded to fp32, then the fp32 quotient and
// reciprocal square root, each rounded once -- and the step count advanced, or, for a skipped guarded step, the skip
// counted and nothing else touched.
__global__ void adam_scalars_kernel(bin_adam_scalars_t* __restrict__ sc) {
  if (sc->audit->skip) {
    sc->skipped += 1;
    return;
  }
  const float step = sc->step + 1.f;
  const float bc1 = (float)(1.0 - pow(sc->beta1, (double)step));
  const float bc2 = (float)(1.0 - pow(sc->beta2, (double)step));
  sc->lr_bc1 = __fdiv_rn(sc->lr, bc1);
  sc->inv_sqrt_bc2 = __fdiv_rn(1.f, __fsqrt_rn(bc2));
  sc->step = step;
}

// ---------------------------------------------------------------------------------------------------------
// Gradient audit of the guarded optimizer step (DESIGN 4i).  grad_audit_kernel walks the Adam table with the Adam
// grid: block b reads its chunk of g once, sums g^2 of the finite elements in fp64 and counts the others, and writes one
// 16-byte partial.  grad_audit_reduce_kernel adds the partials in index order and writes the record the guarded step
// reads.  fp64 because an fp32 sum of squares overflows at |g| ~ 1.8e19, where the gradients are still finite.  Every
// sum has a fixed order (strided per thread, shuffle tree, warp order) and the grids depend on the tensor shapes alone,
// so the record's bytes do not depend on the SM count.  No float atomics.
struct GradAuditPartial {
  double sumsq;
  unsigned nonfinite;
  int first_bad;                                       // this block's tensor if it saw a non-finite element, else INT_MAX
};
static_assert(sizeof(GradAuditPartial) == 16, "bin_grad_audit_scratch_bytes assumes 16-byte partials");
constexpr int kAuditThreads = 256;

__device__ __forceinline__ void audit_one(float g, double& ss, unsigned& bad) {
  if ((__float_as_uint(g) & 0x7f800000u) == 0x7f800000u) {
    ++bad;
  } else {
    const double d = (double)g;
    ss = fma(d, d, ss);
  }
}
// Block sum of (ss, bad) and block minimum of tb in a fixed tree; the result is valid in thread 0.
__device__ __forceinline__ void audit_block_reduce(double& ss, unsigned long long& bad, int& tb) {
  __shared__ double s_ss[kAuditThreads / 32];
  __shared__ unsigned long long s_bad[kAuditThreads / 32];
  __shared__ int s_tb[kAuditThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ss += __shfl_down_sync(0xffffffffu, ss, o);
    bad += __shfl_down_sync(0xffffffffu, bad, o);
    tb = min(tb, __shfl_down_sync(0xffffffffu, tb, o));
  }
  if ((threadIdx.x & 31) == 0) {
    s_ss[threadIdx.x >> 5] = ss;
    s_bad[threadIdx.x >> 5] = bad;
    s_tb[threadIdx.x >> 5] = tb;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kAuditThreads / 32; ++w) {
      ss += s_ss[w];
      bad += s_bad[w];
      tb = min(tb, s_tb[w]);
    }
  }
}
__global__ void __launch_bounds__(kAuditThreads)
grad_audit_kernel(const bin_adam_tensor_t* __restrict__ table, const int* __restrict__ chunk_prefix, int ntensors,
                  GradAuditPartial* __restrict__ partial) {
  __shared__ int s_t;
  if (threadIdx.x == 0) {
    int lo = 0, hi = ntensors - 1;                     // as adam_step_kernel
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (chunk_prefix[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    s_t = lo;
  }
  __syncthreads();
  const int t = s_t;
  const float* __restrict__ G = table[t].g;
  const size_t n = (size_t)table[t].n;
  const size_t base = (size_t)((int)blockIdx.x - chunk_prefix[t]) * kAdamChunk;
  const size_t end = (base + kAdamChunk < n) ? base + kAdamChunk : n;
  double ss = 0.0;
  unsigned nbad = 0;
  size_t tail = base;                                  // first element the scalar loop reads
  if ((((uintptr_t)G) & 15u) == 0) {                   // base is a multiple of 4 elements
    tail = base + ((end - base) & ~(size_t)3);
    for (size_t i = base + threadIdx.x * 4; i < tail; i += kAuditThreads * 4) {
      const float4 g = *reinterpret_cast<const float4*>(G + i);
      audit_one(g.x, ss, nbad);
      audit_one(g.y, ss, nbad);
      audit_one(g.z, ss, nbad);
      audit_one(g.w, ss, nbad);
    }
  }
  for (size_t i = tail + threadIdx.x; i < end; i += kAuditThreads) audit_one(G[i], ss, nbad);
  unsigned long long bad = nbad;
  int tb = nbad ? t : INT_MAX;
  audit_block_reduce(ss, bad, tb);
  if (threadIdx.x == 0) partial[blockIdx.x] = GradAuditPartial{ss, (unsigned)bad, tb};
}
__global__ void __launch_bounds__(kAuditThreads)
grad_audit_reduce_kernel(const GradAuditPartial* __restrict__ partial, int nchunks, float grad_scale, float max_norm,
                         bin_grad_audit_t* __restrict__ audit) {
  double ss = 0.0;
  unsigned long long bad = 0;
  int tb = INT_MAX;
  for (int i = threadIdx.x; i < nchunks; i += kAuditThreads) {
    const GradAuditPartial p = partial[i];
    ss += p.sumsq;
    bad += p.nonfinite;
    tb = min(tb, p.first_bad);
  }
  audit_block_reduce(ss, bad, tb);
  if (threadIdx.x == 0) {
    const float norm = (float)(fabs((double)grad_scale) * sqrt(ss));
    // torch.nn.utils.clip_grad_norm_: clip_coef = max_norm / (total_norm + 1e-6), clamped to 1
    const float coef = isinf(max_norm) ? 1.f : fminf(1.f, __fdiv_rn(max_norm, norm + 1e-6f));
    audit->sumsq = ss;
    audit->nonfinite = bad;
    audit->first_bad = bad ? tb : -1;
    audit->skip = bad != 0;
    audit->norm = norm;
    audit->coef = coef;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Blur synthesis (SURVEY 8f rank 4): create_dataset_blur_N_frames_average.py:108-134.  Blurry frame w is
// uint8(sum_j float32(frame[mid_w - r + j]) / float32(n)) with n = 2r+1 sharp frames around mid_w = first_mid + w*stride
// (float32 sum of <= 256 bytes is exact, one IEEE division, truncation).  One thread = 16 output bytes; the
// overlapping windows (stride 8 of 11) re-read frames from L2, HBM sees each frame once.
__global__ void blur_average_u8_kernel(const uint8_t* __restrict__ frames, size_t frame_bytes, int n, int first, int stride,
                                       int nwin, uint8_t* __restrict__ out, int vec) {
  const size_t per = vec ? (frame_bytes + 15) / 16 : frame_bytes;
  const size_t total = per * (size_t)nwin;
  const float fn = (float)n;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int w = (int)(idx / per);
    const size_t o = idx - (size_t)w * per;
    const uint8_t* src = frames + (size_t)(first + w * stride) * frame_bytes;
    uint8_t* dst = out + (size_t)w * frame_bytes;
    if (vec && (o + 1) * 16 <= frame_bytes) {
      unsigned acc[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) acc[k] = 0;
      for (int j = 0; j < n; ++j) {
        const uint4 q = *reinterpret_cast<const uint4*>(src + (size_t)j * frame_bytes + o * 16);
        const unsigned r[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) acc[k] += (r[k >> 2] >> (8 * (k & 3))) & 0xffu;
      }
      unsigned r[4] = {0, 0, 0, 0};
#pragma unroll
      for (int k = 0; k < 16; ++k) r[k >> 2] |= ((unsigned)(__fdiv_rn((float)acc[k], fn)) & 0xffu) << (8 * (k & 3));
      *reinterpret_cast<uint4*>(dst + o * 16) = make_uint4(r[0], r[1], r[2], r[3]);
    } else {
      const size_t b0 = vec ? o * 16 : o, b1 = vec ? frame_bytes : o + 1;
      for (size_t b = b0; b < b1; ++b) {
        unsigned acc = 0;
        for (int j = 0; j < n; ++j) acc += src[(size_t)j * frame_bytes + b];
        dst[b] = (uint8_t)__fdiv_rn((float)acc, fn);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// x4 flip self-ensemble (utils/test_util.py:110-132 flipx4_forward) over the tensors of a whole window.  Orientation o:
// bit 0 flips W, bit 1 flips H.  blockIdx.y = table entry; one thread = 4 consecutive pixels of one row when vec
// (W % 4 == 0 and 16-byte aligned tensors: a W-flipped float4 is then an aligned float4 with its lanes reversed), else 1.
// Both kernels are memory-bound copies; indices are 64-bit (a 4B batch at 768x1344 is 12.4 M floats per item).
struct FlipTable {
  const float* src[BIN_FLIPX4_MAX_TENSORS];
  float* dst[BIN_FLIPX4_MAX_TENSORS];
};
__device__ __forceinline__ float4 ld4(const float* p, bool rev) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  return rev ? make_float4(v.w, v.z, v.y, v.x) : v;
}
// src (B,3,H,W) -> dst (4B,3,H,W), item o*B + b = orientation o of item b
__global__ void __launch_bounds__(256) flipx4_expand_kernel(const __grid_constant__ FlipTable T, int B, int H, int W, int vec) {
  const float* __restrict__ src = T.src[blockIdx.y];
  float* __restrict__ dst = T.dst[blockIdx.y];
  const int per_row = vec ? W >> 2 : W;
  const size_t orows = (size_t)B * 3 * H;                        // rows of one orientation
  const size_t total = 4 * orows * per_row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(i % per_row);
    const size_t r = i / per_row;                                 // dst row ((o*B + b)*3 + c)*H + y
    const int o = (int)(r / orows);
    const size_t rr = r - (size_t)o * orows;                      // row (b*3 + c)*H + y of src
    const int y = (int)(rr % H);
    const float* s = src + (rr - y + ((o & 2) ? H - 1 - y : y)) * W;
    float* d = dst + r * W;
    if (vec) {
      const int x = 4 * u;
      *reinterpret_cast<float4*>(d + x) = ld4(s + ((o & 1) ? W - 4 - x : x), o & 1);
    } else {
      d[u] = s[(o & 1) ? W - 1 - u : u];
    }
  }
}
// flipx4_forward's accumulation: ((y0 + flipW(y1)) + flipH(y2)) + flipHW(y3), then / 4, each step rounded on its own
__device__ __forceinline__ float flipx4_avg(float a, float b, float c, float d) {
  return __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(a, b), c), d), 4.f);
}
// src (4B,3,H,W) as expand lays it out -> dst (B,3,H,W)
__global__ void __launch_bounds__(256) flipx4_mean_kernel(const __grid_constant__ FlipTable T, int B, int H, int W, int vec) {
  const float* __restrict__ src = T.src[blockIdx.y];
  float* __restrict__ dst = T.dst[blockIdx.y];
  const int per_row = vec ? W >> 2 : W;
  const size_t orows = (size_t)B * 3 * H;
  const size_t ostride = orows * W;                               // floats of one orientation
  const size_t total = orows * per_row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int u = (int)(i % per_row);
    const size_t r = i / per_row;                                 // row (b*3 + c)*H + y
    const int y = (int)(r % H);
    const size_t rf = r - y + (H - 1 - y);                        // the same row, H-flipped
    const float* s0 = src + r * W;
    const float* s1 = src + ostride + r * W;
    const float* s2 = src + 2 * ostride + rf * W;
    const float* s3 = src + 3 * ostride + rf * W;
    if (vec) {
      const int x = 4 * u, xf = W - 4 - x;
      const float4 a = ld4(s0 + x, false), b = ld4(s1 + xf, true), c = ld4(s2 + x, false), d = ld4(s3 + xf, true);
      *reinterpret_cast<float4*>(dst + r * W + x) = make_float4(flipx4_avg(a.x, b.x, c.x, d.x), flipx4_avg(a.y, b.y, c.y, d.y),
                                                                flipx4_avg(a.z, b.z, c.z, d.z), flipx4_avg(a.w, b.w, c.w, d.w));
    } else {
      const int xf = W - 1 - u;
      dst[r * W + u] = flipx4_avg(s0[u], s1[xf], s2[u], s3[xf]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Training batch (data/BIN_dataset.py:62-183 Adobe_BIN_loader + __getitem__ + collation).  grid (row groups, 17 frames,
// B samples); a block walks rows of one (frame, sample) with its threads along x, so each channel plane is stored
// coalesced; the 3 bytes of a pixel are read once for its 3 output planes.  Offsets are 64-bit (row pitch 3W of any
// frame size; a (17,16,3,352,640) batch is 184 M floats).
struct TrainBatchTable {
  bin_train_sample_t s[BIN_TRAIN_MAX_BATCH];
};
__global__ void __launch_bounds__(256) train_batch_u8_kernel(const __grid_constant__ TrainBatchTable T, int h, int w,
                                                             float* __restrict__ dst, int dst_B, int b0) {
  const int f = blockIdx.y, b = blockIdx.z;
  const bin_train_sample_t& S = T.s[b];
  const uint8_t* __restrict__ src = S.src[f];
  const size_t plane = (size_t)h * w;
  float* __restrict__ out = dst + ((size_t)f * dst_B + b0 + b) * 3 * plane;
  const size_t pitch = (size_t)S.W * 3;
  for (int y = blockIdx.x; y < h; y += gridDim.x) {
    const uint8_t* row = src + (size_t)(S.top + y) * pitch + (size_t)S.left * 3;
    float* o = out + (size_t)y * w;
    for (int x = threadIdx.x; x < w; x += blockDim.x) {
      const uint8_t* p = row + (size_t)(S.flip ? w - 1 - x : x) * 3;
      const uint8_t bl = p[0], g = p[1], r = p[2];
      o[x] = __fdiv_rn((float)r, 255.f);
      o[plane + x] = __fdiv_rn((float)g, 255.f);
      o[2 * plane + x] = __fdiv_rn((float)bl, 255.f);
    }
  }
}

static inline int grid_for(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  const size_t cap = (size_t)num_sms() * 16;
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

int launch_nchw_to_p8(const float* x, int C, const bin_act_t& dst, int plane0, cudaStream_t s) {
  const int nplanes = (C + 7) / 8;
  if (plane0 + nplanes > dst.planes) return fail(BIN_ERR_ARG, "nchw_to_p8: plane range exceeds tensor");
  const size_t total = (size_t)dst.B * nplanes * dst.H * dst.W;
  nchw_to_p8_kernel<<<grid_for(total, 256), 256, 0, s>>>(x, C, (__half*)dst.ptr, dst.planes, plane0, nplanes, dst.B,
                                                         dst.H, dst.W);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_p8_to_nchw(const bin_act_t& src, int plane0, int C, float* y, cudaStream_t s) {
  if (plane0 + (C + 7) / 8 > src.planes) return fail(BIN_ERR_ARG, "p8_to_nchw: plane range exceeds tensor");
  const size_t total = (size_t)src.B * C * src.H * src.W;
  p8_to_nchw_kernel<<<grid_for(total, 256), 256, 0, s>>>((const __half*)src.ptr, src.planes, plane0, C, y, src.B,
                                                         src.H, src.W);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_pack_frames(const bin_frames_t& fr, int H, int W, const bin_act_t& dst, cudaStream_t s, int x3) {
  if ((H & 1) || (W & 1)) return fail(BIN_ERR_ARG, "frame height/width must be even (pixel_reshuffle, RDN.py:123-128)");
  if (fr.ncalls < 1 || fr.ncalls > BIN_MAX_CALLS || fr.nframes < 1 || fr.nframes > BIN_MAX_FRAMES)
    return fail(BIN_ERR_ARG, "pack_frames: bad frame table");
  const int lplanes = x3 ? dst.planes / 2 : dst.planes;
  if (dst.B != fr.ncalls * fr.Bc || dst.H != H / 2 || dst.W != W / 2 || lplanes * 8 < 12 * fr.nframes || (x3 && (lplanes & 3)))
    return fail(BIN_ERR_ARG, "pack_frames: destination geometry mismatch");
  const int hw = dst.H * dst.W;
  const dim3 grid((unsigned)((hw + 256 * kPkU - 1) / (256 * kPkU)), (unsigned)lplanes, (unsigned)dst.B);
  pack_frames_kernel<<<grid, 256, 0, s>>>(fr, H, W, (__half*)dst.ptr, lplanes, x3);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
// ---- weight packing
static int pack_batch_blocks(const PackBatch& b) {
  return b.njobs ? b.job[b.njobs - 1].block0 + b.job[b.njobs - 1].nblocks : 0;
}
static int pack_batch_add(PackBatch& b, const PackJob& job, size_t total) {
  if (b.njobs >= kPackMaxJobs) return fail(BIN_ERR_UNSUPPORTED, "pack batch: too many tensors");
  PackJob j = job;
  size_t nb = (total + 256 * 8 - 1) / (256 * 8);               // ~8 elements per thread
  if (nb < 1) nb = 1;
  if (nb > 64) nb = 64;
  j.block0 = pack_batch_blocks(b); j.nblocks = (int)nb;
  b.job[b.njobs++] = j;
  return BIN_OK;
}
int pack_batch_add_weight(PackBatch& b, const float* w, int cout, int cin, int ks, int cout_pad, int cin_pad, int variant,
                          void* packed, int x3) {
  if (cin_pad % kKC || cout_pad % 16 || cout > cout_pad || cin > cin_pad)
    return fail(BIN_ERR_ARG, "pack_conv_weight: cin_pad must be a multiple of 32, cout_pad of 16");
  const int nt = conv_nt(cout_pad);
  if (cout_pad % nt) return fail(BIN_ERR_ARG, "pack_conv_weight: cout_pad must be <=128, or a multiple of 96 or 128");
  PackJob j;
  memset(&j, 0, sizeof(j));
  j.src = w; j.dst = packed; j.cout = cout; j.cin = cin; j.ks = ks; j.cout_pad = cout_pad; j.cin_pad = cin_pad; j.nt = nt;
  j.stackx = (ks == 3 && (cout_pad == 32 || cout_pad == 16) && variant == BIN_CONV_DEFAULT) ? 1 : 0;
  j.x3 = x3;
  return pack_batch_add(b, j, (size_t)cout_pad * cin_pad * ks * ks * (x3 ? 3 : 1));
}
int pack_batch_add_weight_t(PackBatch& b, const float* w, int cout, int cin, int ks, int row0, int nrows, int cout_pad_t,
                            int cin_pad_t, void* packed) {
  if (cin_pad_t % kKC || cout_pad_t % 96 || nrows > cout_pad_t || cout > cin_pad_t || row0 + nrows > cin)
    return fail(BIN_ERR_ARG, "pack_conv_weight_t: bad padding / row range");
  PackJob j;
  memset(&j, 0, sizeof(j));
  j.src = w; j.dst = packed; j.cout = cout; j.cin = cin; j.ks = ks; j.cout_pad = cout_pad_t; j.cin_pad = cin_pad_t; j.nt = 96;
  j.transpose = 1; j.row0 = row0; j.nrows = nrows;
  return pack_batch_add(b, j, (size_t)cout_pad_t * cin_pad_t * ks * ks);
}
int pack_batch_add_bias(PackBatch& b, const float* bias, int cout, int cout_pad, float* dst) {
  PackJob j;
  memset(&j, 0, sizeof(j));
  j.src = bias; j.dst = dst; j.cout = cout; j.cout_pad = cout_pad; j.is_bias = 1;
  return pack_batch_add(b, j, (size_t)cout_pad);
}
int pack_batch_launch(const PackBatch& b, cudaStream_t s) {
  if (b.njobs == 0) return BIN_OK;
  pack_batch_kernel<<<pack_batch_blocks(b), 256, 0, s>>>(b);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(BIN_ERR_CUDA, std::string("pack_batch_kernel: ") + cudaGetErrorString(e));
  return BIN_OK;
}
int launch_convlstm_multi(const LstmCells& cells, int ncells, int B, int H, int W, cudaStream_t s) {
  if (ncells < 1 || ncells > 3) return fail(BIN_ERR_ARG, "convlstm: 1..3 cells per launch");
  bool state = cells.h_prev[0] != nullptr;
  for (int i = 0; i < ncells; ++i) {
    if (!cells.x[i] || !cells.w[i] || !cells.b[i] || !cells.h_out[i]) return fail(BIN_ERR_ARG, "convlstm: null argument");
    if ((cells.c_prev[i] == nullptr) != (cells.h_prev[i] == nullptr))
      return fail(BIN_ERR_ARG, "convlstm: give both c_prev and h_prev or neither");
    if ((cells.h_prev[i] != nullptr) != state) return fail(BIN_ERR_ARG, "convlstm: cells of one launch must all have or all lack a state");
  }
  const int tiles_x = (W + kLsTW - 1) / kLsTW, tiles_y = (H + kLsTH - 1) / kLsTH;
  const dim3 grid((unsigned)(tiles_x * tiles_y * B), 1, (unsigned)ncells);
  if (state) convlstm_kernel<true><<<grid, 256, 0, s>>>(cells, B, H, W, tiles_x, tiles_y);
  else convlstm_kernel<false><<<grid, 256, 0, s>>>(cells, B, H, W, tiles_x, tiles_y);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_p8_add(const bin_act_t& dst, int dplane0, const bin_act_t& src, int splane0, int nplanes, cudaStream_t s) {
  const int hw = dst.H * dst.W;
  const dim3 grid((unsigned)((hw + 511) / 512), (unsigned)nplanes, (unsigned)dst.B);
  p8_add_kernel<<<grid, 256, 0, s>>>((__half*)dst.ptr, dst.planes, dplane0, (const __half*)src.ptr, src.planes, splane0, hw);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_relu_mask(const bin_act_t& dg, int dplane0, const bin_act_t& g, int gplane0, int nplanes, cudaStream_t s) {
  const int hw = dg.H * dg.W;
  const dim3 grid((unsigned)((hw + 511) / 512), (unsigned)nplanes, (unsigned)dg.B);
  p8_relu_mask_kernel<<<grid, 256, 0, s>>>((__half*)dg.ptr, dg.planes, dplane0, (const __half*)g.ptr, g.planes, gplane0, hw);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_pixel_unshuffle(const bin_act_t& du, const bin_act_t& dst, cudaStream_t s) {
  pixel_unshuffle_kernel<<<grid_for((size_t)dst.B * 32 * dst.H * dst.W, 256), 256, 0, s>>>((const __half*)du.ptr,
      (__half*)dst.ptr, dst.B, dst.H, dst.W);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_unpack_frames_grad(const bin_act_t& dx0, const bin_frames_t& dout, const bin_frames_t& dfr, int H, int W,
                              const float* scale, cudaStream_t s) {
  const size_t total = (size_t)dx0.B * dfr.nframes * 3 * (H / 2) * (W / 2);
  unpack_frames_grad_kernel<<<grid_for(total, 256), 256, 0, s>>>((const __half*)dx0.ptr, dx0.planes, dout, dfr, H, W, scale);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_grad_out_to_p8(const bin_frames_t& dout, int H, int W, const bin_act_t& dst, const float* scale, cudaStream_t s) {
  grad_out_to_p8_kernel<<<grid_for((size_t)dst.B * 4 * H * W, 256), 256, 0, s>>>(dout, H, W, (__half*)dst.ptr, scale);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
size_t bias_grad_partial_floats(int B, int hw, int C) { return (size_t)B * ((hw + 1023) / 1024) * C; }
int launch_bias_grad(const bin_act_t& dy, int plane0, int C, const float* scale, float* db, cudaStream_t s, float* partial,
                     size_t partial_floats) {
  const int hw = dy.H * dy.W;
  // run_backbone_bwd checks every conv's partials against the region before its first launch; this is a backstop
  if (partial && bias_grad_partial_floats(dy.B, hw, C) > partial_floats)
    return fail(BIN_ERR_WORKSPACE, "bias_grad: deterministic partial sums do not fit the workspace");
  dim3 grid((unsigned)((hw + 1023) / 1024), (unsigned)((C + 7) / 8), (unsigned)dy.B);
  p8_bias_grad_kernel<<<grid, 256, 0, s>>>((const __half*)dy.ptr, dy.planes, plane0, C, hw, scale, db, partial);
  BIN_CUDA_OK(cudaGetLastError());
  if (partial) {
    bias_grad_reduce_kernel<<<(C + 7) / 8, 256, 0, s>>>(partial, (int)(grid.x * grid.z), C, scale, db);
    BIN_CUDA_OK(cudaGetLastError());
  }
  return BIN_OK;
}
int launch_grad_scale(const float* const* gouts, int n, size_t numel, float target, float* scale_dev, unsigned* tmp_dev,
                      cudaStream_t s) {
  if (n < 1 || n > BIN_MAX_CALLS) return fail(BIN_ERR_ARG, "grad_scale: 1..BIN_MAX_CALLS tensors");
  GradPtrs G;
  memset(&G, 0, sizeof(G));
  G.n = n;
  for (int i = 0; i < n; ++i) {
    if (!gouts[i] || (reinterpret_cast<uintptr_t>(gouts[i]) & 15)) return fail(BIN_ERR_ARG, "grad_scale: null or unaligned gradient");
    G.p[i] = gouts[i];
  }
  BIN_CUDA_OK(cudaMemsetAsync(tmp_dev, 0, sizeof(unsigned), s));
  const dim3 grid((unsigned)grid_for(numel / 4 + 1, 256), (unsigned)n);
  grad_absmax_kernel<<<grid, 256, 0, s>>>(G, numel, tmp_dev);
  BIN_CUDA_OK(cudaGetLastError());
  grad_scale_finalize_kernel<<<1, 1, 0, s>>>(tmp_dev, target, scale_dev);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_tensor2img_u8(const float* x, int Hs, int Ws, int top, int left, int h, int w, uint8_t* out, cudaStream_t s) {
  if (top < 0 || left < 0 || h < 1 || w < 1 || top + h > Hs || left + w > Ws) return fail(BIN_ERR_ARG, "tensor2img: crop outside the image");
  tensor2img_u8_kernel<<<grid_for((size_t)h * w, 256), 256, 0, s>>>(x, Hs, Ws, top, left, h, w, out);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_u8_to_frame(const uint8_t* img, int h, int w, int pl, int pr, int pt, int pb, float* out, cudaStream_t s) {
  if (h < 1 || w < 1 || pl < 0 || pr < 0 || pt < 0 || pb < 0) return fail(BIN_ERR_ARG, "u8_to_frame: bad geometry");
  const int Hp = h + pt + pb, Wp = w + pl + pr;
  u8_to_frame_kernel<<<grid_for((size_t)Hp * Wp, 256), 256, 0, s>>>(img, h, w, pl, pt, Hp, Wp, out);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_adam_step(const bin_adam_tensor_t* table, const int* chunk_prefix, int ntensors, int nchunks, float lr,
                     float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                     float bias_correction2, float grad_scale, const bin_grad_audit_t* audit, bin_adam_scalars_t* sc,
                     cudaStream_t s) {
  if (sc) {
    if (ntensors < 1 || nchunks < 1 || audit) return fail(BIN_ERR_ARG, "adam_step: empty table");
    adam_scalars_kernel<<<1, 1, 0, s>>>(sc);
    BIN_CUDA_OK(cudaGetLastError());
    adam_step_kernel<kAdamDevice><<<nchunks, 256, 0, s>>>(table, chunk_prefix, ntensors, 0.f, beta1, beta2, eps,
                                                          weight_decay, 0.f, grad_scale, nullptr, sc);
    BIN_CUDA_OK(cudaGetLastError());
    return BIN_OK;
  }
  if (ntensors < 1 || nchunks < 1 || !(bias_correction1 > 0.f) || !(bias_correction2 > 0.f))
    return fail(BIN_ERR_ARG, "adam_step: empty table or non-positive bias correction");
  const float lr_bc1 = lr / bias_correction1, inv_sqrt_bc2 = 1.f / sqrtf(bias_correction2);
  if (audit)
    adam_step_kernel<kAdamGuarded><<<nchunks, 256, 0, s>>>(table, chunk_prefix, ntensors, lr_bc1, beta1, beta2, eps,
                                                           weight_decay, inv_sqrt_bc2, grad_scale, audit, nullptr);
  else
    adam_step_kernel<kAdamPlain><<<nchunks, 256, 0, s>>>(table, chunk_prefix, ntensors, lr_bc1, beta1, beta2, eps,
                                                         weight_decay, inv_sqrt_bc2, grad_scale, nullptr, nullptr);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
size_t grad_audit_scratch_bytes(int nchunks) { return nchunks < 1 ? 0 : (size_t)nchunks * sizeof(GradAuditPartial); }
int launch_grad_audit(const bin_adam_tensor_t* table, const int* chunk_prefix, int ntensors, int nchunks, float grad_scale,
                      float max_norm, void* scratch, bin_grad_audit_t* audit, cudaStream_t s) {
  grad_audit_kernel<<<nchunks, kAuditThreads, 0, s>>>(table, chunk_prefix, ntensors, (GradAuditPartial*)scratch);
  BIN_CUDA_OK(cudaGetLastError());
  grad_audit_reduce_kernel<<<1, kAuditThreads, 0, s>>>((const GradAuditPartial*)scratch, nchunks, grad_scale, max_norm,
                                                       audit);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_blur_average_u8(const uint8_t* frames, int T, size_t frame_bytes, int window_size, int first_mid, int stride,
                           int nwin, uint8_t* out, cudaStream_t s) {
  const int r = (window_size - 1) / 2;                 // average_half_range, script :101
  const int n = 2 * r + 1;                             // len(mid_list)
  if (T < 1 || frame_bytes < 1 || window_size < 1 || n > 256 || stride < 0 || nwin < 1 || first_mid - r < 0 ||
      (long long)first_mid + (long long)(nwin - 1) * stride + r >= T)
    return fail(BIN_ERR_ARG, "blur_average: window runs outside the T frames (or window_size > 256)");
  const int vec = ((((uintptr_t)frames) | ((uintptr_t)out) | (uintptr_t)frame_bytes) & 15u) == 0;
  const size_t per = vec ? frame_bytes / 16 : frame_bytes;
  blur_average_u8_kernel<<<grid_for(per * (size_t)nwin, 256), 256, 0, s>>>(frames, frame_bytes, n, first_mid - r, stride,
                                                                          nwin, out, vec);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
static unsigned pixel_loss_blocks(size_t n) {
  return (unsigned)((n + 256 * 16 - 1) / (256 * 16) < 256 ? (n + 256 * 16 - 1) / (256 * 16) : 256);
}
size_t pixel_loss_scratch_bytes(int npairs, size_t n) {
  if (npairs < 1 || npairs > BIN_MAX_LOSS_PAIRS) return 0;
  return (size_t)npairs * pixel_loss_blocks(n) * sizeof(float);
}
int launch_pixel_loss_fwd(const float* const* a, const float* const* b, int npairs, size_t n, int kind, float eps,
                          float* pair_loss, cudaStream_t s, int flags, void* scratch, size_t scratch_bytes) {
  if (npairs < 1 || npairs > BIN_MAX_LOSS_PAIRS || kind < 0 || kind > 2) return fail(BIN_ERR_ARG, "pixel_loss: bad pair count / kind");
  const bool det = flags & BIN_DETERMINISTIC;
  if (det && !scratch) return fail(BIN_ERR_ARG, "pixel_loss: BIN_DETERMINISTIC needs a scratch buffer");
  if (det && scratch_bytes < pixel_loss_scratch_bytes(npairs, n)) return fail(BIN_ERR_WORKSPACE, "pixel_loss: scratch too small");
  LossPairs P;
  memset(&P, 0, sizeof(P));
  P.npairs = npairs;
  for (int k = 0; k < npairs; ++k) { P.a[k] = a[k]; P.b[k] = b[k]; }
  dim3 grid(pixel_loss_blocks(n), npairs);
  if (det) {                                        // every pair_loss[k] has one writer: no memset, no atomics
    pixel_loss_fwd_kernel<true><<<grid, 256, 0, s>>>(P, n, kind, eps, pair_loss, (float*)scratch);
    BIN_CUDA_OK(cudaGetLastError());
    pixel_loss_reduce_kernel<<<(npairs + 7) / 8, 256, 0, s>>>((const float*)scratch, (int)grid.x, npairs, kind, n, pair_loss);
    BIN_CUDA_OK(cudaGetLastError());
    return BIN_OK;
  }
  BIN_CUDA_OK(cudaMemsetAsync(pair_loss, 0, npairs * sizeof(float), s));
  pixel_loss_fwd_kernel<false><<<grid, 256, 0, s>>>(P, n, kind, eps, pair_loss, nullptr);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
int launch_pixel_loss_bwd(const float* const* a, const float* const* b, float* const* da, float* const* db, int npairs,
                          size_t n, int kind, float eps, const float* upstream, cudaStream_t s) {
  if (npairs < 1 || npairs > BIN_MAX_LOSS_PAIRS || kind < 0 || kind > 2) return fail(BIN_ERR_ARG, "pixel_loss: bad pair count / kind");
  LossPairs P;
  memset(&P, 0, sizeof(P));
  P.npairs = npairs;
  for (int k = 0; k < npairs; ++k) { P.a[k] = a[k]; P.b[k] = b[k]; P.da[k] = da[k]; P.db[k] = db ? db[k] : nullptr; }
  dim3 grid((unsigned)((n + 256 * 8 - 1) / (256 * 8) < 512 ? (n + 256 * 8 - 1) / (256 * 8) : 512), npairs);
  pixel_loss_bwd_kernel<<<grid, 256, 0, s>>>(P, n, kind, eps, upstream);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
static unsigned convlstm_wgrad_blocks(size_t total) { return (unsigned)((total + 31) / 32 < 592 ? (total + 31) / 32 : 592); }
size_t convlstm_bwd_scratch_bytes(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return 0;
  return (size_t)convlstm_wgrad_blocks((size_t)B * H * W) * kLstmGradN * sizeof(float);
}
int launch_convlstm_bwd(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                        const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                        float* dw, float* db, int B, int H, int W, cudaStream_t s, int flags, void* scratch,
                        size_t scratch_bytes) {
  if ((c_prev == nullptr) != (h_prev == nullptr)) return fail(BIN_ERR_ARG, "convlstm_bwd: give both c_prev and h_prev or neither");
  // NULL outputs are not asked for: the weight pass runs when dw or db is wanted, the input pass when dx or dh_prev is,
  // and the gates pass (which also writes dc_prev) when anything is.  What runs is unchanged, so its bits are too.
  const bool weights = dw || db, inputs = dx || dh_prev;
  const bool det = (flags & BIN_DETERMINISTIC) && weights;     // the scratch holds the weight pass's partials only
  if (det && !scratch) return fail(BIN_ERR_ARG, "convlstm_bwd: BIN_DETERMINISTIC needs a scratch buffer");
  if (det && scratch_bytes < convlstm_bwd_scratch_bytes(B, H, W)) return fail(BIN_ERR_WORKSPACE, "convlstm_bwd: scratch too small");
  const size_t total = (size_t)B * H * W;
  if (!weights && !inputs && !dc_prev) return BIN_OK;
  convlstm_bwd_gates_kernel<<<grid_for(total, 128), 128, 0, s>>>(x, c_prev, h_prev, w, b, dh, dc, dgates_ws, dc_prev, B, H, W);
  BIN_CUDA_OK(cudaGetLastError());
  if (weights) {
    const unsigned wblocks = convlstm_wgrad_blocks(total);
    convlstm_bwd_weights_kernel<<<wblocks, 288, 0, s>>>(x, h_prev, dgates_ws, dw, db, B, H, W, det ? (float*)scratch : nullptr);
    BIN_CUDA_OK(cudaGetLastError());
    if (det) {
      convlstm_wgrad_reduce_kernel<<<(kLstmGradN + 7) / 8, 256, 0, s>>>((const float*)scratch, (int)wblocks, dw, db);
      BIN_CUDA_OK(cudaGetLastError());
    }
  }
  if (inputs) {
    convlstm_bwd_input_kernel<<<grid_for(total, 128), 128, 0, s>>>(dgates_ws, w, dx, dh_prev, B, H, W);
    BIN_CUDA_OK(cudaGetLastError());
  }
  return BIN_OK;
}
// expand = 1: bin_flipx4_expand, 0: bin_flipx4_mean.  Every check runs before the first CUDA call.
int launch_flipx4(int expand, const float* const* src, float* const* dst, int n, int B, int H, int W, cudaStream_t s) {
  const std::string who = expand ? "flipx4_expand: " : "flipx4_mean: ";
  if (!src || !dst) return fail(BIN_ERR_ARG, who + "null table");
  if (n < 1 || n > BIN_FLIPX4_MAX_TENSORS) return fail(BIN_ERR_ARG, who + "n must be 1..14");
  if (B < 1 || H < 1 || W < 1) return fail(BIN_ERR_ARG, who + "B, H and W must be >= 1");
  if ((double)B * H * W * 12 >= 0x1p62) return fail(BIN_ERR_ARG, who + "tensor too large");
  FlipTable T;
  memset(&T, 0, sizeof(T));
  uintptr_t align = 0;
  for (int i = 0; i < n; ++i) {
    if (!src[i] || !dst[i]) return fail(BIN_ERR_ARG, who + "null table entry");
    for (int j = 0; j < n; ++j) {
      if ((const float*)dst[i] == src[j]) return fail(BIN_ERR_ARG, who + "a dst equals a src (in place would race)");
      if (j < i && dst[j] == dst[i]) return fail(BIN_ERR_ARG, who + "dst entries must be distinct");
    }
    T.src[i] = src[i];
    T.dst[i] = dst[i];
    align |= (uintptr_t)src[i] | (uintptr_t)dst[i];
  }
  const int vec = (W % 4 == 0) && (align & 15) == 0;
  const size_t units = (size_t)(expand ? 4 : 1) * B * 3 * H * (vec ? W / 4 : W);
  const dim3 grid((unsigned)grid_for(units, 256), (unsigned)n);
  if (expand) flipx4_expand_kernel<<<grid, 256, 0, s>>>(T, B, H, W, vec);
  else flipx4_mean_kernel<<<grid, 256, 0, s>>>(T, B, H, W, vec);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
// bin_train_batch_u8.  Every check runs before the first CUDA call.
int launch_train_batch_u8(const bin_train_sample_t* samples, int B, int h, int w, float* dst, int dst_B, int b0,
                          cudaStream_t s) {
  const std::string who = "train_batch_u8: ";
  if (!samples) return fail(BIN_ERR_ARG, who + "null table");
  if (B < 1 || B > BIN_TRAIN_MAX_BATCH) return fail(BIN_ERR_ARG, who + "B must be 1..16");
  if (h < 1 || w < 1) return fail(BIN_ERR_ARG, who + "h and w must be >= 1");
  if (!dst) return fail(BIN_ERR_ARG, who + "null dst");
  if (b0 < 0 || (long long)b0 + B > dst_B) return fail(BIN_ERR_ARG, who + "items [b0, b0+B) must lie inside dst_B");
  if ((double)BIN_TRAIN_FRAMES * dst_B * 3 * h * w * 4 >= 0x1p62) return fail(BIN_ERR_ARG, who + "dst too large");
  TrainBatchTable T;
  memset(&T, 0, sizeof(T));
  for (int i = 0; i < B; ++i) {
    const bin_train_sample_t& S = samples[i];
    for (int f = 0; f < BIN_TRAIN_FRAMES; ++f)
      if (!S.src[f]) return fail(BIN_ERR_ARG, who + "null frame pointer");
    if (S.flip != 0 && S.flip != 1) return fail(BIN_ERR_ARG, who + "flip must be 0 or 1");
    if (S.H < 1 || S.W < 1) return fail(BIN_ERR_ARG, who + "source H and W must be >= 1");
    if ((double)S.H * S.W * 3 >= 0x1p62) return fail(BIN_ERR_ARG, who + "source frame too large");
    if (S.top < 0 || S.left < 0 || (long long)S.top + h > S.H || (long long)S.left + w > S.W)
      return fail(BIN_ERR_ARG, who + "crop outside its source frame");
    T.s[i] = S;
  }
  // about 16 blocks per SM in all, each over whole rows of one (frame, sample)
  const int per = (num_sms() * 16 + BIN_TRAIN_FRAMES * B - 1) / (BIN_TRAIN_FRAMES * B);
  const dim3 grid((unsigned)(h < per ? h : per), BIN_TRAIN_FRAMES, (unsigned)B);
  train_batch_u8_kernel<<<grid, 256, 0, s>>>(T, h, w, dst, dst_B, b0);
  BIN_CUDA_OK(cudaGetLastError());
  return BIN_OK;
}
}  // namespace binb
