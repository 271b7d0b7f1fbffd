// bin_b200 internal declarations shared by the .cu files (not part of the ABI).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <atomic>
#include <string>

#include "../../include/bin_b200.h"

namespace binb {

// ------------------------------------------------------------------ errors
int fail(int code, const std::string& msg);
#define BIN_CUDA_OK(expr)                                                                          \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      return ::binb::fail(BIN_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));      \
  } while (0)
#define BIN_TRY(expr)            \
  do {                           \
    int _r = (expr);             \
    if (_r != BIN_OK) return _r; \
  } while (0)

// cudaFuncSetAttribute acts on the CURRENT device's context: a process that drives several GPUs (nn.DataParallel
// replicas, bin_model.py:40-42) must opt every kernel into its dynamic shared-memory size once per device.
// `mask` is one static per kernel (instantiation); bit d = done on device d.
template <typename Kernel>
inline int ensure_dynamic_smem(Kernel kern, int bytes, std::atomic<unsigned long long>& mask) {
  int dev = 0;
  BIN_CUDA_OK(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(mask.load(std::memory_order_acquire) & bit)) {
    BIN_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));   // idempotent
    mask.fetch_or(bit, std::memory_order_release);
  }
  return BIN_OK;
}

// ------------------------------------------------------------------ SM count
// SM count of the current device (cached per device).  BIN_B200_MAX_SMS=n, read once per process, caps it at n (grid
// sizes only; 0 or unset = no cap), so one card can stand in for one with fewer SMs.
int num_sms();
// Grid of the weight-gradient kernel in deterministic mode (BIN_DETERMINISTIC): a constant, so dW does not depend on
// the SM count.  132 = the SMs of an H100 SXM, where it equals the default grid.
constexpr int kDetCtas = 132;

// ------------------------------------------------------------------ tile geometry of the conv kernel
constexpr int kTWH = 32;   // smem row pitch of an activation tile, in pixels (= 4 core-matrix row groups)
constexpr int kTH = 8;     // output rows per CTA tile
constexpr int kMT = 2;     // 128-row accumulators per CTA tile (kTH*kTWH/128), one per consumer warpgroup
// target wgmma instructions per warpgroup and pipeline stage: an mbarrier round trip costs a few hundred cycles, so a
// stage should carry >= ~12 of them; one 1x1 unit is only 4
constexpr int kStageMmas = 12;
constexpr int kKC = 32;    // input channels per pipeline stage
constexpr int kKPL = 4;    // P8 planes per stage
constexpr int kCtrlBytes = 2048;
constexpr int kSmemMax = 227 * 1024;
constexpr int kMaxStages = 8;
constexpr int kMaxResidentChunks = 8;

// n / d for 0 <= n < 2^31 without a division instruction: q = (umulhi(n, mul) + n) >> shift, with the round-up magic of
// Granlund and Montgomery computed on the host (fast_div).  The conv kernel's tile coordinates then stay on the uniform
// datapath instead of taking vector registers in the epilogue.
struct FastDiv {
  unsigned mul; int shift;
#ifdef __CUDACC__
  __device__ __forceinline__ int div(int n) const { return (int)((__umulhi((unsigned)n, mul) + (unsigned)n) >> shift); }
#endif
};
inline FastDiv fast_div(int d) {   // d >= 1
  int l = 0;
  while ((1u << l) < (unsigned)d) ++l;
  return {(unsigned)((((1ull << 32) * ((1ull << l) - (unsigned)d)) / (unsigned)d) + 1), l};
}

struct alignas(64) ConvParams {
  CUtensorMap tmap0, tmap1;
  int plane0_0, nch0, plane0_1, nch1;  // segment start plane / number of K chunks (X3: 3 per logical chunk)
  int nch0l;                           // logical 32-channel chunks of segment 0
  const __half* w;
  const float* bias;
  int H, W, Btot;                      // conv resolution
  int b0, y0, ny;                      // batch / row sub-range processed by this launch
  int tiles_x, tiles_y, ntiles, nh;    // nh = cout_pad / NT
  FastDiv div_nh, div_tx, div_ty;
  int relu, resident, nstages, cps;
  __half* out; int out_planes, out_plane0, store_planes;
  const __half* res; int res_planes, res_plane0;
  bin_frames_t fr;
};

int launch_conv(const bin_conv_args_t& a, cudaStream_t s);

// up to 3 independent ConvLSTM cells in one launch (aux_kernels.cu)
struct LstmCells {
  const float* x[3]; const float* c_prev[3]; const float* h_prev[3];
  const float* w[3]; const float* b[3];
  float* h_out[3]; float* c_out[3];
};
int launch_convlstm_multi(const LstmCells& cells, int ncells, int B, int H, int W, cudaStream_t s);

// packed-weight geometry
inline int conv_nt(int cout_pad) { return cout_pad % 96 == 0 ? 96 : (cout_pad > 128 ? 128 : cout_pad); }

}  // namespace binb
