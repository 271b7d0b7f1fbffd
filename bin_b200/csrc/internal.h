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

// ------------------------------------------------------------------ process options
// Environment knobs of the library (documented in DESIGN.md), read once per process (no getenv on the launch path).
struct Options {
  int debug;                 // BIN_B200_DEBUG   bit 4: synchronise after each conv launch
  bool fuse_lff;             // BIN_B200_FUSE_LFF=0 runs conv3 and LFF as two launches instead of rdb_tail_kernel
  bool zigzag;               // BIN_B200_ZIGZAG: consecutive RDB launches walk the tiles in opposite directions (L2 reuse)
  int stage_mmas;            // BIN_B200_STAGE_MMAS: target wgmma instructions per pipeline stage of the conv kernel (default 12)
  size_t band_budget;        // BIN_B200_BAND_BUDGET_KB (L2 band walker; default: one band)
};
const Options& options();
int num_sms();               // SM count of the current device (cached per device)

// ------------------------------------------------------------------ tile geometry of the conv kernel
constexpr int kTWH = 32;   // smem row pitch of an activation tile, in pixels (= 4 core-matrix row groups)
constexpr int kTH = 8;     // output rows per CTA tile
constexpr int kMT = 2;     // 128-row accumulators per CTA tile (kTH*kTWH/128), one per consumer warpgroup
constexpr int kKC = 32;    // input channels per pipeline stage
constexpr int kKPL = 4;    // P8 planes per stage
constexpr int kCtrlBytes = 2048;
constexpr int kSmemMax = 227 * 1024;
constexpr int kMaxStages = 8;
constexpr int kMaxResidentChunks = 8;

struct alignas(64) ConvParams {
  CUtensorMap tmap0, tmap1;
  int plane0_0, nch0, plane0_1, nch1;  // segment start plane / number of K chunks (X3: 3 per logical chunk)
  int nch0l;                           // logical 32-channel chunks of segment 0
  const __half* w;
  const float* bias;
  int H, W, Btot;                      // conv resolution
  int b0, y0, ny;                      // batch / row sub-range processed by this launch
  int tiles_x, tiles_y, ntiles, nh;    // nh = cout_pad / NT
  int relu, resident, nstages, cps, reverse;
  __half* out; int out_planes, out_plane0, store_planes;
  const __half* res; int res_planes, res_plane0;
  bin_frames_t fr;
};

int launch_conv(const bin_conv_args_t& a, cudaStream_t s, bool reverse = false);   // reverse: walk the tiles last-to-first

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
