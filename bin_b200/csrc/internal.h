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
  CUtensorMap tmap_out;                // fp16 x-stacked P8 epilogue: the output over the launch's sub-range (TMA stores)
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

// ------------------------------------------------------------------ conv_igemm.cu
int launch_conv(const bin_conv_args_t& a, cudaStream_t s);
// TMA map of a P8 tensor whose box is box_px pixels x box_rows rows x box_planes planes.  With nb, ny > 0 it covers rows
// [y0, y0 + ny) of images [b0, b0 + nb) only: coordinates are then relative to (b0, y0), and a box's parts outside that
// range read as zeros and are not written.
int make_p8_tmap(CUtensorMap* m, const bin_act_t& t, int box_px, int box_rows, int box_planes, int b0 = 0, int nb = 0,
                 int y0 = 0, int ny = 0);

// ------------------------------------------------------------------ rdb_tail.cu
int launch_rdb_tail(int g0, const bin_act_t& x, int x_plane0, const bin_act_t& g, int g_plane0, const void* w_conv,
                    const float* b_conv, const void* w_lff, const float* b_lff, const bin_act_t& out, int out_plane0,
                    int b_begin, int b_count, int y_begin, int y_count, cudaStream_t s);

// ------------------------------------------------------------------ wgrad.cu
// det: the constant grid of kDetCtas CTAs instead of one CTA per SM
int launch_wgrad(const bin_act_t& x0, int x0_plane0, int x0_planes, const bin_act_t& x1, int x1_plane0, int x1_planes,
                 const bin_act_t& dy, int dy_plane0, int cout, int cin, int ks, const float* scale, float* dw,
                 float* partial_ws, cudaStream_t s, bool det = false);

// ------------------------------------------------------------------ aux_kernels.cu
// up to 3 independent ConvLSTM cells in one launch
struct LstmCells {
  const float* x[3]; const float* c_prev[3]; const float* h_prev[3];
  const float* w[3]; const float* b[3];
  float* h_out[3]; float* c_out[3];
};
int launch_convlstm_multi(const LstmCells& cells, int ncells, int B, int H, int W, cudaStream_t s);
size_t convlstm_bwd_scratch_bytes(int B, int H, int W);
int launch_convlstm_bwd(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                        const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                        float* dw, float* db, int B, int H, int W, cudaStream_t s, int flags, void* scratch,
                        size_t scratch_bytes);

// packed-weight geometry
inline int conv_nt(int cout_pad) { return cout_pad % 96 == 0 ? 96 : (cout_pad > 128 ? 128 : cout_pad); }

// Weight packing: pack_batch_kernel packs every job of a PackBatch in one launch.  The pack_batch_add_* calls check
// their arguments and append one tensor each; pack_batch_launch runs the batch.
struct PackJob {            // one conv's weight tensor (or bias vector) of a batched pack launch
  const float* src; void* dst;
  int cout, cin, ks, cout_pad, cin_pad, nt, stackx, transpose, row0, nrows, x3, is_bias;
  int block0, nblocks;     // this job's blocks are [block0, block0 + nblocks) of the launch
};
constexpr int kPackMaxJobs = 136;      // 66 weights + 66 biases (forward blob) / 66 + 48 transposed slabs, + slack
struct PackBatch { PackJob job[kPackMaxJobs]; int njobs = 0; };   // ~10 KB of kernel parameters (limit 32 KB)
int pack_batch_add_weight(PackBatch& b, const float* w, int cout, int cin, int ks, int cout_pad, int cin_pad, int variant,
                          void* packed, int x3);
// data-gradient weights of a conv (cout,cin,ks): output rows [row0,row0+nrows) of the cin axis, padded to
// cout_pad_t (multiple of 96); K = cout padded to cin_pad_t (multiple of 32).
int pack_batch_add_weight_t(PackBatch& b, const float* w, int cout, int cin, int ks, int row0, int nrows, int cout_pad_t,
                            int cin_pad_t, void* packed);
int pack_batch_add_bias(PackBatch& b, const float* bias, int cout, int cout_pad, float* dst);
int pack_batch_launch(const PackBatch& b, cudaStream_t s);

int launch_nchw_to_p8(const float* x, int C, const bin_act_t& dst, int plane0, cudaStream_t s);
int launch_p8_to_nchw(const bin_act_t& src, int plane0, int C, float* y, cudaStream_t s);
int launch_pack_frames(const bin_frames_t& fr, int H, int W, const bin_act_t& dst, cudaStream_t s, int x3 = 0);
// backward of a backbone
int launch_p8_add(const bin_act_t& dst, int dplane0, const bin_act_t& src, int splane0, int nplanes, cudaStream_t s);
int launch_relu_mask(const bin_act_t& dg, int dplane0, const bin_act_t& g, int gplane0, int nplanes, cudaStream_t s);
int launch_pixel_unshuffle(const bin_act_t& du, const bin_act_t& dst, cudaStream_t s);
int launch_unpack_frames_grad(const bin_act_t& dx0, const bin_frames_t& dout, const bin_frames_t& dfr, int H, int W,
                              const float* scale, cudaStream_t s);
int launch_grad_out_to_p8(const bin_frames_t& dout, int H, int W, const bin_act_t& dst, const float* scale, cudaStream_t s);
// partial == NULL: atomic per-block sums; otherwise the deterministic two-launch reduction through `partial`
size_t bias_grad_partial_floats(int B, int hw, int C);
int launch_bias_grad(const bin_act_t& dy, int plane0, int C, const float* scale, float* db, cudaStream_t s,
                     float* partial = nullptr, size_t partial_floats = 0);
int launch_grad_scale(const float* const* gouts, int n, size_t numel, float target, float* scale_dev, unsigned* tmp_dev,
                      cudaStream_t s);
// training step
size_t pixel_loss_scratch_bytes(int npairs, size_t n);
int launch_pixel_loss_fwd(const float* const* a, const float* const* b, int npairs, size_t n, int kind, float eps,
                          float* pair_loss, cudaStream_t s, int flags, void* scratch, size_t scratch_bytes);
int launch_pixel_loss_bwd(const float* const* a, const float* const* b, float* const* da, float* const* db, int npairs,
                          size_t n, int kind, float eps, const float* upstream, cudaStream_t s);
int launch_adam_step(const bin_adam_tensor_t* table, const int* chunk_prefix, int ntensors, int nchunks, float lr,
                     float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                     float bias_correction2, float grad_scale, const bin_grad_audit_t* audit, bin_adam_scalars_t* sc,
                     cudaStream_t s);   // audit: NULL = unguarded; sc: NULL = scalars by value
size_t grad_audit_scratch_bytes(int nchunks);
int launch_grad_audit(const bin_adam_tensor_t* table, const int* chunk_prefix, int ntensors, int nchunks, float grad_scale,
                      float max_norm, void* scratch, bin_grad_audit_t* audit, cudaStream_t s);
// data preparation and evaluation
int launch_blur_average_u8(const uint8_t* frames, int T, size_t frame_bytes, int window_size, int first_mid, int stride,
                           int nwin, uint8_t* out, cudaStream_t s);
int launch_flipx4(int expand, const float* const* src, float* const* dst, int n, int B, int H, int W, cudaStream_t s);
int launch_train_batch_u8(const bin_train_sample_t* samples, int B, int h, int w, float* dst, int dst_B, int b0,
                          cudaStream_t s);
int launch_tensor2img_u8(const float* x, int Hs, int Ws, int top, int left, int h, int w, uint8_t* out, cudaStream_t s);
int launch_u8_to_frame(const uint8_t* img, int h, int w, int pl, int pr, int pt, int pb, float* out, cudaStream_t s);

// ------------------------------------------------------------------ metrics.cu
size_t metrics_workspace_bytes(int h, int w);
int launch_image_metrics_u8(const uint8_t* a, const uint8_t* b, int h, int w, int c, double* out4, void* workspace,
                            size_t workspace_bytes, cudaStream_t s);
size_t metrics_batch_workspace_bytes(int n, int h, int w);
// who: the entry point's name, which starts every error message
int launch_image_metrics_batch_u8(const char* who, const uint8_t* const* a_host, const uint8_t* const* b_host, int n, int h,
                                  int w, int c, int flags, double* out, void* workspace, size_t workspace_bytes,
                                  cudaStream_t s);

// ------------------------------------------------------------------ ssim_loss.cu
size_t ssim_loss_scratch_bytes(int npairs, int planes, int h, int w);
size_t ssim_loss_maps_bytes(int npairs, int planes, int h, int w);
int launch_ssim_loss_fwd(const float* const* a, const float* const* b, int npairs, int planes, int h, int w, float* sums,
                         float* maps, int flags, void* scratch, size_t scratch_bytes, cudaStream_t s);
int launch_ssim_loss_bwd(const float* const* a, const float* const* b, const float* maps, float* const* da,
                         float* const* db, int npairs, int planes, int h, int w, const float* upstream, cudaStream_t s);

// ------------------------------------------------------------------ png.cu
size_t png_max_bytes(int h, int w);
size_t png_workspace_bytes(int n, int h, int w);
int launch_png_encode_u8(const uint8_t* const* imgs_host, int n, int h, int w, uint8_t* out, size_t out_stride,
                         int64_t* sizes, void* workspace, size_t workspace_bytes, cudaStream_t s);

}  // namespace binb
