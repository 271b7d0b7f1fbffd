/* bin_b200 -- C ABI of the Hopper-native (H100, sm_90a) BIN hot path (libbin_b200.so).
 *
 * The reference (laomao0/BIN) has no FFI layer: its boundary for this path is the Python
 * nn.Module contract reached through models/networks.py:9-10 -> models/archs/RDN.py:469-471
 * (SURVEY.md 8b).  This header is the "thin C-ABI extension" north_star asks for: every
 * entry point replaces one reference symbol (cited per function) and is called by the
 * Python mirror in bin_b200/rdn.py through ctypes.  Conventions:
 *   - all data pointers are DEVICE pointers unless the name ends in _host;
 *   - every call is asynchronous on the given CUDA stream (cudaStream_t passed as void*);
 *   - return 0 on success, non-zero error code otherwise; bin_last_error() gives the text
 *     (thread-local, valid until the next failing call on that thread);
 *   - no allocation inside: callers pass workspaces sized by the *_bytes() queries;
 *   - no global mutable state: re-entrant per (device, stream).
 *
 * Device layouts
 *   frames / outputs : fp32 NCHW, exactly what the reference module takes and returns.
 *   "planar-8" (P8)  : fp16 activations [B][C/8][H][W][8]  (8-channel planes; one pixel of one
 *                      plane = 16 B = one wgmma core-matrix row, so any pixel shift of a smem
 *                      tile is a 16-byte descriptor offset -> implicit GEMM without im2col).
 *   packed conv W    : fp16 [Cin_pad/32][kh][kw][4][Cout_pad][8]  (K-major B operand, one
 *                      contiguous slab per 32-channel K chunk), + fp32 bias[Cout_pad].
 *                      3x3 convs with Cout=32 (the RDB convs, 70 % of all FLOPs) use the
 *                      "x-stacked" layout [Cin_pad/32][kh][4][kw*32+cout][8]: the three horizontal
 *                      taps become GEMM columns (N=96) and are re-aligned in the epilogue.
 */
#ifndef BIN_B200_H_
#define BIN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BIN_ABI_VERSION 6
#define BIN_MAX_CALLS 6   /* same-weight backbone calls batched along N */
#define BIN_MAX_FRAMES 5  /* frames per backbone call (2, 3 or 5) */
#define BIN_MAX_LOSS_PAIRS 20 /* (prediction, target) pairs of one fused loss call */

enum { BIN_OK = 0, BIN_ERR_ARG = 1, BIN_ERR_CUDA = 2, BIN_ERR_UNSUPPORTED = 3, BIN_ERR_WORKSPACE = 4 };

/* `flags` of the *_ex entry points.  BIN_DETERMINISTIC: every cross-block sum (the pixel-loss terms, the backbone bias
 * gradients, the ConvLSTM weight and bias gradients) writes one partial per block and adds them in index order, and the
 * backbone weight gradients use a constant grid instead of one CTA per SM, so the result has the same bits from run to
 * run, on any stream and whatever SM count the device has.  0 = the default: float atomics, grids sized by SM count.
 * Any other bit fails with BIN_ERR_ARG. */
#define BIN_DETERMINISTIC 1

typedef void* bin_stream_t; /* cudaStream_t */

int bin_abi_version(void);
const char* bin_last_error(void);
/* 0 if the current device is sm_90 (H100) and the driver exposes cuTensorMapEncodeTiled. */
int bin_check_device(void);

/* ---- P8 activation tensor view ------------------------------------------------------- */
typedef struct {
  void* ptr; /* fp16 [B][planes][H][W][8] */
  int B, planes, H, W;
} bin_act_t;

/* ---- frame pointer table (one row per batched backbone call) --------------------------- */
typedef struct {
  const float* frame[BIN_MAX_CALLS][BIN_MAX_FRAMES]; /* each (Bc,3,H,W) fp32 NCHW */
  float* out[BIN_MAX_CALLS];                          /* each (Bc,3,H,W) fp32 NCHW */
  int ncalls, nframes, Bc;
} bin_frames_t;

/* ---- layout helpers (tests, boundary) ----------------------------------------------- */
/* fp32 NCHW (B,C,H,W) -> P8 planes [plane0, plane0+ceil(C/8)); channels past C are zeroed. */
int bin_nchw_to_p8(const float* x, int C, bin_act_t dst, int plane0, bin_stream_t s);
/* P8 planes -> fp32 NCHW (B,C,H,W). */
int bin_p8_to_nchw(bin_act_t src, int plane0, int C, float* y, bin_stream_t s);

/* RDN.py:107-132 pixel_reshuffle(cat(frames),2) fused with the fp32->fp16 cast and channel
 * padding: dst is P8 (ncalls*Bc, cin_pad/8, H/2, W/2); channel (f*3+rgb)*4 + dy*2+dx. */
int bin_pack_frames(const bin_frames_t* fr, int H, int W, bin_act_t dst, bin_stream_t s);

/* ---- weights ------------------------------------------------------------------------- */
size_t bin_packed_weight_bytes(int cout_pad, int cin_pad, int ksize);
/* nn.Conv2d weight (cout,cin,k,k) fp32 OIHW -> packed fp16; rows/cols past cout/cin are zero. */
/* variant: BIN_CONV_DEFAULT, or BIN_CONV_PLAIN to force the un-stacked layout for 3x3/Cout=32. */
int bin_pack_conv_weight(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int variant,
                         void* packed, bin_stream_t s);
/* Precision-parameterised twins of bin_pack_frames / bin_pack_conv_weight (prec = BIN_PREC_F16 | BIN_PREC_F32X3; the
 * enum is below), for unit-level use of the x3 conv.  F32X3: bin_pack_frames_p writes (hi, lo) = (fp16(v), fp16(v - hi))
 * per 32-channel chunk, 4 hi planes then 4 lo planes, so dst.planes is twice the logical count (a multiple of 8);
 * bin_pack_conv_weight_p writes three slabs per 32-channel K chunk, hi, hi and lo of (w * 2^8), so `packed` needs
 * 3 * bin_packed_weight_bytes.  Any other prec fails with BIN_ERR_ARG. */
int bin_pack_frames_p(const bin_frames_t* fr, int H, int W, bin_act_t dst, int prec, bin_stream_t s);
int bin_pack_conv_weight_p(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int variant,
                           int prec, void* packed, bin_stream_t s);

/* ---- the implicit-GEMM convolution (wgmma) -------------------------------------------- */
enum { BIN_EPI_P8 = 0, BIN_EPI_PIXSHUF = 1, BIN_EPI_FINAL = 2 };
enum { BIN_CONV_DEFAULT = 0, BIN_CONV_PLAIN = 1 };
/* Precision modes: fp16 storage / fp32 accumulate (<=1e-3 parity), or the split-fp16 "fp32-accurate" mode
 * (x = hi + lo, 3 MMAs per product, <=1e-5 parity; ~3x slower -- a correctness mode, not the benchmarked one). */
enum { BIN_PREC_F16 = 0, BIN_PREC_F32X3 = 1 };
typedef struct {
  /* input channels = planes [in0_plane0, +in0_planes) of in0 followed by planes of in1
   * (dense concat without a copy: RDN.py:147 torch.cat((x,out),1)); plane counts multiples of 4. */
  bin_act_t in0; int in0_plane0, in0_planes;
  bin_act_t in1; int in1_plane0, in1_planes; /* in1_planes = 0 -> unused */
  const void* w_packed; const float* bias;   /* bias: fp32[cout_pad] */
  int ksize;     /* 1, 3 or 5; stride 1, zero padding ksize/2 (all convs of RDN.py) */
  int cout_pad;  /* 16, 32, 64, 256 or a multiple of 96 */
  int relu;      /* RDN.py:142 */
  int epilogue;  /* BIN_EPI_* */
  int variant;   /* BIN_CONV_*; must match the variant the weights were packed with */
  /* optional sub-range of the output: batch items [b_begin, b_begin+b_count) and rows
   * [y_begin, y_begin+y_count); counts of 0 mean "to the end". */
  int b_begin, b_count, y_begin, y_count;
  /* BIN_EPI_P8 only: number of output planes actually stored (0 = cout_pad/8); lets a conv whose Cout was
   * zero-padded up to a multiple of 96 (the data-gradient launches) write a narrower tensor. */
  int store_planes;
  /* 1 = fp32-accurate split mode: tensors carry (hi, lo) fp16 pairs -- per 32-channel chunk 4 planes of hi then
   * 4 planes of lo, so bin_act_t.planes is twice the logical plane count while every *_plane0 / *_planes field
   * stays LOGICAL (multiples of 4); weights must have been packed with BIN_PREC_F32X3. */
  int x3;
  /* BIN_EPI_P8: out planes [out_plane0, +cout_pad/8), optional residual (RDN.py:165, :219), except for the x-stacked
   * 3x3 / cout_pad 32 kernel (variant BIN_CONV_DEFAULT), which takes none */
  bin_act_t out; int out_plane0;
  bin_act_t res; int res_plane0; /* res.ptr = NULL -> none */
  /* BIN_EPI_PIXSHUF (RDN.py:206): cout_pad=256 -> out is P8 (B, 8 planes, 2H, 2W) */
  /* BIN_EPI_FINAL (RDN.py:207 + :221/:279/:333): cout_pad=16 (3 used); out = conv + bias +
   * mean(frames) written as fp32 NCHW to fr.out[call] (call = b / fr.Bc, item b % fr.Bc) */
  bin_frames_t fr;
} bin_conv_args_t;
/* Fails with BIN_ERR_ARG, before any tensor map is built or anything is launched, on: a NULL in0 / in1 (when used) /
 * w_packed / bias, or out for the P8 and pixel-shuffle epilogues, or a NULL frame or output pointer of the final one;
 * a negative plane offset or store_planes; an input, output or residual plane range that runs past its tensor (x3: up
 * to the lo plane of the last logical plane); a residual for the x-stacked kernel; relu or a residual with the
 * pixel-shuffle or final epilogue (neither applies them); a batch/row sub-range outside the tensor. */
int bin_conv_fwd(const bin_conv_args_t* a, bin_stream_t s);

/* Fused tail of one RDB (RDN.py:141-147 for the 4th RDB_Conv, :162-165): g3 = ReLU(conv3x3(cat(x, g0..g2))) and
 * out = LFF(cat(x, g0..g3)) + x in one kernel; g3 is never written.  x: 12 planes from x_plane0, g: the 12 planes of
 * g0..g2 from g_plane0, out: 12 planes from out_plane0 (may be other planes of x's tensor).  w_conv / w_lff are the
 * bin_pack_conv_weight outputs of the (32,192,3,3) conv (variant BIN_CONV_DEFAULT) and the (96,224,1,1) LFF; b_conv
 * has 32 floats, b_lff 96.  b/y sub-ranges as in the conv arguments: a count of 0 means "to the end".  fp16 mode only.
 * A NULL argument, a negative plane offset, a plane range past its tensor or a bad sub-range fails with BIN_ERR_ARG
 * before any tensor map is built. */
int bin_rdb_tail_fwd(const bin_act_t* x, int x_plane0, const bin_act_t* g, int g_plane0, const void* w_conv,
                     const float* b_conv, const void* w_lff, const float* b_lff, const bin_act_t* out, int out_plane0,
                     int b_begin, int b_count, int y_begin, int y_count, bin_stream_t s);

/* Data-gradient weights of a conv (cout,cin,k): V[ci][co][ky][kx] = W[co][row0+ci][k-1-ky][k-1-kx] for ci < nrows,
 * packed like a forward conv with Cout' = cout_pad_t (multiple of 96), Cin' = cin_pad_t (multiple of 32):
 * bin_conv_fwd over dY with these weights gives dX[:, row0:row0+nrows]. */
int bin_pack_conv_weight_t(const float* w_oihw, int cout, int cin, int ksize, int row0, int nrows, int cout_pad_t,
                           int cin_pad_t, void* packed, bin_stream_t s);
/* Weight gradient of one conv: dw (cout,cin,k,k fp32 OIHW) += (1/ *scale_dev) * sum_px dY[px][co] X[px+tap][ci];
 * X = planes of x0 followed by planes of x1 (like bin_conv_args_t), dY = planes [dy_plane0, +ceil(cout/16)*2).
 * Segment plane counts are multiples of 4 (x1_planes may be 0), every plane range lies inside its tensor, x1 and dy
 * have the B/H/W of x0 and cin <= 8 * (x0_planes + x1_planes); anything else fails with BIN_ERR_ARG before any launch.
 * workspace: bin_conv_wgrad_workspace_bytes() bytes (per-CTA partial sums, reduced by a second kernel). */
size_t bin_conv_wgrad_workspace_bytes(void);
int bin_conv_wgrad(bin_act_t x0, int x0_plane0, int x0_planes, bin_act_t x1, int x1_plane0, int x1_planes, bin_act_t dy,
                   int dy_plane0, int cout, int cin, int ksize, const float* scale_dev, float* dw, void* workspace,
                   bin_stream_t s);

/* ---- ConvLSTMCell.forward, RDN.py:50-95 ------------------------------------------------ */
/* One cell: x,(c_prev,h_prev): (B,3,H,W) fp32; c_prev/h_prev NULL = zeros (RDN.py:57-68);
 * w: (12,6,3,3), b: (12); writes h_out and (optionally, c_out NULL = not written) c_out. */
typedef struct {
  const float *x, *c_prev, *h_prev, *w, *b;
  float *h_out, *c_out;
} bin_lstm_cell_t;
/* ncells (1..3) independent cells of one (B,3,H,W) shape in one launch (the cells of one recurrent hand-off of the
 * window, RDN.py:451-456); each cell's results have the bits of its own one-cell launch.  cells_host: host array.
 * A NULL table or x / w / b / h_out, a count outside 1..3, half a state, or cells that do not all have (or all lack) a
 * state fail with BIN_ERR_ARG before the launch. */
int bin_convlstm_fwd(const bin_lstm_cell_t* cells_host, int ncells, int B, int H, int W, bin_stream_t s);

/* Backward of the cell: dh/dc = gradients of the two outputs (either may be NULL = zero); dgates_ws = scratch
 * (B,12,H,W) fp32; writes dx (and dc_prev/dh_prev when a state was given), ACCUMULATES into dw (12,6,3,3) and db (12).
 * Any of dx, dc_prev, dh_prev, dw, db may be NULL: that gradient is not computed (no dw and no db skips the weight
 * pass, no dx and no dh_prev the input pass; the others are unchanged). */
int bin_convlstm_bwd(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                     const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                     float* dw, float* db, int B, int H, int W, bin_stream_t s);
/* bin_convlstm_bwd with flags (bin_convlstm_bwd = flags 0, scratch NULL).  With BIN_DETERMINISTIC, scratch (device, at
 * least bin_convlstm_bwd_scratch_bytes(B, H, W) = one 660-float row per weight-gradient block, <= 1.6 MB) receives the
 * per-block sums; a NULL scratch fails with BIN_ERR_ARG and a small one with BIN_ERR_WORKSPACE, before any launch. */
size_t bin_convlstm_bwd_scratch_bytes(int B, int H, int W);
int bin_convlstm_bwd_ex(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                        const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                        float* dw, float* db, int B, int H, int W, int flags, void* scratch, size_t scratch_bytes,
                        bin_stream_t s);

/* ---- one backbone (RDN_residual_interp_{2,2_1,4_1}_input.forward, RDN.py:210-334) ---------- */
/* Every backbone call takes an `arch`: the frame count (2, 3 or 5), the width G0 and the number D of residual dense
 * blocks, as BIN_BACKBONE_ARCH(nframes, g0, d).  g0 is 64 or 96 and d is 1..12; g0 = 0
 * and d = 0 stand for the shipped 96 and 12, so BIN_BACKBONE_ARCH(n, 0, 0) == n and a plain frame count keeps its
 * meaning.  C = 4 growth convs of G = 32 channels per block, as every configuration of the reference.  G0 = 128 is not
 * supported (the fused RDB tail's weights would not fit in shared memory), nor D > 12 (the tables below hold 66 convs).
 * A size query returns 0 and an entry point fails with BIN_ERR_ARG, before any launch, on an arch outside this range. */
#define BIN_BACKBONE_ARCH(nframes, g0, d) ((nframes) | ((g0) << 8) | ((d) << 16))
#define BIN_BACKBONE_NCONV 66 /* convs of the shipped backbone: SFENet1, SFENet2, 12 x (4 conv + LFF), GFF.0, GFF.1,
                                 UPNet.0, UPNet.2; the most any arch has */
/* Convs of a backbone, 5 D + 6 in the order above; -1 for an arch the library rejects. */
int bin_backbone_nconv(int arch);
size_t bin_backbone_packed_bytes(int arch);
/* w[i], b[i]: bin_backbone_nconv(arch) device fp32 parameters in nn.Module registration order (see bin_b200/rdn.py). */
int bin_backbone_pack(int arch, const float* const* w_host, const float* const* b_host, void* blob,
                      bin_stream_t s);
size_t bin_backbone_workspace_bytes(int arch, int Btot, int H, int W);
int bin_backbone_fwd(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* workspace,
                     size_t workspace_bytes, bin_stream_t s);
/* ---- training: forward that keeps the activations + backward (bin_model.optimize_parameters,
 * bin_model.py:130-141 -> l_pix.backward()).  Gradients flow as loss-scaled fp16 P8 tensors:
 * *scale_dev (device float, a power of two chosen by the caller from max|dOut|) multiplies dOut on entry
 * and is divided out of every result (frame gradients, dW, db). */
size_t bin_backbone_packed_t_bytes(int arch);             /* data-gradient (transposed, tap-flipped) weights */
int bin_backbone_pack_t(int arch, const float* const* w_host, void* blob_t, bin_stream_t s);
size_t bin_backbone_train_workspace_bytes(int arch, int Btot, int H, int W);   /* saved activations */
int bin_backbone_fwd_train(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* save_ws,
                           size_t save_ws_bytes, bin_stream_t s);
size_t bin_backbone_grad_workspace_bytes(int arch, int Btot, int H, int W);
size_t bin_backbone_grad_param_floats(int arch);          /* fp32 [w0,b0,w1,b1,...] in nn.Module order */
/* dout->out[k]: dL/d(output of call k), (Bc,3,H,W) fp32.  dframes->frame[k][f]: receives dL/d(frame f of call k)
 * (written, not accumulated; the caller sums frames that feed several calls).  grad_params is ACCUMULATED into. */
int bin_backbone_bwd(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H, int W,
                     const void* save_ws, void* grad_ws, size_t grad_ws_bytes, float* grad_params,
                     const float* scale_dev, bin_stream_t s);
/* The same backward from the INFERENCE workspace (activation recomputation): fwd_ws (fwd_ws_bytes >=
 * bin_backbone_workspace_bytes) is what bin_backbone_fwd with `blob` just left for the same frames, which keeps every
 * activation the backward reads except the growth maps of the D RDBs.  Before each RDB's backward its four growth convs
 * are re-run from its input with `blob`, into the workspace's one RDB of growth scratch.  Every launch then reads the
 * operands that bin_backbone_bwd reads after bin_backbone_fwd_train, so the frame and weight gradients have the same bits.
 * The bias gradients are summed with float atomics in both when flags = 0 (their last bits vary from run to run), and in
 * a fixed order with BIN_DETERMINISTIC (the same bits in both).  grad_ws, grad_params and scale_dev are as there.  A NULL
 * pointer, an undersized or unaligned fwd_ws fail (BIN_ERR_ARG / BIN_ERR_WORKSPACE) before any launch. */
int bin_backbone_bwd_recompute(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                               const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                               void* grad_ws, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                               bin_stream_t s);
/* The two backwards with flags (the calls above = flags 0).  BIN_DETERMINISTIC needs no extra memory: the bias-gradient
 * partials live in the wgrad region of grad_ws, which bin_backbone_grad_workspace_bytes sizes for both. */
int bin_backbone_bwd_ex(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H,
                        int W, const void* save_ws, void* grad_ws, size_t grad_ws_bytes, float* grad_params,
                        const float* scale_dev, int flags, bin_stream_t s);
int bin_backbone_bwd_recompute_ex(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                                  const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                                  void* grad_ws, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                                  int flags, bin_stream_t s);
/* The two backwards for a partly frozen network (the _ex calls above = need_host NULL).  need_host: host array of
 * 2 * bin_backbone_nconv(arch) bytes, nonzero where a gradient is wanted: weight then bias of each conv, the order of
 * grad_params; NULL = all.  A NULL dframes->frame[k][f] = no gradient for that frame.  Gradients not asked for are not
 * computed and their grad_params entries are left untouched; grad_params may be NULL when need_host asks for none.  The
 * data gradient of conv k's input is computed only if a frame or a tensor of a lower-index conv wants a gradient, and
 * the walk stops once none does.  Everything that is computed runs the launches of the full backward on the same
 * operands in the same order, so the gradients that are kept have its bits. */
int bin_backbone_bwd_masked(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H,
                            int W, const void* save_ws, void* grad_ws, size_t grad_ws_bytes, float* grad_params,
                            const float* scale_dev, int flags, const unsigned char* need_host, bin_stream_t s);
int bin_backbone_bwd_recompute_masked(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                                      const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                                      void* grad_ws, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                                      int flags, const unsigned char* need_host, bin_stream_t s);
/* Loss scale for one backbone backward: *scale_dev = 2^floor(log2(target / max_k max|gouts[k]|)) (a power of two, so
 * scaling and un-scaling are exact), computed on the device -- no host synchronisation.  The exponent is exact:
 * scale * max <= target < 2 * scale * max.  NaN elements do not count towards the maximum; a maximum of 0 (all zeros)
 * counts as 1e-30, which keeps the scale finite; an infinite maximum gives scale 0 (the backward's gradients are then
 * NaN).  gouts_host: host array of n (<= BIN_MAX_CALLS) device pointers to fp32 tensors of `numel` elements, 16-byte
 * aligned; tmp4_dev: 4 bytes of scratch. */
int bin_grad_scale(const float* const* gouts_host, int n, size_t numel, float target, float* scale_dev, void* tmp4_dev,
                   bin_stream_t s);

/* Unit-test entry: one RDB (RDN.py:149-165) on fp32 NCHW (B,G0,h,w), using RDB `index` (< D) of a blob packed for
 * `arch`; the block is G0 channels wide. */
int bin_rdb_fwd(const void* blob, int arch, int index, const float* x, float* y, int B, int h, int w,
                void* workspace, size_t workspace_bytes, bin_stream_t s);

/* Precision-parameterised twins of the backbone calls (prec = BIN_PREC_F16 | BIN_PREC_F32X3).  In BIN_PREC_F32X3 the
 * packed blob is 3x and the workspace 2x as large; results match the fp32 reference to <=1e-5. */
size_t bin_backbone_packed_bytes_p(int arch, int prec);
int bin_backbone_pack_p(int arch, const float* const* w_host, const float* const* b_host, void* blob, int prec,
                        bin_stream_t s);
size_t bin_backbone_workspace_bytes_p(int arch, int Btot, int H, int W, int prec);
int bin_backbone_fwd_p(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* workspace,
                       size_t workspace_bytes, int prec, bin_stream_t s);

/* ---- fused pixel loss (SURVEY 8f rank 3): bin_model.get_loss, bin_model.py:395-425 ---------------------- */
/* kind: 0 = nn.L1Loss(reduction='sum') (bin_model.py:55), 1 = nn.MSELoss(reduction='sum') (:57),
 * 2 = CharbonnierLoss mean sqrt(d^2+eps) (loss.py:130-140).  pair_loss[k] (device fp32[npairs]) = cri_pix(a_k, b_k);
 * the caller's loss is their mean.  a_host/b_host: host arrays of npairs device pointers, n elements each. */
enum { BIN_LOSS_L1_SUM = 0, BIN_LOSS_L2_SUM = 1, BIN_LOSS_CHARBONNIER_MEAN = 2 };
int bin_pixel_loss_fwd(const float* const* a_host, const float* const* b_host, int npairs, size_t n, int kind, float eps,
                       float* pair_loss, bin_stream_t s);
/* bin_pixel_loss_fwd with flags (bin_pixel_loss_fwd = flags 0, scratch NULL).  With BIN_DETERMINISTIC each block writes
 * its partial sum to scratch (device, >= bin_pixel_loss_scratch_bytes(npairs, n) <= 20 KB) and a second launch adds
 * them in index order (then divides once by n for the Charbonnier mean).  A NULL scratch fails with BIN_ERR_ARG and a
 * small one with BIN_ERR_WORKSPACE, before any launch. */
size_t bin_pixel_loss_scratch_bytes(int npairs, size_t n);
int bin_pixel_loss_fwd_ex(const float* const* a_host, const float* const* b_host, int npairs, size_t n, int kind, float eps,
                          float* pair_loss, int flags, void* scratch, size_t scratch_bytes, bin_stream_t s);
/* da_k = (upstream/npairs) * d cri_pix / d a_k, db_k = -da_k (db_host or single entries may be NULL). */
int bin_pixel_loss_bwd(const float* const* a_host, const float* const* b_host, float* const* da_host, float* const* db_host,
                       int npairs, size_t n, int kind, float eps, const float* upstream, bin_stream_t s);

/* ---- image boundary of the caller loop (SURVEY 8f rank 2) ------------------------------------ */
/* utils/util.py:113-137 tensor2img + the crop of test.py:394-402 for ONE (3,Hs,Ws) fp32 RGB image:
 * clamp [0,1], *255, round-half-even, uint8 HWC BGR of the (top,left,h,w) window -> out (h*w*3 bytes, device). */
int bin_tensor2img_u8(const float* x, int Hs, int Ws, int top, int left, int h, int w, uint8_t* out, bin_stream_t s);
/* test.py:44-56 read_image + the ReplicationPad2d of test.py:366-371: uint8 HWC BGR (h,w,3) ->
 * fp32 CHW RGB /255 of size (3, h+pad_t+pad_b, w+pad_l+pad_r), edge-replicated. */
int bin_u8_to_frame(const uint8_t* img, int h, int w, int pad_l, int pad_r, int pad_t, int pad_b, float* out, bin_stream_t s);

/* ---- optimizer step (SURVEY 8f rank 3): torch.optim.Adam as bin_model.py:97-100 builds it and :141 steps it ----- */
/* One launch over every parameter tensor.  table (device): ntensors entries; chunk_prefix (device int[ntensors+1]):
 * chunk_prefix[t] = number of BIN_ADAM_CHUNK-element blocks before tensor t, chunk_prefix[ntensors] = nchunks.
 * Semantics of torch.optim.Adam(amsgrad=False, maximize=False): g' = grad_scale*g + weight_decay*p;
 * m += (g'-m)(1-beta1); v = beta2 v + (1-beta2) g'^2; p -= lr/bias_correction1 * m / (sqrt(v)/sqrt(bias_correction2) + eps)
 * with bias_correction_i = 1 - beta_i^step computed by the caller (as torch does, on the host). */
#define BIN_ADAM_CHUNK 4096
typedef struct {
  float* p;                 /* parameter (updated in place)        */
  const float* g;           /* gradient                            */
  float* m;                 /* exp_avg                             */
  float* v;                 /* exp_avg_sq                          */
  unsigned long long n;     /* elements                            */
} bin_adam_tensor_t;
int bin_adam_step(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks, float lr,
                  float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                  float bias_correction2, float grad_scale, bin_stream_t s);

/* ---- guarded optimizer step: a device-side audit of all gradients, then an Adam step that obeys it --------------- */
/* bin_grad_audit makes one pass over the g column of an Adam table (two launches: one block per chunk, then one block)
 * and leaves this record on the device.  Every sum is fp64 in a fixed order and the grids depend on the tensor shapes
 * alone, so the record's bytes are reproducible.  sumsq and norm cover the finite elements. */
typedef struct {
  double sumsq;                 /* sum of g^2 over every finite element of every tensor                              */
  unsigned long long nonfinite; /* elements that are inf or NaN                                                     */
  int first_bad;                /* lowest table index of a tensor with such an element, -1 if none                  */
  int skip;                     /* nonfinite != 0: bin_adam_step_guarded writes nothing                              */
  float norm;                   /* |grad_scale| * sqrt(sumsq): the global L2 norm of the gradients Adam would see    */
  float coef;                   /* min(1, max_norm / (norm + 1e-6)) as torch's clip_grad_norm_; 1 if max_norm is inf  */
} bin_grad_audit_t;
/* Bytes of per-chunk partial sums (device, 16-byte aligned); 0 if nchunks < 1. */
size_t bin_grad_audit_scratch_bytes(int nchunks);
/* table / chunk_prefix as bin_adam_step takes them; one table may span every parameter group, so that one record
 * decides for the whole optimizer.  max_norm > 0, INFINITY for no clipping.  NULL, misaligned or empty arguments fail
 * with BIN_ERR_ARG and a small scratch with BIN_ERR_WORKSPACE, before any launch. */
int bin_grad_audit(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks,
                   float grad_scale, float max_norm, void* scratch, size_t scratch_bytes, bin_grad_audit_t* audit_dev,
                   bin_stream_t s);
/* bin_adam_step that reads audit_dev on the device: if skip, p, m and v keep their bits; otherwise the step runs with
 * grad_scale * coef in place of grad_scale (coef == 1 gives bin_adam_step's bits).  No host synchronisation. */
int bin_adam_step_guarded(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks,
                          float lr, float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                          float bias_correction2, float grad_scale, const bin_grad_audit_t* audit_dev, bin_stream_t s);

/* ---- training-data synthesis (SURVEY 8f rank 4): create_dataset_blur_N_frames_average.py:108-134 ------------------ */
/* frames: device uint8 [T][frame_bytes] (consecutive sharp frames, any pixel layout); out: [nwin][frame_bytes].
 * out[w] = uint8( sum_{j=-r..r} float32(frames[first_mid + w*stride + j]) / float32(2r+1) ), r = (window_size-1)/2
 * (script: window_size 11, first_mid 16, stride 8, nwin = floor(T/8) - 2). */
int bin_blur_average_u8(const uint8_t* frames, int T, size_t frame_bytes, int window_size, int first_mid, int stride,
                        int nwin, uint8_t* out, bin_stream_t s);

/* ---- evaluation metrics of the caller loop: test.py:404-458 (utils/util.py:201-250, skimage.measure) -------------- */
/* Bytes of per-tile partial sums for an (h, w) pair (0 if h or w is outside [7, 65535]). */
size_t bin_image_metrics_workspace_bytes(int h, int w);
/* a, b: uint8 (h,w,c) contiguous, c = 1 or 3, 7 <= h,w <= 65535, h*w*c < 2^31.  out4 (device fp64[4]) = { sum|a-b|,
 * sum (a-b)^2, mean Gaussian-11 SSIM (utils/util.py:211-231; NaN if h or w < 11), mean box-7 SSIM (skimage compare_ssim
 * defaults) }.  Bit-reproducible: the tiling depends only on (h, w) and every sum has a fixed order.  Every argument
 * is checked (BIN_ERR_ARG) before the first CUDA call. */
int bin_image_metrics_u8(const uint8_t* a, const uint8_t* b, int h, int w, int c, double* out4,
                         void* workspace, size_t workspace_bytes, bin_stream_t s);
/* Up to BIN_METRICS_MAX_BATCH pairs of one shape in one tile launch (tiles x pairs) and one reduce launch (one CTA per
 * pair), with no host synchronisation.  a_host[i], b_host[i]: device pointers as for bin_image_metrics_u8; pairs may
 * share an operand.  out (device fp64[4n]): out[4i..4i+3] = the four values bin_image_metrics_u8 writes for pair i, bit
 * for bit; out[4n..] is not written.  flags: BIN_METRICS_BGR (c = 3 only) stages source channel 2-ch as channel ch, so a
 * BGR image scores exactly what its RGB view scores (the SSIM sums run over the channels in order).  Workspace:
 * bin_image_metrics_batch_workspace_bytes(n, h, w) (0 if n, h or w is out of range).  Every argument is checked
 * (BIN_ERR_ARG) before the first CUDA call. */
#define BIN_METRICS_MAX_BATCH 16
#define BIN_METRICS_BGR 1
size_t bin_image_metrics_batch_workspace_bytes(int n, int h, int w);
int bin_image_metrics_batch_u8(const uint8_t* const* a_host, const uint8_t* const* b_host, int n, int h, int w, int c,
                               int flags, double* out, void* workspace, size_t workspace_bytes, bin_stream_t s);

/* ---- x4 flip self-ensemble: utils/test_util.py:110-132 flipx4_forward, for a whole 6-frame window ---------------- */
/* Orientation o of an image x: 0 = x, 1 = flip W (torch.flip(x, (-1,))), 2 = flip H ((-2,)), 3 = flip H and W ((-2, -1)).
 * Each flip is its own inverse.  One launch handles a table of n <= BIN_FLIPX4_MAX_TENSORS tensors (the 6 frames or the
 * 14 outputs of a window).
 * expand: src[i] (B,3,H,W) fp32 NCHW -> dst[i] (4B,3,H,W), orientation-major: item o*B + b = orientation o of src item b,
 *         so dst[i] + o*B*3*H*W is a contiguous (B,3,H,W) batch.
 * mean:   src[i] (4B,3,H,W), laid out as expand writes it -> dst[i] (B,3,H,W) =
 *         (((y0 + flipW(y1)) + flipH(y2)) + flipHW(y3)) / 4 with y_o = items [o*B, o*B+B) of src[i]: flipx4_forward's
 *         order, every step one correctly rounded fp32 operation (no contraction), so it equals the torch expression.
 * Fails with BIN_ERR_ARG before the first CUDA call if n is outside 1..BIN_FLIPX4_MAX_TENSORS, B, H or W < 1, a table or
 * an entry is NULL, or a dst pointer equals a src pointer or another dst pointer (in place would race). */
#define BIN_FLIPX4_MAX_TENSORS 14
int bin_flipx4_expand(const float* const* src_host, float* const* dst_host, int n, int B, int H, int W, bin_stream_t s);
int bin_flipx4_mean(const float* const* src_host, float* const* dst_host, int n, int B, int H, int W, bin_stream_t s);

/* ---- training batches: data/BIN_dataset.py:30-54,62-183 BINDataset.__getitem__ + DataLoader collation ------------ */
/* One sample: its 17 source frames in output order (6 LQs, 6 GTenh, 5 GTinp; the caller applies the order draw), each a
 * device uint8 (H,W,3) BGR image with row pitch 3W, as cv2.imread returns it; the crop (top, left) and the fliplr draw. */
#define BIN_TRAIN_MAX_BATCH 16
#define BIN_TRAIN_FRAMES 17
typedef struct {
  const uint8_t* src[BIN_TRAIN_FRAMES];
  int H, W;
  int top, left, flip;
} bin_train_sample_t;
/* Writes samples[0..B) as items [b0, b0+B) of dst, an fp32 (17, dst_B, 3, h, w) tensor (rows 0-5 LQs, 6-11 GTenh,
 * 12-16 GTinp; each row is a contiguous (dst_B,3,h,w) batch):
 *   dst[f][b0+b][c][y][x] = src_f[top+y][left + (flip ? w-1-x : x)][2-c] / 255
 * as one correctly rounded fp32 division (numpy's float32 `/ 255.`), so the bits equal read_img + the crop, np.fliplr,
 * BGR->RGB and torch.stack of the reference.  The table travels in the kernel parameters: one launch per call.
 * Fails with BIN_ERR_ARG before the first CUDA call if B is outside 1..BIN_TRAIN_MAX_BATCH, h or w < 1, the table,
 * a frame pointer or dst is NULL, [b0, b0+B) is not inside [0, dst_B), flip is not 0 or 1, a crop lies outside its
 * source frame, or a size overflows. */
int bin_train_batch_u8(const bin_train_sample_t* samples_host, int B, int h, int w, float* dst, int dst_B, int b0,
                       bin_stream_t s);

/* ---- PNG output of the caller loop: test.py / demo.py cv2.imwrite(path.png, uint8 BGR image) ------------------- */
/* Each file holds IHDR (8-bit truecolour), 8192-byte IDAT chunks and IEND; its inflated payload is the one cv2.imwrite
 * writes (RGB; filter type 1, Sub, on every row, 0 when w = 1; deflate with literals and distance-1 matches as zlib's
 * Z_RLE parses them), so any decoder returns the same pixels.  The bytes depend only on the pixels and (h, w). */
#define BIN_PNG_MAX_BATCH 16
/* Exact worst-case file size (every deflate block stored); 0 if (h, w) is out of range. */
size_t bin_png_max_bytes(int h, int w);
size_t bin_png_workspace_bytes(int n, int h, int w);   /* 0 if n, h or w is out of range */
/* imgs_host: n device pointers to uint8 (h,w,3) BGR, row pitch 3w (what bin_tensor2img_u8 writes and cv2.imwrite
 * takes).  out: device, n slots of out_stride >= bin_png_max_bytes(h,w) bytes; slot i receives a complete PNG file
 * and sizes[i] (device int64) its length.  1 <= n <= BIN_PNG_MAX_BATCH, 1 <= h,w <= 65535, h*(3w+1) < 2^31.
 * workspace: 256-byte aligned.  A null pointer, a bad n, h or w, an undersized or overflowing stride fail with
 * BIN_ERR_ARG and a small workspace with BIN_ERR_WORKSPACE, before the first CUDA call.  Nothing outside
 * [out, out + n*out_stride), sizes[0..n) and the workspace is written. */
int bin_png_encode_u8(const uint8_t* const* imgs_host, int n, int h, int w, uint8_t* out, size_t out_stride,
                      int64_t* sizes, void* workspace, size_t workspace_bytes, bin_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* BIN_B200_H_ */
