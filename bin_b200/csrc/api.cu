// bin_b200 -- extern "C" entry points (include/bin_b200.h) and the host-side orchestration of
// one batched backbone stage.  Host code only: every arithmetic step is a kernel in
// conv_igemm.cu / aux_kernels.cu.  The six-frame window and the pyramids are scheduled in bin_b200/rdn.py.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "internal.h"

namespace binb {

static thread_local std::string g_err;
int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

int num_sms() {
  static const int cap = [] {                   // read once per process, not on the launch path
    const char* e = getenv("BIN_B200_MAX_SMS");
    const int n = (e && *e) ? atoi(e) : 0;
    return n > 0 ? n : 0;
  }();
  static std::atomic<int> cache[64];
  int dev = 0;
  cudaGetDevice(&dev);
  int v = cache[dev & 63].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (v <= 0) v = 132;
    if (cap > 0 && cap < v) v = cap;            // lowers the grids the library picks, nothing on the device
    cache[dev & 63].store(v, std::memory_order_relaxed);
  }
  return v;
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ------------------------------------------------------------------ backbone configuration
// A backbone is 2, 3 or 5 frames wide, G0 = 64 or 96 channels, and D = 1..12 residual dense blocks of C = 4 growth
// convs with G = 32 channels each (RDN.py:167-334).  The arch value of the C ABI carries all three
// (BIN_BACKBONE_ARCH); its g0 and d fields are 0 for the shipped 96 and 12, so the shipped arch equals nframes.
constexpr int kCgrow = 4, kG = 32;

struct Arch {
  int nframes, g0, d;
  int nconv() const { return 5 * d + 6; }      // SFENet1, SFENet2, D x (4 conv + LFF), GFF.0, GFF.1, UPNet.0, UPNet.2
  int planes() const { return g0 / 8; }        // P8 planes of one G0-channel feature map
};

static bool valid_nframes(int n) { return n == 2 || n == 3 || n == 5; }

static bool decode_arch(int arch, Arch& a) {
  if (arch < 0 || (arch >> 24) != 0) return false;
  const int g0 = (arch >> 8) & 0xff, d = (arch >> 16) & 0xff;
  a.nframes = arch & 0xff;
  a.g0 = g0 ? g0 : 96;
  a.d = d ? d : 12;
  return valid_nframes(a.nframes) && (a.g0 == 64 || a.g0 == 96) && a.d >= 1 && a.d <= 12;
}
// decode_arch for an entry point: BIN_ERR_ARG, with `who` in the message, for an arch it rejects
static int arch_or_fail(int arch, const char* who, Arch& a) {
  if (decode_arch(arch, a)) return BIN_OK;
  if (!valid_nframes(arch & 0xff)) return fail(BIN_ERR_ARG, std::string(who) + ": nframes must be 2, 3 or 5");
  return fail(BIN_ERR_ARG, std::string(who) + ": G0 must be 64 or 96 and D 1..12 (BIN_BACKBONE_ARCH)");
}

// ------------------------------------------------------------------ backbone conv table
// Order = nn.Module registration order of the reference backbones (RDN.py:187-208): SFENet1,
// SFENet2, RDBs.{i}.convs.{0..3}, RDBs.{i}.LFF, GFF.0, GFF.1, UPNet.0, UPNet.2.
struct ConvSpec {
  int cin, cout, ks, cin_pad, cout_pad;
  size_t w_off, b_off;
};

struct BackboneLayout {
  ConvSpec conv[BIN_BACKBONE_NCONV];   // the first a.nconv() entries are used
  size_t bytes;
};

static BackboneLayout backbone_layout(const Arch& A, int x3 = 0) {
  BackboneLayout L;
  int k = 0;
  auto add = [&](int cin, int cout, int ks, int cout_pad) {
    ConvSpec c;
    c.cin = cin; c.cout = cout; c.ks = ks;
    c.cin_pad = (int)align_up(cin, kKC);
    c.cout_pad = cout_pad;
    c.w_off = c.b_off = 0;
    L.conv[k++] = c;
  };
  const int g0 = A.g0;
  add(12 * A.nframes, g0, 5, g0);
  add(g0, g0, 3, g0);
  for (int i = 0; i < A.d; ++i) {
    for (int c = 0; c < kCgrow; ++c) add(g0 + c * kG, kG, 3, 32);
    add(g0 + kCgrow * kG, g0, 1, g0);
  }
  add(A.d * g0, g0, 1, g0);
  add(g0, g0, 3, g0);
  add(g0, 256, 3, 256);
  add(64, 3, 3, 16);
  size_t off = 0;
  for (int i = 0; i < A.nconv(); ++i) {
    ConvSpec& c = L.conv[i];
    c.w_off = off;
    off = align_up(off + (size_t)c.cout_pad * c.cin_pad * c.ks * c.ks * sizeof(__half) * (x3 ? 3 : 1), 256);
    c.b_off = off;
    off = align_up(off + (size_t)c.cout_pad * sizeof(float), 256);
  }
  L.bytes = off;
  return L;
}

// ------------------------------------------------------------------ workspaces
// Lays P8 tensors of B items out one after another from `base`, each at a 256-byte boundary; `off` is the bytes used so
// far.  A NULL base only sizes the layout.  Each tensor gets plane_mult times the planes asked for.
struct P8Carver {
  void* base;
  int B, plane_mult;
  size_t off;
  bin_act_t operator()(int planes, int h, int w) {
    bin_act_t t;
    t.ptr = base ? (void*)((uint8_t*)base + off) : nullptr;
    t.B = B; t.planes = planes * plane_mult; t.H = h; t.W = w;
    off = align_up(off + (size_t)B * t.planes * h * w * 16, 256);
    return t;
  }
};

struct BackboneWs {
  bin_act_t x0, f1, f2, cat, g, t1, t2, u;
  size_t bytes;
};
static BackboneWs backbone_ws(const Arch& A, int Btot, int H, int W, void* base, bool train = false, int x3 = 0) {
  BackboneWs w;
  const int h = H / 2, wd = W / 2, P = A.planes();
  P8Carver carve{base, Btot, x3 ? 2 : 1, 0};      // x3: hi + lo plane groups
  w.x0 = carve((int)align_up(12 * A.nframes, kKC) / 8, h, wd);
  w.f1 = carve(P, h, wd);
  w.f2 = carve(P, h, wd);
  w.cat = carve(P * A.d, h, wd);
  w.g = carve(train ? 16 * A.d : 16, h, wd);   // training keeps the growth maps of all D RDBs for the backward
  w.t1 = carve(P, h, wd);
  w.t2 = carve(P, h, wd);
  w.u = carve(8, H, W);
  w.bytes = carve.off;
  return w;
}

static bin_conv_args_t conv_args(const void* blob, const ConvSpec& c, int x3 = 0) {
  bin_conv_args_t a;
  memset(&a, 0, sizeof(a));
  a.x3 = x3;
  a.w_packed = (const uint8_t*)blob + c.w_off;
  a.bias = (const float*)((const uint8_t*)blob + c.b_off);
  a.ksize = c.ks;
  a.cout_pad = c.cout_pad;
  return a;
}

// The first `nconv` growth convs of RDB i (RDN.py:141-147): conv3x3 + ReLU of cat(x, g planes so far) into g planes
// [g_plane0 + 4c, +4).  The forward runs them in run_rdb; the recomputing backward runs all four again.
static int run_growth(const Arch& A, const void* blob, const BackboneLayout& L, int i, const bin_act_t& xin, int x_plane0,
                      const bin_act_t& g, int g_plane0, int nconv, cudaStream_t s, int x3) {
  const int base = 2 + i * (kCgrow + 1);
  for (int c = 0; c < nconv; ++c) {
    bin_conv_args_t a = conv_args(blob, L.conv[base + c], x3);
    a.in0 = xin; a.in0_plane0 = x_plane0; a.in0_planes = A.planes();
    a.in1 = g; a.in1_plane0 = g_plane0; a.in1_planes = 4 * c;
    a.relu = 1; a.epilogue = BIN_EPI_P8;
    a.out = g; a.out_plane0 = g_plane0 + 4 * c;
    BIN_TRY(launch_conv(a, s));
  }
  return BIN_OK;
}

// One RDB: 4 x (conv3x3+ReLU -> growth planes) + LFF 1x1 + residual (RDN.py:149-165).
// The last conv and the LFF run as one kernel (rdb_tail.cu) in fp16 inference; training keeps them apart because the
// backward needs the fourth growth map, and the split-fp16 mode has no fused variant.
static int run_rdb(const Arch& A, const void* blob, const BackboneLayout& L, int i, const bin_act_t& xin, int x_plane0,
                   const bin_act_t& g, const bin_act_t& out, int out_plane0, cudaStream_t s, int g_plane0 = 0, int x3 = 0,
                   bool keep_growth = false) {
  const int base = 2 + i * (kCgrow + 1);
  const bool fuse = !x3 && !keep_growth;
  BIN_TRY(run_growth(A, blob, L, i, xin, x_plane0, g, g_plane0, fuse ? kCgrow - 1 : kCgrow, s, x3));
  if (fuse) {
    const ConvSpec& c3 = L.conv[base + kCgrow - 1];
    const ConvSpec& lf = L.conv[base + kCgrow];
    return launch_rdb_tail(A.g0, xin, x_plane0, g, g_plane0, (const uint8_t*)blob + c3.w_off,
                           (const float*)((const uint8_t*)blob + c3.b_off), (const uint8_t*)blob + lf.w_off,
                           (const float*)((const uint8_t*)blob + lf.b_off), out, out_plane0, 0, 0, 0, 0, s);
  }
  bin_conv_args_t a = conv_args(blob, L.conv[base + kCgrow], x3);
  a.in0 = xin; a.in0_plane0 = x_plane0; a.in0_planes = A.planes();
  a.in1 = g; a.in1_plane0 = g_plane0; a.in1_planes = 16;
  a.epilogue = BIN_EPI_P8;
  a.out = out; a.out_plane0 = out_plane0;
  a.res = xin; a.res_plane0 = x_plane0;
  return launch_conv(a, s);
}

static int run_backbone(int arch, const void* blob, const bin_frames_t& fr, int H, int W, void* workspace,
                        size_t workspace_bytes, cudaStream_t s, bool train = false, int x3 = 0) {
  Arch A;
  BIN_TRY(arch_or_fail(arch, "backbone", A));
  if (fr.nframes != A.nframes) return fail(BIN_ERR_ARG, "backbone: nframes must be 2, 3 or 5");
  if (fr.ncalls < 1 || fr.ncalls > BIN_MAX_CALLS || fr.Bc < 1) return fail(BIN_ERR_ARG, "backbone: bad call table");
  if ((H & 1) || (W & 1) || H < 2 || W < 2) return fail(BIN_ERR_ARG, "backbone: H and W must be even (RDN.py:123-128)");
  const int Btot = fr.ncalls * fr.Bc;
  if (train && x3) return fail(BIN_ERR_UNSUPPORTED, "backbone: training runs in the fp16 mode only");
  const BackboneLayout L = backbone_layout(A, x3);
  const BackboneWs ws = backbone_ws(A, Btot, H, W, workspace, train, x3);
  if (ws.bytes > workspace_bytes) return fail(BIN_ERR_WORKSPACE, "backbone: workspace too small");
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) return fail(BIN_ERR_ARG, "backbone: workspace must be 256-byte aligned");
  const int P = A.planes(), nc = A.nconv();

  BIN_TRY(launch_pack_frames(fr, H, W, ws.x0, s, x3));                           // RDN.py:211
  {
    bin_conv_args_t a = conv_args(blob, L.conv[0], x3);                              // SFENet1 (RDN.py:212)
    a.in0 = ws.x0; a.in0_planes = ws.x0.planes / (x3 ? 2 : 1); a.epilogue = BIN_EPI_P8; a.out = ws.f1;
    BIN_TRY(launch_conv(a, s));
  }
  {
    bin_conv_args_t a = conv_args(blob, L.conv[1], x3);                              // SFENet2 (RDN.py:213)
    a.in0 = ws.f1; a.in0_planes = P; a.epilogue = BIN_EPI_P8; a.out = ws.f2;
    BIN_TRY(launch_conv(a, s));
  }
  for (int i = 0; i < A.d; ++i) {                                                // RDN.py:215-217
    const int gp0 = train ? 16 * i : 0;
    if (i == 0) BIN_TRY(run_rdb(A, blob, L, i, ws.f2, 0, ws.g, ws.cat, 0, s, gp0, x3, train));
    else BIN_TRY(run_rdb(A, blob, L, i, ws.cat, P * (i - 1), ws.g, ws.cat, P * i, s, gp0, x3, train));
  }
  {
    bin_conv_args_t a = conv_args(blob, L.conv[nc - 4], x3);                         // GFF.0 on the D*G0-ch concat (RDN.py:218)
    a.in0 = ws.cat; a.in0_planes = P * A.d; a.epilogue = BIN_EPI_P8; a.out = ws.t1;
    BIN_TRY(launch_conv(a, s));
  }
  {
    bin_conv_args_t a = conv_args(blob, L.conv[nc - 3], x3);                         // GFF.1, x += f__1 (RDN.py:219)
    a.in0 = ws.t1; a.in0_planes = P; a.epilogue = BIN_EPI_P8; a.out = ws.t2; a.res = ws.f1;
    BIN_TRY(launch_conv(a, s));
  }
  {
    bin_conv_args_t a = conv_args(blob, L.conv[nc - 2], x3);                         // UPNet.0 + PixelShuffle (RDN.py:205-206)
    a.in0 = ws.t2; a.in0_planes = P; a.epilogue = BIN_EPI_PIXSHUF; a.out = ws.u;
    BIN_TRY(launch_conv(a, s));
  }
  {
    bin_conv_args_t a = conv_args(blob, L.conv[nc - 1], x3);                         // UPNet.2 + mean(frames) (RDN.py:207,221)
    a.in0 = ws.u; a.in0_planes = 8; a.epilogue = BIN_EPI_FINAL; a.fr = fr;
    BIN_TRY(launch_conv(a, s));
  }
  return BIN_OK;
}

// ------------------------------------------------------------------ backward of one backbone
// Data gradients reuse conv_igemm_kernel: for a stride-1 / pad k/2 conv, dX = conv(dY, V) with
// V[ci][co][ky][kx] = W[co][ci][k-1-ky][k-1-kx] (packed by pack_batch_add_weight_t, Cout' padded to a
// multiple of 96 and clipped by store_planes; at G0 = 64 the G0-row parts run as 96-row launches that store 8 planes).  Gradients are fp16 P8 tensors scaled by *scale (loss
// scaling, a device scalar) and un-scaled when they leave the backbone (frame grads, dW, db).

// per-CTA accumulator slabs: grid = #SMs by default, kDetCtas in deterministic mode
static size_t wgrad_partial_bytes() {
  const int ctas = num_sms() > kDetCtas ? num_sms() : kDetCtas;
  return (size_t)ctas * 128 * 512 * sizeof(float);
}

struct TSpec {          // one data-gradient conv: output rows [row0,row0+nrows) of the forward conv's Cin axis
  int conv, row0, nrows, cout_pad_t, cin_pad_t, ks;
  size_t off;
};
struct BackboneLayoutT {
  TSpec x[BIN_BACKBONE_NCONV];      // x part / whole input
  TSpec g[BIN_BACKBONE_NCONV];      // growth part (RDB convs c>=1 and LFF); nrows = 0 if absent
  size_t zero_bias_off, bytes;
};
static BackboneLayoutT backbone_layout_t(const Arch& A) {
  const BackboneLayout L = backbone_layout(A);
  BackboneLayoutT T;
  size_t off = 0;
  auto mk = [&](int conv, int row0, int nrows) {
    TSpec t;
    t.conv = conv; t.row0 = row0; t.nrows = nrows; t.ks = L.conv[conv].ks;
    t.cout_pad_t = nrows > 0 ? (int)align_up(nrows, 96) : 0;
    t.cin_pad_t = (int)align_up(L.conv[conv].cout, kKC);
    t.off = off;
    if (nrows > 0) off = align_up(off + (size_t)t.cout_pad_t * t.cin_pad_t * t.ks * t.ks * sizeof(__half), 256);
    return t;
  };
  for (int i = 0; i < A.nconv(); ++i) {
    const ConvSpec& c = L.conv[i];
    const bool in_rdb = i >= 2 && i < 2 + A.d * (kCgrow + 1);
    if (in_rdb) {
      T.x[i] = mk(i, 0, A.g0);
      T.g[i] = mk(i, A.g0, c.cin - A.g0);        // 0 rows for conv 0 of each RDB
    } else {
      T.x[i] = mk(i, 0, c.cin);
      T.g[i] = mk(i, 0, 0);
    }
  }
  T.zero_bias_off = off;                     // zero bias of the widest data-gradient launch, GFF.0's D*G0 <= 1152 rows
  off = align_up(off + 1152 * sizeof(float), 256);
  T.bytes = off;
  return T;
}

struct GradWs {
  bin_act_t dout16, du, dup0, dt2, dt1, dcat, df2, dg, dx0;
  float* wg_partial;          // wgrad slabs; in deterministic mode also the bias-gradient partials (stream-ordered reuse)
  size_t wg_partial_floats;
  size_t bytes;
};
// Largest bias-gradient partial array of one backward: UPNet.2 (3 channels, full resolution) or UPNet.0 (256 channels,
// low resolution).  It fits the wgrad slabs for every shape a card can train; the region grows if it does not.
static size_t bias_partial_bytes(int Btot, int H, int W) {
  const size_t a = bias_grad_partial_floats(Btot, H * W, 3), b = bias_grad_partial_floats(Btot, (H / 2) * (W / 2), 256);
  return (a > b ? a : b) * sizeof(float);
}
static GradWs grad_ws(const Arch& A, int Btot, int H, int W, void* base) {
  GradWs w;
  const int h = H / 2, wd = W / 2, P = A.planes();
  P8Carver carve{base, Btot, 1, 0};
  w.dout16 = carve(4, H, W);
  w.du = carve(8, H, W);
  w.dup0 = carve(32, h, wd);
  w.dt2 = carve(P, h, wd);
  w.dt1 = carve(P, h, wd);
  w.dcat = carve(P * A.d, h, wd);
  w.df2 = carve(P, h, wd);
  w.dg = carve(16, h, wd);
  w.dx0 = carve((int)align_up(12 * A.nframes, kKC) / 8, h, wd);
  w.wg_partial = base ? (float*)((uint8_t*)base + carve.off) : nullptr;
  const size_t wgb = wgrad_partial_bytes(), bb = bias_partial_bytes(Btot, H, W);
  w.wg_partial_floats = (wgb > bb ? wgb : bb) / sizeof(float);
  w.bytes = align_up(carve.off + w.wg_partial_floats * sizeof(float), 256);
  return w;
}

struct GradParamLayout { size_t w[BIN_BACKBONE_NCONV], b[BIN_BACKBONE_NCONV], floats; };
static GradParamLayout grad_param_layout(const Arch& A) {
  const BackboneLayout L = backbone_layout(A);
  GradParamLayout g;
  size_t off = 0;
  for (int i = 0; i < A.nconv(); ++i) {
    g.w[i] = off; off += (size_t)L.conv[i].cout * L.conv[i].cin * L.conv[i].ks * L.conv[i].ks;
    g.b[i] = off; off += (size_t)L.conv[i].cout;
  }
  g.floats = off;
  return g;
}

// act_ws holds the forward's activations.  recompute_blob == NULL: the saving layout of bin_backbone_fwd_train, with the
// growth maps of all D RDBs (its size is the caller's; act_ws_bytes is not checked).  Otherwise: the inference layout
// that bin_backbone_fwd left, checked against act_ws_bytes; before RDB i's backward its four growth convs are re-run
// from cat[i-1] (f2 for RDB 0) with the forward weights in recompute_blob, into growth planes 0..15.  Same inputs, same
// weights and the same launches as the saving forward, so the rebuilt maps have the same bits, and every launch of the
// backward reads the same operands in both layouts.
//
// need (host, 2 * A.nconv() bytes, weight then bias of each conv in grad_param_layout order; NULL = all) and the
// NULL entries of dfr.frame say which gradients the caller reads.  Conv k's input depends on every conv with a lower
// index, so the gradient with respect to it is needed iff a frame or some tensor of a lower conv needs one: U[k] below.
// The backward walks the convs from the top; a weight or bias gradient nobody needs is not launched, a data gradient
// runs only where U holds at the input it feeds, and the walk stops once U is false.  Whatever runs is the launch the full
// backward makes, on the same operands and in the same order, so every gradient that is kept has the same bits.
static int run_backbone_bwd(int arch, const void* blob_t, const bin_frames_t& dout, const bin_frames_t& dfr, int H,
                            int W, const void* act_ws, size_t act_ws_bytes, const void* recompute_blob, void* gws_ptr,
                            size_t gws_bytes, float* gparams, const float* scale, cudaStream_t s, int flags,
                            const unsigned char* need) {
  Arch A;
  BIN_TRY(arch_or_fail(arch, "backbone_bwd", A));
  if (dfr.nframes != A.nframes) return fail(BIN_ERR_ARG, "backbone_bwd: nframes must be 2, 3 or 5");
  if (flags & ~BIN_DETERMINISTIC) return fail(BIN_ERR_ARG, "backbone_bwd: unknown flags");
  const bool det = flags & BIN_DETERMINISTIC;
  if (dout.ncalls != dfr.ncalls || dout.Bc != dfr.Bc || dout.ncalls < 1 || dout.ncalls > BIN_MAX_CALLS)
    return fail(BIN_ERR_ARG, "backbone_bwd: bad call tables");
  const int nc = A.nconv(), P = A.planes(), nframes = A.nframes;
  bool need_w[BIN_BACKBONE_NCONV], need_b[BIN_BACKBONE_NCONV], U[BIN_BACKBONE_NCONV + 1];
  bool any_param = false;
  for (int i = 0; i < nc; ++i) {
    need_w[i] = !need || need[2 * i];
    need_b[i] = !need || need[2 * i + 1];
    any_param = any_param || need_w[i] || need_b[i];
  }
  if (any_param && !gparams) return fail(BIN_ERR_ARG, "backbone_bwd: null argument");
  U[0] = false;                                                // U[0]: some frame of some call wants its gradient
  for (int k = 0; k < dfr.ncalls; ++k)
    for (int f = 0; f < nframes; ++f) U[0] = U[0] || dfr.frame[k][f] != nullptr;
  for (int i = 0; i < nc; ++i) U[i + 1] = U[i] || need_w[i] || need_b[i];
  const int Btot = dout.ncalls * dout.Bc;
  const bool recompute = recompute_blob != nullptr;
  const BackboneWs ws = backbone_ws(A, Btot, H, W, const_cast<void*>(act_ws), !recompute);
  if (recompute && ws.bytes > act_ws_bytes) return fail(BIN_ERR_WORKSPACE, "backbone_bwd: forward workspace too small");
  if (recompute && (reinterpret_cast<uintptr_t>(act_ws) & 255) != 0)
    return fail(BIN_ERR_ARG, "backbone_bwd: forward workspace must be 256-byte aligned");
  const BackboneLayout L = backbone_layout(A);
  const BackboneLayoutT T = backbone_layout_t(A);
  const GradParamLayout GP = grad_param_layout(A);
  const GradWs gw = grad_ws(A, Btot, H, W, gws_ptr);
  if (gw.bytes > gws_bytes) return fail(BIN_ERR_WORKSPACE, "backbone_bwd: gradient workspace too small");
  // Deterministic bias partials of every conv must fit the slab region before the first launch (grad_ws sizes it from
  // bias_partial_bytes; this keeps that invariant explicit should a conv with more partials ever be added).
  if (det)
    for (int i = 0; i < nc; ++i) {
      const int hw = i == nc - 1 ? H * W : (H / 2) * (W / 2);   // UPNet.2 runs at full resolution
      if (bias_grad_partial_floats(Btot, hw, L.conv[i].cout) > gw.wg_partial_floats)
        return fail(BIN_ERR_WORKSPACE, "backbone_bwd: deterministic bias partials do not fit the gradient workspace");
    }
  const float* zero_bias = (const float*)((const uint8_t*)blob_t + T.zero_bias_off);

  // dX (+)= conv(dY planes [dy_plane0, +dy_planes), V): writes `nstore` planes of `out` at out_plane0
  auto dgrad = [&](const TSpec& t, const bin_act_t& dy, int dy_plane0, int dy_planes, const bin_act_t& out, int out_plane0,
                   int nstore, bool accumulate) -> int {
    bin_conv_args_t a;
    memset(&a, 0, sizeof(a));
    a.in0 = dy; a.in0_plane0 = dy_plane0; a.in0_planes = dy_planes;
    a.w_packed = (const uint8_t*)blob_t + t.off; a.bias = zero_bias;
    a.ksize = t.ks; a.cout_pad = t.cout_pad_t; a.epilogue = BIN_EPI_P8;
    a.out = out; a.out_plane0 = out_plane0; a.store_planes = nstore;
    if (accumulate) { a.res = out; a.res_plane0 = out_plane0; }
    return launch_conv(a, s);
  };
  // dW += X^T dY, db += sum dY for forward conv `idx`.  Deterministic mode: the bias partials use the wgrad slabs, which
  // the stream frees again before the wgrad that follows writes them.
  auto wgrad = [&](int idx, const bin_act_t& x0, int x0p, int x0n, const bin_act_t& x1, int x1p, int x1n,
                   const bin_act_t& dy, int dyp) -> int {
    const ConvSpec& c = L.conv[idx];
    if (need_b[idx])
      BIN_TRY(launch_bias_grad(dy, dyp, c.cout, scale, gparams + GP.b[idx], s, det ? gw.wg_partial : nullptr,
                               gw.wg_partial_floats));
    if (!need_w[idx]) return BIN_OK;
    return launch_wgrad(x0, x0p, x0n, x1, x1p, x1n, dy, dyp, c.cout, c.cin, c.ks, scale, gparams + GP.w[idx], gw.wg_partial,
                        s, det);
  };
  const bin_act_t none = {nullptr, 0, 0, 0, 0};

  if (!U[nc]) return BIN_OK;                                                     // nothing asked for
  const int up2 = nc - 1, up0 = nc - 2, gff1 = nc - 3, gff0 = nc - 4;
  BIN_TRY(launch_grad_out_to_p8(dout, H, W, gw.dout16, scale, s));
  BIN_TRY(wgrad(up2, ws.u, 0, 8, none, 0, 0, gw.dout16, 0));                         // UPNet.2
  if (!U[up2]) return BIN_OK;
  BIN_TRY(dgrad(T.x[up2], gw.dout16, 0, 4, gw.du, 0, 8, false));
  BIN_TRY(launch_pixel_unshuffle(gw.du, gw.dup0, s));                               // nn.PixelShuffle backward
  BIN_TRY(wgrad(up0, ws.t2, 0, P, none, 0, 0, gw.dup0, 0));                          // UPNet.0
  if (!U[up0]) return BIN_OK;
  BIN_TRY(dgrad(T.x[up0], gw.dup0, 0, 32, gw.dt2, 0, P, false));
  BIN_TRY(wgrad(gff1, ws.t1, 0, P, none, 0, 0, gw.dt2, 0));                          // GFF.1
  if (!U[gff1]) return BIN_OK;
  BIN_TRY(dgrad(T.x[gff1], gw.dt2, 0, P, gw.dt1, 0, P, false));                      // dt2 doubles as d f__1 (RDN.py:219)
  BIN_TRY(wgrad(gff0, ws.cat, 0, P * A.d, none, 0, 0, gw.dt1, 0));                   // GFF.0
  if (!U[gff0]) return BIN_OK;
  BIN_TRY(dgrad(T.x[gff0], gw.dt1, 0, P, gw.dcat, 0, P * A.d, false));
  if (U[2]) BIN_CUDA_OK(cudaMemsetAsync(gw.df2.ptr, 0, (size_t)Btot * P * (H / 2) * (W / 2) * 16, s));
  // Reaching RDB i means U holds at its output (base + 5).  Inside it, the growth-map gradients dg feed the growth convs
  // below the current one and the RDB input, so they are needed while U holds at the current conv; the parts that land
  // in the input gradient dxin (residual, x rows of every conv) are needed iff U holds at the RDB input.
  for (int i = A.d - 1; i >= 0; --i) {
    const int base = 2 + i * (kCgrow + 1);
    const bin_act_t& xin = i == 0 ? ws.f2 : ws.cat;           // forward input of RDB i
    const int xin_p = i == 0 ? 0 : P * (i - 1);
    const bin_act_t& dxin = i == 0 ? gw.df2 : gw.dcat;        // its gradient (accumulated)
    const int dxin_p = i == 0 ? 0 : P * (i - 1);
    const int dxo_p = P * i;                                  // d x_{i+1}, complete at this point
    const int gp0 = recompute ? 0 : 16 * i;                   // growth maps of RDB i
    const bool dx_in = U[base];
    // recomputing: rebuild the growth maps, which the LFF's wgrad and, below it, the growth-map dgrads and ReLU masks
    // read; the LFF's bias gradient alone reads only dcat.  The saving layout already holds them, in planes 16 i.
    if (recompute && (need_w[base + kCgrow] || U[base + kCgrow]))
      BIN_TRY(run_growth(A, recompute_blob, L, i, xin, xin_p, ws.g, 0, kCgrow, s, 0));
    BIN_TRY(wgrad(base + kCgrow, xin, xin_p, P, ws.g, gp0, 16, gw.dcat, dxo_p));                      // LFF
    if (!U[base + kCgrow]) return BIN_OK;
    if (dx_in) {
      BIN_TRY(launch_p8_add(dxin, dxin_p, gw.dcat, dxo_p, P, s));                                     // residual (RDN.py:165)
      BIN_TRY(dgrad(T.x[base + kCgrow], gw.dcat, dxo_p, P, dxin, dxin_p, P, true));
    }
    BIN_TRY(dgrad(T.g[base + kCgrow], gw.dcat, dxo_p, P, gw.dg, 0, 16, false));
    for (int c = kCgrow - 1; c >= 0; --c) {
      BIN_TRY(launch_relu_mask(gw.dg, 4 * c, ws.g, gp0 + 4 * c, 4, s));                               // RDN.py:142
      BIN_TRY(wgrad(base + c, xin, xin_p, P, ws.g, gp0, 4 * c, gw.dg, 4 * c));
      if (!U[base + c]) return BIN_OK;
      if (dx_in) BIN_TRY(dgrad(T.x[base + c], gw.dg, 4 * c, 4, dxin, dxin_p, P, true));
      if (c > 0) BIN_TRY(dgrad(T.g[base + c], gw.dg, 4 * c, 4, gw.dg, 0, 4 * c, true));
    }
  }
  BIN_TRY(wgrad(1, ws.f1, 0, P, none, 0, 0, gw.df2, 0));                             // SFENet2
  if (!U[1]) return BIN_OK;
  BIN_TRY(dgrad(T.x[1], gw.df2, 0, P, gw.dt2, 0, P, true));                          // d f__1 complete
  BIN_TRY(wgrad(0, ws.x0, 0, ws.x0.planes, none, 0, 0, gw.dt2, 0));                  // SFENet1
  if (!U[0]) return BIN_OK;
  BIN_TRY(dgrad(T.x[0], gw.dt2, 0, P, gw.dx0, 0, gw.dx0.planes, false));
  return launch_unpack_frames_grad(gw.dx0, dout, dfr, H, W, scale, s);
}

}  // namespace binb

using namespace binb;

extern "C" {

int bin_abi_version(void) { return BIN_ABI_VERSION; }
const char* bin_last_error(void) { return g_err.c_str(); }

int bin_check_device(void) {
  int dev = 0;
  BIN_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  BIN_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9) return fail(BIN_ERR_UNSUPPORTED, std::string("bin_b200 needs an sm_90 device, found sm_") +
                                                          std::to_string(prop.major) + std::to_string(prop.minor));
  return BIN_OK;
}

int bin_nchw_to_p8(const float* x, int C, bin_act_t dst, int plane0, bin_stream_t s) {
  return launch_nchw_to_p8(x, C, dst, plane0, (cudaStream_t)s);
}
int bin_p8_to_nchw(bin_act_t src, int plane0, int C, float* y, bin_stream_t s) {
  return launch_p8_to_nchw(src, plane0, C, y, (cudaStream_t)s);
}
int bin_pack_frames(const bin_frames_t* fr, int H, int W, bin_act_t dst, bin_stream_t s) {
  if (!fr) return fail(BIN_ERR_ARG, "pack_frames: null frame table");
  return launch_pack_frames(*fr, H, W, dst, (cudaStream_t)s);
}
size_t bin_packed_weight_bytes(int cout_pad, int cin_pad, int ksize) {
  return (size_t)cout_pad * cin_pad * ksize * ksize * sizeof(__half);
}
int bin_pack_conv_weight(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int variant,
                         void* packed, bin_stream_t s) {
  return bin_pack_conv_weight_p(w_oihw, cout, cin, ksize, cout_pad, cin_pad, variant, BIN_PREC_F16, packed, s);
}
int bin_pack_frames_p(const bin_frames_t* fr, int H, int W, bin_act_t dst, int prec, bin_stream_t s) {
  if (!fr) return fail(BIN_ERR_ARG, "pack_frames: null frame table");
  if (prec != BIN_PREC_F16 && prec != BIN_PREC_F32X3) return fail(BIN_ERR_ARG, "pack_frames: unknown precision");
  return launch_pack_frames(*fr, H, W, dst, (cudaStream_t)s, prec == BIN_PREC_F32X3);
}
int bin_pack_conv_weight_p(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int variant,
                           int prec, void* packed, bin_stream_t s) {
  if (prec != BIN_PREC_F16 && prec != BIN_PREC_F32X3) return fail(BIN_ERR_ARG, "pack_conv_weight: unknown precision");
  PackBatch b;
  BIN_TRY(pack_batch_add_weight(b, w_oihw, cout, cin, ksize, cout_pad, cin_pad, variant, packed, prec == BIN_PREC_F32X3));
  return pack_batch_launch(b, (cudaStream_t)s);
}
int bin_pack_conv_weight_t(const float* w_oihw, int cout, int cin, int ksize, int row0, int nrows, int cout_pad_t,
                           int cin_pad_t, void* packed, bin_stream_t s) {
  PackBatch b;
  BIN_TRY(pack_batch_add_weight_t(b, w_oihw, cout, cin, ksize, row0, nrows, cout_pad_t, cin_pad_t, packed));
  return pack_batch_launch(b, (cudaStream_t)s);
}
size_t bin_conv_wgrad_workspace_bytes(void) { return wgrad_partial_bytes(); }
int bin_conv_wgrad(bin_act_t x0, int x0_plane0, int x0_planes, bin_act_t x1, int x1_plane0, int x1_planes, bin_act_t dy,
                   int dy_plane0, int cout, int cin, int ksize, const float* scale_dev, float* dw, void* workspace,
                   bin_stream_t s) {
  return launch_wgrad(x0, x0_plane0, x0_planes, x1, x1_plane0, x1_planes, dy, dy_plane0, cout, cin, ksize, scale_dev, dw,
                      (float*)workspace, (cudaStream_t)s);
}
int bin_conv_fwd(const bin_conv_args_t* a, bin_stream_t s) {
  if (!a) return fail(BIN_ERR_ARG, "conv: null args");
  return launch_conv(*a, (cudaStream_t)s);
}
int bin_convlstm_fwd(const bin_lstm_cell_t* cells_host, int ncells, int B, int H, int W, bin_stream_t s) {
  if (!cells_host) return fail(BIN_ERR_ARG, "convlstm: null cell table");
  if (ncells < 1 || ncells > 3) return fail(BIN_ERR_ARG, "convlstm: 1..3 cells per launch");
  LstmCells c;
  memset(&c, 0, sizeof(c));
  for (int i = 0; i < ncells; ++i) {
    const bin_lstm_cell_t& e = cells_host[i];
    c.x[i] = e.x; c.c_prev[i] = e.c_prev; c.h_prev[i] = e.h_prev; c.w[i] = e.w; c.b[i] = e.b;
    c.h_out[i] = e.h_out; c.c_out[i] = e.c_out;
  }
  return launch_convlstm_multi(c, ncells, B, H, W, (cudaStream_t)s);
}

size_t bin_pixel_loss_scratch_bytes(int npairs, size_t n) { return pixel_loss_scratch_bytes(npairs, n); }
int bin_pixel_loss_fwd_ex(const float* const* a_host, const float* const* b_host, int npairs, size_t n, int kind, float eps,
                          float* pair_loss, int flags, void* scratch, size_t scratch_bytes, bin_stream_t s) {
  if (!a_host || !b_host || !pair_loss) return fail(BIN_ERR_ARG, "pixel_loss_fwd: null argument");
  if (flags & ~BIN_DETERMINISTIC) return fail(BIN_ERR_ARG, "pixel_loss_fwd: unknown flags");
  return launch_pixel_loss_fwd(a_host, b_host, npairs, n, kind, eps, pair_loss, (cudaStream_t)s, flags, scratch,
                               scratch_bytes);
}
int bin_pixel_loss_fwd(const float* const* a_host, const float* const* b_host, int npairs, size_t n, int kind, float eps,
                       float* pair_loss, bin_stream_t s) {
  return bin_pixel_loss_fwd_ex(a_host, b_host, npairs, n, kind, eps, pair_loss, 0, nullptr, 0, s);
}
int bin_pixel_loss_bwd(const float* const* a_host, const float* const* b_host, float* const* da_host, float* const* db_host,
                       int npairs, size_t n, int kind, float eps, const float* upstream, bin_stream_t s) {
  if (!a_host || !b_host || !da_host || !upstream) return fail(BIN_ERR_ARG, "pixel_loss_bwd: null argument");
  return launch_pixel_loss_bwd(a_host, b_host, da_host, db_host, npairs, n, kind, eps, upstream, (cudaStream_t)s);
}
int bin_tensor2img_u8(const float* x, int Hs, int Ws, int top, int left, int h, int w, uint8_t* out, bin_stream_t s) {
  if (!x || !out) return fail(BIN_ERR_ARG, "tensor2img: null argument");
  return launch_tensor2img_u8(x, Hs, Ws, top, left, h, w, out, (cudaStream_t)s);
}
int bin_u8_to_frame(const uint8_t* img, int h, int w, int pad_l, int pad_r, int pad_t, int pad_b, float* out, bin_stream_t s) {
  if (!img || !out) return fail(BIN_ERR_ARG, "u8_to_frame: null argument");
  return launch_u8_to_frame(img, h, w, pad_l, pad_r, pad_t, pad_b, out, (cudaStream_t)s);
}
size_t bin_convlstm_bwd_scratch_bytes(int B, int H, int W) { return convlstm_bwd_scratch_bytes(B, H, W); }
int bin_convlstm_bwd_ex(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                        const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                        float* dw, float* db, int B, int H, int W, int flags, void* scratch, size_t scratch_bytes,
                        bin_stream_t s) {
  if (!x || !w || !b || !dgates_ws) return fail(BIN_ERR_ARG, "convlstm_bwd: null argument");
  if (flags & ~BIN_DETERMINISTIC) return fail(BIN_ERR_ARG, "convlstm_bwd: unknown flags");
  return launch_convlstm_bwd(x, c_prev, h_prev, w, b, dh, dc, dgates_ws, dx, dc_prev, dh_prev, dw, db, B, H, W,
                             (cudaStream_t)s, flags, scratch, scratch_bytes);
}
int bin_convlstm_bwd(const float* x, const float* c_prev, const float* h_prev, const float* w, const float* b,
                     const float* dh, const float* dc, float* dgates_ws, float* dx, float* dc_prev, float* dh_prev,
                     float* dw, float* db, int B, int H, int W, bin_stream_t s) {
  return bin_convlstm_bwd_ex(x, c_prev, h_prev, w, b, dh, dc, dgates_ws, dx, dc_prev, dh_prev, dw, db, B, H, W, 0, nullptr,
                             0, s);
}

int bin_backbone_nconv(int arch) {
  Arch A;
  return decode_arch(arch, A) ? A.nconv() : -1;
}

size_t bin_backbone_packed_bytes(int arch) {
  Arch A;
  return decode_arch(arch, A) ? backbone_layout(A).bytes : 0;
}

// all weights + biases of a backbone in ONE launch
static int pack_backbone(int arch, const float* const* w_host, const float* const* b_host, void* blob, int x3,
                         cudaStream_t s) {
  Arch A;
  BIN_TRY(arch_or_fail(arch, "backbone_pack", A));
  if (!w_host || !b_host || !blob) return fail(BIN_ERR_ARG, "backbone_pack: null argument");
  const BackboneLayout L = backbone_layout(A, x3);
  PackBatch b;
  for (int i = 0; i < A.nconv(); ++i) {
    const ConvSpec& c = L.conv[i];
    BIN_TRY(pack_batch_add_weight(b, w_host[i], c.cout, c.cin, c.ks, c.cout_pad, c.cin_pad, BIN_CONV_DEFAULT,
                                  (uint8_t*)blob + c.w_off, x3));
    BIN_TRY(pack_batch_add_bias(b, b_host[i], c.cout, c.cout_pad, (float*)((uint8_t*)blob + c.b_off)));
  }
  return pack_batch_launch(b, s);
}

int bin_backbone_pack(int arch, const float* const* w_host, const float* const* b_host, void* blob,
                      bin_stream_t s) {
  return pack_backbone(arch, w_host, b_host, blob, 0, (cudaStream_t)s);
}

size_t bin_backbone_workspace_bytes(int arch, int Btot, int H, int W) {
  Arch A;
  return decode_arch(arch, A) ? backbone_ws(A, Btot, H, W, nullptr).bytes : 0;
}

int bin_backbone_fwd(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* workspace,
                     size_t workspace_bytes, bin_stream_t s) {
  if (!fr || !blob) return fail(BIN_ERR_ARG, "backbone_fwd: null argument");
  return run_backbone(arch, blob, *fr, H, W, workspace, workspace_bytes, (cudaStream_t)s);
}

size_t bin_backbone_packed_t_bytes(int arch) {
  Arch A;
  return decode_arch(arch, A) ? backbone_layout_t(A).bytes : 0;
}

int bin_backbone_pack_t(int arch, const float* const* w_host, void* blob_t, bin_stream_t s) {
  Arch A;
  BIN_TRY(arch_or_fail(arch, "backbone_pack_t", A));
  const BackboneLayout L = backbone_layout(A);
  const BackboneLayoutT T = backbone_layout_t(A);
  PackBatch b;
  for (int i = 0; i < A.nconv(); ++i) {
    const ConvSpec& c = L.conv[i];
    const TSpec* parts[2] = {&T.x[i], &T.g[i]};
    for (const TSpec* t : parts) {
      if (t->nrows <= 0) continue;
      BIN_TRY(pack_batch_add_weight_t(b, w_host[i], c.cout, c.cin, c.ks, t->row0, t->nrows, t->cout_pad_t, t->cin_pad_t,
                                      (uint8_t*)blob_t + t->off));
    }
  }
  BIN_TRY(pack_batch_launch(b, (cudaStream_t)s));
  BIN_CUDA_OK(cudaMemsetAsync((uint8_t*)blob_t + T.zero_bias_off, 0, 1152 * sizeof(float), (cudaStream_t)s));
  return BIN_OK;
}

size_t bin_backbone_train_workspace_bytes(int arch, int Btot, int H, int W) {
  Arch A;
  return decode_arch(arch, A) ? backbone_ws(A, Btot, H, W, nullptr, true).bytes : 0;
}
int bin_backbone_fwd_train(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* save_ws,
                           size_t save_ws_bytes, bin_stream_t s) {
  if (!fr || !blob) return fail(BIN_ERR_ARG, "backbone_fwd_train: null argument");
  return run_backbone(arch, blob, *fr, H, W, save_ws, save_ws_bytes, (cudaStream_t)s, true);
}
size_t bin_backbone_grad_workspace_bytes(int arch, int Btot, int H, int W) {
  Arch A;
  return decode_arch(arch, A) ? grad_ws(A, Btot, H, W, nullptr).bytes : 0;
}
size_t bin_backbone_grad_param_floats(int arch) {
  Arch A;
  return decode_arch(arch, A) ? grad_param_layout(A).floats : 0;
}
int bin_backbone_bwd_masked(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H,
                            int W, const void* save_ws, void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params,
                            const float* scale_dev, int flags, const unsigned char* need_host, bin_stream_t s) {
  if (!blob_t || !dout || !dframes || !save_ws || !scale_dev) return fail(BIN_ERR_ARG, "backbone_bwd: null argument");
  return run_backbone_bwd(arch, blob_t, *dout, *dframes, H, W, save_ws, 0, nullptr, grad_ws_ptr, grad_ws_bytes,
                          grad_params, scale_dev, (cudaStream_t)s, flags, need_host);
}
int bin_backbone_bwd_ex(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H,
                        int W, const void* save_ws, void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params,
                        const float* scale_dev, int flags, bin_stream_t s) {
  return bin_backbone_bwd_masked(arch, blob_t, dout, dframes, H, W, save_ws, grad_ws_ptr, grad_ws_bytes, grad_params,
                                 scale_dev, flags, nullptr, s);
}
int bin_backbone_bwd(int arch, const void* blob_t, const bin_frames_t* dout, const bin_frames_t* dframes, int H, int W,
                     const void* save_ws, void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params,
                     const float* scale_dev, bin_stream_t s) {
  return bin_backbone_bwd_ex(arch, blob_t, dout, dframes, H, W, save_ws, grad_ws_ptr, grad_ws_bytes, grad_params,
                             scale_dev, 0, s);
}
int bin_backbone_bwd_recompute_masked(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                                      const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                                      void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                                      int flags, const unsigned char* need_host, bin_stream_t s) {
  if (!blob || !blob_t || !dout || !dframes || !fwd_ws || !scale_dev) return fail(BIN_ERR_ARG, "backbone_bwd: null argument");
  return run_backbone_bwd(arch, blob_t, *dout, *dframes, H, W, fwd_ws, fwd_ws_bytes, blob, grad_ws_ptr, grad_ws_bytes,
                          grad_params, scale_dev, (cudaStream_t)s, flags, need_host);
}
int bin_backbone_bwd_recompute_ex(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                                  const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                                  void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                                  int flags, bin_stream_t s) {
  return bin_backbone_bwd_recompute_masked(arch, blob, blob_t, dout, dframes, H, W, fwd_ws, fwd_ws_bytes, grad_ws_ptr,
                                           grad_ws_bytes, grad_params, scale_dev, flags, nullptr, s);
}
int bin_backbone_bwd_recompute(int arch, const void* blob, const void* blob_t, const bin_frames_t* dout,
                               const bin_frames_t* dframes, int H, int W, const void* fwd_ws, size_t fwd_ws_bytes,
                               void* grad_ws_ptr, size_t grad_ws_bytes, float* grad_params, const float* scale_dev,
                               bin_stream_t s) {
  return bin_backbone_bwd_recompute_ex(arch, blob, blob_t, dout, dframes, H, W, fwd_ws, fwd_ws_bytes, grad_ws_ptr,
                                       grad_ws_bytes, grad_params, scale_dev, 0, s);
}

int bin_grad_scale(const float* const* gouts_host, int n, size_t numel, float target, float* scale_dev, void* tmp4_dev,
                   bin_stream_t s) {
  if (!gouts_host || !scale_dev || !tmp4_dev) return fail(BIN_ERR_ARG, "grad_scale: null argument");
  return launch_grad_scale(gouts_host, n, numel, target, scale_dev, (unsigned*)tmp4_dev, (cudaStream_t)s);
}

int bin_rdb_fwd(const void* blob, int arch, int index, const float* x, float* y, int B, int h, int w,
                void* workspace, size_t workspace_bytes, bin_stream_t s) {
  Arch A;
  if (!decode_arch(arch, A) || index < 0 || index >= A.d) return fail(BIN_ERR_ARG, "rdb_fwd: bad nframes/index");
  const BackboneLayout L = backbone_layout(A);
  P8Carver carve{workspace, B, 1, 0};
  bin_act_t xin = carve(A.planes(), h, w), g = carve(16, h, w), out = carve(A.planes(), h, w);
  if (carve.off > workspace_bytes) return fail(BIN_ERR_WORKSPACE, "rdb_fwd: workspace too small");
  BIN_TRY(launch_nchw_to_p8(x, A.g0, xin, 0, (cudaStream_t)s));
  BIN_TRY(run_rdb(A, blob, L, index, xin, 0, g, out, 0, (cudaStream_t)s));
  return launch_p8_to_nchw(out, 0, A.g0, y, (cudaStream_t)s);
}

/* precision-parameterised twins (BIN_PREC_*) */
size_t bin_backbone_packed_bytes_p(int arch, int prec) {
  Arch A;
  return decode_arch(arch, A) ? backbone_layout(A, prec ? 1 : 0).bytes : 0;
}
int bin_backbone_pack_p(int arch, const float* const* w_host, const float* const* b_host, void* blob, int prec,
                        bin_stream_t s) {
  return pack_backbone(arch, w_host, b_host, blob, prec ? 1 : 0, (cudaStream_t)s);
}
size_t bin_backbone_workspace_bytes_p(int arch, int Btot, int H, int W, int prec) {
  Arch A;
  return decode_arch(arch, A) ? backbone_ws(A, Btot, H, W, nullptr, false, prec ? 1 : 0).bytes : 0;
}
int bin_backbone_fwd_p(int arch, const void* blob, const bin_frames_t* fr, int H, int W, void* workspace,
                       size_t workspace_bytes, int prec, bin_stream_t s) {
  if (!fr || !blob) return fail(BIN_ERR_ARG, "backbone_fwd: null argument");
  return run_backbone(arch, blob, *fr, H, W, workspace, workspace_bytes, (cudaStream_t)s, false, prec ? 1 : 0);
}

int bin_rdb_tail_fwd(const bin_act_t* x, int x_plane0, const bin_act_t* g, int g_plane0, const void* w_conv,
                     const float* b_conv, const void* w_lff, const float* b_lff, const bin_act_t* out, int out_plane0,
                     int b_begin, int b_count, int y_begin, int y_count, bin_stream_t s) {
  if (!x || !g || !out) return fail(BIN_ERR_ARG, "rdb_tail_fwd: null argument");
  return launch_rdb_tail(96, *x, x_plane0, *g, g_plane0, w_conv, b_conv, w_lff, b_lff, *out, out_plane0, b_begin, b_count,
                         y_begin, y_count, (cudaStream_t)s);
}
int bin_adam_step(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks, float lr,
                  float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                  float bias_correction2, float grad_scale, bin_stream_t s) {
  if (!table_dev || !chunk_prefix_dev) return fail(BIN_ERR_ARG, "adam_step: null argument");
  return launch_adam_step(table_dev, chunk_prefix_dev, ntensors, nchunks, lr, beta1, beta2, eps, weight_decay,
                          bias_correction1, bias_correction2, grad_scale, nullptr, (cudaStream_t)s);
}
int bin_adam_step_guarded(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks,
                          float lr, float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                          float bias_correction2, float grad_scale, const bin_grad_audit_t* audit_dev, bin_stream_t s) {
  if (!table_dev || !chunk_prefix_dev || !audit_dev) return fail(BIN_ERR_ARG, "adam_step_guarded: null argument");
  if (reinterpret_cast<uintptr_t>(audit_dev) & 7) return fail(BIN_ERR_ARG, "adam_step_guarded: audit record not 8-byte aligned");
  return launch_adam_step(table_dev, chunk_prefix_dev, ntensors, nchunks, lr, beta1, beta2, eps, weight_decay,
                          bias_correction1, bias_correction2, grad_scale, audit_dev, (cudaStream_t)s);
}
size_t bin_grad_audit_scratch_bytes(int nchunks) { return grad_audit_scratch_bytes(nchunks); }
int bin_grad_audit(const bin_adam_tensor_t* table_dev, const int* chunk_prefix_dev, int ntensors, int nchunks,
                   float grad_scale, float max_norm, void* scratch, size_t scratch_bytes, bin_grad_audit_t* audit_dev,
                   bin_stream_t s) {
  if (!table_dev || !chunk_prefix_dev || !scratch || !audit_dev) return fail(BIN_ERR_ARG, "grad_audit: null argument");
  if (ntensors < 1 || nchunks < 1) return fail(BIN_ERR_ARG, "grad_audit: empty table");
  if (!(max_norm > 0.f) || !isfinite(grad_scale))
    return fail(BIN_ERR_ARG, "grad_audit: max_norm must be positive (INFINITY = no clipping) and grad_scale finite");
  if ((reinterpret_cast<uintptr_t>(scratch) & 15) || (reinterpret_cast<uintptr_t>(audit_dev) & 7))
    return fail(BIN_ERR_ARG, "grad_audit: scratch must be 16-byte and the record 8-byte aligned");
  if (scratch_bytes < grad_audit_scratch_bytes(nchunks)) return fail(BIN_ERR_WORKSPACE, "grad_audit: scratch too small");
  return launch_grad_audit(table_dev, chunk_prefix_dev, ntensors, nchunks, grad_scale, max_norm, scratch, audit_dev,
                           (cudaStream_t)s);
}
int bin_blur_average_u8(const uint8_t* frames, int T, size_t frame_bytes, int window_size, int first_mid, int stride,
                        int nwin, uint8_t* out, bin_stream_t s) {
  if (!frames || !out) return fail(BIN_ERR_ARG, "blur_average: null argument");
  return launch_blur_average_u8(frames, T, frame_bytes, window_size, first_mid, stride, nwin, out, (cudaStream_t)s);
}
size_t bin_image_metrics_workspace_bytes(int h, int w) { return metrics_workspace_bytes(h, w); }
int bin_image_metrics_u8(const uint8_t* a, const uint8_t* b, int h, int w, int c, double* out4, void* workspace,
                         size_t workspace_bytes, bin_stream_t s) {
  return launch_image_metrics_u8(a, b, h, w, c, out4, workspace, workspace_bytes, (cudaStream_t)s);
}
size_t bin_image_metrics_batch_workspace_bytes(int n, int h, int w) { return metrics_batch_workspace_bytes(n, h, w); }
int bin_image_metrics_batch_u8(const uint8_t* const* a_host, const uint8_t* const* b_host, int n, int h, int w, int c,
                               int flags, double* out, void* workspace, size_t workspace_bytes, bin_stream_t s) {
  return launch_image_metrics_batch_u8("image_metrics_batch", a_host, b_host, n, h, w, c, flags, out, workspace,
                                       workspace_bytes, (cudaStream_t)s);
}
int bin_flipx4_expand(const float* const* src_host, float* const* dst_host, int n, int B, int H, int W, bin_stream_t s) {
  return launch_flipx4(1, src_host, dst_host, n, B, H, W, (cudaStream_t)s);
}
int bin_flipx4_mean(const float* const* src_host, float* const* dst_host, int n, int B, int H, int W, bin_stream_t s) {
  return launch_flipx4(0, src_host, dst_host, n, B, H, W, (cudaStream_t)s);
}
int bin_train_batch_u8(const bin_train_sample_t* samples_host, int B, int h, int w, float* dst, int dst_B, int b0,
                       bin_stream_t s) {
  return launch_train_batch_u8(samples_host, B, h, w, dst, dst_B, b0, (cudaStream_t)s);
}
size_t bin_png_max_bytes(int h, int w) { return png_max_bytes(h, w); }
size_t bin_png_workspace_bytes(int n, int h, int w) { return png_workspace_bytes(n, h, w); }
int bin_png_encode_u8(const uint8_t* const* imgs_host, int n, int h, int w, uint8_t* out, size_t out_stride,
                      int64_t* sizes, void* workspace, size_t workspace_bytes, bin_stream_t s) {
  return launch_png_encode_u8(imgs_host, n, h, w, out, out_stride, sizes, workspace, workspace_bytes, (cudaStream_t)s);
}

}  // extern "C"
