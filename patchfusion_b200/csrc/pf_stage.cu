// Stage-level sequencing of the PatchFusion hot path (SURVEY.md §8b): the kernel order behind the reference's
// coarse_forward / fine_forward / fusion_forward / G2L, issued from C++ over caller-owned weights and ONE workspace.
// Every intermediate is bump-allocated from the workspace in program order, so for given (weights, batch) the
// addresses never change: tensor maps are cached, the call is CUDA-graph capturable, and the workspace size is found by
// running the same code in "dry" mode (no launches).  Reference lines are cited at each step.
#include <cuda_bf16.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "pf_kernels.h"

namespace pf {

typedef __nv_bfloat16 bf16;

static inline int pad_to(int n, int m) { return (n + m - 1) / m * m; }

struct Map {            // NHWC bf16 activation
  bf16* p; int B, H, W, C, ld;
  long long rows() const { return static_cast<long long>(B) * H * W; }
};
struct MapF {           // NHWC fp32 activation (metric-bins tail)
  float* p; int B, H, W, C, ld;
};

struct Ctx {
  uint8_t* base; size_t cap, off;
  bool dry;
  void* stream;
  int err;
  pf_tap_fn tap; void* tap_user;
  int n_e4m3;           // FP8 convs issued so far (names their debug taps)
  const char* lname;    // name of the layer being issued (the engine's weight key), for the calibration and layer taps
  char lbuf[48];

  void* alloc(size_t bytes) {
    off = (off + 255) & ~static_cast<size_t>(255);
    void* p = dry ? nullptr : base + off;
    off += bytes;
    if (!dry && off > cap && !err) err = set_error("workspace too small: need > %zu bytes, have %zu", off, cap);
    return p;
  }
  bool live() const { return !dry && !err; }
  Map map(int B, int H, int W, int C) {
    Map m; m.B = B; m.H = H; m.W = W; m.C = C; m.ld = pad_to(C, 8);
    m.p = static_cast<bf16*>(alloc(static_cast<size_t>(B) * H * W * m.ld * 2));
    return m;
  }
  MapF mapf(int B, int H, int W, int C, int ld) {
    MapF m; m.B = B; m.H = H; m.W = W; m.C = C; m.ld = ld;
    m.p = static_cast<float*>(alloc(static_cast<size_t>(B) * H * W * ld * 4));
    return m;
  }
  void chk(int rc) { if (rc && !err) err = rc; }
  void tap_out(const char* name, const void* ptr, int is_f32, long long rows, int cols, int ld) {
    if (tap && live()) tap(tap_user, name, ptr, is_f32, rows, cols, ld);
  }
  // names the next GEMM / conv (every call site names its layer, so no launch inherits another's name)
  void name(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(lbuf, sizeof(lbuf), fmt, ap);
    va_end(ap);
    lname = lbuf;
  }
  // layer tap "L.<lname>.<part>" of a bf16 GEMM / conv (tests/test_gpu_stage_layers.py checks each layer on exactly
  // these inputs).  Taps issued before the launch (in<s>, res1, res2, x) are copied by the callback in stream order, so
  // they hold what the kernel read.
  bool ltaps() const { return tap != nullptr && lname != nullptr && live(); }
  void ltap(const char* part, const void* ptr, int is_f32, long long rows, int cols, int ld) {
    char nm[64];
    snprintf(nm, sizeof(nm), "L.%s.%s", lname, part);
    tap_out(nm, ptr, is_f32, rows, cols, ld);
  }
};

static Map from_pf(const pf_map& m) {
  Map r; r.p = static_cast<bf16*>(m.ptr); r.B = m.B; r.H = m.H; r.W = m.W; r.C = m.C; r.ld = m.ld;
  return r;
}
static pf_map to_pf(const Map& m) {
  pf_map r; r.ptr = m.p; r.B = m.B; r.H = m.H; r.W = m.W; r.C = m.C; r.ld = m.ld;
  return r;
}

// ---------------------------------------------------------------------------------------------------- gemm wrappers
struct GemmOpt {
  int act = PF_ACT_NONE;
  const Map* res1 = nullptr; const Map* res2 = nullptr;
  const float* gamma = nullptr;
  Map* relu_copy = nullptr;            // second output = relu(v)
  bf16* vt = nullptr; int vt_col0 = 0, vt_seq = 0, vt_seq_pad = 0;
  bool tail = false; int act2 = PF_ACT_NONE; float* out3 = nullptr; int out3_ld = 0; bool skip_main = false;
  int ps_B = 0, ps_H = 0, ps_W = 0;    // ConvTranspose input grid
};

// rows x K matrix sources (a_mode 0) or NHWC images (a_mode 1)
static void gemm_desc_common(pf_gemm_desc& d, const pf_layer& L, const GemmOpt& o, void* out, int out_f32, int out_ld) {
  d.taps = L.taps;
  d.w_ptr = L.w; d.N = L.N; d.Ktot = L.Ktot; d.block_n = 0;
  d.bias = L.bias; d.act = o.act;
  if (o.res1) { d.res1 = o.res1->p; d.res_ld = o.res1->ld; }
  if (o.res2) d.res2 = o.res2->p;
  d.gamma = o.gamma;
  d.out = out; d.out_f32 = out_f32; d.out_ld = out_ld; d.out_col0 = 0;
  if (o.relu_copy) { d.out2 = o.relu_copy->p; d.out2_ld = o.relu_copy->ld; }
  d.ps = L.ps > 1 ? L.ps : 1; d.ps_cout = L.ps_cout;
  if (o.vt) { d.vt = o.vt; d.vt_col0 = o.vt_col0; d.vt_seq = o.vt_seq; d.vt_seq_pad = o.vt_seq_pad; d.vt_dim = L.N - o.vt_col0; }
  if (o.tail) {
    d.w2 = L.w2; d.b2 = L.b2; d.n2 = L.n2; d.act2 = o.act2; d.skip_main = o.skip_main ? 1 : 0;
    d.out3 = o.out3; d.out3_ld = o.out3_ld;
  }
}

// layer taps around a bf16 launch: the residuals and the fp32 stream a gamma update accumulates into before it, the
// outputs after it (out: the main store, out2: the ReLU copy, out3: the fused tail, vt: the qkv's V^T)
static void ltap_pre(Ctx& c, const pf_layer& L, const GemmOpt& o, long long rows, const void* out, int out_ld) {
  if (!c.ltaps()) return;
  if (o.res1) c.ltap("res1", o.res1->p, 0, rows, L.N, o.res1->ld);
  if (o.res2) c.ltap("res2", o.res2->p, 0, rows, L.N, o.res1->ld);
  if (o.gamma) c.ltap("x", out, 1, rows, L.N, out_ld);
}
static void ltap_post(Ctx& c, const pf_layer& L, const GemmOpt& o, long long rows, const void* out, int out_f32,
                      int out_ld) {
  if (!c.ltaps()) return;
  const int ps = L.ps > 1 ? L.ps : 1;
  if (!o.skip_main)
    c.ltap("out", out, out_f32, rows * ps * ps, ps > 1 ? L.ps_cout : (o.vt ? o.vt_col0 : L.N), out_ld);
  if (o.relu_copy) c.ltap("out2", o.relu_copy->p, 0, rows, L.N, o.relu_copy->ld);
  if (o.tail) c.ltap("out3", o.out3, 1, rows, L.n2, o.out3_ld);
  if (o.vt) c.ltap("vt", o.vt, 0, rows / o.vt_seq * (L.N - o.vt_col0), o.vt_seq, o.vt_seq_pad);
}

// D[M, N] = A[M, K] W^T : A is a bf16 matrix with `cols` logical columns and row stride ld
static void linear(Ctx& c, const pf_layer& L, const bf16* A, long long M, int cols, int ld, void* out, int out_f32,
                   int out_ld, const GemmOpt& o = GemmOpt()) {
  if (!c.live()) return;
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = 1; d.a_mode = 0;
  d.a_ptr[0] = A; d.a_c[0] = pad_to(cols, 8); d.a_ld[0] = ld;
  d.M = static_cast<int32_t>(M);
  if (L.ps > 1) { d.NB = o.ps_B; d.H = o.ps_H; d.W = o.ps_W; }
  gemm_desc_common(d, L, o, out, out_f32, out_ld);
  if (c.ltaps()) c.ltap("in0", A, 0, M, cols, ld);
  ltap_pre(c, L, o, M, out, out_ld);
  c.chk(pf_gemm(&d, c.stream));
  ltap_post(c, L, o, M, out, out_f32, out_ld);
}

// FP8 3x3 conv (a layer packed with pf_pack_weight_e4m3: fusion_precision 'fp8'): the sources are quantized with one
// scale per tile (batch index) into one e4m3 map, which the E4M3 halo conv reads.  The map, the scales and the partial
// maxima are bump-allocated here, so only FP8 layers change the workspace.
static void conv_into_e4m3(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, void* out, int out_ld,
                           const GemmOpt& o) {
  const int T = srcs[0]->B, H = srcs[0]->H, W = srcs[0]->W;
  int kc = 0;
  for (int i = 0; i < ns; ++i) kc += pad_to(srcs[i]->C, 64);
  void* q = c.alloc(static_cast<size_t>(T) * H * W * kc);
  float* s_a = static_cast<float*>(c.alloc(static_cast<size_t>(T) * 4));
  float* part = static_cast<float*>(c.alloc(static_cast<size_t>(T) * PF_QUANT_PARTS * 4));
  if (!c.live()) return;
  if (out_ld % 8 || o.res1 || o.res2 || o.relu_copy || o.tail || o.gamma)
    c.chk(set_error("FP8 conv: plain bf16 output only"));
  const void* p[3] = {nullptr, nullptr, nullptr};
  int32_t cc[3] = {0, 0, 0}, ld[3] = {0, 0, 0};
  for (int i = 0; i < ns; ++i) { p[i] = srcs[i]->p; cc[i] = srcs[i]->C; ld[i] = srcs[i]->ld; }
  if (c.live()) c.chk(pf_quantize_e4m3_tiles(ns, p, cc, ld, T, H, W, part, q, s_a, c.stream));
  if (!c.live()) return;
  // calibration tap "amax.<layer>": the tiles' partial maxima [T, PF_QUANT_PARTS] of the input this conv quantized
  if (c.tap != nullptr && c.lname != nullptr) {
    char an[32];
    snprintf(an, sizeof(an), "amax.%s", c.lname);
    c.tap_out(an, part, 1, T, PF_QUANT_PARTS, PF_QUANT_PARTS);
  }
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = ns; d.a_mode = 1;
  d.a_ptr[0] = q;
  for (int i = 0; i < ns; ++i) { d.a_c[i] = pad_to(srcs[i]->C, 8); d.a_ld[i] = kc; }
  d.NB = T; d.H = H; d.W = W;
  gemm_desc_common(d, L, o, out, 0, out_ld);
  d.w_ptr = L.w8;
  d.a_e4m3 = 1; d.s_a = s_a; d.s_w = L.w_scale;
  c.chk(pf_gemm(&d, c.stream));
  // debug taps "e4m3.<k>.src<i>.<H>x<W>" / "e4m3.<k>.out.<H>x<W>": the k-th FP8 conv's bf16 inputs and its output, so a
  // test can check each conv against a reference on exactly the input the kernel saw
  if (c.tap != nullptr && c.live()) {
    char nm[48];
    for (int i = 0; i < ns; ++i) {
      snprintf(nm, sizeof(nm), "e4m3.%d.src%d.%dx%d", c.n_e4m3, i, H, W);
      c.tap_out(nm, srcs[i]->p, 0, srcs[i]->rows(), srcs[i]->C, srcs[i]->ld);
    }
    snprintf(nm, sizeof(nm), "e4m3.%d.out.%dx%d", c.n_e4m3, H, W);
    c.tap_out(nm, out, 0, static_cast<long long>(T) * H * W, L.N, out_ld);
  }
  ++c.n_e4m3;
}

// ---- fusion_precision 'fp8_static': one calibrated amax per conv input (pf_layer.a_amax), fixed before the forward.
// r = 448 / amax and scale = amax / 448, one IEEE fp32 division each, as the kernels' per-tile rule.
static float static_ratio(float amax) { return amax == 0.f ? 0.f : 448.f / amax; }
static float static_scale(float amax) { return amax / 448.f; }

// the sources quantized at L's static ratio into one e4m3 map of kc bytes per pixel (one launch)
static void* quant_static(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, int* kc) {
  const int T = srcs[0]->B, H = srcs[0]->H, W = srcs[0]->W;
  *kc = 0;
  for (int i = 0; i < ns; ++i) *kc += pad_to(srcs[i]->C, 64);
  void* q = c.alloc(static_cast<size_t>(T) * H * W * *kc);
  if (!c.live()) return q;
  const void* p[3] = {nullptr, nullptr, nullptr};
  int32_t cc[3] = {0, 0, 0}, ld[3] = {0, 0, 0};
  for (int i = 0; i < ns; ++i) { p[i] = srcs[i]->p; cc[i] = srcs[i]->C; ld[i] = srcs[i]->ld; }
  c.chk(pf_quantize_e4m3_static(ns, p, cc, ld, T, H, W, static_ratio(*L.a_amax), q, c.stream));
  return q;
}

// the static-scale E4M3 conv (pf_conv3_halo_e4m3_q8_kernel) over the e4m3 map q (sources of src_c channels, kc bytes
// per pixel) with ReLU: a bf16 output, or, when `next` is given, next's e4m3 operand map (out_ld = its kc bytes) at
// next's static ratio.  Debug taps "e4m3s.<layer>.in.<H>x<W>" (the e4m3 map the conv read) and
// "e4m3s.<layer>.out.<H>x<W>" (what it wrote), so a test can check each conv on exactly its input.
static void conv_static_e4m3(Ctx& c, const pf_layer& L, const void* q, int kc, const int* src_c, int ns, int T, int H,
                             int W, void* out, int out_ld, const pf_layer* next) {
  if (!c.live()) return;
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = ns; d.a_mode = 1;
  d.a_ptr[0] = q;
  for (int i = 0; i < ns; ++i) { d.a_c[i] = pad_to(src_c[i], 8); d.a_ld[i] = kc; }
  d.NB = T; d.H = H; d.W = W;
  GemmOpt o; o.act = PF_ACT_RELU;
  gemm_desc_common(d, L, o, out, 0, out_ld);
  d.w_ptr = L.w8;
  d.a_e4m3 = 1; d.s_w = L.w_scale;
  d.a_static = 1; d.a_scale = static_scale(*L.a_amax);
  if (next != nullptr) { d.out_e4m3 = 1; d.out_ratio = static_ratio(*next->a_amax); }
  c.chk(pf_gemm(&d, c.stream));
  if (c.tap != nullptr && c.live() && c.lname != nullptr) {
    char nm[48];
    const long long rows = static_cast<long long>(T) * H * W;
    snprintf(nm, sizeof(nm), "e4m3s.%s.in.%dx%d", c.lname, H, W);
    c.tap_out(nm, q, 2, rows, kc, kc);
    snprintf(nm, sizeof(nm), "e4m3s.%s.out.%dx%d", c.lname, H, W);
    if (next != nullptr) c.tap_out(nm, out, 2, rows, out_ld, out_ld);
    else c.tap_out(nm, out, 0, rows, L.N, out_ld);
  }
}

// ---- vit_precision 'fp8_static': a ViT linear layer on the E4M3 ping-pong GEMM (pf_gemm_pp_e4m3_kernel) over the
// e4m3 matrix A [M, K bytes] at L's static scale; a bf16 / fp32 / gamma / V^T output as `linear`, or, when `next` is
// given, next's e4m3 operand matrix (out_ld bytes) at next's static ratio.
static bool vit_block_fp8(const pf_vit_block& b) {
  return b.qkv.w8 && b.qkv.a_amax && b.fc1.w8 && b.fc1.a_amax && b.fc2.w8 && b.fc2.a_amax;
}
static void linear_e4m3(Ctx& c, const pf_layer& L, const void* A, long long M, int K, void* out, int out_f32, int out_ld,
                        const GemmOpt& o, const pf_layer* next) {
  if (!c.live()) return;
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = 1; d.a_mode = 0;
  d.a_ptr[0] = A; d.a_c[0] = K; d.a_ld[0] = K;
  d.M = static_cast<int32_t>(M);
  gemm_desc_common(d, L, o, out, out_f32, out_ld);
  d.w_ptr = L.w8;
  d.a_e4m3 = 1; d.s_w = L.w_scale;
  d.a_static = 1; d.a_scale = static_scale(*L.a_amax);
  if (next != nullptr) { d.out_e4m3 = 1; d.out_ratio = static_ratio(*next->a_amax); }
  c.chk(pf_gemm(&d, c.stream));
}

// ---- dpt_precision 'fp8_static': the DPT decoder's 19 covered 3x3 convs (the four reassemble convs, the 14 RCU convs
// that run, output_conv1), each with e4m3 panels and a calibrated input amax.  All or none of them run E4M3.
static bool dpt_fp8(const pf_branch& b) {
  const pf_layer* L[19] = {&b.rn[0], &b.rn[1], &b.rn[2], &b.rn[3], &b.ff_c1[3][1], &b.ff_c2[3][1], &b.oc1};
  int n = 7;
  for (int i = 0; i < 3; ++i)
    for (int u = 0; u < 2; ++u) { L[n++] = &b.ff_c1[i][u]; L[n++] = &b.ff_c2[i][u]; }
  for (int i = 0; i < n; ++i)
    if (!L[i]->w8 || !L[i]->w_scale || !L[i]->a_amax || L[i]->taps != 9 || L[i]->num_src != 1) return false;
  return true;
}

// One covered DPT conv on the e4m3 map q (one source of L.src_c[0] channels, kc bytes per pixel) at L's static scale,
// activation `act`.  next != nullptr: the output is next's e4m3 operand map (out_ld bytes; the RCU conv1 -> conv2 hand-
// off, pf_conv3_halo_e4m3_q8_kernel).  Otherwise a bf16 `out` plus the residuals res1 / res2 and, when copy_next is
// given, the e4m3 ReLU copy `copy` (copy_ld bytes) at copy_next's ratio (pf_conv3_halo_e4m3_res_kernel; the q8 kernel
// when there is neither).  Debug taps "e4m3d.<name>.in" (the e4m3 map read), ".out" (bf16, or e4m3 with next),
// ".res1" / ".res2" (the residuals read) and ".copy" (the e4m3 ReLU copy), so a test can check each conv on exactly its
// own inputs.
static void conv_dpt_e4m3(Ctx& c, const char* name, const pf_layer& L, const void* q, int kc, int T, int H, int W, int act,
                          void* out, int out_ld, const pf_layer* next, const Map* res1, const Map* res2, void* copy,
                          int copy_ld, const pf_layer* copy_next) {
  if (!c.live()) return;
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = 1; d.a_mode = 1;
  d.a_ptr[0] = q;
  d.a_c[0] = pad_to(L.src_c[0], 8); d.a_ld[0] = kc;
  d.NB = T; d.H = H; d.W = W;
  GemmOpt o; o.act = act; o.res1 = res1; o.res2 = res2;
  gemm_desc_common(d, L, o, out, 0, out_ld);
  d.w_ptr = L.w8;
  d.a_e4m3 = 1; d.s_w = L.w_scale;
  d.a_static = 1; d.a_scale = static_scale(*L.a_amax);
  if (next != nullptr) { d.out_e4m3 = 1; d.out_ratio = static_ratio(*next->a_amax); }
  if (copy_next != nullptr) { d.out2 = copy; d.out2_ld = copy_ld; d.out2_e4m3 = 1; d.out2_ratio = static_ratio(*copy_next->a_amax); }
  c.chk(pf_gemm(&d, c.stream));
  if (c.tap != nullptr && c.live()) {
    char nm[64];
    const long long rows = static_cast<long long>(T) * H * W;
    snprintf(nm, sizeof(nm), "e4m3d.%s.in", name);
    c.tap_out(nm, q, 2, rows, kc, kc);
    snprintf(nm, sizeof(nm), "e4m3d.%s.out", name);
    if (next != nullptr) c.tap_out(nm, out, 2, rows, out_ld, out_ld);
    else c.tap_out(nm, out, 0, rows, L.N, out_ld);
    const Map* rs[2] = {res1, res2};
    for (int i = 0; i < 2; ++i)
      if (rs[i] != nullptr) {
        snprintf(nm, sizeof(nm), "e4m3d.%s.res%d", name, i + 1);
        c.tap_out(nm, rs[i]->p, 0, rows, rs[i]->C, rs[i]->ld);
      }
    if (copy_next != nullptr) {
      snprintf(nm, sizeof(nm), "e4m3d.%s.copy", name);
      c.tap_out(nm, copy, 2, rows, copy_ld, copy_ld);
    }
  }
}

// layer taps "in<s>": a conv's sources as the kernel reads them (a fused-resample conv's at their own size)
static void ltap_srcs(Ctx& c, const Map* const* srcs, int ns) {
  if (!c.ltaps()) return;
  for (int i = 0; i < ns; ++i) {
    char p[8];
    snprintf(p, sizeof(p), "in%d", i);
    c.ltap(p, srcs[i]->p, 0, srcs[i]->rows(), srcs[i]->C, srcs[i]->ld);
  }
}

// 3x3 / 1x1 conv over up to three channel-concatenated NHWC sources
static void conv_into(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, void* out, int out_f32, int out_ld,
                      const GemmOpt& o = GemmOpt()) {
  if (L.w_scale != nullptr && L.a_amax != nullptr && L.taps == 9 && !out_f32) {
    // a static conv whose producer wrote bf16 (the second conv after a fused-resample first one): one quantize pass
    if (o.act != PF_ACT_RELU || o.res1 || o.res2 || o.relu_copy || o.tail || o.gamma) {
      c.chk(set_error("static FP8 conv: plain ReLU output only"));
      return;
    }
    int kc = 0;
    void* q = quant_static(c, L, srcs, ns, &kc);
    int cs[3] = {0, 0, 0};
    for (int i = 0; i < ns; ++i) cs[i] = srcs[i]->C;
    conv_static_e4m3(c, L, q, kc, cs, ns, srcs[0]->B, srcs[0]->H, srcs[0]->W, out, out_ld, nullptr);
    return;
  }
  if (L.w_scale != nullptr && L.taps == 9 && !out_f32) {
    conv_into_e4m3(c, L, srcs, ns, out, out_ld, o);
    return;
  }
  if (!c.live()) return;
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = ns; d.a_mode = 1;
  for (int i = 0; i < ns; ++i) { d.a_ptr[i] = srcs[i]->p; d.a_c[i] = pad_to(srcs[i]->C, 8); d.a_ld[i] = srcs[i]->ld; }
  d.NB = srcs[0]->B; d.H = srcs[0]->H; d.W = srcs[0]->W;
  gemm_desc_common(d, L, o, out, out_f32, out_ld);
  ltap_srcs(c, srcs, ns);
  ltap_pre(c, L, o, srcs[0]->rows(), out, out_ld);
  c.chk(pf_gemm(&d, c.stream));
  ltap_post(c, L, o, srcs[0]->rows(), out, out_f32, out_ld);
}

// 3x3 conv whose sources are read THROUGH F.interpolate(mode='bilinear', align_corners=True) to (H, W): sources of
// another size are resampled inside the conv kernel's operand stage (pf_gemm_desc.rs_h / rs_w) instead of being
// materialised; sources already at (H, W) are read directly.  Opt-in (PF_OPT_FUSED_RESAMPLE = 1): two producer warps per
// CTA cannot keep up with the tensor pipe (measured 215 -> 317 ms per 4K image), so the default materialises them.
static Map resize(Ctx& c, const Map& x, int OH, int OW);
static Map conv_resampled(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, int H, int W, const GemmOpt& o) {
  Map out = c.map(srcs[0]->B, H, W, L.N);
  if (L.taps != 9 || !option(PF_OPT_FUSED_RESAMPLE)) {
    Map tmp[3];
    const Map* a[3];
    for (int i = 0; i < ns; ++i) { tmp[i] = resize(c, *srcs[i], H, W); a[i] = &tmp[i]; }
    conv_into(c, L, a, ns, out.p, 0, out.ld, o);
    return out;
  }
  if (!c.live()) return out;
  // an FP8 layer reads its bf16 panel here: the resample is produced inside the conv, there is no input to quantize
  if (L.w == nullptr) {
    c.chk(set_error("fused-resample conv: layer has no bf16 panel"));
    return out;
  }
  pf_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.num_src = ns; d.a_mode = 1;
  for (int i = 0; i < ns; ++i) {
    d.a_ptr[i] = srcs[i]->p; d.a_c[i] = pad_to(srcs[i]->C, 8); d.a_ld[i] = srcs[i]->ld;
    if (srcs[i]->H != H || srcs[i]->W != W) { d.rs_h[i] = srcs[i]->H; d.rs_w[i] = srcs[i]->W; }
  }
  d.NB = srcs[0]->B; d.H = H; d.W = W;
  gemm_desc_common(d, L, o, out.p, 0, out.ld);
  ltap_srcs(c, srcs, ns);
  ltap_pre(c, L, o, out.rows(), out.p, out.ld);
  c.chk(pf_gemm(&d, c.stream));
  ltap_post(c, L, o, out.rows(), out.p, 0, out.ld);
  return out;
}

static Map conv(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, const GemmOpt& o = GemmOpt()) {
  Map out = c.map(srcs[0]->B, srcs[0]->H, srcs[0]->W, L.N);
  conv_into(c, L, srcs, ns, out.p, 0, out.ld, o);
  return out;
}
static Map conv1(Ctx& c, const pf_layer& L, const Map& s, const GemmOpt& o = GemmOpt()) {
  const Map* a[1] = {&s};
  return conv(c, L, a, 1, o);
}

// One DoubleConv of the U-Net, X.0 -> ReLU -> X.1 -> ReLU (guided_fusion_model.py DoubleConv), over sources read at
// (H, W) (resampled: through F.interpolate(bilinear, align_corners=True) when their size differs).  `name` is the
// DoubleConv's name in FP8_LAYERS (inc, down<i>, up<i>, cv<i>).  When both convs have static scales ('fp8_static') X.0
// reads its sources through one pf_quantize_e4m3_static and writes X.1's e4m3 operand directly: X.0's output has no
// other consumer, so no bf16 map of it exists.  Otherwise (and for a fused-resample X.0, which stays bf16) the two convs
// run one after the other as before.
static Map resize(Ctx& c, const Map& x, int OH, int OW);
static Map conv_resampled(Ctx& c, const pf_layer& L, const Map* const* srcs, int ns, int H, int W, const GemmOpt& o);
static Map double_conv(Ctx& c, const pf_layer& L0, const pf_layer& L1, const Map* const* srcs, int ns, int H, int W,
                       bool resampled, const char* name) {
  GemmOpt gr; gr.act = PF_ACT_RELU;
  char n0[24], n1[24];
  snprintf(n0, sizeof(n0), "%s.0", name);
  snprintf(n1, sizeof(n1), "%s.1", name);
  const bool st = L0.w_scale && L1.w_scale && L0.a_amax && L1.a_amax && L0.taps == 9 && L1.taps == 9;
  if (!st || (resampled && option(PF_OPT_FUSED_RESAMPLE))) {
    c.lname = n0;
    Map y = resampled ? conv_resampled(c, L0, srcs, ns, H, W, gr) : conv(c, L0, srcs, ns, gr);
    c.lname = n1;
    Map x = conv1(c, L1, y, gr);
    c.lname = nullptr;
    return x;
  }
  Map tmp[3];
  const Map* a[3];
  int cs[3] = {0, 0, 0};
  for (int i = 0; i < ns; ++i) {
    tmp[i] = resampled ? resize(c, *srcs[i], H, W) : *srcs[i];
    a[i] = &tmp[i];
    cs[i] = srcs[i]->C;
  }
  const int T = srcs[0]->B;
  int kc0 = 0;
  void* q0 = quant_static(c, L0, a, ns, &kc0);
  const int kc1 = pad_to(L0.N, 64);
  void* q1 = c.alloc(static_cast<size_t>(T) * H * W * kc1);
  Map out = c.map(T, H, W, L1.N);
  c.lname = n0;
  conv_static_e4m3(c, L0, q0, kc0, cs, ns, T, H, W, q1, kc1, &L1);
  c.lname = n1;
  const int c1[1] = {L0.N};
  conv_static_e4m3(c, L1, q1, kc1, c1, 1, T, H, W, out.p, out.ld, nullptr);
  c.lname = nullptr;
  return out;
}

// F.interpolate(mode='bilinear', align_corners=True)
static Map resize(Ctx& c, const Map& x, int OH, int OW) {
  if (x.H == OH && x.W == OW) return x;
  Map out = c.map(x.B, OH, OW, x.C);
  if (c.live()) c.chk(pf_resize_bilinear(x.p, x.B, x.H, x.W, pad_to(x.C, 8), x.ld, OH, OW, out.p, out.ld, 0, c.stream));
  return out;
}

// ---------------------------------------------------------------------------------------------------- metric-bins head
// zoedepth_v1.py:173-219 (branch heads, with the relative-depth condition) / patchfusion.py:297-339 (fusion head)
static void metric_head(Ctx& c, const pf_head& Hd, const Map& x, const Map* x_blocks, const Map& last, const MapF* rel,
                        float* depth_out) {
  const int B = x.B, nb = Hd.n_bins, E = Hd.bin_embedding_dim;
  // two-layer 1x1 MLP `_net` (localbins_layers.py:84-89,110-114, attractor.py:157-162)
  // `mod`: the module's name in the engine's head weights (layer taps "L.head.<mod>.0|2")
  auto mlp_bf16 = [&](const pf_layer& L0, const pf_layer& L2, const Map& src, const char* mod) -> Map {
    GemmOpt o0; o0.act = PF_ACT_RELU;
    c.name("head.%s.0", mod);
    Map t = conv1(c, L0, src, o0);
    c.name("head.%s.2", mod);
    return conv1(c, L2, t);
  };
  auto mlp_f32 = [&](const pf_layer& L0, const pf_layer& L2, const Map& src, int act2, const char* mod) -> MapF {
    const int n_out = L0.n2 > 0 ? L0.n2 : L2.N;
    MapF o = c.mapf(B, src.H, src.W, n_out, pad_to(pad_to(n_out, 8), 32));
    c.name("head.%s.0", mod);
    if (L0.n2 > 0) {       // narrow second layer fused into the first layer's epilogue
      GemmOpt g; g.act = PF_ACT_RELU; g.tail = true; g.act2 = act2; g.out3 = o.p; g.out3_ld = o.ld; g.skip_main = true;
      conv1(c, L0, src, g);
    } else {
      GemmOpt o0; o0.act = PF_ACT_RELU;
      Map t = conv1(c, L0, src, o0);
      const Map* a[1] = {&t};
      GemmOpt g2; g2.act = act2;
      c.name("head.%s.2", mod);
      conv_into(c, L2, a, 1, o.p, 1, o.ld, g2);
    }
    return o;
  };
  // bin_centers_type (zoedepth_v1.py:90-105): SeedBinRegressor ends in ReLU and normalises widths into centres,
  // AttractorLayer ends in ReLU and sorts and clips its metric output.  The softplus head launches and allocates exactly
  // as if the type did not exist: the extra buffers below come only with the other types.
  const int type = Hd.bin_centers_type;
  if (type < PF_BINS_SOFTPLUS || type > PF_BINS_HYBRID2) {
    c.chk(set_error("metric head: unknown bin_centers_type %d", type));
    return;
  }
  const bool normed_seed = type == PF_BINS_NORMED || type == PF_BINS_HYBRID1;
  const bool normed_att = type == PF_BINS_NORMED || type == PF_BINS_HYBRID2;
  MapF b_prev = mlp_f32(Hd.seed0, Hd.seed2, x, normed_seed ? PF_ACT_RELU : PF_ACT_SOFTPLUS,   // fp32 [B,h,w,64]
                        "seed_bin_regressor");
  const float* b_t = b_prev.p;
  if (type != PF_BINS_SOFTPLUS) {     // seed centres; normalised to [0, 1] for the normed attractors (zoedepth_v1.py:176-181)
    const long long px = static_cast<long long>(B) * x.H * x.W;
    float* sb = static_cast<float*>(c.alloc(static_cast<size_t>(px) * nb * 4));
    if (c.live())
      c.chk(pf_seed_bins(b_prev.p, b_prev.ld, px, nb, (normed_seed ? PF_SEED_NORMED : 0) | (normed_att ? PF_SEED_TO_UNIT : 0),
                         Hd.min_depth, Hd.max_depth, sb, c.stream));
    b_t = sb;
    c.tap_out("seed", sb, 1, px, nb, nb);
  }
  Map prev_emb = mlp_bf16(Hd.seedproj0, Hd.seedproj2, x, "seed_projector");
  const float* centers = nullptr;
  int ph = x.H, pw = x.W;
  for (int i = 0; i < 4; ++i) {
    const Map& xb = x_blocks[i];
    char mod[16];
    snprintf(mod, sizeof(mod), "projectors.%d", i);
    Map emb = mlp_bf16(Hd.proj0[i], Hd.proj2[i], xb, mod);
    Map s = c.map(B, xb.H, xb.W, E);
    if (c.live()) c.chk(pf_add_upsampled(emb.p, B, xb.H, xb.W, E, prev_emb.p, prev_emb.H, prev_emb.W, s.p, c.stream));
    snprintf(mod, sizeof(mod), "attractors.%d", i);
    MapF A = mlp_f32(Hd.att0[i], Hd.att2[i], s, normed_att ? PF_ACT_RELU : PF_ACT_SOFTPLUS, mod);
    const size_t bytes = static_cast<size_t>(B) * xb.H * xb.W * nb * 4;
    float* b_new = static_cast<float*>(c.alloc(bytes));
    if (normed_att) {
      // only the last level's sorted metric centres are read (zoedepth_v1.py:217-219)
      float* cen = i == 3 ? static_cast<float*>(c.alloc(bytes)) : nullptr;
      if (c.live())
        c.chk(pf_attractor_normed(A.p, A.ld, Hd.n_attractors[i], b_t, ph, pw, B, xb.H, xb.W, nb, Hd.attractor_flags,
                                  Hd.min_depth, Hd.max_depth, b_new, cen, c.stream));
      if (cen != nullptr) centers = cen;
    } else if (c.live()) {
      c.chk(pf_attractor(A.p, A.ld, Hd.n_attractors[i], b_t, ph, pw, B, xb.H, xb.W, nb, Hd.attractor_flags, b_new, c.stream));
    }
    b_t = b_new; ph = xb.H; pw = xb.W; prev_emb = emb;
    char nm[8];
    snprintf(nm, sizeof(nm), "b%d", i);
    c.tap_out(nm, b_new, 1, static_cast<long long>(B) * xb.H * xb.W, nb, nb);
  }
  if (normed_att) {
    c.tap_out("centers", centers, 1, static_cast<long long>(B) * ph * pw, nb, nb);
    b_t = centers;
  }
  const int H = last.H, W = last.W;
  Map emb_up = resize(c, prev_emb, H, W);
  float* pt = nullptr;
  GemmOpt g; g.act = PF_ACT_GELU; g.tail = true; g.act2 = PF_ACT_SOFTPLUS; g.out3_ld = 8; g.skip_main = true;
  c.name("head.clb.0");
  if (rel != nullptr) {
    Map relb = c.map(B, H, W, 1);
    if (c.live()) c.chk(pf_f32_to_bf16(rel->p, static_cast<int64_t>(B) * H * W * rel->ld, relb.p, c.stream));
    pt = static_cast<float*>(c.alloc(static_cast<size_t>(B) * H * W * 8 * 4));
    g.out3 = pt;
    const Map* a[3] = {&last, &relb, &emb_up};
    conv(c, Hd.clb0, a, 3, g);         // CLB MLP: 1x1 (161->80) + GELU with 80->4 + Softplus fused (dist_layers.py:91-98)
  } else {
    pt = static_cast<float*>(c.alloc(static_cast<size_t>(B) * H * W * 8 * 4));
    g.out3 = pt;
    const Map* a[2] = {&last, &emb_up};
    conv(c, Hd.clb0, a, 2, g);
  }
  if (c.live())
    c.chk(pf_logbinom_depth(pt, 8, b_t, ph, pw, B, H, W, nb, Hd.min_temp, Hd.max_temp, depth_out, c.stream));
}

// ---------------------------------------------------------------------------------------------------- one branch
static void branch_run(Ctx& c, const pf_branch& Wb, const float* images, int B, pf_branch_out* out) {
  const int H = Wb.H, W = Wb.W, gh = H / 14, gw = W / 14;
  const int D = Wb.dim, C = Wb.features;
  const int npatch = gh * gw, seq = npatch + 1, seq_pad = pad_to(seq, 8);
  const long long rows = static_cast<long long>(B) * seq;
  // ---- tokens: normalise + 14x14 patch gather, patch-embed GEMM, cls + pos (vision_transformer.py:212-219)
  bf16* a0 = static_cast<bf16*>(c.alloc(static_cast<size_t>(B) * npatch * 592 * 2));
  if (c.live()) c.chk(pf_patch_im2col(images, B, H, W, a0, 592, c.stream));
  float* patch = static_cast<float*>(c.alloc(static_cast<size_t>(B) * npatch * D * 4));
  c.name("patch");
  linear(c, Wb.patch, a0, static_cast<long long>(B) * npatch, 592, 592, patch, 1, D);
  float* x = static_cast<float*>(c.alloc(static_cast<size_t>(rows) * D * 4));
  if (c.live()) c.chk(pf_assemble_tokens(patch, Wb.cls, Wb.pos, B, npatch, D, x, c.stream));
  c.tap_out("tokens", x, 1, rows, D, D);
  bf16* hbuf = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * D * 2));
  bf16* qk = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * 2 * D * 2));
  bf16* vt = static_cast<bf16*>(c.alloc(static_cast<size_t>(B) * D * seq_pad * 2));
  bf16* att = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * D * 2));
  bf16* hid = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * 4 * D * 2));
  if (c.live() && seq_pad > seq) {
    // V^T pad columns [seq, seq_pad): the attention kernel never reads them (its V^T tensor map is seq wide, so TMA
    // zero-fills the last KV tile; tests/test_gpu_attn_parity.py runs it with NaN there).  Zeroed anyway as defence in
    // depth: the qkv GEMM writes only columns < seq, and a NaN here would turn any future reader's P = 0 into NaN.
    cudaError_t e = cudaMemset2DAsync(vt + seq, static_cast<size_t>(seq_pad) * 2, 0, static_cast<size_t>(seq_pad - seq) * 2,
                                      static_cast<size_t>(B) * D, static_cast<cudaStream_t>(c.stream));
    if (e != cudaSuccess) c.chk(set_error("cudaMemset2DAsync(vt pad): %s", cudaGetErrorString(e)));
  }
  // vit_precision 'fp8_static' (blocks whose qkv, fc1 and fc2 carry e4m3 panels and calibrated input amax): the e4m3
  // operands of qkv / fc1 ([rows, D] bytes, written by LN1 / LN2) and of fc2 ([rows, 4D] bytes, written by fc1).  Only
  // such a branch allocates them, so the bf16 workspace is what it was.
  bool any_fp8 = false;
  for (int i = 0; i < Wb.depth; ++i) any_fp8 = any_fp8 || vit_block_fp8(Wb.blocks[i]);
  uint8_t* h8 = any_fp8 ? static_cast<uint8_t*>(c.alloc(static_cast<size_t>(rows) * D)) : nullptr;
  uint8_t* hid8 = any_fp8 ? static_cast<uint8_t*>(c.alloc(static_cast<size_t>(rows) * 4 * D)) : nullptr;
  Map feats[4];
  int nf = 0;
  char nm[32];
  for (int i = 0; i < Wb.depth; ++i) {
    const pf_vit_block& bw = Wb.blocks[i];
    // x += ls1 * proj(attn(LN(x)));  x += ls2 * fc2(gelu(fc1(LN(x))))   (dinov2/layers/block.py:82-107)
    GemmOpt oq; oq.vt = vt; oq.vt_col0 = 2 * D; oq.vt_seq = seq; oq.vt_seq_pad = seq_pad;
    GemmOpt o1; o1.gamma = bw.ls1;
    GemmOpt of; of.act = PF_ACT_GELU;
    GemmOpt o2; o2.gamma = bw.ls2;
    if (vit_block_fp8(bw)) {
      // LN1 -> e4m3 at qkv's ratio, qkv on the e4m3 GEMM, attention, proj in bf16 (its input comes from the attention
      // kernel), LN2 -> e4m3 at fc1's ratio, fc1 + GELU -> fc2's e4m3 operand, fc2 + gamma reduce-add into x.  Debug
      // taps "e4m3v.<i>.<lin>.in" (the e4m3 operand the linear read) and "e4m3v.<i>.<lin>.out" (what it wrote; qkv's V^T
      // third is "e4m3v.<i>.qkv.vt", fc2's residual stream before its update "e4m3v.<i>.fc2.x").
      if (c.live())
        c.chk(pf_layernorm_e4m3(x, D, bw.n1w, bw.n1b, 1e-6f, static_cast<int32_t>(rows), D, static_ratio(*bw.qkv.a_amax), h8,
                                D, c.stream));
      linear_e4m3(c, bw.qkv, h8, rows, D, qk, 0, 2 * D, oq, nullptr);
      if (c.tap != nullptr) {
        snprintf(nm, sizeof(nm), "e4m3v.%d.qkv.in", i);
        c.tap_out(nm, h8, 2, rows, D, D);
        snprintf(nm, sizeof(nm), "e4m3v.%d.qkv.out", i);
        c.tap_out(nm, qk, 0, rows, 2 * D, 2 * D);
        snprintf(nm, sizeof(nm), "e4m3v.%d.qkv.vt", i);
        c.tap_out(nm, vt, 0, static_cast<long long>(B) * D, seq_pad, seq_pad);
      }
      if (c.live()) c.chk(pf_attention(qk, 2 * D, vt, B, seq, seq_pad, Wb.heads, 0.125f, att, D, c.stream));
      c.name("b%d.proj", i);
      linear(c, bw.proj, att, rows, D, D, x, 1, D, o1);
      if (c.live())
        c.chk(pf_layernorm_e4m3(x, D, bw.n2w, bw.n2b, 1e-6f, static_cast<int32_t>(rows), D, static_ratio(*bw.fc1.a_amax), h8,
                                D, c.stream));
      linear_e4m3(c, bw.fc1, h8, rows, D, hid8, 0, 4 * D, of, &bw.fc2);
      if (c.tap != nullptr) {
        snprintf(nm, sizeof(nm), "e4m3v.%d.fc1.in", i);
        c.tap_out(nm, h8, 2, rows, D, D);
        snprintf(nm, sizeof(nm), "e4m3v.%d.fc1.out", i);
        c.tap_out(nm, hid8, 2, rows, 4 * D, 4 * D);
        snprintf(nm, sizeof(nm), "e4m3v.%d.fc2.in", i);
        c.tap_out(nm, hid8, 2, rows, 4 * D, 4 * D);
        snprintf(nm, sizeof(nm), "e4m3v.%d.fc2.x", i);
        c.tap_out(nm, x, 1, rows, D, D);
      }
      linear_e4m3(c, bw.fc2, hid8, rows, 4 * D, x, 1, D, o2, nullptr);
      snprintf(nm, sizeof(nm), "e4m3v.%d.fc2.out", i);
      c.tap_out(nm, x, 1, rows, D, D);
    } else {
      // the calibration taps "amaxv.<i>.<lin>": the bf16 inputs of qkv, fc1 and fc2, whose amax 'fp8_static' runs with
      if (c.live()) c.chk(pf_layernorm(x, D, bw.n1w, bw.n1b, 1e-6f, static_cast<int32_t>(rows), D, hbuf, D, c.stream));
      if (c.tap != nullptr) {
        snprintf(nm, sizeof(nm), "amaxv.%d.qkv", i);
        c.tap_out(nm, hbuf, 0, rows, D, D);
      }
      c.name("b%d.qkv", i);
      linear(c, bw.qkv, hbuf, rows, D, D, qk, 0, 2 * D, oq);
      if (c.live()) c.chk(pf_attention(qk, 2 * D, vt, B, seq, seq_pad, Wb.heads, 0.125f, att, D, c.stream));
      c.name("b%d.proj", i);
      linear(c, bw.proj, att, rows, D, D, x, 1, D, o1);
      if (c.live()) c.chk(pf_layernorm(x, D, bw.n2w, bw.n2b, 1e-6f, static_cast<int32_t>(rows), D, hbuf, D, c.stream));
      if (c.tap != nullptr) {
        snprintf(nm, sizeof(nm), "amaxv.%d.fc1", i);
        c.tap_out(nm, hbuf, 0, rows, D, D);
      }
      c.name("b%d.fc1", i);
      linear(c, bw.fc1, hbuf, rows, D, D, hid, 0, 4 * D, of);
      if (c.tap != nullptr) {
        snprintf(nm, sizeof(nm), "amaxv.%d.fc2", i);
        c.tap_out(nm, hid, 0, rows, 4 * D, 4 * D);
      }
      c.name("b%d.fc2", i);
      linear(c, bw.fc2, hid, rows, 4 * D, 4 * D, x, 1, D, o2);
    }
    snprintf(nm, sizeof(nm), "block%d", i);
    c.tap_out(nm, x, 1, rows, D, D);
    if (i >= Wb.depth - 4) {
      // get_intermediate_layers(x, 4): final LayerNorm of the LAST four blocks' patch tokens, cls dropped
      // (dpt.py:149, vision_transformer.py:297-321) - one batched launch over all images
      Map f = c.map(B, gh, gw, D);
      if (c.live()) c.chk(pf_layernorm_grouped(x, D, Wb.nw, Wb.nb, 1e-6f, B, seq, 1, npatch, D, f.p, D, c.stream));
      feats[nf++] = f;
    }
  }
  // ---- DPT head (dpt.py:97-130, blocks.py:69-153)
  const int* oc = Wb.out_channels;
  Map lay[4];
  for (int i = 0; i < 4; ++i) {
    Map p = c.map(B, gh, gw, oc[i]);
    c.name("proj%d", i);
    linear(c, Wb.proj[i], feats[i].p, feats[i].rows(), D, feats[i].ld, p.p, 0, p.ld);
    if (i == 0 || i == 1) {
      const int k = i == 0 ? 4 : 2;
      Map o = c.map(B, gh * k, gw * k, oc[i]);
      GemmOpt g; g.ps_B = B; g.ps_H = gh; g.ps_W = gw;
      c.name("rs%d", i);
      linear(c, i == 0 ? Wb.rs0 : Wb.rs1, p.p, p.rows(), oc[i], p.ld, o.p, 0, o.ld, g);
      lay[i] = o;
    } else if (i == 2) {
      lay[i] = p;
    } else {
      const int oh = (gh - 1) / 2 + 1, ow = (gw - 1) / 2 + 1;
      bf16* col = static_cast<bf16*>(c.alloc(static_cast<size_t>(B) * oh * ow * 9 * oc[3] * 2));
      if (c.live()) c.chk(pf_im2col_3x3_s2(p.p, B, gh, gw, oc[3], p.ld, col, c.stream));
      Map o = c.map(B, oh, ow, oc[3]);
      c.name("rs3");
      linear(c, Wb.rs3, col, static_cast<long long>(B) * oh * ow, 9 * oc[3], 9 * oc[3], o.p, 0, o.ld);
      lay[i] = o;
    }
  }
  // dpt_precision 'fp8_static' (dpt_fp8): layer{i}_rn reads lay[i] through one static quantize and writes the bf16
  // rn[i] and the e4m3 ReLU copy of it that the first RCU conv1 reading it takes; an RCU conv1 reads that copy and
  // writes its conv2's e4m3 operand; conv2 adds x (and the path) and writes bf16 y, plus the e4m3 ReLU copy the next
  // unit's conv1 reads; output_conv1 reads the resized p1 through one static quantize.  No bf16 ReLU copy or t map of
  // a covered conv exists.  The bf16 path keeps the calibration taps "amaxd.<conv>" on each covered conv's bf16 input.
  const bool f8 = dpt_fp8(Wb);
  static const char* const kRn[4] = {"layer1_rn", "layer2_rn", "layer3_rn", "layer4_rn"};
  char dn[48];
  auto amax_tap = [&](const char* conv, const Map& m) {
    if (c.tap == nullptr) return;
    char an[64];
    snprintf(an, sizeof(an), "amaxd.%s", conv);
    c.tap_out(an, m.p, 0, m.rows(), m.C, m.ld);
  };
  // the conv1 that reads rn[i]'s ReLU: refinenet4's only unit for rn[3], the first unit of refinenet{i+1} otherwise
  auto rn_reader = [&](int i) -> const pf_layer& { return i == 3 ? Wb.ff_c1[3][1] : Wb.ff_c1[i][0]; };
  Map rn[4], rn_relu[4];
  uint8_t* rn8[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int i = 0; i < 4; ++i) {
    if (f8) {
      int kc = 0;
      const Map* a[1] = {&lay[i]};
      void* q = quant_static(c, Wb.rn[i], a, 1, &kc);
      rn[i] = c.map(lay[i].B, lay[i].H, lay[i].W, C);
      rn8[i] = static_cast<uint8_t*>(c.alloc(static_cast<size_t>(rn[i].rows()) * pad_to(C, 64)));
      conv_dpt_e4m3(c, kRn[i], Wb.rn[i], q, kc, lay[i].B, lay[i].H, lay[i].W, PF_ACT_NONE, rn[i].p, rn[i].ld, nullptr,
                    nullptr, nullptr, rn8[i], pad_to(C, 64), &rn_reader(i));
    } else {
      amax_tap(kRn[i], lay[i]);
      rn_relu[i] = c.map(lay[i].B, lay[i].H, lay[i].W, C);
      GemmOpt g; g.relu_copy = &rn_relu[i];
      c.name("rn%d", i);
      rn[i] = conv1(c, Wb.rn[i], lay[i], g);
    }
  }
  // ResidualConvUnit: y = conv2(relu(conv1(relu(x)))) + x (+ extra); optionally also relu(y)
  auto rcu = [&](int wi, int u, const Map& xin, const Map& xrelu, const Map* extra, Map* relu_copy) -> Map {
    char n1[48], n2[48];
    snprintf(n1, sizeof(n1), "refinenet%d.resConfUnit%d.conv1", wi, u);
    snprintf(n2, sizeof(n2), "refinenet%d.resConfUnit%d.conv2", wi, u);
    amax_tap(n1, xrelu);
    GemmOpt g1; g1.act = PF_ACT_RELU;
    c.name("ff%d.u%d.c1", wi, u);
    Map t = conv1(c, Wb.ff_c1[wi - 1][u - 1], xrelu, g1);
    amax_tap(n2, t);
    GemmOpt g2; g2.res1 = &xin; g2.res2 = extra;
    if (relu_copy) { *relu_copy = c.map(xin.B, xin.H, xin.W, C); g2.relu_copy = relu_copy; }
    c.name("ff%d.u%d.c2", wi, u);
    return conv1(c, Wb.ff_c2[wi - 1][u - 1], t, g2);
  };
  // the same unit in FP8: x8 is the e4m3 ReLU copy of xin at conv1's ratio; copy8 (when given) receives y's e4m3 ReLU
  // copy at the ratio of the next unit's conv1
  auto rcu8 = [&](int wi, int u, const Map& xin, const uint8_t* x8, const Map* extra, uint8_t** copy8) -> Map {
    const pf_layer& c1 = Wb.ff_c1[wi - 1][u - 1];
    const pf_layer& c2 = Wb.ff_c2[wi - 1][u - 1];
    const int kc = pad_to(C, 64);
    uint8_t* t8 = static_cast<uint8_t*>(c.alloc(static_cast<size_t>(xin.rows()) * kc));
    snprintf(dn, sizeof(dn), "refinenet%d.resConfUnit%d.conv1", wi, u);
    conv_dpt_e4m3(c, dn, c1, x8, kc, xin.B, xin.H, xin.W, PF_ACT_RELU, t8, kc, &c2, nullptr, nullptr, nullptr, 0, nullptr);
    Map y = c.map(xin.B, xin.H, xin.W, C);
    if (copy8 != nullptr) *copy8 = static_cast<uint8_t*>(c.alloc(static_cast<size_t>(xin.rows()) * kc));
    snprintf(dn, sizeof(dn), "refinenet%d.resConfUnit%d.conv2", wi, u);
    conv_dpt_e4m3(c, dn, c2, t8, kc, xin.B, xin.H, xin.W, PF_ACT_NONE, y.p, y.ld, nullptr, &xin, extra,
                  copy8 != nullptr ? *copy8 : nullptr, kc, copy8 != nullptr ? &Wb.ff_c1[wi - 1][1] : nullptr);
    return y;
  };
  // FeatureFusionBlock; the 1x1 out_conv commutes with the bilinear upsample and runs at the low resolution
  auto ffb = [&](int wi, const Map* path, int i, int OH, int OW) -> Map {
    Map s = rn[i], y;
    if (f8) {
      uint8_t* s8 = rn8[i];
      if (path != nullptr) s = rcu8(wi, 1, rn[i], rn8[i], path, &s8);
      y = rcu8(wi, 2, s, s8, nullptr, nullptr);
    } else {
      Map s_relu = rn_relu[i];
      if (path != nullptr) s = rcu(wi, 1, rn[i], rn_relu[i], path, &s_relu);
      y = rcu(wi, 2, s, s_relu, nullptr, nullptr);
    }
    c.name("ff%d.out", wi);
    y = conv1(c, Wb.ff_out[wi - 1], y);
    return resize(c, y, OH, OW);
  };
  Map p4 = ffb(4, nullptr, 3, rn[2].H, rn[2].W);
  Map p3 = ffb(3, &p4, 2, rn[1].H, rn[1].W);
  Map p2 = ffb(2, &p3, 1, rn[0].H, rn[0].W);
  Map p1 = ffb(1, &p2, 0, rn[0].H * 2, rn[0].W * 2);
  Map o;
  if (f8) {
    int kc = 0;
    const Map* a[1] = {&p1};
    void* q = quant_static(c, Wb.oc1, a, 1, &kc);
    o = c.map(p1.B, p1.H, p1.W, Wb.oc1.N);
    conv_dpt_e4m3(c, "output_conv1", Wb.oc1, q, kc, p1.B, p1.H, p1.W, PF_ACT_NONE, o.p, o.ld, nullptr, nullptr, nullptr,
                  nullptr, 0, nullptr);
  } else {
    amax_tap("output_conv1", p1);
    c.name("oc1");
    o = conv1(c, Wb.oc1, p1);
  }
  o = resize(c, o, H, W);
  MapF rel = c.mapf(B, H, W, 1, 8);
  if (c.live()) {     // only column 0 is produced (fused 32 -> 1 layer); the 7 pad columns feed zero weights and must be finite
    cudaError_t e = cudaMemsetAsync(rel.p, 0, static_cast<size_t>(B) * H * W * 8 * 4, static_cast<cudaStream_t>(c.stream));
    if (e != cudaSuccess) c.chk(set_error("cudaMemsetAsync(rel): %s", cudaGetErrorString(e)));
  }
  // output_conv2: 3x3 C/2 -> 32 + ReLU (the hooked `out_conv` tap) with the 1x1 32 -> 1 + ReLU fused in its epilogue
  GemmOpt go; go.act = PF_ACT_RELU; go.tail = true; go.act2 = PF_ACT_RELU; go.out3 = rel.p; go.out3_ld = rel.ld;
  c.name("oc2.0");
  Map out_conv = conv1(c, Wb.oc2, o, go);
  c.name("conv2");
  Map x_d0 = conv1(c, Wb.conv2, rn[3]);
  c.tap_out("rel", rel.p, 1, static_cast<long long>(B) * H * W, 1, 8);
  float* depth = static_cast<float*>(c.alloc(static_cast<size_t>(B) * H * W * 4));
  Map blocks[4] = {p4, p3, p2, p1};
  metric_head(c, Wb.head, x_d0, blocks, out_conv, &rel, depth);
  if (out != nullptr && !c.dry) {
    out->depth = depth;
    out->feats[0] = to_pf(x_d0); out->feats[1] = to_pf(p4); out->feats[2] = to_pf(p3); out->feats[3] = to_pf(p2);
    out->feats[4] = to_pf(p1); out->feats[5] = to_pf(out_conv);
  }
}

// ---------------------------------------------------------------------------------------------------- G2L
// B whole images at once (B = coarse[i].B): every op below is one launch over the batch.  Row-wise ops and GEMMs see
// B*n (or B*Hp*Wp) rows, window attention and the pad / crop kernels take the image as a grid dimension.
static void g2l_run(Ctx& c, const pf_fusion& Wf, const pf_map* coarse, pf_map* outs) {
  const int WS = 12;
  const int B = coarse[0].B;
  for (int i = 0; i < 6; ++i) {
    const pf_g2l_level& L = Wf.g2l[i];
    const Map f = from_pf(coarse[i]);
    const int cc = L.C, h = f.H, w = f.W, n = h * w;
    const int Hp = (h + WS - 1) / WS * WS, Wp = (w + WS - 1) / WS * WS;
    const long long rows = static_cast<long long>(B) * n, prow = static_cast<long long>(B) * Hp * Wp;
    if (!c.dry && L.ape_rows != n && !c.err)
      c.err = set_error("guided_fusion.num_patches[%d] = %d does not match the %dx%d coarse map", i, L.ape_rows, h, w);
    if (f.B != B && !c.err) c.err = set_error("pf_g2l_forward: coarse map %d has batch %d, map 0 has %d", i, f.B, B);
    float* x = static_cast<float*>(c.alloc(static_cast<size_t>(rows) * cc * 4));
    if (c.live()) c.chk(pf_g2l_embed_batched(f.p, f.ld, L.ape, B, n, cc, x, c.stream));
    bf16* npad = static_cast<bf16*>(c.alloc(static_cast<size_t>(prow) * cc * 2));
    bf16* qkv = static_cast<bf16*>(c.alloc(static_cast<size_t>(prow) * 3 * cc * 2));
    bf16* att = static_cast<bf16*>(c.alloc(static_cast<size_t>(prow) * cc * 2));
    float* prj = static_cast<float*>(c.alloc(static_cast<size_t>(prow) * cc * 4));
    bf16* hb = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * cc * 2));
    bf16* hid = static_cast<bf16*>(c.alloc(static_cast<size_t>(rows) * 4 * cc * 2));
    for (int b = 0; b < L.depth; ++b) {
      const pf_g2l_block& bw = L.blocks[b];
      const int shift = (b % 2 == 0) ? 0 : WS / 2;
      if (c.live()) c.chk(pf_swin_norm_pad_batched(x, bw.n1w, bw.n1b, 1e-5f, B, h, w, Hp, Wp, cc, npad, c.stream));
      c.name("g2l%d.b%d.qkv", i, b);
      linear(c, bw.qkv, npad, prow, cc, cc, qkv, 0, 3 * cc);
      if (c.live()) c.chk(pf_window_attention_batched(qkv, bw.table, B, Hp, Wp, cc, L.heads, shift, att, c.stream));
      c.name("g2l%d.b%d.proj", i, b);
      linear(c, bw.proj, att, prow, cc, cc, prj, 1, cc);
      if (c.live()) c.chk(pf_swin_residual_crop_batched(x, prj, B, h, w, Hp, Wp, cc, c.stream));
      if (c.live()) c.chk(pf_layernorm(x, cc, bw.n2w, bw.n2b, 1e-5f, static_cast<int32_t>(rows), cc, hb, cc, c.stream));
      GemmOpt g1; g1.act = PF_ACT_GELU;
      c.name("g2l%d.b%d.fc1", i, b);
      linear(c, bw.fc1, hb, rows, cc, cc, hid, 0, 4 * cc, g1);
      GemmOpt g2; g2.gamma = L.ones;
      c.name("g2l%d.b%d.fc2", i, b);
      linear(c, bw.fc2, hid, rows, 4 * cc, 4 * cc, x, 1, cc, g2);
    }
    Map o = c.map(B, h, w, cc);
    if (c.live()) c.chk(pf_layernorm(x, cc, L.nw, L.nb, 1e-5f, static_cast<int32_t>(rows), cc, o.p, o.ld, c.stream));
    if (!c.dry && outs) outs[i] = to_pf(o);
  }
}

// ---------------------------------------------------------------------------------------------------- fusion
// tile_image (nullable): tile t crops image tile_image[t] of the batch-B coarse depth, coarse maps and G2L maps
static void fusion_run(Ctx& c, const pf_fusion& Wf, const float* crops, const float* boxes, const int32_t* tile_image,
                       int T, const float* fine_depth, const pf_map* fine_feats, const float* coarse_depth,
                       const pf_map* coarse_feats, const pf_map* g2l_maps, float* depth_out) {
  const int H = Wf.H, W = Wf.W;
  // ROI crop-zoom of the whole-image coarse maps + fused 3x3 convs with the fine maps (patchfusion.py:240-267)
  Map guide[5];
  for (int i = 0; i < 5; ++i) {
    const Map cf = from_pf(coarse_feats[i]);
    const Map ff = from_pf(fine_feats[i]);
    Map roi = c.map(T, cf.H, cf.W, cf.C);
    if (c.live())
      c.chk(pf_roi_crop_zoom_batched(cf.p, 0, cf.H, cf.W, pad_to(cf.C, 8), cf.ld, tile_image, boxes, T,
                                     static_cast<float>(cf.H) / H, roi.p, roi.ld, 0, c.stream));
    const Map* a[2] = {&roi, &ff};
    c.name("fc%d", i);
    guide[i] = conv(c, Wf.fc[i], a, 2);
  }
  float* droi = static_cast<float*>(c.alloc(static_cast<size_t>(T) * H * W * 4));
  if (c.live())
    c.chk(pf_roi_crop_zoom_batched(coarse_depth, 1, H, W, 1, 1, tile_image, boxes, T, 1.0f, droi, 1, 0, c.stream));
  Map u = c.map(T, H, W, 5);
  if (c.live()) c.chk(pf_pack_unet_input(droi, fine_depth, crops, T, H, W, u.p, u.ld, c.stream));
  // encoder (guided_fusion_model.py:179-184)
  const Map* ui[1] = {&u};
  Map x = double_conv(c, Wf.inc[0], Wf.inc[1], ui, 1, H, W, false, "inc");
  Map enc[6];
  enc[5] = x;
  for (int i = 0; i < 5; ++i) {
    Map p = c.map(T, x.H / 2, x.W / 2, x.C);
    if (c.live()) c.chk(pf_maxpool2(x.p, T, x.H, x.W, pad_to(x.C, 8), x.ld, p.p, p.ld, c.stream));
    const Map* pi[1] = {&p};
    char nm[8];
    snprintf(nm, sizeof(nm), "down%d", i);
    x = double_conv(c, Wf.down[i][0], Wf.down[i][1], pi, 1, p.H, p.W, false, nm);
    enc[4 - i] = x;
  }
  // decoder, low -> high resolution (guided_fusion_model.py:188-205)
  Map outs[6], prev;
  for (int i = 0; i < 6; ++i) {
    const Map gm = from_pf(g2l_maps[i]);
    const int h = gm.H, w = gm.W;
    // F.interpolate(enc / previous level / guide, size=(h, w), bilinear, align_corners=True) feeding the 3x3 convs
    // (guided_fusion_model.py:98-99,191-203)
    Map e = enc[i];
    char nm[8];
    if (i > 0) {
      const Map* a[3] = {&enc[i], &prev, &guide[i - 1]};
      snprintf(nm, sizeof(nm), "up%d", i);
      e = double_conv(c, Wf.up[i - 1][0], Wf.up[i - 1][1], a, 3, h, w, true, nm);
    }
    Map cr = c.map(T, h, w, gm.C);
    if (c.live())
      c.chk(pf_roi_crop_zoom_batched(gm.p, 0, h, w, pad_to(gm.C, 8), gm.ld, tile_image, boxes, T, static_cast<float>(h) / H,
                                     cr.p, cr.ld, 0, c.stream));
    const Map* a2[2] = {&e, &cr};
    snprintf(nm, sizeof(nm), "cv%d", i);
    prev = double_conv(c, Wf.cv[i][0], Wf.cv[i][1], a2, 2, h, w, true, nm);
    outs[i] = prev;
    snprintf(nm, sizeof(nm), "fuse%d", i);
    c.tap_out(nm, prev.p, 0, prev.rows(), prev.C, prev.ld);
  }
  metric_head(c, Wf.head, outs[0], &outs[1], outs[5], nullptr, depth_out);
}

static Ctx make_ctx(void* ws, size_t bytes, bool dry, void* stream, pf_tap_fn tap, void* user) {
  Ctx c;
  c.base = static_cast<uint8_t*>(ws); c.cap = bytes; c.off = 0; c.dry = dry; c.stream = stream; c.err = 0;
  c.tap = tap; c.tap_user = user; c.n_e4m3 = 0; c.lname = nullptr;
  return c;
}

}  // namespace pf

using namespace pf;

extern "C" {

size_t pf_branch_workspace_bytes(const pf_branch* w, int32_t B) {
  Ctx c = make_ctx(nullptr, 0, true, nullptr, nullptr, nullptr);
  branch_run(c, *w, nullptr, B, nullptr);
  return c.off + 256;
}

int pf_branch_forward(const pf_branch* w, const float* images, int32_t B, void* ws, size_t ws_bytes, pf_branch_out* out,
                      pf_tap_fn tap, void* tap_user, void* stream) {
  if (!w || !images || !ws || !out || B < 1) return set_error("pf_branch_forward: null argument");
  if (w->H % 14 || w->W % 14) return set_error("pf_branch_forward: patch_process_shape must be a multiple of 14");
  if (reinterpret_cast<uintptr_t>(ws) & 255) return set_error("pf_branch_forward: workspace must be 256-byte aligned");
  Ctx c = make_ctx(ws, ws_bytes, false, stream, tap, tap_user);
  branch_run(c, *w, images, B, out);
  return c.err;
}

size_t pf_g2l_workspace_bytes(const pf_fusion* w, const pf_map* coarse_feats) {
  Ctx c = make_ctx(nullptr, 0, true, nullptr, nullptr, nullptr);
  g2l_run(c, *w, coarse_feats, nullptr);
  return c.off + 256;
}

int pf_g2l_forward(const pf_fusion* w, const pf_map* coarse_feats, void* ws, size_t ws_bytes, pf_map* out, pf_tap_fn tap,
                   void* tap_user, void* stream) {
  if (!w || !coarse_feats || !ws || !out) return set_error("pf_g2l_forward: null argument");
  if (reinterpret_cast<uintptr_t>(ws) & 255) return set_error("pf_g2l_forward: workspace must be 256-byte aligned");
  Ctx c = make_ctx(ws, ws_bytes, false, stream, tap, tap_user);
  g2l_run(c, *w, coarse_feats, out);
  return c.err;
}

size_t pf_fusion_workspace_bytes(const pf_fusion* w, int32_t T, const pf_map* g2l_maps) {
  Ctx c = make_ctx(nullptr, 0, true, nullptr, nullptr, nullptr);
  // shapes only: the fine / coarse maps share the G2L maps' geometry and channel counts
  pf_map fine[6];
  for (int i = 0; i < 6; ++i) { fine[i] = g2l_maps[i]; fine[i].B = T; fine[i].ptr = nullptr; }
  fusion_run(c, *w, nullptr, nullptr, nullptr, T, nullptr, fine, nullptr, g2l_maps, g2l_maps, nullptr);
  return c.off + 256;
}

int pf_fusion_forward_batched(const pf_fusion* w, const float* crops, const float* boxes, const int32_t* tile_image,
                              int32_t T, const float* fine_depth, const pf_map* fine_feats, const float* coarse_depth,
                              const pf_map* coarse_feats, const pf_map* g2l_maps, void* ws, size_t ws_bytes,
                              float* depth_out, pf_tap_fn tap, void* tap_user, void* stream) {
  if (!w || !crops || !boxes || !fine_depth || !fine_feats || !coarse_depth || !coarse_feats || !g2l_maps || !ws ||
      !depth_out || T < 1)
    return set_error("pf_fusion_forward: null argument");
  if (reinterpret_cast<uintptr_t>(ws) & 255) return set_error("pf_fusion_forward: workspace must be 256-byte aligned");
  Ctx c = make_ctx(ws, ws_bytes, false, stream, tap, tap_user);
  fusion_run(c, *w, crops, boxes, tile_image, T, fine_depth, fine_feats, coarse_depth, coarse_feats, g2l_maps, depth_out);
  return c.err;
}

int pf_fusion_forward(const pf_fusion* w, const float* crops, const float* boxes, int32_t T, const float* fine_depth,
                      const pf_map* fine_feats, const float* coarse_depth, const pf_map* coarse_feats,
                      const pf_map* g2l_maps, void* ws, size_t ws_bytes, float* depth_out, pf_tap_fn tap,
                      void* tap_user, void* stream) {
  return pf_fusion_forward_batched(w, crops, boxes, nullptr, T, fine_depth, fine_feats, coarse_depth, coarse_feats,
                                   g2l_maps, ws, ws_bytes, depth_out, tap, tap_user, stream);
}

}  // extern "C"
