/* pf_b200.h — C ABI of libpf_b200.so: the H100 (sm_90a) kernels behind PatchFusion's per-tile inference hot path.
 *
 * Boundary (SURVEY.md §8b): the reference is pure Python/PyTorch and has no FFI; the drop-in class
 * `estimator.models.patchfusion.PatchFusion` (reference `estimator/models/patchfusion.py:55-453`) keeps its Python
 * surface and its methods call the entry points below through ctypes (patchfusion_b200/lib.py; the stub a reference
 * maintainer would add is shown in INTEGRATION.md).  Conventions:
 *   - plain pointers and ints only; every pointer is a DEVICE pointer unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued asynchronously on it (CUDA-graph capturable);
 *   - no allocation, no synchronisation, no global mutable state besides one-time kernel attribute setup and a
 *     tensor-map cache keyed by (pointer, shape);
 *   - return 0 on success, non-zero on error with a message in pf_last_error() (thread-local);
 *   - activations are bf16, channels-last (NHWC, row stride `ld` elements); the ViT residual stream, LayerNorm
 *     statistics, softmax, the metric-bins tail and the stitch canvases are fp32.
 * Each entry point cites the reference code it replaces (paths relative to the reference repo root).
 */
#ifndef PF_B200_H_
#define PF_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PF_ACT_NONE 0
#define PF_ACT_RELU 1
#define PF_ACT_GELU 2      /* exact erf GELU (nn.GELU default) */
#define PF_ACT_SOFTPLUS 3  /* beta 1, threshold 20 */

/* ---- library ------------------------------------------------------------------------------------------------ */
const char* pf_last_error(void);
int pf_version(void);
/* number of kernels launched by this library since process start (bench.py's gpu_launches) */
long long pf_launch_count(void);
/* Per-launch profiler: between start and stop every kernel this library launches on `stream` is bracketed by CUDA
 * events (duration i = event i - event i-1).  pf_profile_stop returns the record count; pf_profile_get returns a
 * record's kernel name, shape label, algorithmic flops (0 for HBM kernels) and milliseconds. */
/* Tuning switches (defaults in parentheses; each is also read once from the environment variable of the same name):
 *   PF_OPT_TMA_EPILOGUE (1)   pf_gemm_kernel and pf_conv3_halo_kernel epilogue through shared memory + bulk tensor
 *                             stores / reduce-add
 *   PF_OPT_HALO_MULTICAST (1) pf_conv3_halo_kernel in clusters of 2 (value 1) or 4 (value 2) CTAs sharing the weight
 *                             tiles by TMA multicast
 *   PF_OPT_GEMM_MULTICAST (1) the same for the linear layers of pf_gemm_kernel
 *   PF_OPT_FUSED_RESAMPLE (0) pf_fusion_forward: bilinear resamples feeding the U-Net's 3x3 convs are produced in the
 *                             conv's operand stage (pf_gemm_desc.rs_h / rs_w) instead of being materialised.  Correct
 *                             and parity-tested; off by default: only two warps of the CTA are free to produce it.
 *   PF_OPT_PDL (0)            programmatic dependent launch for the persistent kernels
 *   PF_OPT_RESIZE_SEPARABLE (0) tiled bilinear resample: x blend once per source row, then one y blend per output row
 *                             (3x fewer ALU instructions)
 * Changing one invalidates nothing inside the library; callers holding CUDA graphs must re-capture. */
#define PF_OPT_TMA_EPILOGUE 0
#define PF_OPT_HALO_MULTICAST 1
#define PF_OPT_GEMM_MULTICAST 2
#define PF_OPT_FUSED_RESAMPLE 3
#define PF_OPT_PDL 4
#define PF_OPT_RESIZE_SEPARABLE 5
int pf_set_option(int32_t option, int32_t value);
int pf_profile_start(void* stream);
int pf_profile_stop(void);
int pf_profile_get(int32_t i, const char** name, const char** label, double* flops, float* ms);
/* pf_gemm_kernel / pf_conv3_halo_kernel phase timeline, in libraries built with -DPF_GEMM_TIMELINE (any other build
 * returns an error): synchronises the device, copies the PF_GEMM_TIMELINE_SLOTS clock64 sums accumulated by every launch
 * of either kernel since the last reset into host array `out` (may be NULL) and zeroes them if `reset`.  Slots: producer tiles, producer
 * cycles waiting for an empty stage, producer loop cycles; then per consumer warpgroup: tiles, cycles waiting for a
 * full stage, mainloop cycles (waits included), epilogue cycles, loop cycles. */
#define PF_GEMM_TIMELINE_SLOTS 8
int pf_gemm_timeline(unsigned long long* out, int32_t reset);

/* ---- dense contractions: one wgmma/TMA implicit-GEMM kernel ----------------------------------------------------
 * Replaces every nn.Linear / nn.Conv2d(1x1, 3x3 s1 p1) / nn.ConvTranspose2d(k==s) on the path:
 *   external/torchhub/facebookresearch_dinov2_main/dinov2/layers/attention.py:51,60  mlp.py:36-39
 *   external/depth_anything/dpt.py:30-60,87-95  blocks.py:53-58,123  estimator/models/patchfusion.py:122-127,263-267
 *   estimator/models/blocks/guided_fusion_model.py:41-47,59-66  swin_layers.py:45-48,140,162
 *   external/zoedepth/models/layers/{localbins_layers.py:84-89,110-114, attractor.py:157-162, dist_layers.py:91-98}
 */
typedef struct pf_gemm_desc {
  /* A operand: up to 3 channel-concatenated sources (torch.cat(dim=1) is never materialised) */
  int32_t num_src;        /* 1..3 */
  int32_t a_mode;         /* 0: rows x K matrix; 1: NHWC image, 3x3 or 1x1 window */
  int32_t taps;           /* 1 or 9 (3x3, stride 1, zero pad 1) */
  int32_t chunks[3];      /* ceil(C_src / 64) */
  const void* a_ptr[3];   /* bf16 */
  int32_t a_c[3];         /* channels (columns) of each source, multiple of 8 */
  int32_t a_ld[3];        /* row (pixel) stride in elements, multiple of 8 */
  /* M geometry */
  int32_t M;              /* a_mode 0: rows */
  int32_t NB, H, W;       /* a_mode 1: batch and image size; also the input grid for pixel-shuffle (ps > 1) */
  int32_t bh, bw;         /* a_mode 1: pixel tile, bh*bw == 128 (0 = choose) */
  int32_t tiles_y, tiles_x, m_tiles;   /* filled by the library */
  /* B operand: packed weights [N_pad, Ktot] bf16 K-major from pf_pack_weight */
  const void* w_ptr;
  int32_t N, Ktot;
  int32_t block_n, n_tiles;            /* block_n: 0 = choose; multiple of 32, <= 256 */
  /* epilogue: v = act(acc + bias); v += res1 + res2; then one of {bf16 store, f32 store, x += gamma*v} */
  const float* bias;
  int32_t act;
  const void* res1; const void* res2; int32_t res_ld;   /* bf16, same row mapping as out */
  const float* gamma;                                    /* LayerScale: out (fp32) += gamma * v */
  void* out; int32_t out_f32; int32_t out_ld; int32_t out_col0;
  void* out2; int32_t out2_ld;                           /* optional second bf16 output = relu(v) */
  int32_t ps, ps_cout;                                   /* ConvTranspose k==s as GEMM + pixel shuffle (ps = k) */
  void* vt; int32_t vt_col0, vt_seq, vt_seq_pad, vt_dim; /* attention V columns written transposed */
  /* fused trailing 1x1 layer on the activated row (e.g. the 80->4 / 128->nA / 32->1 heads): out3[row, i] =
   * act2(b2[i] + sum_j w2[i*N + j] * v[j]), i < n2 <= 16; needs N <= block_n (one N tile).  skip_main != 0
   * suppresses the main store. */
  const float* w2; const float* b2; int32_t n2, act2, skip_main; float* out3; int32_t out3_ld;
  /* Fused bilinear resample of a 3x3 conv's input (F.interpolate(mode='bilinear', align_corners=True) feeding the
   * conv, guided_fusion_model.py:98-99,191-203): rs_h[i] > 0 means source i is a [NB, rs_h, rs_w, a_ld] map that the
   * conv reads THROUGH the resample to (H, W); the up-sampled tensor is never written to memory - a producer warp of
   * the halo-tile kernel interpolates each 18 x 10 pixel halo straight into the swizzled operand tile. */
  int32_t rs_h[3], rs_w[3];
  /* E4M3 operands (a_e4m3 != 0; 3x3 halo-tile convs with materialised sources and a plain bf16 output only): a_ptr[0]
   * is ONE e4m3 NHWC map [NB, H, W, a_ld[0] bytes] holding the num_src sources back to back, each padded to 64 channels
   * (pf_quantize_e4m3_tiles); a_c[] still give the sources' channels.  w_ptr is an e4m3 panel (pf_pack_weight_e4m3).
   * The epilogue computes act(fl(acc * fl(s_a[img] * s_w[n])) + bias[n]): s_a one fp32 scale per image of the batch,
   * s_w one per output channel.
   * Linear layers (vit_precision 'fp8_static'; a_e4m3 and a_static set, a_mode 0, taps 1): a_ptr[0] is an e4m3 matrix
   * [M, a_ld[0] bytes] of K = a_c[0] columns, K and N multiples of 128, one source, w_ptr the e4m3 panel [N_pad, K]; the
   * outputs are the plain linear layer's (bf16, fp32, the gamma residual update, the V^T third of a fused qkv
   * projection) or the e4m3 output below, after bias -> none / GELU / ReLU.  They run on pf_gemm_pp_e4m3_kernel. */
  int32_t a_e4m3;
  const float* s_a;
  const float* s_w;
  /* Static input scale (fusion_precision 'fp8_static'; a_e4m3 != 0): a_static != 0 replaces s_a[img] by the one value
   * a_scale (amax / 448 of the conv's calibrated input amax) for the whole launch: act(fl(acc * fl(a_scale * s_w[n])) +
   * bias[n]).  s_a may then be NULL.
   * E4M3 output (out_e4m3 != 0; needs a_static): the activated fp32 value v is written as q = e4m3_rn(sat(v * out_ratio))
   * (the consumer's r = 448 / amax, pf_quantize_e4m3_static's rule) into `out`, an e4m3 NHWC map [NB, H, W, out_ld
   * bytes] whose columns N .. 64 ceil(N / 64) - 1 are written as zero: the operand map of a one-source E4M3 conv.  For
   * a linear layer `out` is the e4m3 matrix [M, out_ld bytes] the next E4M3 linear layer reads (fc1 -> fc2).
   * out_ld a multiple of 16 >= 64 ceil(N / 64), out_col0 0, `out` 16-byte aligned, a plain output (no residual, second
   * output, trailing layer or fp32), and block_n 32 only when N <= 32. */
  int32_t a_static;
  float a_scale;
  int32_t out_e4m3;
  float out_ratio;
  /* Residuals and an e4m3 ReLU copy on a static-scale E4M3 3x3 conv (dpt_precision 'fp8_static': the DPT decoder's
   * ResidualConvUnits and reassemble convs; pf_conv3_halo_e4m3_res_kernel): with a_static set and a bf16 `out`,
   * res1 / res2 (bf16, even res_ld >= N, 4-byte aligned) are added as in the bf16 path, v = act(fl(acc * fl(a_scale *
   * s_w[n])) + bias[n]), then + res1, then + res2 in fp32, and out2_e4m3 != 0 makes out2 an e4m3 NHWC map [NB, H, W,
   * out2_ld bytes] that receives q = e4m3_rn(sat(max(bf16(v), 0) * out2_ratio)), quantized from the bf16-rounded output
   * (so q is pf_quantize_e4m3_static of the output's ReLU at r = out2_ratio), columns N .. 64 ceil(N / 64) - 1 zero.
   * out2_ld a multiple of 16 >= 64 ceil(N / 64), out2 16-byte aligned, out_col0 0, block_n 0, 64 or 128. */
  int32_t out2_e4m3;
  float out2_ratio;
} pf_gemm_desc;

int pf_gemm(pf_gemm_desc* desc, void* stream);

/* Repack an fp32 PyTorch weight into the K-major bf16 panel pf_gemm consumes.
 *   w: [N, C_total, kh, kw] (Conv2d) or [N, C_total] (Linear, kh=kw=1); `src_c[i]` = channels of concat source i.
 *   dst: [N_pad, Ktot] bf16, Ktot = sum_i taps * 64*ceil(src_c[i]/64); rows >= N and pad channels are zero.
 *   scale (nullable, [N]): per-output-channel factor folded into the weights (eval-mode BatchNorm). */
int pf_pack_weight(const float* w, int32_t N, int32_t N_pad, int32_t num_src, const int32_t* src_c, int32_t taps,
                   const float* scale, void* dst, void* stream);
/* ConvTranspose2d(k==s) weight [Cin, Cout, k, k] -> [k*k*Cp, Cin_pad64] bf16, Cp = pad32(Cout),
 * row = (ky*k + kx)*Cp + co (rows co >= Cout are zero).  Use with pf_gemm ps=k, ps_cout=Cout, N=k*k*Cp. */
int pf_pack_weight_convT(const float* w, int32_t Cin, int32_t Cout, int32_t k, void* dst, void* stream);

/* ---- E4M3 (FP8) operands of the Guided-Fusion U-Net's 3x3 convs (model config fusion_precision = 'fp8') ----------
 * Rounding rule shared by both entry points, all in IEEE fp32 without contraction:
 *   amax  = max |v| over the group (a NaN anywhere makes it NaN, an infinity makes it +inf)
 *   r     = 448 / amax, or 0 when amax == 0
 *   q     = e4m3_rn(v * r)    round to nearest even to float8_e4m3fn (torch.float8_e4m3fn; |v * r| <= 448, so no
 *                             saturation happens; the sign of zero is kept; NaN stays NaN)
 *   scale = amax / 448        so that v ~= q * scale; an all-zero group gets scale 0 and q = 0
 * Non-finite data propagate: a group holding NaN gets scale NaN and q NaN everywhere (r = NaN); a group holding an
 * infinity gets scale +inf, q = 0 for its finite values and NaN for the infinities (r = 0).  The conv's accumulator times
 * such a scale is NaN; what the activation makes of a NaN is as in the bf16 path (ReLU's fmaxf returns 0). */
/* pf_pack_weight's panel and K order (source, tap, 64-channel chunk; pad channels and rows >= N zero) with one group
 * per output channel: v = w[n, ...] * scale[n] (BatchNorm folded first, when scale != NULL), dst e4m3 [N_pad, Ktot],
 * s_w[n] (n < N) the channel's scale. */
int pf_pack_weight_e4m3(const float* w, int32_t N, int32_t N_pad, int32_t num_src, const int32_t* src_c, int32_t taps,
                        const float* scale, void* dst, float* s_w, void* stream);
/* One group per TILE (batch index t of the U-Net maps) over all of a conv's sources: src[i] (host array of device
 * pointers) is a bf16 NHWC map [T, H, W, src_ld[i]] of which the first src_c[i] channels are read (src_ld[i] a multiple
 * of 8 >= src_c[i], 16-byte aligned).  out: e4m3 [T, H, W, Kc], Kc = sum_i 64 ceil(src_c[i] / 64), the sources back to
 * back with zero pad channels (the map pf_gemm reads with a_e4m3); s_a[t] the tile's scale.  Two launches: per-block
 * partial maxima into `partial` (T * PF_QUANT_PARTS floats), then the scales and the map.  A max does not depend on
 * the order it is taken in, so the result is deterministic and tile t's bytes depend on tile t's data only. */
#define PF_QUANT_PARTS 32
int pf_quantize_e4m3_tiles(int32_t num_src, const void* const* src, const int32_t* src_c, const int32_t* src_ld,
                           int32_t T, int32_t H, int32_t W, float* partial, void* out, float* s_a, void* stream);
/* ---- Static E4M3 activations (fusion_precision = 'fp8_static'): one calibrated amax per conv input ---------------
 *   r = 448 / amax (one IEEE fp32 division), or 0 when amax == 0;   scale = amax / 448
 *   q = e4m3_rn(sat(v * r))   cvt.rn.satfinite: |v * r| beyond 448 (the input may exceed the calibrated amax) gives
 *                             +-448, an infinity too; NaN stays NaN; the sign of zero is kept
 * pf_quantize_e4m3_tiles' sources and output map (each source padded to 64 channels, pad channels zero) at the given
 * ratio r for every tile: ONE launch that reads each bf16 source once, no amax pass.  A tile's bytes depend on the tile
 * only. */
int pf_quantize_e4m3_static(int32_t num_src, const void* const* src, const int32_t* src_c, const int32_t* src_ld,
                            int32_t T, int32_t H, int32_t W, float ratio, void* out, void* stream);

/* ---- ViT pieces --------------------------------------------------------------------------------------------- */
/* LayerNorm over the last dim, fp32 in -> bf16 out (dinov2/layers/block.py:84,87; vision_transformer.py:311;
 * swin_layers.py:222,265,428).  rows x C; x_ld/out_ld in elements. */
int pf_layernorm(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t rows, int32_t C,
                 void* out, int32_t out_ld, void* stream);
/* pf_layernorm's statistics with an e4m3 output (vit_precision 'fp8_static': the operand of the qkv / fc1 linear):
 * out[r, c] = e4m3_rn(sat(y * ratio)), y the fp32 affine value (no bf16 rounding in between), ratio = 448 / amax of the
 * consumer's calibrated input amax (pf_quantize_e4m3_static's rule).  out is [rows, out_ld bytes], out_ld >= C. */
int pf_layernorm_e4m3(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t rows, int32_t C,
                      float ratio, void* out, int32_t out_ld, void* stream);
/* Fused softmax(QK^T * scale) V for the DINOv2 blocks (dinov2/layers/attention.py:49-62): qk is the [B*seq, 2*D]
 * bf16 Q|K part of the qkv GEMM output (row stride qk_ld), vt the transposed V written by pf_gemm;
 * out [B*seq, D] bf16.  head_dim == 64. */
int pf_attention(const void* qk, int32_t qk_ld, const void* vt, int32_t B, int32_t seq, int32_t seq_pad,
                 int32_t heads, float scale, void* out, int32_t out_ld, void* stream);
/* Normalise (ImageNet mean/std, depth_anything.py:184-190) + 14x14 patch gather (patch_embed.py:76-78) of
 * B planar fp32 RGB images [B,3,H,W] in [0,1] -> bf16 [B*(H/14)*(W/14), ld] (cols = c*196 + py*14 + px). */
int pf_patch_im2col(const float* img, int32_t B, int32_t H, int32_t W, void* out, int32_t ld, void* stream);
/* tokens[b, 0] = cls + pos[0]; tokens[b, 1+i] = patch[b, i] + pos[1+i]  (vision_transformer.py:216-217); fp32 */
int pf_assemble_tokens(const float* patch, const float* cls, const float* pos, int32_t B, int32_t n_patch, int32_t D,
                       float* tokens, void* stream);

/* ---- HBM-bound image ops (NHWC bf16 unless noted) ------------------------------------------------------------- */
/* F.interpolate(mode='bilinear', align_corners=True) (blocks.py:147-149, dpt.py:127,154, guided_fusion_model.py:98,
 * 192-193, attractor.py:175-183).  Writes into out[..., out_col0:out_col0+C] of a buffer with row stride out_ld. */
int pf_resize_bilinear(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, int32_t OH,
                       int32_t OW, void* out, int32_t out_ld, int32_t out_col0, void* stream);
int pf_resize_bilinear_f32(const float* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t OH, int32_t OW,
                           float* out, void* stream);
/* torchvision.ops.roi_align(feat.repeat(T), boxes, (h,w), h/Hp, aligned=True) with one tap per bin
 * (patchfusion.py:240-257, guided_fusion_model.py:202).  feat: batch-1 map [h,w,ld]; boxes: T x 4 fp32
 * (x1,y1,x2,y2, patch_process units) on the device; out [T,h,w,out_ld] at channel offset out_col0.
 * in_f32 != 0 reads an fp32 map (the coarse depth). */
int pf_roi_crop_zoom(const void* feat, int32_t in_f32, int32_t h, int32_t w, int32_t C, int32_t in_ld,
                     const float* boxes, int32_t T, float spatial_scale, void* out, int32_t out_ld,
                     int32_t out_col0, void* stream);
/* The same over a batch: feat is a [B,h,w,in_ld] map (fp32 when in_f32) and box t samples image tile_image[t]
 * (int32 [T] on the device, values in [0, B); the batch column of the reference's bboxs_feat, patchfusion.py:240-257).
 * tile_image == NULL reads image 0 for every box, i.e. pf_roi_crop_zoom. */
int pf_roi_crop_zoom_batched(const void* feat, int32_t in_f32, int32_t h, int32_t w, int32_t C, int32_t in_ld,
                             const int32_t* tile_image, const float* boxes, int32_t T, float spatial_scale, void* out,
                             int32_t out_ld, int32_t out_col0, void* stream);
/* nn.MaxPool2d(2) (guided_fusion_model.py:78) */
int pf_maxpool2(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, void* out,
                int32_t out_ld, void* stream);
/* stride-2 3x3 pad-1 window gather for dpt.py:54-59 (resize_layers[3]): out [B*OH*OW, 9*C] */
int pf_im2col_3x3_s2(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, void* out,
                     void* stream);
/* Crop T tiles from the planar fp32 image [3,H,W] and resize each to (ph,pw) with bilinear align_corners=True
 * (baseline_pretrain.py:258-264, depth_anything/transform.py:127-129): origins int32 (y,x) pairs on the device.
 * out_planar [T,3,ph,pw] fp32 (the tensor the reference hands to fine_forward). */
int pf_crop_resize(const float* img, int32_t H, int32_t W, const int32_t* origins, int32_t T, int32_t th, int32_t tw,
                   int32_t ph, int32_t pw, float* out_planar, void* stream);
/* The same from a batch of images [B,3,H,W]: tile t is cropped from image tile_image[t] (int32 [T] on the device,
 * values in [0, B)), so one call may mix tiles of different images.  tile_image == NULL: image 0 (pf_crop_resize). */
int pf_crop_resize_batched(const float* img, int32_t H, int32_t W, const int32_t* origins, const int32_t* tile_image,
                           int32_t T, int32_t th, int32_t tw, int32_t ph, int32_t pw, float* out_planar, void* stream);
/* One image of a mixed-geometry batch: its planar fp32 [3,H,W] pixels and the th x tw size of its tiles. */
typedef struct pf_crop_image {
  const float* img;
  int32_t H, W;
  int32_t th, tw;
} pf_crop_image;
/* The same over images of different sizes and tile grids: `images` is a device table of descriptors and tile t is a
 * th x tw crop of images[tile_image[t]] at origins[t], resized to (ph, pw) with the arithmetic of
 * pf_crop_resize_batched (equal geometry gives equal bits).  tile_image is required. */
int pf_crop_resize_multi(const pf_crop_image* images, const int32_t* origins, const int32_t* tile_image, int32_t T,
                         int32_t ph, int32_t pw, float* out_planar, void* stream);
/* U-Net input cat[coarse_depth_roi, fine_depth, rgb] (patchfusion.py:269) as NHWC bf16 with `ld` channels */
int pf_pack_unet_input(const float* coarse_depth_roi, const float* fine_depth, const float* rgb_planar, int32_t T,
                       int32_t H, int32_t W, void* out, int32_t ld, void* stream);
/* tokens [B, n, D] bf16 rows -> skip cls handled by caller; generic strided row copy / convert helpers */
int pf_f32_to_bf16(const float* in, int64_t n, void* out, void* stream);

/* ---- callers either side of the path (SURVEY.md §8f-1 / f-2) ------------------------------------------------- */
/* uint8 HWC image (bgr != 0: cv2.imread channel order) -> planar RGB fp32 in [0,1] resized with bicubic
 * align_corners=True to (OH, OW): estimator/datasets/general_dataset.py:40-45. */
int pf_ingest_u8(const uint8_t* img_hwc, int32_t H, int32_t W, int32_t bgr, int32_t OH, int32_t OW, float* out_planar,
                 void* stream);
/* depth canvas -> uint16: nearest resize to (OH, OW) (tools/test_single_forward.py:26) then saturating
 * (depth * scale) cast (estimator/tester/tester.py:75-76, scale 256). */
int pf_depth_to_u16(const float* depth, int32_t H, int32_t W, int32_t OH, int32_t OW, float scale, uint16_t* out,
                    void* stream);
/* U4K raw frame: uint8 HWC (bgr != 0: stored BGR) -> planar RGB fp32 u8 / 255 at the same size, correctly rounded,
 * no resample (estimator/datasets/u4k_dataset.py:115-129). */
int pf_ingest_raw_u8(const uint8_t* img_hwc, int32_t H, int32_t W, int32_t bgr, float* out_planar, void* stream);
/* Evaluation ground truth in one pass over a source map [H, W]: depth [H, W] fp32 and boundary [H, W] uint8, where a
 * pixel is an edge when |e[p] - e[q]| > th for a 4-neighbour q (get_boundaries(e, th, dilation=0),
 * estimator/utils/image_ops.py:25-31; a NaN difference is no edge).  kind (PF_GT_*) picks the dataset branch:
 *   U4K        src fp32 disparity; e = src; depth = factor / src
 *   MID        src fp32 disparity; e = src with +inf -> 0; depth = factor / (src + doffs) / 1000, +inf src -> 0
 *   ETH3D      src fp32 depth; depth = e = nan_to_num(src, nan=0, posinf=0, neginf=0)
 *   CITYSCAPES src uint16 disparity x; x > 0 -> (x - 1) / 256; depth = e = nan_to_num(factor / x)
 * factor and doffs are the float32 roundings of the reference's Python floats; all arithmetic is IEEE fp32. */
#define PF_GT_U4K 0
#define PF_GT_MID 1
#define PF_GT_ETH3D 2
#define PF_GT_CITYSCAPES 3
int pf_gt_prepare(const void* src, int32_t kind, int32_t H, int32_t W, float factor, float doffs, float th,
                  float* depth, uint8_t* boundary, void* stream);

/* compute_metrics / compute_errors / soft_edge_error (estimator/utils/metric.py:10-50, 67-72, 97-148) as one fused
 * reduction over the ground-truth grid.  pred [PH,PW] fp32 is resampled (bilinear, align_corners=False, metric.py:101-104)
 * when its shape differs from gt [H,W]; clamped to [min_eval, max_eval] (inf -> max, nan -> min); valid pixels are
 * min_eval < gt < max_eval (and extra_mask != 0 when given).  edges (nullable, uint8 [H,W]): boundary mask for the
 * soft edge error.  partials: workspace of nblocks * 12 doubles (device); out: 12 doubles (device), summed in a fixed
 * order: {n, #thresh<1.25, #<1.25^2, #<1.25^3, sum|gt-p|/gt, sum(gt-p)^2/gt, sum(gt-p)^2, sum(ln gt - ln p)^2,
 * sum(ln p - ln gt), sum|log10 gt - log10 p|, n_edge, sum see}.  patchfusion_b200/metrics.py turns them into the
 * reference's dict (a1,a2,a3,abs_rel,rmse,log_10,rmse_log,silog,sq_rel,see). */
int pf_depth_metrics(const float* pred, int32_t PH, int32_t PW, const float* gt, int32_t H, int32_t W, float min_eval,
                     float max_eval, const uint8_t* edges, const uint8_t* extra_mask, double* partials, int32_t nblocks,
                     double* out, void* stream);
/* colorize (estimator/utils/color.py:95-140) after the percentile normalisation: x = (d - vmin)/(vmax - vmin),
 * LUT index int(x*256) clipped to [0,255] (matplotlib Colormap.__call__(bytes=True)), d == invalid_val or NaN ->
 * background (128,128,128); lut_rgb: 256 x 3 uint8 (device); out [n,3] uint8, channel order BGR when bgr != 0
 * (tester.py:67-69 writes `[:, :, [2,1,0]]` through cv2). */
int pf_colorize_u8(const float* depth, int64_t n, float vmin, float vmax, float invalid_val, const uint8_t* lut_rgb,
                   int32_t bgr, uint8_t* out, void* stream);

/* ---- Swin / G2L (estimator/models/blocks/swin_layers.py) ------------------------------------------------------ */
/* x[h*w, C] fp32 = NHWC bf16 feature + absolute_pos_embed (swin_layers.py:419-422) */
int pf_g2l_embed(const void* feat, int32_t feat_ld, const float* ape, int32_t n, int32_t C, float* x, void* stream);
/* LayerNorm(eps) of x[H*W, C] written into the zero-padded (Hp x Wp) token grid, bf16 (swin_layers.py:222-230) */
int pf_swin_norm_pad(const float* x, const float* w, const float* b, float eps, int32_t H, int32_t W, int32_t Hp,
                     int32_t Wp, int32_t C, void* out, void* stream);
/* Window attention on the padded grid with cyclic shift, relative-position bias and the -100 shift mask
 * (swin_layers.py:133-164, 232-258, 327-345).  qkv [Hp*Wp, 3C] bf16; bias_table [529, heads] fp32;
 * out [Hp*Wp, C] bf16 in un-shifted token order. */
int pf_window_attention(const void* qkv, const float* bias_table, int32_t Hp, int32_t Wp, int32_t C, int32_t heads,
                        int32_t shift, void* out, void* stream);
/* x[H*W, C] += y[(padded grid), C] cropped (swin_layers.py:260-264); y fp32 */
int pf_swin_residual_crop(float* x, const float* y, int32_t H, int32_t W, int32_t Wp, int32_t C, void* stream);
/* Batched forms of the four ops above, one launch for B images: feat / x hold B maps of n = H*W rows back to back,
 * the padded grids are [B, Hp*Wp, .] and the same ape is added to every image.  B = 1 is the single-image call. */
int pf_g2l_embed_batched(const void* feat, int32_t feat_ld, const float* ape, int32_t B, int32_t n, int32_t C, float* x,
                         void* stream);
int pf_swin_norm_pad_batched(const float* x, const float* w, const float* b, float eps, int32_t B, int32_t H, int32_t W,
                             int32_t Hp, int32_t Wp, int32_t C, void* out, void* stream);
int pf_window_attention_batched(const void* qkv, const float* bias_table, int32_t B, int32_t Hp, int32_t Wp, int32_t C,
                                int32_t heads, int32_t shift, void* out, void* stream);
int pf_swin_residual_crop_batched(float* x, const float* y, int32_t B, int32_t H, int32_t W, int32_t Hp, int32_t Wp,
                                  int32_t C, void* stream);

/* ---- metric-bins tail (zoedepth_v1.py:173-219, attractor.py:164-208, dist_layers.py:36-121) -------------------- */
/* x = emb + up(prev_emb) (attractor.py:175-178), NHWC bf16 */
int pf_add_upsampled(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, const void* prev, int32_t PH,
                     int32_t PW, void* out, void* stream);
/* b_new = up(b_prev) + agg_a dist(A_a - up(b_prev)), alpha=300, gamma=2 (the TorchScript defaults the layer always
 * runs with, attractor.py:186-195); fp32 [B,H,W,nbins]; A: fp32 [B*H*W, A_ld] (first nA columns used).
 * flags: PF_ATTRACTOR_MEAN (kind='mean', else 'sum') | PF_ATTRACTOR_EXP (attractor_type='exp', else 'inv'). */
#define PF_ATTRACTOR_MEAN 1
#define PF_ATTRACTOR_EXP 2
int pf_attractor(const float* A, int32_t A_ld, int32_t nA, const float* b_prev, int32_t PH, int32_t PW, int32_t B, int32_t H,
                 int32_t W, int32_t nbins, int32_t flags, float* b_out, void* stream);
/* AttractorLayer (attractor.py:100-135, the normed and hybrid2 heads): as pf_attractor with the attractor points
 * A + 1e-3, A holding the even `_net` channels only (attractor.py:105-106).  b_out receives the normalised, unsorted
 * b_new; centers (nullable; the last level) clip(sort((max - min) b_new + min), min, max) per pixel. */
int pf_attractor_normed(const float* A, int32_t A_ld, int32_t nA, const float* b_prev, int32_t PH, int32_t PW, int32_t B,
                        int32_t H, int32_t W, int32_t nbins, int32_t flags, float min_depth, float max_depth, float* b_out,
                        float* centers, void* stream);
/* seed bin centres from the seed regressor's `_net` output S [pixels, S_ld] (fp32; ReLU'd for PF_SEED_NORMED, else
 * softplus'd) into out [pixels, nbins].  PF_SEED_NORMED: SeedBinRegressor (localbins_layers.py:51-67): widths
 * (max - min) (S + 1e-3) / sum, centres the midpoints of min + cumsum(widths); else the centres are S.
 * PF_SEED_TO_UNIT: then (c - min) / (max - min) (zoedepth_v1.py:176-181). */
#define PF_SEED_NORMED 1
#define PF_SEED_TO_UNIT 2
int pf_seed_bins(const float* S, int32_t S_ld, int64_t pixels, int32_t nbins, int32_t flags, float min_depth,
                 float max_depth, float* out, void* stream);
/* depth = sum_k softmax_k(logbinom(p)/t) * up(b_centers)_k from the 4-channel softplus'd pt map */
int pf_logbinom_depth(const float* pt, int32_t pt_ld, const float* b_centers, int32_t BH, int32_t BW, int32_t B, int32_t H, int32_t W,
                      int32_t nbins, float min_temp, float max_temp, float* depth, void* stream);

/* ---- stitch (baseline_pretrain.py:310-326, estimator/models/utils.py:21-36 in closed form) --------------------- */
/* num[y0+i, x0+j] += mask[i,j]*d[t,i,j]; den += mask  — touches only the tile footprints; tiles of one call may
 * overlap (atomics).  origins: T (y,x) int32 pairs on the device.  up_h/up_w > 0: tiles are nearest-upsampled to
 * (up_h, up_w) first (random_tile, baseline_pretrain.py:203). */
int pf_stitch_accumulate(float* num, float* den, int32_t CH, int32_t CW, const float* tiles, int32_t T, int32_t th,
                         int32_t tw, const int32_t* origins, const float* mask, int32_t up_h, int32_t up_w,
                         void* stream);
/* Deterministic stitch (the product path; no atomics): every canvas pixel sums, in list order, mask * prediction over
 * the tiles covering it.  tiles: n x {origin_y, origin_x, slot} int32 (device); tile i's prediction is
 * preds[slot_i] ([*, th, tw] fp32 - e.g. the all-gathered per-rank blocks of the tile-sharded run, so the result is
 * bit-identical for any rank count and micro-batch grouping).  up_h/up_w > 0: nearest-upsample each tile first
 * (random_tile).  base_num/base_den (nullable): canvases to continue from (RunningAverageMap.resize output).
 * Outputs (each nullable): num, den, avg = num / den. */
int pf_stitch_gather(const float* preds, const int32_t* tiles, int32_t n, int32_t th, int32_t tw, const float* mask,
                     int32_t up_h, int32_t up_w, const float* base_num, const float* base_den, int32_t CH, int32_t CW,
                     float* num_out, float* den_out, float* avg_out, void* stream);
int pf_stitch_finalize(const float* num, const float* den, int64_t n, float* out, void* stream);
/* Multi-GPU tile sharding: `stack` is the all-gathered [world][2][n] (num, den) canvases; sums over ranks in rank
 * order into stack[0] (deterministic for a fixed world size). */
int pf_stitch_reduce(float* stack, int32_t world, int64_t n, void* stream);
/* RunningAverageMap.resize (utils.py:32-36): num' = nearest(avg) * bilinear_ac(cnt), den' = bilinear_ac(cnt) */
int pf_stitch_resize(const float* num, const float* den, int32_t H, int32_t W, int32_t OH, int32_t OW, float* num_out,
                     float* den_out, void* stream);

/* ---- depth to 3D (external/zoedepth/utils/geometry.py) --------------------------------------------------------- */
/* depth_to_points (geometry.py:39-72) of depth [H, W] fp32: points [H*W, 3] fp32, p = R M d K^-1 [x, y, 1]^T + t with
 * K = get_intrinsics(H, W) (55 degree FOV, f = W / 2 / tan(27.5 deg), principal point (W/2, H/2); inv_f = fp32 1/f)
 * and M = diag(-1, -1, 1).  rt_host (nullable: identity and zero): 12 host floats, R row-major then t.  image
 * (nullable, with colors): planar RGB [3, H, W] fp32; colors [H*W, 3] uint8 = round-half-even(255 clamp(v, 0, 1)),
 * NaN -> 0, written by the same pass. */
int pf_depth_to_points(const float* depth, int32_t H, int32_t W, float inv_f, const float* rt_host, const float* image,
                       float* points, uint8_t* colors, void* stream);
/* Vertex mask [H, W] uint8 (H, W >= 2): 1 where d is finite, d > 0 and hypot(gy, gx) <= threshold, with (gy, gx) =
 * np.gradient(d) in fp32 (central differences / 2 inside, one-sided differences at the borders). */
int pf_depth_edge_mask(const float* depth, int32_t H, int32_t W, float threshold, uint8_t* mask, void* stream);
/* create_triangles (geometry.py:75-98) with a vertex mask [h, w] (uint8 / bool, nonzero = set), in two calls with one
 * read of the total between them.  Quads are row-major; quad q's triangles are (tl, bl, tr) then (br, tr, bl), and a
 * triangle is kept when its three vertices are set.
 * pf_mesh_quad_counts: flags [(h-1)(w-1)] uint8 (bit 0 / bit 1: first / second triangle kept) and block_offsets
 * [ceil((h-1)(w-1) / PF_MESH_SCAN_BLOCK) + 1] int64: the exclusive offset of every block of PF_MESH_SCAN_BLOCK quads,
 * then the total.  Deterministic (no atomics).
 * pf_mesh_triangles: faces [n, 3] int32 in numpy boolean-indexing order; nothing is written at or past row `cap`.
 * flags == NULL: every triangle, 2 (h-1)(w-1) rows (cap must hold them), block_offsets unused. */
#define PF_MESH_SCAN_BLOCK 64
int pf_mesh_quad_counts(const uint8_t* mask, int32_t h, int32_t w, uint8_t* flags, int64_t* block_offsets,
                        void* stream);
int pf_mesh_triangles(const uint8_t* flags, const int64_t* block_offsets, int32_t h, int32_t w, int32_t* faces,
                      int64_t cap, void* stream);
/* Binary little-endian PLY records, out 16-byte aligned: vertices 15 bytes each (float x, y, z; uchar r, g, b) from
 * points [n, 3] fp32 and colors [n, 3] uint8; faces 13 bytes each (uchar 3; int32 a, b, c) from faces [n, 3] int32. */
int pf_ply_pack_vertices(const float* points, const uint8_t* colors, int64_t n, uint8_t* out, void* stream);
int pf_ply_pack_faces(const int32_t* faces, int64_t n, uint8_t* out, void* stream);


/* ================================================================================================================
 * STAGE-LEVEL ENTRY POINTS (SURVEY.md §8b): the kernel sequences behind the reference's methods, issued by the
 * library itself from caller-owned weights and ONE caller-owned workspace per call (no allocation inside; every
 * intermediate is bump-allocated from the workspace in a fixed order, so addresses are a function of (weights, batch)
 * only: TMA tensor maps are cached and the whole call is CUDA-graph capturable).
 *
 *   pf_branch_forward   PatchFusion.coarse_forward / fine_forward  (estimator/models/patchfusion.py:189-225) =
 *                       ZoeDepth.forward (zoedepth_v1.py:125-233) over DepthAnythingCore (depth_anything.py:262-278),
 *                       DPT_DINOv2 (dpt.py:97-157) and DinoVisionTransformer.get_intermediate_layers
 *                       (vision_transformer.py:297-321)
 *   pf_g2l_forward      G2LFusion.forward on the six whole-image coarse maps (swin_layers.py:410-432), once per image
 *   pf_fusion_forward   PatchFusion.fusion_forward (patchfusion.py:259-340) incl. coarse_postprocess_test's ROI
 *                       crop-zoom (:240-257) and GuidedFusionPatchFusion.forward (guided_fusion_model.py:163-207)
 * ================================================================================================================ */

/* one packed dense layer: the panel written by pf_pack_weight / pf_pack_weight_convT + its fp32 bias */
typedef struct pf_layer {
  const void* w;            /* bf16 [N_pad, Ktot] K-major */
  const float* bias;        /* [N] or NULL */
  int32_t N, Ktot, taps;    /* taps: 1 or 9 */
  int32_t num_src;          /* concat sources the panel was packed for */
  int32_t src_c[3];         /* logical channels of each */
  int32_t ps, ps_cout;      /* ConvTranspose k == stride: k and Cout (else 0) */
  const float* w2;          /* optional trailing 1x1 layer fused into the epilogue: fp32 [n2, N] */
  const float* b2;          /* [n2] or NULL */
  int32_t n2;
  /* FP8 (3x3 convs of the Guided-Fusion U-Net, fusion_precision = 'fp8'): when w_scale != NULL the conv quantizes its
   * input per tile (pf_quantize_e4m3_tiles) and runs on the e4m3 panel w8 with per-channel scales w_scale
   * (pf_pack_weight_e4m3).  w (bf16) may then be NULL unless the conv can run through the fused resample
   * (PF_OPT_FUSED_RESAMPLE), which has no materialised input to quantize and stays bf16. */
  const void* w8;
  const float* w_scale;
  /* fusion_precision 'fp8_static': a HOST pointer to the calibrated amax of the conv's input (NULL: per-tile scales as
   * above).  The stage then quantizes the input with pf_quantize_e4m3_static at r = 448 / amax and runs the conv with the
   * static scale amax / 448; the first conv of a U-Net DoubleConv whose second conv is static too writes the second's
   * e4m3 operand map directly (pf_gemm_desc.out_e4m3).  Read when the stage is issued.
   * vit_precision 'fp8_static': set on a ViT block's qkv, fc1 and fc2 (with w8 / w_scale), the amax of the linear's
   * input.  LN1 / LN2 then write qkv's / fc1's e4m3 operand (pf_layernorm_e4m3) and fc1 writes fc2's (out_e4m3). */
  const float* a_amax;
} pf_layer;

typedef struct pf_vit_block {             /* dinov2/layers/block.py:82-107 */
  const float* n1w; const float* n1b; const float* n2w; const float* n2b;
  const float* ls1; const float* ls2;     /* LayerScale gammas */
  pf_layer qkv, proj, fc1, fc2;
} pf_vit_block;

typedef struct pf_head {                  /* metric-bins head: zoedepth_v1.py:173-219 / patchfusion.py:297-339 */
  pf_layer seed0, seed2;                  /* seed_bin_regressor._net.{0,2} */
  pf_layer seedproj0, seedproj2;          /* seed_projector */
  pf_layer proj0[4], proj2[4];            /* projectors.N */
  pf_layer att0[4], att2[4];              /* attractors.N (att0 carries the fused N<=16 second layer) */
  pf_layer clb0;                          /* conditional_log_binomial.mlp.0 (+ fused mlp.2) */
  int32_t n_attractors[4];
  int32_t n_bins, bin_embedding_dim;
  int32_t attractor_flags;                /* PF_ATTRACTOR_MEAN | PF_ATTRACTOR_EXP */
  int32_t has_rel;                        /* CLB input carries the relative-depth channel (branch heads) */
  float min_temp, max_temp;
  int32_t bin_centers_type;               /* PF_BINS_*: seed regressor and attractor form (zoedepth_v1.py:90-105) */
  float min_depth, max_depth;             /* the head's depth range (branch config; top-level for the fusion head) */
} pf_head;
#define PF_BINS_SOFTPLUS 0                /* SeedBinRegressorUnnormed + AttractorLayerUnnormed */
#define PF_BINS_NORMED 1                  /* SeedBinRegressor + AttractorLayer */
#define PF_BINS_HYBRID1 2                 /* SeedBinRegressor + AttractorLayerUnnormed */
#define PF_BINS_HYBRID2 3                 /* SeedBinRegressorUnnormed + AttractorLayer */

typedef struct pf_branch {                /* one ZoeDepth(Depth-Anything) branch */
  int32_t H, W;                           /* patch_process_shape (multiples of 14) */
  int32_t dim, depth, heads, features;
  int32_t out_channels[4];
  pf_layer patch;                         /* patch_embed.proj as a K=592 GEMM */
  const float* pos;                       /* [1 + gh*gw, dim] pos_embed already resampled (vision_transformer.py:189-210) */
  const float* cls;                       /* [dim] */
  const pf_vit_block* blocks;             /* host array [depth] */
  const float* nw; const float* nb;       /* final norm */
  pf_layer proj[4];                       /* depth_head.projects */
  pf_layer rs0, rs1, rs3;                 /* resize_layers 0,1 (ConvTranspose), 3 (3x3 s2 as GEMM over pf_im2col_3x3_s2) */
  pf_layer rn[4];                         /* scratch.layerN_rn */
  pf_layer ff_out[4];                     /* refinenet{1..4}.out_conv (index = N-1) */
  pf_layer ff_c1[4][2], ff_c2[4][2];      /* refinenetN.resConfUnit{1,2}.conv{1,2} */
  pf_layer oc1, oc2;                      /* output_conv1, output_conv2.0 (+ fused output_conv2.2) */
  pf_layer conv2;
  pf_head head;
} pf_branch;

typedef struct pf_g2l_block {             /* SwinTransformerBlock, swin_layers.py:218-268 */
  const float* n1w; const float* n1b; const float* n2w; const float* n2b;
  const float* table;                     /* relative_position_bias_table [529, heads] */
  pf_layer qkv, proj, fc1, fc2;
} pf_g2l_block;

typedef struct pf_g2l_level {
  int32_t C, heads, depth;
  const float* ape;                       /* absolute_pos_embed [h*w, C] */
  int32_t ape_rows;
  const float* nw; const float* nb;       /* g2l_layer_norm */
  const float* ones;                      /* [C] of 1.0 (plain residual through the LayerScale epilogue) */
  const pf_g2l_block* blocks;             /* host array [depth] */
} pf_g2l_level;

typedef struct pf_fusion {
  int32_t H, W;                           /* patch_process_shape */
  pf_layer fc[5];                         /* fusion_conv_list.0..4 */
  pf_layer inc[2];                        /* guided_fusion.inc (BatchNorm folded) */
  pf_layer down[5][2];
  pf_layer up[5][2];                      /* up_conv_list.N.conv.double_conv.{0,2} */
  pf_layer cv[6][2];                      /* convs.N */
  pf_g2l_level g2l[6];                    /* low -> high resolution */
  pf_head head;
} pf_fusion;

typedef struct pf_map { void* ptr; int32_t B, H, W, C, ld; } pf_map;     /* NHWC bf16 activation */
typedef struct pf_branch_out { float* depth; pf_map feats[6]; } pf_branch_out;   /* x_d0, r4, r3, r2, r1, out_conv */

/* debug tap: called (synchronously, while enqueuing) after the named intermediate has been produced.  The layer taps
 * "L.<layer>.<part>" of the bf16 GEMMs and convs (<layer>: the engine's weight key) also name what a launch is about
 * to read (in<s>, res1, res2, x), emitted just before it: a callback that copies on the stream sees those values. */
typedef void (*pf_tap_fn)(void* user, const char* name, const void* ptr, int32_t is_f32, int64_t rows, int32_t cols,
                          int32_t ld);

size_t pf_branch_workspace_bytes(const pf_branch* w, int32_t B);
/* images: planar fp32 [B,3,H,W] in [0,1], un-normalised.  out->depth [B,H,W] fp32 and the six taps live inside ws. */
int pf_branch_forward(const pf_branch* w, const float* images, int32_t B, void* ws, size_t ws_bytes, pf_branch_out* out,
                      pf_tap_fn tap, void* tap_user, void* stream);
/* coarse_feats: the six coarse maps of B whole images (every map's B must agree); out: the six G2L maps, batch B.
 * Every op runs once over the batch (the GEMMs and LayerNorms over B*n rows), so a batch costs the launches of one
 * image and image b equals its batch-1 result bit for bit. */
size_t pf_g2l_workspace_bytes(const pf_fusion* w, const pf_map* coarse_feats);
int pf_g2l_forward(const pf_fusion* w, const pf_map* coarse_feats, void* ws, size_t ws_bytes, pf_map* out,
                   pf_tap_fn tap, void* tap_user, void* stream);
size_t pf_fusion_workspace_bytes(const pf_fusion* w, int32_t T, const pf_map* g2l_maps);
/* crops planar fp32 [T,3,H,W]; boxes fp32 [T,4] (x1,y1,x2,y2 in patch_process units, device); fine_* = the fine
 * branch's outputs for the same T tiles; coarse_* / g2l_maps = the whole-image (batch 1) outputs; depth_out [T,H,W]. */
int pf_fusion_forward(const pf_fusion* w, const float* crops, const float* boxes, int32_t T, const float* fine_depth,
                      const pf_map* fine_feats, const float* coarse_depth, const pf_map* coarse_feats,
                      const pf_map* g2l_maps, void* ws, size_t ws_bytes, float* depth_out, pf_tap_fn tap,
                      void* tap_user, void* stream);
/* The same for tiles of several images: coarse_depth [B,H,W], coarse_feats and g2l_maps are batch-B maps and tile t
 * reads image tile_image[t] of them (int32 [T] on the device, values in [0, B)).  tile_image == NULL: image 0 for
 * every tile (pf_fusion_forward).  pf_fusion_workspace_bytes applies unchanged. */
int pf_fusion_forward_batched(const pf_fusion* w, const float* crops, const float* boxes, const int32_t* tile_image,
                              int32_t T, const float* fine_depth, const pf_map* fine_feats, const float* coarse_depth,
                              const pf_map* coarse_feats, const pf_map* g2l_maps, void* ws, size_t ws_bytes,
                              float* depth_out, pf_tap_fn tap, void* tap_user, void* stream);
/* LayerNorm of rows [skip, skip + rows_out) of each group of rows_in rows (the patch tokens of every image, cls
 * dropped: vision_transformer.py:309-312): out row g*rows_out + i <- x row g*rows_in + skip + i */
int pf_layernorm_grouped(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t groups,
                         int32_t rows_in, int32_t skip, int32_t rows_out, int32_t C, void* out, int32_t out_ld,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PF_B200_H_ */
