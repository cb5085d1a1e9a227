// Internal declarations shared by the translation units of libpf_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "../../include/pf_b200.h"

namespace pf {

// Kernel-side view of pf_gemm_desc (device pointers typed, host-only fields dropped).
struct GemmDesc {
  int num_src, a_mode, taps;
  int halo;              // 3x3 conv through the halo-tile kernel (bh=16, bw=8)
  int halo_cl;           // halo kernel: CTAs per weight-multicast cluster (1, 2 or 4)
  int chunks[3];
  int k_true[3];         // logical channels of each source (profiler flop count)
  int M, NB, H, W, bh, bw, tiles_y, tiles_x, m_tiles;
  int N, block_n, n_tiles;
  const float* bias;
  int act;
  const __nv_bfloat16* res1;
  const __nv_bfloat16* res2;
  int res_ld;
  const float* gamma;
  void* out;
  int out_f32, out_ld, out_col0;
  int wide;              // every bf16 row pitch / column offset is a multiple of 16 elements: 256-bit accesses are aligned
  __nv_bfloat16* out2;
  int out2_ld;
  int ps, ps_cout_pad;   // pixel shuffle factor, per-tap column stride of the packed weight
  int n_logical;         // logical output channels (N, or Cout for pixel shuffle)
  __nv_bfloat16* vt;
  int vt_col0, vt_seq, vt_seq_pad, vt_dim;
  // fused trailing 1x1 layer (n2 <= 16 outputs per row, whole row in one N tile)
  const float* w2;
  const float* b2;
  int n2, act2, skip_main;
  float* out3;
  int out3_ld;
  // fused bilinear resample of halo-kernel sources (rs_h > 0): low-resolution map, its size / pitch and the
  // align_corners scales (in - 1) / (out - 1)
  const __nv_bfloat16* rs_ptr[3];
  int rs_h[3], rs_w[3], rs_ld[3];
  float rs_sy[3], rs_sx[3];
  int rs_any;
  int tma_out;           // pf_gemm_kernel epilogue through shared memory + TMA: 0 direct, 1 bf16 output, 2 fp32 output / residual stream
  int pp;                // plain linear layer through pf_gemm_pp_kernel (128 x 128 tiles, one per consumer warpgroup)
  // E4M3 halo conv (pf_conv3_halo_kernel<CL, BN, true>): the sources are 64-channel-padded segments of ONE e4m3 map
  // (pf_quantize_e4m3_tiles) read through tmA[0], the weights an e4m3 panel; acc * s_a[img] * s_w[col] before the bias
  int a_e4m3;
  const float* s_a;
  const float* s_w;
  // static input scale (pf_conv3_halo_e4m3_q8_kernel): a_scale for every tile instead of s_a[img]; out_e4m3: the output
  // is an e4m3 map written as e4m3_rn(sat(v * out_ratio)) through a uint8 tensor map, pad columns up to 64 ceil(N / 64)
  // zero
  int a_static;
  float a_scale;
  int out_e4m3;
  float out_ratio;       // pf_conv3_halo_e4m3_res_kernel (bf16 output): the ratio of its e4m3 ReLU copy out2
};

int set_error(const char* fmt, ...);
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count are per DEVICE: one-time setup is keyed by the
// current device so one process can drive engines on several GPUs.
constexpr int kMaxDevices = 64;
inline int current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return (d < 0 || d >= kMaxDevices) ? 0 : d;
}
// multiprocessors of the current device (cached per device)
inline int sm_count() {
  static int counts[kMaxDevices] = {0};
  const int dev = current_device();
  if (counts[dev] == 0) cudaDeviceGetAttribute(&counts[dev], cudaDevAttrMultiProcessorCount, dev);
  return counts[dev] > 0 ? counts[dev] : 1;
}
bool pdl_enabled();
int option(int which);          // PF_OPT_* tuning switches (pf_set_option / environment)

// <<<>>> replacement that sets the programmatic-stream-serialization attribute (kernels launched through it call
// pdl_wait() before touching global memory).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
void count_launch(const char* name);
// profiler hint for the NEXT launch: algorithmic flops + a printf-style shape label (no-op unless profiling)
void note_work(double flops, const char* fmt, ...);
int check_launch(const char* what);

// n-tile widths pf_gemm_kernel is compiled for (each consumer warpgroup holds a 64 x block_n fp32 accumulator tile in
// registers)
constexpr int kGemmWidths[] = {32, 64, 96, 128, 192, 256};

// n-tile width of pf_gemm_pp_kernel (d.pp): each consumer warpgroup owns whole 128 x 128 tiles; a block_n = 256 work
// item is two of them
constexpr int kPpBN = 128;

// tmBh != nullptr selects the weight-multicast variant (clusters of 2 CTAs): a {64, block_n / 2} box map of the weights
// ({64, 128} and {64, 64} boxes for d.pp)
// tmOut: output tensor map when d.tma_out != 0
int gemm_launch(const GemmDesc& d, const CUtensorMap* tmA, const CUtensorMap& tmB, const CUtensorMap* tmBh,
                const CUtensorMap* tmOut, cudaStream_t stream,
                const CUtensorMap* tmOut2 = nullptr);

// Tensor maps (driver entry point fetched at run time; cached by key).
int tmap_2d_bf16(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_cols,
                 uint32_t box_rows);
int tmap_2d_f32(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_cols,
                uint32_t box_rows);
int tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t ld1_elems,
                 uint64_t ld2_elems, uint32_t b0, uint32_t b1, uint32_t b2);
// 8-bit elements (e4m3 operands): rows of 64 bytes use SWIZZLE_64B
int tmap_2d_u8(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_bytes, uint32_t box_cols,
               uint32_t box_rows);
int tmap_4d_nhwc_u8(CUtensorMap* out, const void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint64_t ld_bytes,
                    uint32_t box_c, uint32_t box_w, uint32_t box_h);
int tmap_4d_nhwc_bf16(CUtensorMap* out, const void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N,
                      uint64_t ld_elems, uint32_t box_c, uint32_t box_w, uint32_t box_h);

}  // namespace pf
