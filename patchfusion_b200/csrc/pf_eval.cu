// Evaluation-data preparation on the device (the per-image host work of the reference's dataset classes):
//
//   pf_gt_prepare     ground-truth depth + get_boundaries(x, th, dilation=0) in one pass over the source map, one branch
//                     per dataset: `estimator/datasets/u4k_dataset.py:118-119,168`, `general_dataset.py:66-79` (u4k),
//                     `:93-121` (mid), `:88-96` (eth3d), `:126-136` (cityscapes), edges `estimator/utils/image_ops.py:25-31`.
//   pf_ingest_raw_u8  the U4K raw frame: HWC uint8 BGR -> planar RGB fp32 u8 / 255, no resample
//                     (`u4k_dataset.py:115-129`, `general_dataset.py:23-25`).
//
// Every result is bit-identical to the reference's numpy arithmetic: under numpy 2 promotion a Python float combined
// with a float32 array is rounded to float32 first, so the constants arrive as host-rounded floats and every operation
// is an explicitly rounded IEEE fp32 operation (no contraction, no approximate division).
#include "pf_common.cuh"
#include "pf_kernels.h"

namespace pf {

enum GtKind { kGtU4k = 0, kGtMid = 1, kGtEth3d = 2, kGtCityscapes = 3 };

__device__ __forceinline__ float nan_to_num0(float v) { return (isnan(v) || isinf(v)) ? 0.0f : v; }

template <int KIND>
__device__ __forceinline__ float gt_source(const void* src, long long i) {
  if constexpr (KIND == kGtCityscapes) return static_cast<float>(static_cast<const uint16_t*>(src)[i]);
  else return static_cast<const float*>(src)[i];
}

// depth_gt of one source value
template <int KIND>
__device__ __forceinline__ float gt_depth(float x, float factor, float doffs) {
  if constexpr (KIND == kGtU4k) {
    return __fdiv_rn(factor, x);                                       // zero disparity -> inf, as in the reference
  } else if constexpr (KIND == kGtMid) {
    if (x == INFINITY) return 0.0f;
    return __fdiv_rn(__fdiv_rn(factor, __fadd_rn(x, doffs)), 1000.0f);
  } else if constexpr (KIND == kGtEth3d) {
    return nan_to_num0(x);
  } else {
    if (x > 0.0f) x = __fdiv_rn(__fsub_rn(x, 1.0f), 256.0f);
    return nan_to_num0(__fdiv_rn(factor, x));
  }
}

// the map the boundary is detected on
template <int KIND>
__device__ __forceinline__ float gt_edge_value(float x, float factor, float doffs) {
  if constexpr (KIND == kGtU4k) return x;
  else if constexpr (KIND == kGtMid) return x == INFINITY ? 0.0f : x;
  else return gt_depth<KIND>(x, factor, doffs);
}

// one thread per pixel; the four neighbours are re-read (L1) and re-transformed rather than staged
template <int KIND>
__global__ void __launch_bounds__(256) gt_prepare_kernel(const void* __restrict__ src, int H, int W, float factor,
                                                         float doffs, float th, float* __restrict__ depth,
                                                         uint8_t* __restrict__ boundary) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const long long i = static_cast<long long>(y) * W + x;
  const float s = gt_source<KIND>(src, i);
  const float e = gt_edge_value<KIND>(s, factor, doffs);
  // |e - q| > th compares as numpy does: a NaN difference (NaN input, inf - inf) is not an edge
  bool edge = false;
  if (y > 0) edge |= fabsf(__fsub_rn(e, gt_edge_value<KIND>(gt_source<KIND>(src, i - W), factor, doffs))) > th;
  if (y + 1 < H) edge |= fabsf(__fsub_rn(e, gt_edge_value<KIND>(gt_source<KIND>(src, i + W), factor, doffs))) > th;
  if (x > 0) edge |= fabsf(__fsub_rn(e, gt_edge_value<KIND>(gt_source<KIND>(src, i - 1), factor, doffs))) > th;
  if (x + 1 < W) edge |= fabsf(__fsub_rn(e, gt_edge_value<KIND>(gt_source<KIND>(src, i + 1), factor, doffs))) > th;
  depth[i] = gt_depth<KIND>(s, factor, doffs);
  boundary[i] = edge ? 1 : 0;
}

__global__ void __launch_bounds__(256) ingest_raw_u8_kernel(const uint8_t* __restrict__ img, long long n, int bgr,
                                                            float* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint8_t* px = img + 3 * i;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(bgr ? 2 - c : c) * n + i] = __fdiv_rn(static_cast<float>(px[c]), 255.0f);
}

}  // namespace pf

using namespace pf;

extern "C" {

int pf_gt_prepare(const void* src, int32_t kind, int32_t H, int32_t W, float factor, float doffs, float th,
                  float* depth, uint8_t* boundary, void* stream) {
  if (H < 1 || W < 1) return set_error("pf_gt_prepare: bad shape %d x %d", H, W);
  const dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (kind) {
    case kGtU4k: gt_prepare_kernel<kGtU4k><<<grid, block, 0, st>>>(src, H, W, factor, doffs, th, depth, boundary); break;
    case kGtMid: gt_prepare_kernel<kGtMid><<<grid, block, 0, st>>>(src, H, W, factor, doffs, th, depth, boundary); break;
    case kGtEth3d:
      gt_prepare_kernel<kGtEth3d><<<grid, block, 0, st>>>(src, H, W, factor, doffs, th, depth, boundary);
      break;
    case kGtCityscapes:
      gt_prepare_kernel<kGtCityscapes><<<grid, block, 0, st>>>(src, H, W, factor, doffs, th, depth, boundary);
      break;
    default: return set_error("pf_gt_prepare: unknown kind %d", kind);
  }
  return check_launch("gt_prepare_kernel");
}

int pf_ingest_raw_u8(const uint8_t* img_hwc, int32_t H, int32_t W, int32_t bgr, float* out_planar, void* stream) {
  if (H < 1 || W < 1) return set_error("pf_ingest_raw_u8: bad shape %d x %d", H, W);
  const long long n = static_cast<long long>(H) * W;
  ingest_raw_u8_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      img_hwc, n, bgr, out_planar);
  return check_launch("ingest_raw_u8_kernel");
}

}  // extern "C"
