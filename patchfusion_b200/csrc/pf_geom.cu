// Depth to 3D on the device: the geometry helpers of `external/zoedepth/utils/geometry.py` on a depth canvas.
//
//   pf_depth_to_points    depth_to_points (:39-72): p = R M d K^-1 [x, y, 1]^T + t per pixel, with the pixel's colour
//                         round(255 clamp(v, 0, 1)) from the planar image in the same pass
//   pf_depth_edge_mask    hypot(np.gradient(d)) <= threshold and finite d > 0 (the vertex mask that drops the stretched
//                         triangles at depth discontinuities)
//   pf_mesh_quad_counts   create_triangles (:75-98) with a mask, first half: the kept triangles of every quad, their
//                         per-block sums and a scan of those into per-block output offsets
//   pf_mesh_triangles     second half: every kept triangle written at its offset (or, without a mask, all of them)
//   pf_ply_pack_vertices / pf_ply_pack_faces  binary little-endian PLY records, so the host only streams bytes
//
// Everything here is HBM-bound: one thread per pixel, quad or 16 output bytes, 16-byte accesses where alignment
// allows, and no shared-memory staging beyond the scans' partial sums.  The mesh compaction is deterministic: no
// atomics, and the kept triangles come out in numpy's boolean-indexing order.
#include "pf_common.cuh"
#include "pf_kernels.h"

namespace pf {

// R (row-major), t, 1/f and the principal point of get_intrinsics (:27-37), passed by value
struct PointXform {
  float r[9];
  float t[3];
  float inv_f, cx, cy;
};

// d K^-1 [x, y, 1]^T, then the x/y flip M, then R p + t
__device__ __forceinline__ void lift(const PointXform& p, float d, int x, int y, float* o) {
  const float px = -__fmul_rn(d, __fmul_rn(static_cast<float>(x) - p.cx, p.inv_f));
  const float py = -__fmul_rn(d, __fmul_rn(static_cast<float>(y) - p.cy, p.inv_f));
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = fmaf(p.r[3 * i], px, fmaf(p.r[3 * i + 1], py, fmaf(p.r[3 * i + 2], d, p.t[i])));
}

// round(255 clamp(v, 0, 1)), half to even (np.rint); NaN -> 0
__device__ __forceinline__ uint32_t to_u8(float v) {
  return static_cast<uint32_t>(rintf(__fmul_rn(255.0f, fminf(fmaxf(v, 0.0f), 1.0f))));
}

// VEC: four consecutive pixels per thread (n % 4 == 0, every pointer 16-byte aligned; colors 4-byte aligned): one
// float4 depth load, three float4 point stores, three float4 image loads and three 32-bit colour stores
template <bool VEC>
__global__ void __launch_bounds__(256) depth_to_points_kernel(const float* __restrict__ depth, int W, long long n,
                                                              PointXform p, const float* __restrict__ image,
                                                              float* __restrict__ points,
                                                              uint8_t* __restrict__ colors) {
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if constexpr (VEC) {
    const long long i0 = 4 * tid;
    if (i0 >= n) return;
    const float4 d4 = *reinterpret_cast<const float4*>(depth + i0);
    const float d[4] = {d4.x, d4.y, d4.z, d4.w};
    float o[12];
    int y = static_cast<int>(i0 / W), x = static_cast<int>(i0 - static_cast<long long>(y) * W);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lift(p, d[k], x, y, o + 3 * k);
      if (++x == W) { x = 0; ++y; }
    }
    float4* po = reinterpret_cast<float4*>(points + 3 * i0);
    po[0] = make_float4(o[0], o[1], o[2], o[3]);
    po[1] = make_float4(o[4], o[5], o[6], o[7]);
    po[2] = make_float4(o[8], o[9], o[10], o[11]);
    if (image != nullptr) {
      uint32_t c[12];
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float4 v = *reinterpret_cast<const float4*>(image + ch * n + i0);
        c[ch] = to_u8(v.x); c[3 + ch] = to_u8(v.y); c[6 + ch] = to_u8(v.z); c[9 + ch] = to_u8(v.w);
      }
      uint32_t* co = reinterpret_cast<uint32_t*>(colors + 3 * i0);
#pragma unroll
      for (int w = 0; w < 3; ++w)
        co[w] = c[4 * w] | (c[4 * w + 1] << 8) | (c[4 * w + 2] << 16) | (c[4 * w + 3] << 24);
    }
  } else {
    if (tid >= n) return;
    const int y = static_cast<int>(tid / W), x = static_cast<int>(tid - static_cast<long long>(y) * W);
    float o[3];
    lift(p, depth[tid], x, y, o);
#pragma unroll
    for (int i = 0; i < 3; ++i) points[3 * tid + i] = o[i];
    if (image != nullptr) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) colors[3 * tid + ch] = static_cast<uint8_t>(to_u8(image[ch * n + tid]));
    }
  }
}

// np.gradient along one axis with unit spacing, in fp32: (f[i+1] - f[i-1]) / 2 inside, one-sided at the borders
__device__ __forceinline__ float np_gradient(const float* __restrict__ f, long long i, int pos, int len, long long step,
                                             float here) {
  if (pos == 0) return __fsub_rn(f[i + step], here);
  if (pos == len - 1) return __fsub_rn(here, f[i - step]);
  return __fmul_rn(__fsub_rn(f[i + step], f[i - step]), 0.5f);
}

// one thread per pixel; the neighbours are re-read through L1 rather than staged
__global__ void __launch_bounds__(256) depth_edge_mask_kernel(const float* __restrict__ depth, int H, int W,
                                                              float threshold, uint8_t* __restrict__ mask) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  const long long i = static_cast<long long>(y) * W + x;
  const float d = depth[i];
  const float gy = np_gradient(depth, i, y, H, W, d), gx = np_gradient(depth, i, x, W, 1, d);
  // both squares are exact in fp64 and the sum is rounded once: hypotf's correctly rounded result but for double
  // rounding; a NaN or infinite gradient fails the comparison
  const double g2 = static_cast<double>(gy) * gy + static_cast<double>(gx) * gx;
  const float g = __double2float_rn(sqrt(g2));
  mask[i] = (isfinite(d) && d > 0.0f && g <= threshold) ? 1 : 0;
}

constexpr int kMeshBlock = PF_MESH_SCAN_BLOCK;        // quads per scan block (one per thread)
static_assert(kMeshBlock == 64, "the block scans below combine two warps");

struct Quad {
  int tl, tr, bl, br;
};

__device__ __forceinline__ Quad quad_at(long long q, int w) {
  const int y = static_cast<int>(q / (w - 1)), x = static_cast<int>(q - static_cast<long long>(y) * (w - 1));
  const int tl = y * w + x;
  return {tl, tl + 1, tl + w, tl + w + 1};
}

// flags of one quad: bit 0 keeps (tl, bl, tr), bit 1 keeps (br, tr, bl); the per-block sums of their popcounts
__global__ void __launch_bounds__(kMeshBlock) mesh_quad_counts_kernel(const uint8_t* __restrict__ mask, int w,
                                                                      long long nq, uint8_t* __restrict__ flags,
                                                                      long long* __restrict__ block_sums) {
  __shared__ int warp_sum[2];
  const long long q = blockIdx.x * static_cast<long long>(kMeshBlock) + threadIdx.x;
  int c = 0;
  if (q < nq) {
    const Quad v = quad_at(q, w);
    const bool tl = mask[v.tl] != 0, tr = mask[v.tr] != 0, bl = mask[v.bl] != 0, br = mask[v.br] != 0;
    const int f = ((tl && bl && tr) ? 1 : 0) | ((br && tr && bl) ? 2 : 0);
    flags[q] = static_cast<uint8_t>(f);
    c = __popc(f);
  }
  const int s = static_cast<int>(__reduce_add_sync(0xffffffffu, static_cast<unsigned>(c)));
  if (lane_id() == 0) warp_sum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) block_sums[blockIdx.x] = warp_sum[0] + warp_sum[1];
}

// in-place exclusive scan of nb block sums by one CTA, chunk after chunk in a fixed order; off[nb] = the total
constexpr int kScanThreads = 1024, kScanItems = 8;

__global__ void __launch_bounds__(kScanThreads) mesh_scan_kernel(long long* __restrict__ off, long long nb) {
  __shared__ long long warp_tot[kScanThreads / 32];
  __shared__ long long carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = lane_id(), warp = threadIdx.x >> 5;
  for (long long base = 0; base < nb; base += static_cast<long long>(kScanThreads) * kScanItems) {
    const long long i0 = base + static_cast<long long>(threadIdx.x) * kScanItems;
    long long v[kScanItems], sum = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      v[k] = i0 + k < nb ? off[i0 + k] : 0;
      sum += v[k];
    }
    long long inc = sum;                               // inclusive scan of the thread sums within the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      long long t = warp_tot[lane], wi = t;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += u;
      }
      warp_tot[lane] = wi - t;                         // exclusive warp offsets
    }
    __syncthreads();
    long long run = carry_s + warp_tot[warp] + inc - sum;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      if (i0 + k < nb) off[i0 + k] = run;
      run += v[k];
    }
    __syncthreads();                                   // every thread has read carry_s and warp_tot
    if (threadIdx.x == kScanThreads - 1) carry_s = run;
    __syncthreads();
  }
  if (threadIdx.x == 0) off[nb] = carry_s;
}

__device__ __forceinline__ void put_tri(int* __restrict__ faces, long long t, long long cap, int a, int b, int c) {
  if (t >= cap) return;
  faces[3 * t] = a; faces[3 * t + 1] = b; faces[3 * t + 2] = c;
}

// every kept triangle at block offset + the exclusive scan of the kept counts within the block
__global__ void __launch_bounds__(kMeshBlock) mesh_triangles_kernel(const uint8_t* __restrict__ flags,
                                                                    const long long* __restrict__ off, int w,
                                                                    long long nq, long long cap,
                                                                    int* __restrict__ faces) {
  __shared__ int warp_sum[2];
  const long long q = blockIdx.x * static_cast<long long>(kMeshBlock) + threadIdx.x;
  const int f = q < nq ? flags[q] : 0, c = __popc(f), lane = lane_id();
  int inc = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_sum[threadIdx.x >> 5] = inc;
  __syncthreads();
  if (f == 0) return;
  long long t = off[blockIdx.x] + inc - c + ((threadIdx.x >> 5) ? warp_sum[0] : 0);
  const Quad v = quad_at(q, w);
  if (f & 1) put_tri(faces, t++, cap, v.tl, v.bl, v.tr);
  if (f & 2) put_tri(faces, t, cap, v.br, v.tr, v.bl);
}

// every triangle (no mask): two quads (12 indices, 48 bytes) per thread; VEC: faces 16-byte aligned, three int4 stores
template <bool VEC>
__global__ void __launch_bounds__(256) mesh_all_triangles_kernel(int w, long long nq, int* __restrict__ faces) {
  const long long q0 = 2 * (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x);
  if (q0 >= nq) return;
  const bool pair = q0 + 1 < nq;
  const Quad a = quad_at(q0, w), b = quad_at(pair ? q0 + 1 : q0, w);
  const int v[12] = {a.tl, a.bl, a.tr, a.br, a.tr, a.bl, b.tl, b.bl, b.tr, b.br, b.tr, b.bl};
  int* o = faces + 6 * q0;
  if (VEC && pair) {
    int4* o4 = reinterpret_cast<int4*>(o);
    o4[0] = make_int4(v[0], v[1], v[2], v[3]);
    o4[1] = make_int4(v[4], v[5], v[6], v[7]);
    o4[2] = make_int4(v[8], v[9], v[10], v[11]);
  } else {
    const int m = pair ? 12 : 6;
#pragma unroll
    for (int k = 0; k < 12; ++k)
      if (k < m) o[k] = v[k];
  }
}

// 16 bytes of the PLY record stream per thread.  Faces (R = 13): uchar 3, then the three int32 indices; vertices
// (R = 15): float x, y, z, then uchar r, g, b.  `a` is the int32 / fp32 array viewed as bytes (little-endian, as the
// device is), `b` the colours.
template <int R>
__device__ __forceinline__ uint8_t ply_byte(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                            long long rec, int o) {
  if constexpr (R == 13) return o == 0 ? 3 : a[12 * rec + o - 1];
  else return o < 12 ? a[12 * rec + o] : b[3 * rec + o - 12];
}

template <int R>
__global__ void __launch_bounds__(256) ply_pack_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b,
                                                       long long nrec, uint8_t* __restrict__ out) {
  const long long total = nrec * R;
  const long long j0 = 16 * (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x);
  if (j0 >= total) return;
  long long rec = j0 / R;
  int o = static_cast<int>(j0 - rec * R);
  uint32_t word[4] = {0, 0, 0, 0};
  const int m = total - j0 < 16 ? static_cast<int>(total - j0) : 16;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    if (k < m) word[k >> 2] |= static_cast<uint32_t>(ply_byte<R>(a, b, rec, o)) << (8 * (k & 3));
    if (++o == R) { o = 0; ++rec; }
  }
  if (m == 16) {
    *reinterpret_cast<uint4*>(out + j0) = make_uint4(word[0], word[1], word[2], word[3]);
  } else {
    for (int k = 0; k < m; ++k) out[j0 + k] = static_cast<uint8_t>(word[k >> 2] >> (8 * (k & 3)));
  }
}

inline bool aligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

inline unsigned grid_for(long long items, int block) { return static_cast<unsigned>((items + block - 1) / block); }

}  // namespace pf

using namespace pf;

extern "C" {

int pf_depth_to_points(const float* depth, int32_t H, int32_t W, float inv_f, const float* rt_host, const float* image,
                       float* points, uint8_t* colors, void* stream) {
  if (H < 1 || W < 1) return set_error("pf_depth_to_points: bad shape %d x %d", H, W);
  if (depth == nullptr || points == nullptr) return set_error("pf_depth_to_points: null depth or points");
  if ((image == nullptr) != (colors == nullptr)) return set_error("pf_depth_to_points: image and colors go together");
  PointXform p = {};
  for (int i = 0; i < 9; ++i) p.r[i] = rt_host ? rt_host[i] : (i % 4 == 0 ? 1.0f : 0.0f);
  for (int i = 0; i < 3; ++i) p.t[i] = rt_host ? rt_host[9 + i] : 0.0f;
  p.inv_f = inv_f;
  p.cx = 0.5f * static_cast<float>(W);
  p.cy = 0.5f * static_cast<float>(H);
  const long long n = static_cast<long long>(H) * W;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = n % 4 == 0 && aligned(depth, 16) && aligned(points, 16) &&
                   (image == nullptr || (aligned(image, 16) && aligned(colors, 4)));
  if (vec) depth_to_points_kernel<true><<<grid_for(n / 4, 256), 256, 0, st>>>(depth, W, n, p, image, points, colors);
  else depth_to_points_kernel<false><<<grid_for(n, 256), 256, 0, st>>>(depth, W, n, p, image, points, colors);
  return check_launch("depth_to_points_kernel");
}

int pf_depth_edge_mask(const float* depth, int32_t H, int32_t W, float threshold, uint8_t* mask, void* stream) {
  if (H < 2 || W < 2) return set_error("pf_depth_edge_mask: np.gradient needs at least 2 x 2 pixels, got %d x %d", H, W);
  const dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8);
  depth_edge_mask_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(depth, H, W, threshold, mask);
  return check_launch("depth_edge_mask_kernel");
}

int pf_mesh_quad_counts(const uint8_t* mask, int32_t h, int32_t w, uint8_t* flags, int64_t* block_offsets,
                        void* stream) {
  if (h < 2 || w < 2) return set_error("pf_mesh_quad_counts: a mesh needs at least 2 x 2 vertices, got %d x %d", h, w);
  const long long nq = static_cast<long long>(h - 1) * (w - 1);
  const long long nb = (nq + kMeshBlock - 1) / kMeshBlock;
  long long* off = reinterpret_cast<long long*>(block_offsets);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  mesh_quad_counts_kernel<<<static_cast<unsigned>(nb), kMeshBlock, 0, st>>>(mask, w, nq, flags, off);
  if (int e = check_launch("mesh_quad_counts_kernel")) return e;
  mesh_scan_kernel<<<1, kScanThreads, 0, st>>>(off, nb);
  return check_launch("mesh_scan_kernel");
}

int pf_mesh_triangles(const uint8_t* flags, const int64_t* block_offsets, int32_t h, int32_t w, int32_t* faces,
                      int64_t cap, void* stream) {
  if (h < 2 || w < 2) return set_error("pf_mesh_triangles: a mesh needs at least 2 x 2 vertices, got %d x %d", h, w);
  const long long nq = static_cast<long long>(h - 1) * (w - 1);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (flags == nullptr) {
    if (cap < 2 * nq) return set_error("pf_mesh_triangles: room for %lld triangles, %lld needed", (long long)cap, 2 * nq);
    const unsigned grid = grid_for((nq + 1) / 2, 256);
    if (aligned(faces, 16)) mesh_all_triangles_kernel<true><<<grid, 256, 0, st>>>(w, nq, faces);
    else mesh_all_triangles_kernel<false><<<grid, 256, 0, st>>>(w, nq, faces);
    return check_launch("mesh_all_triangles_kernel");
  }
  if (cap <= 0) return 0;
  const long long nb = (nq + kMeshBlock - 1) / kMeshBlock;
  mesh_triangles_kernel<<<static_cast<unsigned>(nb), kMeshBlock, 0, st>>>(
      flags, reinterpret_cast<const long long*>(block_offsets), w, nq, cap, faces);
  return check_launch("mesh_triangles_kernel");
}

int pf_ply_pack_vertices(const float* points, const uint8_t* colors, int64_t n, uint8_t* out, void* stream) {
  if (n < 0 || !aligned(out, 16)) return set_error("pf_ply_pack_vertices: bad count or unaligned output");
  if (n == 0) return 0;
  ply_pack_kernel<15><<<grid_for((15 * n + 15) / 16, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint8_t*>(points), colors, n, out);
  return check_launch("ply_pack_vertices_kernel");
}

int pf_ply_pack_faces(const int32_t* faces, int64_t n, uint8_t* out, void* stream) {
  if (n < 0 || !aligned(out, 16)) return set_error("pf_ply_pack_faces: bad count or unaligned output");
  if (n == 0) return 0;
  ply_pack_kernel<13><<<grid_for((13 * n + 15) / 16, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint8_t*>(faces), nullptr, n, out);
  return check_launch("ply_pack_faces_kernel");
}

}  // extern "C"
