// HBM-bound kernels of the PatchFusion hot path: normalisation, resampling, ROI crop-zoom, pooling, token assembly,
// Swin window attention (tiny head_dim -> CUDA cores), the metric-bins tail and the scatter-stitch.
// Layout: activations NHWC bf16 (row stride `ld`), 8 channels (16 B) per thread where the op is per-pixel.
#include "pf_common.cuh"
#include "pf_kernels.h"

namespace pf {

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 t = __bfloat1622float2(p[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static inline unsigned nblocks(long long n, int threads) { return static_cast<unsigned>((n + threads - 1) / threads); }

// ------------------------------------------------------------------------------------------------ LayerNorm
// one warp per row; the row lives in registers (C <= 1024) so HBM is touched once: mean, centred variance (two-pass
// like ATen), normalise, bf16 store.
__device__ __forceinline__ void ln_row(const float* __restrict__ xr, const float* __restrict__ w,
                                       const float* __restrict__ b, float eps, int C, bf16* __restrict__ orow, int lane) {
  float4 v[8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) { v[i] = *reinterpret_cast<const float4*>(xr + c); s += v[i].x + v[i].y + v[i].z + v[i].w; }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) {
      float a = v[i].x - mean, bb = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
      q += a * a + bb * bb + cc * cc + d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) {
      float4 g = __ldg(reinterpret_cast<const float4*>(w + c));
      float4 be = __ldg(reinterpret_cast<const float4*>(b + c));
      uint2 pk = make_uint2(pack_bf16((v[i].x - mean) * rstd * g.x + be.x, (v[i].y - mean) * rstd * g.y + be.y),
                            pack_bf16((v[i].z - mean) * rstd * g.z + be.z, (v[i].w - mean) * rstd * g.w + be.w));
      *reinterpret_cast<uint2*>(orow + c) = pk;
    }
  }
}

// pf_layernorm_e4m3: ln_row's statistics, and each fp32 affine value y (the same expression as ln_row's, before any
// bf16 rounding) written as e4m3_rn(sat(y * ratio)) with cvt.rn.satfinite, four bytes per store
__device__ __forceinline__ void ln_row_e4m3(const float* __restrict__ xr, const float* __restrict__ w,
                                            const float* __restrict__ b, float eps, int C, float ratio,
                                            uint8_t* __restrict__ orow, int lane) {
  float4 v[8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) { v[i] = *reinterpret_cast<const float4*>(xr + c); s += v[i].x + v[i].y + v[i].z + v[i].w; }
  }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) {
      float a = v[i].x - mean, bb = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
      q += a * a + bb * bb + cc * cc + d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane * 4 + i * 128;
    if (c < C) {
      float4 g = __ldg(reinterpret_cast<const float4*>(w + c));
      float4 be = __ldg(reinterpret_cast<const float4*>(b + c));
      const float y0 = (v[i].x - mean) * rstd * g.x + be.x, y1 = (v[i].y - mean) * rstd * g.y + be.y;
      const float y2 = (v[i].z - mean) * rstd * g.z + be.z, y3 = (v[i].w - mean) * rstd * g.w + be.w;
      uint16_t lo, hi;
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(__fmul_rn(y1, ratio)), "f"(__fmul_rn(y0, ratio)));
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(__fmul_rn(y3, ratio)), "f"(__fmul_rn(y2, ratio)));
      *reinterpret_cast<uint32_t*>(orow + c) = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
    }
  }
}
__global__ void layernorm_e4m3_kernel(const float* __restrict__ x, int x_ld, const float* __restrict__ w,
                                      const float* __restrict__ b, float eps, int rows, int C, float ratio,
                                      uint8_t* __restrict__ out, int out_ld) {
  pdl_wait();
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  ln_row_e4m3(x + static_cast<long long>(row) * x_ld, w, b, eps, C, ratio, out + static_cast<long long>(row) * out_ld,
              threadIdx.x & 31);
}

// rows_out > 0: output row r comes from input row (r / rows_out) * rows_in + skip + r % rows_out (per-image patch
// tokens with the cls row dropped); rows_out == 0: identity mapping.
__global__ void layernorm_kernel(const float* __restrict__ x, int x_ld, const float* __restrict__ w,
                                 const float* __restrict__ b, float eps, int rows, int C, bf16* __restrict__ out,
                                 int out_ld, int rows_in, int skip, int rows_out) {
  pdl_wait();
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  long long src = row;
  if (rows_out > 0) {
    const int g = row / rows_out;
    src = static_cast<long long>(g) * rows_in + skip + (row - g * rows_out);
  }
  ln_row(x + src * x_ld, w, b, eps, C, out + static_cast<long long>(row) * out_ld, threadIdx.x & 31);
}

// LayerNorm into the zero-padded (Hp x Wp) Swin token grid, one grid per image of x[B, H*W, C].
__global__ void swin_norm_pad_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                     const float* __restrict__ b, float eps, int B, int H, int W, int Hp, int Wp, int C,
                                     bf16* __restrict__ out) {
  long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= static_cast<long long>(B) * Hp * Wp) return;
  const int img = static_cast<int>(row / (Hp * Wp));
  const int r = static_cast<int>(row - static_cast<long long>(img) * Hp * Wp);
  int y = r / Wp, xx = r - y * Wp;
  bf16* orow = out + row * C;
  if (y >= H || xx >= W) {
    for (int c = lane * 4; c < C; c += 128) *reinterpret_cast<uint2*>(orow + c) = make_uint2(0u, 0u);
    return;
  }
  ln_row(x + ((static_cast<long long>(img) * H + y) * W + xx) * C, w, b, eps, C, orow, lane);
}

// ------------------------------------------------------------------------------------------------ ViT input
__global__ void patch_im2col_kernel(const float* __restrict__ img, int B, int H, int W, bf16* __restrict__ out, int ld) {
  const int gh = H / 14, gw = W / 14;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * gh * gw * ld;
  if (idx >= total) return;
  int col = static_cast<int>(idx % ld);
  long long row = idx / ld;
  float v = 0.f;
  if (col < 588) {
    int c = col / 196, rr = col - c * 196, py = rr / 14, px = rr - py * 14;
    int gx = static_cast<int>(row % gw);
    long long t = row / gw;
    int gy = static_cast<int>(t % gh);
    int b = static_cast<int>(t / gh);
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    float p = img[((static_cast<long long>(b) * 3 + c) * H + gy * 14 + py) * W + gx * 14 + px];
    v = (p - mean[c]) / stdv[c];
  }
  out[idx] = __float2bfloat16(v);
}

__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, int B, int n_patch, int D,
                                       float* __restrict__ tokens) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * (n_patch + 1) * D;
  if (idx >= total) return;
  int d = static_cast<int>(idx % D);
  long long t = idx / D;
  int tok = static_cast<int>(t % (n_patch + 1));
  int b = static_cast<int>(t / (n_patch + 1));
  float v = tok == 0 ? cls[d] : patch[(static_cast<long long>(b) * n_patch + tok - 1) * D + d];
  tokens[idx] = v + pos[static_cast<long long>(tok) * D + d];
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, long long n, bf16* __restrict__ out) {
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = __float2bfloat16(in[i]);
}

// ------------------------------------------------------------------------------------------------ resampling
// align_corners=True source coordinate exactly as ATen: scale = (in-1)/(out-1) (0 when out == 1), src = scale*dst.
__host__ __device__ __forceinline__ float ac_scale(int in, int out) {
  return out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1) : 0.f;
}
__device__ __forceinline__ void ac_coord_s(int dst, int in, float scale, int& lo, int& hi, float& frac) {
  float src = scale * dst;
  lo = static_cast<int>(src);
  if (lo > in - 1) lo = in - 1;
  hi = lo + (lo < in - 1 ? 1 : 0);
  frac = src - lo;
}
__device__ __forceinline__ void ac_coord(int dst, int in, int out, int& lo, int& hi, float& frac) {
  float scale = ac_scale(in, out);
  float src = scale * dst;
  lo = static_cast<int>(src);
  if (lo > in - 1) lo = in - 1;
  hi = lo + (lo < in - 1 ? 1 : 0);
  frac = src - lo;
}

// grid: (ceil(OW*cg / 256), OH, B); thread = (output pixel x, 8-channel group).  32-bit index math only, row
// coordinates and scales hoisted (the 64-bit div/mod version spent most of its time on address arithmetic).
__global__ void resize_bilinear_kernel(const bf16* __restrict__ in, int H, int W, int cg, int in_ld, int OH, int OW,
                                       float sy, float sx, bf16* __restrict__ out, int out_ld, int out_col0) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= OW * cg) return;
  const int ox = t / cg, g = t - ox * cg;
  const int oy = blockIdx.y, b = blockIdx.z;
  int y0, y1, x0, x1; float fy, fx;
  ac_coord_s(oy, H, sy, y0, y1, fy);
  ac_coord_s(ox, W, sx, x0, x1, fx);
  const bf16* base = in + static_cast<size_t>(b) * H * W * in_ld + g * 8;
  const bf16* r0 = base + static_cast<size_t>(y0) * W * in_ld;
  const bf16* r1 = base + static_cast<size_t>(y1) * W * in_ld;
  const uint4 u00 = __ldg(reinterpret_cast<const uint4*>(r0 + static_cast<size_t>(x0) * in_ld));
  const uint4 u01 = __ldg(reinterpret_cast<const uint4*>(r0 + static_cast<size_t>(x1) * in_ld));
  const uint4 u10 = __ldg(reinterpret_cast<const uint4*>(r1 + static_cast<size_t>(x0) * in_ld));
  const uint4 u11 = __ldg(reinterpret_cast<const uint4*>(r1 + static_cast<size_t>(x1) * in_ld));
  float a[8], bb[8], c[8], d[8], o[8];
  unpack8(u00, a); unpack8(u01, bb); unpack8(u10, c); unpack8(u11, d);
  const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = w00 * a[i] + w01 * bb[i] + w10 * c[i] + w11 * d[i];
  const size_t p = (static_cast<size_t>(b) * OH + oy) * OW + ox;
  *reinterpret_cast<uint4*>(out + p * out_ld + out_col0 + g * 8) = pack8(o);
}

// Shared-memory tiled variant for up-sampling (scale <= 1) of >= 64-channel maps: a block produces an 8 x 32 output
// pixel tile of one 64-channel slab from the <= 10 x 34 input patch it needs, so every input element is fetched from
// L2 once per tile instead of once per tap (4x), and both the patch loads and the output stores are 128-B segments.
constexpr int kRsTH = 8, kRsTW = 32, kRsPH = 10, kRsPW = 34;
__global__ void __launch_bounds__(256) resize_bilinear_tiled_kernel(const bf16* __restrict__ in, int H, int W, int in_ld,
                                                                     int OH, int OW, float sy, float sx, int slabs,
                                                                     bf16* __restrict__ out, int out_ld, int out_col0,
                                                                     int separable) {
  __shared__ uint4 patch[kRsPH * kRsPW * 8];
  __shared__ int s_y0[kRsTH], s_y1[kRsTH];
  __shared__ float s_fy[kRsTH];
  const int b = blockIdx.z;
  const int oy0 = blockIdx.y * kRsTH, ox0 = blockIdx.x * kRsTW;
  const int ylo = static_cast<int>(sy * oy0), xlo = static_cast<int>(sx * ox0);
  const int oy1 = min(oy0 + kRsTH, OH) - 1, ox1 = min(ox0 + kRsTW, OW) - 1;
  const int yhi = min(static_cast<int>(sy * oy1) + 1, H - 1), xhi = min(static_cast<int>(sx * ox1) + 1, W - 1);
  const int ph = yhi - ylo + 1, pw = xhi - xlo + 1;          // <= kRsPH x kRsPW for sy, sx <= 1
  // thread -> (16-byte channel chunk, output column); rows of the tile are looped: the x taps are per-thread
  // constants, the y taps per-row constants shared through smem
  const int ch = threadIdx.x & 7, tx = threadIdx.x >> 3;
  const int ox = ox0 + tx;
  int x0, x1; float fx;
  ac_coord_s(min(ox, OW - 1), W, sx, x0, x1, fx);
  x0 -= xlo; x1 -= xlo;
  if (threadIdx.x < kRsTH) {
    int y0, y1; float fy;
    ac_coord_s(min(oy0 + static_cast<int>(threadIdx.x), OH - 1), H, sy, y0, y1, fy);
    s_y0[threadIdx.x] = y0 - ylo; s_y1[threadIdx.x] = y1 - ylo; s_fy[threadIdx.x] = fy;
  }
  const bf16* base = in + static_cast<size_t>(b) * H * W * in_ld;
  for (int slab = 0; slab < slabs; ++slab) {
    __syncthreads();                                         // previous slab's patch fully consumed / tables ready
    for (int i = threadIdx.x; i < ph * pw * 8; i += 256) {
      const int c8 = i & 7, pix = i >> 3;
      const int py = pix / pw, px = pix - py * pw;
      patch[(py * kRsPW + px) * 8 + c8] = __ldg(reinterpret_cast<const uint4*>(
          base + (static_cast<size_t>(ylo + py) * W + xlo + px) * in_ld + slab * 64) + c8);
    }
    __syncthreads();
    if (ox < OW) {
      if (separable) {
        // Separable, streaming form (the order ATen itself uses: h0 * (w0 a + w1 b) + h1 * (w0 c + w1 d)): the x taps are
        // per-thread constants, so a source row is blended along x ONCE (r0 / r1, fp32 pairs in registers) and re-used by
        // every output row that reads it; an output row is then one y blend.  ~30 instead of ~95 instructions per 16-byte
        // output piece - the 4-tap form was ALU-bound (bf16 <-> fp32 conversion), not HBM-bound.
        const uint64_t pfx = pack2f(fx, fx), pgx = pack2f(1.f - fx, 1.f - fx);
        uint64_t r0[4], r1[4];
        int cy0 = -1, cy1 = -1;
        auto hrow = [&](int y, uint64_t (&r)[4]) {
          const uint4 ua = patch[(y * kRsPW + x0) * 8 + ch], ub = patch[(y * kRsPW + x1) * 8 + ch];
          const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {ub.x, ub.y, ub.z, ub.w};
#pragma unroll
          for (int k = 0; k < 4; ++k)
            r[k] = fma2(pfx, pack2(wb[k] << 16, wb[k] & 0xffff0000u), mul2(pgx, pack2(wa[k] << 16, wa[k] & 0xffff0000u)));
        };
#pragma unroll 2
        for (int ty = 0; ty < kRsTH; ++ty) {
          const int oy = oy0 + ty;
          if (oy >= OH) break;
          const int y0 = s_y0[ty], y1 = s_y1[ty];             // block-uniform: no divergence in the row bookkeeping
          const float fy = s_fy[ty];
          if (y0 != cy0) {
            if (y0 == cy1) {
#pragma unroll
              for (int k = 0; k < 4; ++k) r0[k] = r1[k];
            } else {
              hrow(y0, r0);
            }
            cy0 = y0;
          }
          if (y1 != cy1) {
            if (y1 == cy0) {
#pragma unroll
              for (int k = 0; k < 4; ++k) r1[k] = r0[k];
            } else {
              hrow(y1, r1);
            }
            cy1 = y1;
          }
          const uint64_t pfy = pack2f(fy, fy), pgy = pack2f(1.f - fy, 1.f - fy);
          uint32_t ow[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float lo, hi;
            unpack2f(fma2(pfy, r1[k], mul2(pgy, r0[k])), lo, hi);
            ow[k] = pack_bf16(lo, hi);
          }
          const size_t p = (static_cast<size_t>(b) * OH + oy) * OW + ox;
          *reinterpret_cast<uint4*>(out + p * out_ld + out_col0 + slab * 64 + ch * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
        continue;
      }
#pragma unroll 2
      for (int ty = 0; ty < kRsTH; ++ty) {
        const int oy = oy0 + ty;
        if (oy >= OH) break;
        const int y0 = s_y0[ty], y1 = s_y1[ty];
        const float fy = s_fy[ty];
        // blend on fp32 pairs: a bf16 pair widens to an fp32 pair with a shift and a mask (this kernel was ALU-bound:
        // ncu r01 sm__throughput 75 % at 41 % of DRAM peak)
        const uint4 ua = patch[(y0 * kRsPW + x0) * 8 + ch], ub = patch[(y0 * kRsPW + x1) * 8 + ch];
        const uint4 uc = patch[(y1 * kRsPW + x0) * 8 + ch], ud = patch[(y1 * kRsPW + x1) * 8 + ch];
        const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
        const uint64_t p00 = pack2f(w00, w00), p01 = pack2f(w01, w01), p10 = pack2f(w10, w10), p11 = pack2f(w11, w11);
        const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {ub.x, ub.y, ub.z, ub.w};
        const uint32_t wc[4] = {uc.x, uc.y, uc.z, uc.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
        uint32_t ow[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          uint64_t r = mul2(p00, pack2(wa[k] << 16, wa[k] & 0xffff0000u));
          r = fma2(p01, pack2(wb[k] << 16, wb[k] & 0xffff0000u), r);
          r = fma2(p10, pack2(wc[k] << 16, wc[k] & 0xffff0000u), r);
          r = fma2(p11, pack2(wd[k] << 16, wd[k] & 0xffff0000u), r);
          float lo, hi;
          unpack2f(r, lo, hi);
          ow[k] = pack_bf16(lo, hi);
        }
        const size_t p = (static_cast<size_t>(b) * OH + oy) * OW + ox;
        *reinterpret_cast<uint4*>(out + p * out_ld + out_col0 + slab * 64 + ch * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
    }
  }
}

__global__ void resize_bilinear_f32_kernel(const float* __restrict__ in, int B, int H, int W, int C, int OH, int OW,
                                           float* __restrict__ out) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * OH * OW * C;
  if (idx >= total) return;
  int c = static_cast<int>(idx % C);
  long long p = idx / C;
  int ox = static_cast<int>(p % OW);
  long long t = p / OW;
  int oy = static_cast<int>(t % OH);
  int b = static_cast<int>(t / OH);
  int y0, y1, x0, x1; float fy, fx;
  ac_coord(oy, H, OH, y0, y1, fy);
  ac_coord(ox, W, OW, x0, x1, fx);
  const float* base = in + static_cast<long long>(b) * H * W * C + c;
  float v00 = base[(static_cast<long long>(y0) * W + x0) * C], v01 = base[(static_cast<long long>(y0) * W + x1) * C];
  float v10 = base[(static_cast<long long>(y1) * W + x0) * C], v11 = base[(static_cast<long long>(y1) * W + x1) * C];
  out[idx] = (1.f - fy) * ((1.f - fx) * v00 + fx * v01) + fy * ((1.f - fx) * v10 + fx * v11);
}

// torchvision roi_align bilinear tap with its edge rules (aligned=True, one sample per bin).
__device__ __forceinline__ bool roi_coord(float c, int size, int& lo, int& hi, float& frac) {
  if (c < -1.0f || c > static_cast<float>(size)) return false;
  if (c <= 0.f) c = 0.f;
  lo = static_cast<int>(c);
  if (lo >= size - 1) { lo = hi = size - 1; c = static_cast<float>(lo); } else { hi = lo + 1; }
  frac = c - lo;
  return true;
}

// grid: (ceil(w*cg / 256), h, T); thread = (output pixel x, 8-channel group [bf16] or channel [fp32]).
// tile_image (nullable): box t samples image tile_image[t] of the [B, h, w, in_ld] map (NULL: image 0).
template <bool F32>
__global__ void roi_crop_zoom_kernel(const void* __restrict__ feat, int h, int w, int cg, int in_ld,
                                     const int* __restrict__ tile_image, const float* __restrict__ boxes, float scale,
                                     void* __restrict__ out, int out_ld, int out_col0) {
  const int tt = blockIdx.x * blockDim.x + threadIdx.x;
  if (tt >= w * cg) return;
  const int ox = tt / cg, g = tt - ox * cg;
  const int oy = blockIdx.y, t = blockIdx.z;
  const size_t img = tile_image != nullptr ? static_cast<size_t>(__ldg(tile_image + t)) * h * w * in_ld : 0;
  const float x1 = __ldg(boxes + t * 4 + 0) * scale - 0.5f, y1 = __ldg(boxes + t * 4 + 1) * scale - 0.5f;
  const float x2 = __ldg(boxes + t * 4 + 2) * scale - 0.5f, y2 = __ldg(boxes + t * 4 + 3) * scale - 0.5f;
  const float bw = (x2 - x1) / w, bh = (y2 - y1) / h;
  const float sy = y1 + (oy + 0.5f) * bh, sx = x1 + (ox + 0.5f) * bw;
  int yl, yh, xl, xh; float fy, fx;
  bool ok = roi_coord(sy, h, yl, yh, fy);
  ok = roi_coord(sx, w, xl, xh, fx) && ok;
  const size_t p = (static_cast<size_t>(t) * h + oy) * w + ox;
  if (F32) {
    const float* f = static_cast<const float*>(feat) + img + g;
    float v = 0.f;
    if (ok) {
      float v00 = f[(static_cast<size_t>(yl) * w + xl) * in_ld], v01 = f[(static_cast<size_t>(yl) * w + xh) * in_ld];
      float v10 = f[(static_cast<size_t>(yh) * w + xl) * in_ld], v11 = f[(static_cast<size_t>(yh) * w + xh) * in_ld];
      v = (1.f - fy) * (1.f - fx) * v00 + (1.f - fy) * fx * v01 + fy * (1.f - fx) * v10 + fy * fx * v11;
    }
    static_cast<float*>(out)[p * out_ld + out_col0 + g] = v;
  } else {
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
    if (ok) {
      const bf16* f = static_cast<const bf16*>(feat) + img + g * 8;
      float a[8], bb[8], c[8], d[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(f + (static_cast<size_t>(yl) * w + xl) * in_ld)), a);
      unpack8(__ldg(reinterpret_cast<const uint4*>(f + (static_cast<size_t>(yl) * w + xh) * in_ld)), bb);
      unpack8(__ldg(reinterpret_cast<const uint4*>(f + (static_cast<size_t>(yh) * w + xl) * in_ld)), c);
      unpack8(__ldg(reinterpret_cast<const uint4*>(f + (static_cast<size_t>(yh) * w + xh) * in_ld)), d);
      const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = w00 * a[i] + w01 * bb[i] + w10 * c[i] + w11 * d[i];
    }
    *reinterpret_cast<uint4*>(static_cast<bf16*>(out) + p * out_ld + out_col0 + g * 8) = pack8(o);
  }
}

__global__ void maxpool2_kernel(const bf16* __restrict__ in, int B, int H, int W, int C, int in_ld,
                                bf16* __restrict__ out, int out_ld) {
  const int OH = H / 2, OW = W / 2, cg = C >> 3;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * OH * OW * cg;
  if (idx >= total) return;
  int g = static_cast<int>(idx % cg);
  long long p = idx / cg;
  int ox = static_cast<int>(p % OW);
  long long t = p / OW;
  int oy = static_cast<int>(t % OH);
  int b = static_cast<int>(t / OH);
  const bf16* base = in + ((static_cast<long long>(b) * H + oy * 2) * W + ox * 2) * in_ld + g * 8;
  float a[8], bb[8], c[8], d[8], o[8];
  unpack8(*reinterpret_cast<const uint4*>(base), a);
  unpack8(*reinterpret_cast<const uint4*>(base + in_ld), bb);
  unpack8(*reinterpret_cast<const uint4*>(base + static_cast<long long>(W) * in_ld), c);
  unpack8(*reinterpret_cast<const uint4*>(base + static_cast<long long>(W + 1) * in_ld), d);
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = fmaxf(fmaxf(a[i], bb[i]), fmaxf(c[i], d[i]));
  *reinterpret_cast<uint4*>(out + p * out_ld + g * 8) = pack8(o);
}

__global__ void im2col_3x3_s2_kernel(const bf16* __restrict__ in, int B, int H, int W, int C, int in_ld,
                                     bf16* __restrict__ out) {
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1, cg = C >> 3;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * OH * OW * 9 * cg;
  if (idx >= total) return;
  int g = static_cast<int>(idx % cg);
  long long t = idx / cg;
  int tap = static_cast<int>(t % 9);
  long long p = t / 9;
  int ox = static_cast<int>(p % OW);
  long long t2 = p / OW;
  int oy = static_cast<int>(t2 % OH);
  int b = static_cast<int>(t2 / OH);
  int iy = oy * 2 - 1 + tap / 3, ix = ox * 2 - 1 + tap % 3;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W)
    v = *reinterpret_cast<const uint4*>(in + ((static_cast<long long>(b) * H + iy) * W + ix) * in_ld + g * 8);
  *reinterpret_cast<uint4*>(out + p * (9LL * C) + static_cast<long long>(tap) * C + g * 8) = v;
}

// tile_image (nullable): tile ti is cropped from image tile_image[ti] of img [B,3,H,W] (NULL: image 0).
__global__ void crop_resize_kernel(const float* __restrict__ img, int H, int W, const int* __restrict__ origins,
                                   const int* __restrict__ tile_image, int T, int th, int tw, int ph, int pw,
                                   float* __restrict__ out) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(T) * 3 * ph * pw;
  if (idx >= total) return;
  int ox = static_cast<int>(idx % pw);
  long long t = idx / pw;
  int oy = static_cast<int>(t % ph);
  t /= ph;
  int c = static_cast<int>(t % 3);
  int ti = static_cast<int>(t / 3);
  int y0, y1, x0, x1; float fy, fx;
  ac_coord(oy, th, ph, y0, y1, fy);
  ac_coord(ox, tw, pw, x0, x1, fx);
  const long long plane = (tile_image != nullptr ? tile_image[ti] * 3LL : 0LL) + c;
  const float* base = img + (plane * H + origins[ti * 2]) * W + origins[ti * 2 + 1];
  float v00 = base[static_cast<long long>(y0) * W + x0], v01 = base[static_cast<long long>(y0) * W + x1];
  float v10 = base[static_cast<long long>(y1) * W + x0], v11 = base[static_cast<long long>(y1) * W + x1];
  out[idx] = (1.f - fy) * ((1.f - fx) * v00 + fx * v01) + fy * ((1.f - fx) * v10 + fx * v11);
}

// crop_resize_kernel over images of different sizes: tile ti reads descriptor images[tile_image[ti]] (its own planar
// [3,H,W] image and crop size th x tw).  Same index order and bilinear arithmetic, so equal geometry gives equal bits.
__global__ void crop_resize_multi_kernel(const pf_crop_image* __restrict__ images, const int* __restrict__ origins,
                                         const int* __restrict__ tile_image, int T, int ph, int pw,
                                         float* __restrict__ out) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(T) * 3 * ph * pw;
  if (idx >= total) return;
  int ox = static_cast<int>(idx % pw);
  long long t = idx / pw;
  int oy = static_cast<int>(t % ph);
  t /= ph;
  int c = static_cast<int>(t % 3);
  int ti = static_cast<int>(t / 3);
  const pf_crop_image d = images[tile_image[ti]];
  const int H = d.H, W = d.W;
  int y0, y1, x0, x1; float fy, fx;
  ac_coord(oy, d.th, ph, y0, y1, fy);
  ac_coord(ox, d.tw, pw, x0, x1, fx);
  const float* base = d.img + (static_cast<long long>(c) * H + origins[ti * 2]) * W + origins[ti * 2 + 1];
  float v00 = base[static_cast<long long>(y0) * W + x0], v01 = base[static_cast<long long>(y0) * W + x1];
  float v10 = base[static_cast<long long>(y1) * W + x0], v11 = base[static_cast<long long>(y1) * W + x1];
  // The blend of crop_resize_kernel with its FMA contraction spelled out (nvcc fuses the first product of each a*b + c*d
  // there): left to the compiler, this kernel fused the other product of one row and differed in the last bit.
  const float top = __fmaf_rn(1.f - fx, v00, __fmul_rn(fx, v01));
  const float bot = __fmaf_rn(1.f - fx, v10, __fmul_rn(fx, v11));
  out[idx] = __fmaf_rn(1.f - fy, top, __fmul_rn(fy, bot));
}

__global__ void pack_unet_input_kernel(const float* __restrict__ cd, const float* __restrict__ fd,
                                       const float* __restrict__ rgb, int T, int H, int W, bf16* __restrict__ out,
                                       int ld) {
  long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(T) * H * W;
  if (p >= total) return;
  long long hw = static_cast<long long>(H) * W;
  int t = static_cast<int>(p / hw);
  long long r = p - t * hw;
  float f[8] = {cd[p], fd[p], rgb[(t * 3LL + 0) * hw + r], rgb[(t * 3LL + 1) * hw + r], rgb[(t * 3LL + 2) * hw + r],
                0.f, 0.f, 0.f};
  *reinterpret_cast<uint4*>(out + p * ld) = pack8(f);
}

// ------------------------------------------------------------------------------------------------ image ingest / output
// (SURVEY.md §8f-1/f-2: the callers either side of the hot path)
// uint8 HWC (BGR as cv2.imread returns it, or RGB) -> planar RGB fp32 in [0,1], bicubic (A = -0.75, align_corners=True,
// border taps clamped) to (OH, OW): `estimator/datasets/general_dataset.py:40-45` (cv2 decode -> /255 -> F.interpolate).
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }

__global__ void ingest_u8_kernel(const uint8_t* __restrict__ img, int H, int W, int bgr, int OH, int OW, float sy, float sx,
                                 float* __restrict__ out) {
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= OW) return;
  const float A = -0.75f;
  const float ry = sy * oy, rx = sx * ox;
  const int iy = static_cast<int>(floorf(ry)), ix = static_cast<int>(floorf(rx));
  const float ty = ry - iy, tx = rx - ix;
  const float wy[4] = {cubic2(ty + 1.f, A), cubic1(ty, A), cubic1(1.f - ty, A), cubic2(2.f - ty, A)};
  const float wx[4] = {cubic2(tx + 1.f, A), cubic1(tx, A), cubic1(1.f - tx, A), cubic2(2.f - tx, A)};
  float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int yy = min(max(iy - 1 + a, 0), H - 1);
    float row[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int xx = min(max(ix - 1 + b, 0), W - 1);
      const uint8_t* px = img + (static_cast<size_t>(yy) * W + xx) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) row[c] += wx[b] * (static_cast<float>(px[c]) * (1.0f / 255.0f));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += wy[a] * row[c];
  }
  const size_t plane = static_cast<size_t>(OH) * OW, o = static_cast<size_t>(oy) * OW + ox;
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(bgr ? 2 - c : c) * plane + o] = acc[c];
}

// depth canvas -> uint16 image: nearest resize (F.interpolate default, `tools/test_single_forward.py:26`) then
// (depth * scale).astype(uint16) as `estimator/tester/tester.py:75-76` (scale 256), saturating.
__global__ void depth_to_u16_kernel(const float* __restrict__ d, int H, int W, int OH, int OW, float scale,
                                    uint16_t* __restrict__ out) {
  const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
  if (ox >= OW) return;
  const int sy = min(static_cast<int>(floorf(oy * (static_cast<float>(H) / OH))), H - 1);
  const int sx = min(static_cast<int>(floorf(ox * (static_cast<float>(W) / OW))), W - 1);
  const float v = d[static_cast<size_t>(sy) * W + sx] * scale;
  out[static_cast<size_t>(oy) * OW + ox] = static_cast<uint16_t>(fminf(fmaxf(v, 0.f), 65535.f));
}

// ------------------------------------------------------------------------------------------------ Swin / G2L
// x[B, n, C] = feat rows + ape[n, C], the same embedding added to every image
__global__ void g2l_embed_kernel(const bf16* __restrict__ feat, int feat_ld, const float* __restrict__ ape, int B, int n,
                                 int C, float* __restrict__ x) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long per = static_cast<long long>(n) * C;
  if (idx >= B * per) return;
  int c = static_cast<int>(idx % C);
  long long t = idx / C;
  x[idx] = __bfloat162float(feat[t * feat_ld + c]) + ape[idx % per];
}

// One CTA per (window, head); thread i < 144 owns query row i.  K / V of the window live in shared memory as fp32
// PAIRS so both the q.k dot product and the p.v accumulation run on fp32 pairs (all lanes read the same key: the
// shared-memory reads are broadcasts).  Scores are kept in the log2 domain (scale * log2e folded into q, log2e into
// the bias table and the -100 shift mask) and the online softmax rescales only when the running maximum moves - one
// ex2 per key instead of two exps and an unconditional rescale (r01: 4.7 ms per image in this kernel).
// blockIdx.z = image: qkv / out hold B padded grids back to back.
template <int HD>
__global__ void __launch_bounds__(160) window_attention_kernel(const bf16* __restrict__ qkv,
                                                               const float* __restrict__ bias_table, int Hp, int Wp,
                                                               int C, int heads, int shift, bf16* __restrict__ out) {
  qkv += static_cast<long long>(blockIdx.z) * Hp * Wp * (3 * C);
  out += static_cast<long long>(blockIdx.z) * Hp * Wp * C;
  constexpr int WS = 12, NT = 144, HP = HD / 2;
  constexpr float kLog2e = 1.4426950408889634f;
  __shared__ uint64_t sk[NT][HP];
  __shared__ uint64_t sv[NT][HP];
  __shared__ float sb[529];
  __shared__ int stok[NT];
  __shared__ int sreg[NT];
  const int head = blockIdx.y;
  const int win = blockIdx.x;
  const int wpr = Wp / WS;
  const int wy = win / wpr, wx = win - wy * wpr;
  const int tid = threadIdx.x;
  for (int i = tid; i < 529; i += blockDim.x) sb[i] = bias_table[i * heads + head] * kLog2e;
  if (tid < NT) {
    int iy = tid / WS, ix = tid - iy * WS;
    int ry = wy * WS + iy, rx = wx * WS + ix;                      // position in the rolled frame
    int oy = (ry + shift) % Hp, ox = (rx + shift) % Wp;            // source position (torch.roll by -shift)
    stok[tid] = oy * Wp + ox;
    int hr = ry < Hp - WS ? 0 : (ry < Hp - shift ? 1 : 2);
    int wr = rx < Wp - WS ? 0 : (rx < Wp - shift ? 1 : 2);
    sreg[tid] = shift > 0 ? hr * 3 + wr : 0;
  }
  __syncthreads();
  for (int i = tid; i < NT * HP; i += blockDim.x) {
    int t = i / HP, d = i - t * HP;
    const bf16* row = qkv + static_cast<long long>(stok[t]) * (3 * C) + head * HD + 2 * d;
    const float2 kk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + C));
    const float2 vv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 2 * C));
    sk[t][d] = pack2f(kk.x, kk.y);
    sv[t][d] = pack2f(vv.x, vv.y);
  }
  __syncthreads();
  if (tid >= NT) return;
  const float scale = rsqrtf(static_cast<float>(HD)) * kLog2e;
  uint64_t q[HP], acc[HP];
  {
    const bf16* row = qkv + static_cast<long long>(stok[tid]) * (3 * C) + head * HD;
#pragma unroll
    for (int d = 0; d < HP; ++d) {
      const float2 qq = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + 2 * d));
      q[d] = pack2f(qq.x * scale, qq.y * scale);
      acc[d] = 0;                                                  // (+0.0f, +0.0f)
    }
  }
  const int iy = tid / WS, ix = tid - iy * WS, myreg = sreg[tid];
  const float* brow = sb + (iy + WS - 1) * (2 * WS - 1) + (ix + WS - 1);
  float m = -INFINITY, l = 0.f;
  int jy = 0, jx = 0;
  for (int j = 0; j < NT; ++j) {
    uint64_t s2 = 0;
#pragma unroll
    for (int d = 0; d < HP; ++d) s2 = fma2(q[d], sk[j][d], s2);
    float s0, s1;
    unpack2f(s2, s0, s1);
    float s = s0 + s1 + brow[-(jy * (2 * WS - 1) + jx)];
    if (sreg[j] != myreg) s -= 100.0f * kLog2e;
    if (++jx == WS) { jx = 0; ++jy; }
    if (s > m) {                                                   // running maximum moves (rare after the first keys)
      float a;
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(a) : "f"(m - s));
      const uint64_t a2 = pack2f(a, a);
#pragma unroll
      for (int d = 0; d < HP; ++d) acc[d] = mul2(acc[d], a2);
      l *= a;
      m = s;
    }
    float p;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(p) : "f"(s - m));
    l += p;
    const uint64_t p2 = pack2f(p, p);
#pragma unroll
    for (int d = 0; d < HP; ++d) acc[d] = fma2(p2, sv[j][d], acc[d]);
  }
  const float inv = 1.f / l;
  bf16* orow = out + static_cast<long long>(stok[tid]) * C + head * HD;
#pragma unroll
  for (int d = 0; d < HP; ++d) {
    float a0, a1;
    unpack2f(acc[d], a0, a1);
    *reinterpret_cast<uint32_t*>(orow + 2 * d) = pack_bf16(a0 * inv, a1 * inv);
  }
}

// x[B, H*W, C] += y[B, Hp*Wp, C] cropped to the top-left H x W of each padded grid
__global__ void swin_residual_crop_kernel(float* __restrict__ x, const float* __restrict__ y, int B, int H, int W,
                                          int Hp, int Wp, int C) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(B) * H * W * C) return;
  int c = static_cast<int>(idx % C);
  long long t = idx / C;
  int xx = static_cast<int>(t % W);
  t /= W;
  int yy = static_cast<int>(t % H), img = static_cast<int>(t / H);
  x[idx] += y[((static_cast<long long>(img) * Hp + yy) * Wp + xx) * C + c];
}

// ------------------------------------------------------------------------------------------------ metric-bins tail
__global__ void add_upsampled_kernel(const bf16* __restrict__ a, int B, int H, int W, int C, const bf16* __restrict__ prev,
                                     int PH, int PW, bf16* __restrict__ out) {
  const int cg = C >> 3;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(B) * H * W * cg;
  if (idx >= total) return;
  int g = static_cast<int>(idx % cg);
  long long p = idx / cg;
  int ox = static_cast<int>(p % W);
  long long t = p / W;
  int oy = static_cast<int>(t % H);
  int b = static_cast<int>(t / H);
  int y0, y1, x0, x1; float fy, fx;
  ac_coord(oy, PH, H, y0, y1, fy);
  ac_coord(ox, PW, W, x0, x1, fx);
  const bf16* base = prev + static_cast<long long>(b) * PH * PW * C + g * 8;
  float q0[8], q1[8], q2[8], q3[8], s[8], o[8];
  unpack8(*reinterpret_cast<const uint4*>(base + (static_cast<long long>(y0) * PW + x0) * C), q0);
  unpack8(*reinterpret_cast<const uint4*>(base + (static_cast<long long>(y0) * PW + x1) * C), q1);
  unpack8(*reinterpret_cast<const uint4*>(base + (static_cast<long long>(y1) * PW + x0) * C), q2);
  unpack8(*reinterpret_cast<const uint4*>(base + (static_cast<long long>(y1) * PW + x1) * C), q3);
  unpack8(*reinterpret_cast<const uint4*>(a + p * C + g * 8), s);
  const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = s[i] + w00 * q0[i] + w01 * q1[i] + w10 * q2[i] + w11 * q3[i];
  *reinterpret_cast<uint4*>(out + p * C + g * 8) = pack8(o);
}

// one warp per pixel (grid-stride), 2 bins per lane (nbins == 64): b = up(b_prev); b += mean_a|sum_a( dist(dx) ),
// dx = A_a - b, dist = inverse (dx / (1 + 300 dx^2)) or exponential (exp(-300 dx^2) dx) attractor.  The <= 16 attractor points of the pixel are read once per warp.
// NORMED (AttractorLayer, attractor.py:100-135): the attractor points are A + 1e-3 (A holds the even `_net` channels
// only: A_normed is overwritten by A[:, :, 0], attractor.py:105-106), and `centers`, when given, receives
// clip(sort((max - min) b + min), min, max), sorted per pixel by a bitonic network over the warp's 64 values.
template <bool NORMED>
__device__ __forceinline__ void attractor_body(const float* __restrict__ A, int A_ld, int nA, const float* __restrict__ b_prev,
                                               int PH, int PW, int B, int H, int W, int nbins, int kind_mean, int type_exp,
                                               float sy, float sx, float* __restrict__ b_out, float min_d, float max_d,
                                               float* __restrict__ centers) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const int total = B * H * W, hw = H * W;
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < total; p += warps) {
    const int b = p / hw, rem = p - b * hw;
    const int oy = rem / W, ox = rem - oy * W;
    int y0, y1, x0, x1; float fy, fx;
    ac_coord_s(oy, PH, sy, y0, y1, fy);
    ac_coord_s(ox, PW, sx, x0, x1, fx);
    const float* base = b_prev + static_cast<size_t>(b) * PH * PW * nbins;
    const float* r00 = base + (static_cast<size_t>(y0) * PW + x0) * nbins;
    const float* r01 = base + (static_cast<size_t>(y0) * PW + x1) * nbins;
    const float* r10 = base + (static_cast<size_t>(y1) * PW + x0) * nbins;
    const float* r11 = base + (static_cast<size_t>(y1) * PW + x1) * nbins;
    float av = lane < nA ? __ldg(A + static_cast<size_t>(p) * A_ld + lane) : 0.f;
    if (NORMED) av += 1e-3f;
    float bc[2], s[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = lane + 32 * i;
      bc[i] = (1.f - fy) * ((1.f - fx) * __ldg(r00 + k) + fx * __ldg(r01 + k)) +
              fy * ((1.f - fx) * __ldg(r10 + k) + fx * __ldg(r11 + k));
    }
    for (int a = 0; a < nA; ++a) {
      const float aa = __shfl_sync(0xffffffffu, av, a);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float dx = aa - bc[i];
        // attractor.py:44-57 / 29-41 with the TorchScript defaults alpha=300, gamma=2 (the layer never forwards the
        // configured values, attractor.py:191-195)
        s[i] += type_exp ? __expf(-300.f * dx * dx) * dx : dx / (1.f + 300.f * dx * dx);
      }
    }
    float v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (kind_mean) s[i] /= nA;
      v[i] = bc[i] + s[i];
      b_out[static_cast<size_t>(p) * nbins + lane + 32 * i] = v[i];
    }
    if (NORMED && centers != nullptr) {
      const float range = max_d - min_d;
#pragma unroll
      for (int i = 0; i < 2; ++i) v[i] = range * v[i] + min_d;
      // bitonic sort of the 64 values, element k = lane + 32 i: every (size, stride) step pairs k with k ^ stride and
      // keeps the smaller value at the lower index where (k & size) == 0 (ascending run), the larger elsewhere.  The
      // stride-32 partner is the lane's other register; the others live in lane ^ stride.
#pragma unroll
      for (int size = 2; size <= 64; size <<= 1) {
#pragma unroll
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
          if (stride == 32) {
            const float lo = fminf(v[0], v[1]), hi = fmaxf(v[0], v[1]);
            v[0] = lo; v[1] = hi;
          } else {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const int k = lane + 32 * i;
              const float o = __shfl_xor_sync(0xffffffffu, v[i], stride);
              const bool up = (k & size) == 0, lower = (k & stride) == 0;
              v[i] = (up == lower) ? fminf(v[i], o) : fmaxf(v[i], o);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i)
        centers[static_cast<size_t>(p) * nbins + lane + 32 * i] = fminf(fmaxf(v[i], min_d), max_d);
    }
  }
}

__global__ void attractor_kernel(const float* __restrict__ A, int A_ld, int nA, const float* __restrict__ b_prev, int PH,
                                 int PW, int B, int H, int W, int nbins, int kind_mean, int type_exp, float sy, float sx,
                                 float* __restrict__ b_out) {
  attractor_body<false>(A, A_ld, nA, b_prev, PH, PW, B, H, W, nbins, kind_mean, type_exp, sy, sx, b_out, 0.f, 0.f, nullptr);
}

__global__ void attractor_normed_kernel(const float* __restrict__ A, int A_ld, int nA, const float* __restrict__ b_prev,
                                        int PH, int PW, int B, int H, int W, int nbins, int kind_mean, int type_exp,
                                        float sy, float sx, float* __restrict__ b_out, float min_d, float max_d,
                                        float* __restrict__ centers) {
  attractor_body<true>(A, A_ld, nA, b_prev, PH, PW, B, H, W, nbins, kind_mean, type_exp, sy, sx, b_out, min_d, max_d,
                       centers);
}

// SeedBinRegressor's centres (localbins_layers.py:51-67) from its `_net` output S (ReLU'd), one warp per pixel
// (grid-stride), 2 bins per lane (nbins == 64): w_k = (max - min) (S_k + 1e-3) / sum_j (S_j + 1e-3), edges = min +
// cumsum(w) (the min_depth pad in front), c_k = (edge_k + edge_k+1) / 2.  The sum is a butterfly; the cumsum a
// Hillis-Steele scan of each 32-bin half, the upper half offset by the lower half's total.  PF_SEED_NORMED off: the
// centres are S itself (SeedBinRegressorUnnormed).  PF_SEED_TO_UNIT: (c - min) / (max - min), the b_prev of the
// normed attractors (zoedepth_v1.py:176-181).
__global__ void seed_bins_kernel(const float* __restrict__ S, int S_ld, long long total, int normed, int to_unit,
                                 float min_d, float max_d, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const float range = max_d - min_d;
  for (long long p = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; p < total; p += warps) {
    float c[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) c[i] = __ldg(S + p * S_ld + lane + 32 * i);
    if (normed) {
      float w[2], sum;
#pragma unroll
      for (int i = 0; i < 2; ++i) w[i] = c[i] + 1e-3f;
      sum = w[0] + w[1];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      float inc[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        w[i] = range * (w[i] / sum);
        inc[i] = w[i];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float t = __shfl_up_sync(0xffffffffu, inc[i], o);
          if (lane >= o) inc[i] += t;
        }
      }
      // exclusive prefix = the left neighbour's inclusive one, so bin k's upper edge is bin k+1's lower edge bit for bit
      float exc[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        exc[i] = __shfl_up_sync(0xffffffffu, inc[i], 1);
        if (lane == 0) exc[i] = 0.f;
      }
      const float half = __shfl_sync(0xffffffffu, inc[0], 31);
      exc[1] = lane == 0 ? half : exc[1] + half;
      inc[1] += half;
#pragma unroll
      for (int i = 0; i < 2; ++i) c[i] = 0.5f * ((min_d + exc[i]) + (min_d + inc[i]));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (to_unit) c[i] = (c[i] - min_d) / range;
      out[p * 64 + lane + 32 * i] = c[i];
    }
  }
}

// 8 lanes per pixel (4 pixels per warp, grid-stride), lane j owns bins 8j..8j+7 (two 16-byte loads per bilinear tap,
// nbins == 64); the Stirling log C(K-1,k) terms depend on the lane only and are computed once per thread; the
// softmax reductions are 3-step butterflies inside the 8-lane group.
__global__ void logbinom_depth_kernel(const float* __restrict__ pt, int pt_ld, const float* __restrict__ bc, int BH, int BW,
                                      int B, int H, int W, int nbins, float min_t, float max_t, float sy, float sx,
                                      float* __restrict__ depth) {
  const int lane = threadIdx.x & 31, j = lane & 7;
  const int groups = (gridDim.x * blockDim.x) >> 3;
  const int total = B * H * W;
  const float Km1 = static_cast<float>(nbins - 1);
  float logc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float n_ = Km1 + 1e-7f, k_ = static_cast<float>(8 * j + i) + 1e-7f;
    logc[i] = n_ * logf(n_) - k_ * logf(k_) - (n_ - k_) * logf(n_ - k_ + 1e-7f);
  }
  const int hw = H * W;
  const int iters = (total + groups - 1) / groups;
  int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  for (int it = 0; it < iters; ++it, p += groups) {
    const bool act = p < total;                  // keep the whole warp in the loop for the shuffles
    const int pp = act ? p : total - 1;
    const int b = pp / hw, rem = pp - b * hw;
    const int oy = rem / W, ox = rem - oy * W;
    const float4 q = __ldg(reinterpret_cast<const float4*>(pt + static_cast<size_t>(pp) * pt_ld));
    float p0 = q.x + 1e-4f, p1 = q.y + 1e-4f, t0 = q.z + 1e-4f, t1 = q.w + 1e-4f;
    float pr = __fdividef(p0, p0 + p1);
    float tt = __fdividef(t0, t0 + t1);
    tt = (max_t - min_t) * tt + min_t;
    float om = fminf(fmaxf(1.f - pr, 1e-4f), 1.f);
    pr = fminf(fmaxf(pr, 1e-4f), 1.f);
    const float inv_t = __fdividef(1.f, tt);
    const float lp = __logf(pr) * inv_t, lq = __logf(om) * inv_t;
    int y0, y1, x0, x1; float fy, fx;
    ac_coord_s(oy, BH, sy, y0, y1, fy);
    ac_coord_s(ox, BW, sx, x0, x1, fx);
    const float* base = bc + static_cast<size_t>(b) * BH * BW * nbins + 8 * j;
    const float4* r00 = reinterpret_cast<const float4*>(base + (static_cast<size_t>(y0) * BW + x0) * nbins);
    const float4* r01 = reinterpret_cast<const float4*>(base + (static_cast<size_t>(y0) * BW + x1) * nbins);
    const float4* r10 = reinterpret_cast<const float4*>(base + (static_cast<size_t>(y1) * BW + x0) * nbins);
    const float4* r11 = reinterpret_cast<const float4*>(base + (static_cast<size_t>(y1) * BW + x1) * nbins);
    const float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
    float cv[8], yv[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 a = __ldg(r00 + h), bq = __ldg(r01 + h), c = __ldg(r10 + h), d = __ldg(r11 + h);
      cv[4 * h + 0] = w00 * a.x + w01 * bq.x + w10 * c.x + w11 * d.x;
      cv[4 * h + 1] = w00 * a.y + w01 * bq.y + w10 * c.y + w11 * d.y;
      cv[4 * h + 2] = w00 * a.z + w01 * bq.z + w10 * c.z + w11 * d.z;
      cv[4 * h + 3] = w00 * a.w + w01 * bq.w + w10 * c.w + w11 * d.w;
    }
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float kf = static_cast<float>(8 * j + i);
      yv[i] = fmaf(logc[i], inv_t, fmaf(kf, lp, (Km1 - kf) * lq));
      mx = fmaxf(mx, yv[i]);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float den = 0.f, num = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float e = __expf(yv[i] - mx);
      den += e;
      num = fmaf(e, cv[i], num);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      den += __shfl_xor_sync(0xffffffffu, den, o);
      num += __shfl_xor_sync(0xffffffffu, num, o);
    }
    if (act && j == 0) depth[p] = __fdividef(num, den);
  }
}

// ------------------------------------------------------------------------------------------------ stitch
__global__ void stitch_accumulate_kernel(float* __restrict__ num, float* __restrict__ den, int CH, int CW,
                                         const float* __restrict__ tiles, int T, int th, int tw,
                                         const int* __restrict__ origins, const float* __restrict__ mask, int uh, int uw) {
  const int oh = uh > 0 ? uh : th, ow = uw > 0 ? uw : tw;
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(T) * oh * ow;
  if (idx >= total) return;
  int x = static_cast<int>(idx % ow);
  long long t2 = idx / ow;
  int y = static_cast<int>(t2 % oh);
  int t = static_cast<int>(t2 / oh);
  int sy = y, sx = x;
  if (uh > 0) {   // F.interpolate default 'nearest': src = floor(dst * in/out)
    sy = min(static_cast<int>(floorf(y * (static_cast<float>(th) / uh))), th - 1);
    sx = min(static_cast<int>(floorf(x * (static_cast<float>(tw) / uw))), tw - 1);
  }
  float d = tiles[(static_cast<long long>(t) * th + sy) * tw + sx];
  float m = mask[static_cast<long long>(y) * ow + x];
  int cy = origins[t * 2] + y, cx = origins[t * 2 + 1] + x;
  if (cy < CH && cx < CW) {
    long long o = static_cast<long long>(cy) * CW + cx;
    atomicAdd(num + o, m * d);
    atomicAdd(den + o, m);
  }
}

// Deterministic stitch: each canvas pixel sums, in tile-list order, the (mask-weighted) predictions of the tiles
// that cover it - no atomics, so the canvas is bit-identical for any micro-batch grouping and any rank count (the
// list order is the single-device order; `slot` says where tile i's prediction sits in the gathered blocks).
// tiles: n x {origin y, origin x, slot}.  base_*: canvases of a previous phase to continue from (nullable).
__global__ void stitch_gather_kernel(const float* __restrict__ preds, const int* __restrict__ tiles, int n, int th, int tw,
                                     const float* __restrict__ mask, int uh, int uw, const float* __restrict__ base_num,
                                     const float* __restrict__ base_den, int CH, int CW, float* __restrict__ num_out,
                                     float* __restrict__ den_out, float* __restrict__ avg_out) {
  extern __shared__ int s_tiles[];
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 3 * n; i += blockDim.x * blockDim.y) s_tiles[i] = tiles[i];
  __syncthreads();
  const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
  if (cx >= CW || cy >= CH) return;
  const int oh = uh > 0 ? uh : th, ow = uw > 0 ? uw : tw;
  const float ry = static_cast<float>(th) / oh, rx = static_cast<float>(tw) / ow;
  const long long o = static_cast<long long>(cy) * CW + cx;
  float num = base_num ? base_num[o] : 0.f, den = base_den ? base_den[o] : 0.f;
  for (int i = 0; i < n; ++i) {
    const int y = cy - s_tiles[3 * i], x = cx - s_tiles[3 * i + 1];
    if (static_cast<unsigned>(y) < static_cast<unsigned>(oh) && static_cast<unsigned>(x) < static_cast<unsigned>(ow)) {
      int sy = y, sx = x;
      if (uh > 0) {   // F.interpolate default 'nearest' (baseline_pretrain.py:203): src = floor(dst * in/out)
        sy = min(static_cast<int>(floorf(y * ry)), th - 1);
        sx = min(static_cast<int>(floorf(x * rx)), tw - 1);
      }
      const float d = preds[(static_cast<long long>(s_tiles[3 * i + 2]) * th + sy) * tw + sx];
      const float m = mask[static_cast<long long>(y) * ow + x];
      num += m * d;
      den += m;
    }
  }
  if (num_out) num_out[o] = num;
  if (den_out) den_out[o] = den;
  if (avg_out) avg_out[o] = num / den;
}

__global__ void stitch_finalize_kernel(const float* __restrict__ num, const float* __restrict__ den, long long n,
                                       float* __restrict__ out) {
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = num[i] / den[i];
}

// num[0] <- sum_r num[r], den[0] <- sum_r den[r] over the all-gathered per-rank canvases (fixed rank order).
__global__ void stitch_reduce_kernel(float* __restrict__ stack, int world, long long n) {
  long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= 2 * n) return;
  float s = 0.f;
  for (int r = 0; r < world; ++r) s += stack[static_cast<long long>(r) * 2 * n + i];
  stack[i] = s;
}

__global__ void stitch_resize_kernel(const float* __restrict__ num, const float* __restrict__ den, int H, int W, int OH,
                                     int OW, float* __restrict__ num_out, float* __restrict__ den_out) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(OH) * OW) return;
  int ox = static_cast<int>(idx % OW), oy = static_cast<int>(idx / OW);
  int sy = min(static_cast<int>(floorf(oy * (static_cast<float>(H) / OH))), H - 1);
  int sx = min(static_cast<int>(floorf(ox * (static_cast<float>(W) / OW))), W - 1);
  long long s = static_cast<long long>(sy) * W + sx;
  float avg = num[s] / den[s];
  int y0, y1, x0, x1; float fy, fx;
  ac_coord(oy, H, OH, y0, y1, fy);
  ac_coord(ox, W, OW, x0, x1, fx);
  float c = (1.f - fy) * ((1.f - fx) * den[static_cast<long long>(y0) * W + x0] + fx * den[static_cast<long long>(y0) * W + x1]) +
            fy * ((1.f - fx) * den[static_cast<long long>(y1) * W + x0] + fx * den[static_cast<long long>(y1) * W + x1]);
  num_out[idx] = avg * c;
  den_out[idx] = c;
}

}  // namespace pf

using namespace pf;
#define ST static_cast<cudaStream_t>(stream)

extern "C" {

int pf_layernorm(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t rows, int32_t C,
                 void* out, int32_t out_ld, void* stream) {
  if (C % 4 || x_ld % 4 || out_ld % 4 || C > 1024) return set_error("pf_layernorm: C (<= 1024) and strides must be multiples of 4");
  cudaError_t le = launch_pdl(layernorm_kernel, dim3(nblocks(rows, 8)), dim3(256), 0, ST, x, x_ld, w, b, eps, rows, C,
                              static_cast<bf16*>(out), out_ld, 0, 0, 0);
  if (le != cudaSuccess) return set_error("layernorm_kernel launch: %s", cudaGetErrorString(le));
  return check_launch("layernorm_kernel");
}

int pf_layernorm_e4m3(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t rows, int32_t C,
                      float ratio, void* out, int32_t out_ld, void* stream) {
  if (C % 4 || x_ld % 4 || out_ld % 4 || out_ld < C || C > 1024 || rows < 0 || !(ratio >= 0.f) ||
      reinterpret_cast<uintptr_t>(out) % 4)
    return set_error("pf_layernorm_e4m3: C (<= 1024) and strides must be multiples of 4, out_ld >= C, out 4-byte "
                     "aligned, ratio >= 0");
  cudaError_t le = launch_pdl(layernorm_e4m3_kernel, dim3(nblocks(rows, 8)), dim3(256), 0, ST, x, x_ld, w, b, eps, rows,
                              C, ratio, static_cast<uint8_t*>(out), out_ld);
  if (le != cudaSuccess) return set_error("layernorm_e4m3_kernel launch: %s", cudaGetErrorString(le));
  return check_launch("layernorm_e4m3_kernel");
}

int pf_layernorm_grouped(const float* x, int32_t x_ld, const float* w, const float* b, float eps, int32_t groups,
                         int32_t rows_in, int32_t skip, int32_t rows_out, int32_t C, void* out, int32_t out_ld,
                         void* stream) {
  if (C % 4 || x_ld % 4 || out_ld % 4 || C > 1024) return set_error("pf_layernorm_grouped: C (<= 1024) and strides must be multiples of 4");
  if (groups < 1 || rows_out < 1 || skip < 0 || skip + rows_out > rows_in) return set_error("pf_layernorm_grouped: bad row mapping");
  const int rows = groups * rows_out;
  cudaError_t le = launch_pdl(layernorm_kernel, dim3(nblocks(rows, 8)), dim3(256), 0, ST, x, x_ld, w, b, eps, rows, C,
                              static_cast<bf16*>(out), out_ld, rows_in, skip, rows_out);
  if (le != cudaSuccess) return set_error("layernorm_kernel launch: %s", cudaGetErrorString(le));
  return check_launch("layernorm_kernel");
}

int pf_patch_im2col(const float* img, int32_t B, int32_t H, int32_t W, void* out, int32_t ld, void* stream) {
  if (H % 14 || W % 14 || ld < 588) return set_error("pf_patch_im2col: image must be a multiple of 14, ld >= 588");
  long long total = static_cast<long long>(B) * (H / 14) * (W / 14) * ld;
  patch_im2col_kernel<<<nblocks(total, 256), 256, 0, ST>>>(img, B, H, W, static_cast<bf16*>(out), ld);
  return check_launch("patch_im2col_kernel");
}

int pf_assemble_tokens(const float* patch, const float* cls, const float* pos, int32_t B, int32_t n_patch, int32_t D,
                       float* tokens, void* stream) {
  long long total = static_cast<long long>(B) * (n_patch + 1) * D;
  assemble_tokens_kernel<<<nblocks(total, 256), 256, 0, ST>>>(patch, cls, pos, B, n_patch, D, tokens);
  return check_launch("assemble_tokens_kernel");
}

int pf_f32_to_bf16(const float* in, int64_t n, void* out, void* stream) {
  f32_to_bf16_kernel<<<nblocks(n, 256), 256, 0, ST>>>(in, n, static_cast<bf16*>(out));
  return check_launch("f32_to_bf16_kernel");
}

int pf_resize_bilinear(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, int32_t OH,
                       int32_t OW, void* out, int32_t out_ld, int32_t out_col0, void* stream) {
  if (C % 8 || in_ld % 8 || out_ld % 8 || out_col0 % 8) return set_error("pf_resize_bilinear: channel counts/strides must be multiples of 8");
  const int cg = C / 8;
  const float sy = ac_scale(H, OH), sx = ac_scale(W, OW);
  if (C % 64 == 0 && sy <= 1.0f && sx <= 1.0f && OH * OW >= 4096) {
    dim3 tgrid((OW + kRsTW - 1) / kRsTW, (OH + kRsTH - 1) / kRsTH, B);
    resize_bilinear_tiled_kernel<<<tgrid, 256, 0, ST>>>(static_cast<const bf16*>(in), H, W, in_ld, OH, OW, sy, sx,
                                                        C / 64, static_cast<bf16*>(out), out_ld, out_col0,
                                                        option(PF_OPT_RESIZE_SEPARABLE));
    return check_launch("resize_bilinear_tiled_kernel");
  }
  dim3 grid(nblocks(static_cast<long long>(OW) * cg, 256), OH, B);
  resize_bilinear_kernel<<<grid, 256, 0, ST>>>(static_cast<const bf16*>(in), H, W, cg, in_ld, OH, OW, ac_scale(H, OH),
                                               ac_scale(W, OW), static_cast<bf16*>(out), out_ld, out_col0);
  return check_launch("resize_bilinear_kernel");
}

int pf_resize_bilinear_f32(const float* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t OH, int32_t OW,
                           float* out, void* stream) {
  long long total = static_cast<long long>(B) * OH * OW * C;
  resize_bilinear_f32_kernel<<<nblocks(total, 256), 256, 0, ST>>>(in, B, H, W, C, OH, OW, out);
  return check_launch("resize_bilinear_f32_kernel");
}

int pf_roi_crop_zoom_batched(const void* feat, int32_t in_f32, int32_t h, int32_t w, int32_t C, int32_t in_ld,
                             const int32_t* tile_image, const float* boxes, int32_t T, float spatial_scale, void* out,
                             int32_t out_ld, int32_t out_col0, void* stream) {
  if (in_f32) {
    dim3 grid(nblocks(static_cast<long long>(w) * C, 256), h, T);
    roi_crop_zoom_kernel<true><<<grid, 256, 0, ST>>>(feat, h, w, C, in_ld, tile_image, boxes, spatial_scale, out, out_ld,
                                                     out_col0);
  } else {
    if (C % 8 || in_ld % 8 || out_ld % 8 || out_col0 % 8) return set_error("pf_roi_crop_zoom: channels/strides must be multiples of 8");
    dim3 grid(nblocks(static_cast<long long>(w) * (C / 8), 256), h, T);
    roi_crop_zoom_kernel<false><<<grid, 256, 0, ST>>>(feat, h, w, C / 8, in_ld, tile_image, boxes, spatial_scale, out,
                                                      out_ld, out_col0);
  }
  return check_launch("roi_crop_zoom_kernel");
}

int pf_roi_crop_zoom(const void* feat, int32_t in_f32, int32_t h, int32_t w, int32_t C, int32_t in_ld,
                     const float* boxes, int32_t T, float spatial_scale, void* out, int32_t out_ld, int32_t out_col0,
                     void* stream) {
  return pf_roi_crop_zoom_batched(feat, in_f32, h, w, C, in_ld, nullptr, boxes, T, spatial_scale, out, out_ld, out_col0, stream);
}

int pf_maxpool2(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, void* out, int32_t out_ld,
                void* stream) {
  if (C % 8 || in_ld % 8 || out_ld % 8) return set_error("pf_maxpool2: channels/strides must be multiples of 8");
  long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 8);
  maxpool2_kernel<<<nblocks(total, 256), 256, 0, ST>>>(static_cast<const bf16*>(in), B, H, W, C, in_ld,
                                                        static_cast<bf16*>(out), out_ld);
  return check_launch("maxpool2_kernel");
}

int pf_im2col_3x3_s2(const void* in, int32_t B, int32_t H, int32_t W, int32_t C, int32_t in_ld, void* out,
                     void* stream) {
  if (C % 8 || in_ld % 8) return set_error("pf_im2col_3x3_s2: channels/strides must be multiples of 8");
  long long total = static_cast<long long>(B) * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * 9 * (C / 8);
  im2col_3x3_s2_kernel<<<nblocks(total, 256), 256, 0, ST>>>(static_cast<const bf16*>(in), B, H, W, C, in_ld,
                                                             static_cast<bf16*>(out));
  return check_launch("im2col_3x3_s2_kernel");
}

int pf_crop_resize_batched(const float* img, int32_t H, int32_t W, const int32_t* origins, const int32_t* tile_image,
                           int32_t T, int32_t th, int32_t tw, int32_t ph, int32_t pw, float* out_planar, void* stream) {
  long long total = static_cast<long long>(T) * 3 * ph * pw;
  crop_resize_kernel<<<nblocks(total, 256), 256, 0, ST>>>(img, H, W, origins, tile_image, T, th, tw, ph, pw, out_planar);
  return check_launch("crop_resize_kernel");
}

int pf_crop_resize(const float* img, int32_t H, int32_t W, const int32_t* origins, int32_t T, int32_t th, int32_t tw,
                   int32_t ph, int32_t pw, float* out_planar, void* stream) {
  return pf_crop_resize_batched(img, H, W, origins, nullptr, T, th, tw, ph, pw, out_planar, stream);
}

int pf_crop_resize_multi(const pf_crop_image* images, const int32_t* origins, const int32_t* tile_image, int32_t T,
                         int32_t ph, int32_t pw, float* out_planar, void* stream) {
  if (images == nullptr || tile_image == nullptr) return set_error("pf_crop_resize_multi: images and tile_image are required");
  if (T <= 0) return 0;
  long long total = static_cast<long long>(T) * 3 * ph * pw;
  crop_resize_multi_kernel<<<nblocks(total, 256), 256, 0, ST>>>(images, origins, tile_image, T, ph, pw, out_planar);
  return check_launch("crop_resize_multi_kernel");
}

int pf_pack_unet_input(const float* coarse_depth_roi, const float* fine_depth, const float* rgb_planar, int32_t T,
                       int32_t H, int32_t W, void* out, int32_t ld, void* stream) {
  if (ld % 8) return set_error("pf_pack_unet_input: ld must be a multiple of 8");
  long long total = static_cast<long long>(T) * H * W;
  pack_unet_input_kernel<<<nblocks(total, 256), 256, 0, ST>>>(coarse_depth_roi, fine_depth, rgb_planar, T, H, W,
                                                               static_cast<bf16*>(out), ld);
  return check_launch("pack_unet_input_kernel");
}

int pf_ingest_u8(const uint8_t* img_hwc, int32_t H, int32_t W, int32_t bgr, int32_t OH, int32_t OW, float* out_planar,
                 void* stream) {
  dim3 grid(nblocks(OW, 256), OH);
  ingest_u8_kernel<<<grid, 256, 0, ST>>>(img_hwc, H, W, bgr, OH, OW, ac_scale(H, OH), ac_scale(W, OW), out_planar);
  return check_launch("ingest_u8_kernel");
}

int pf_depth_to_u16(const float* depth, int32_t H, int32_t W, int32_t OH, int32_t OW, float scale, uint16_t* out,
                    void* stream) {
  dim3 grid(nblocks(OW, 256), OH);
  depth_to_u16_kernel<<<grid, 256, 0, ST>>>(depth, H, W, OH, OW, scale, out);
  return check_launch("depth_to_u16_kernel");
}

int pf_g2l_embed_batched(const void* feat, int32_t feat_ld, const float* ape, int32_t B, int32_t n, int32_t C, float* x,
                         void* stream) {
  if (B < 1) return set_error("pf_g2l_embed: B must be >= 1");
  g2l_embed_kernel<<<nblocks(static_cast<long long>(B) * n * C, 256), 256, 0, ST>>>(static_cast<const bf16*>(feat),
                                                                                     feat_ld, ape, B, n, C, x);
  return check_launch("g2l_embed_kernel");
}

int pf_g2l_embed(const void* feat, int32_t feat_ld, const float* ape, int32_t n, int32_t C, float* x, void* stream) {
  return pf_g2l_embed_batched(feat, feat_ld, ape, 1, n, C, x, stream);
}

int pf_swin_norm_pad_batched(const float* x, const float* w, const float* b, float eps, int32_t B, int32_t H, int32_t W,
                             int32_t Hp, int32_t Wp, int32_t C, void* out, void* stream) {
  if (C % 4 || C > 1024) return set_error("pf_swin_norm_pad: C (<= 1024) must be a multiple of 4");
  if (B < 1) return set_error("pf_swin_norm_pad: B must be >= 1");
  swin_norm_pad_kernel<<<nblocks(static_cast<long long>(B) * Hp * Wp, 8), 256, 0, ST>>>(x, w, b, eps, B, H, W, Hp, Wp, C,
                                                                                         static_cast<bf16*>(out));
  return check_launch("swin_norm_pad_kernel");
}

int pf_swin_norm_pad(const float* x, const float* w, const float* b, float eps, int32_t H, int32_t W, int32_t Hp,
                     int32_t Wp, int32_t C, void* out, void* stream) {
  return pf_swin_norm_pad_batched(x, w, b, eps, 1, H, W, Hp, Wp, C, out, stream);
}

int pf_window_attention(const void* qkv, const float* bias_table, int32_t Hp, int32_t Wp, int32_t C, int32_t heads,
                        int32_t shift, void* out, void* stream) {
  return pf_window_attention_batched(qkv, bias_table, 1, Hp, Wp, C, heads, shift, out, stream);
}

int pf_window_attention_batched(const void* qkv, const float* bias_table, int32_t B, int32_t Hp, int32_t Wp, int32_t C,
                                int32_t heads, int32_t shift, void* out, void* stream) {
  if (Hp % 12 || Wp % 12) return set_error("pf_window_attention: padded grid must be a multiple of the 12x12 window");
  if (B < 1 || B > 65535) return set_error("pf_window_attention: B must be in [1, 65535]");
  dim3 grid((Hp / 12) * (Wp / 12), heads, B);
  const bf16* q = static_cast<const bf16*>(qkv);
  bf16* o = static_cast<bf16*>(out);
  switch (C / heads) {
    case 2: window_attention_kernel<2><<<grid, 160, 0, ST>>>(q, bias_table, Hp, Wp, C, heads, shift, o); break;
    case 4: window_attention_kernel<4><<<grid, 160, 0, ST>>>(q, bias_table, Hp, Wp, C, heads, shift, o); break;
    case 8: window_attention_kernel<8><<<grid, 160, 0, ST>>>(q, bias_table, Hp, Wp, C, heads, shift, o); break;
    case 16: window_attention_kernel<16><<<grid, 160, 0, ST>>>(q, bias_table, Hp, Wp, C, heads, shift, o); break;
    case 32: window_attention_kernel<32><<<grid, 160, 0, ST>>>(q, bias_table, Hp, Wp, C, heads, shift, o); break;
    default: return set_error("pf_window_attention: unsupported head_dim %d", C / heads);
  }
  return check_launch("window_attention_kernel");
}

int pf_swin_residual_crop_batched(float* x, const float* y, int32_t B, int32_t H, int32_t W, int32_t Hp, int32_t Wp,
                                  int32_t C, void* stream) {
  if (B < 1) return set_error("pf_swin_residual_crop: B must be >= 1");
  swin_residual_crop_kernel<<<nblocks(static_cast<long long>(B) * H * W * C, 256), 256, 0, ST>>>(x, y, B, H, W, Hp, Wp, C);
  return check_launch("swin_residual_crop_kernel");
}

int pf_swin_residual_crop(float* x, const float* y, int32_t H, int32_t W, int32_t Wp, int32_t C, void* stream) {
  // one grid: its height never enters the address arithmetic
  return pf_swin_residual_crop_batched(x, y, 1, H, W, H, Wp, C, stream);
}

int pf_add_upsampled(const void* a, int32_t B, int32_t H, int32_t W, int32_t C, const void* prev, int32_t PH, int32_t PW,
                     void* out, void* stream) {
  if (C % 8) return set_error("pf_add_upsampled: C must be a multiple of 8");
  long long total = static_cast<long long>(B) * H * W * (C / 8);
  add_upsampled_kernel<<<nblocks(total, 256), 256, 0, ST>>>(static_cast<const bf16*>(a), B, H, W, C,
                                                             static_cast<const bf16*>(prev), PH, PW, static_cast<bf16*>(out));
  return check_launch("add_upsampled_kernel");
}

int pf_attractor(const float* A, int32_t A_ld, int32_t nA, const float* b_prev, int32_t PH, int32_t PW, int32_t B,
                 int32_t H, int32_t W, int32_t nbins, int32_t flags, float* b_out, void* stream) {
  if (nbins != 64 || nA > 32) return set_error("pf_attractor: n_bins must be 64 and n_attractors <= 32");
  if (flags & ~3) return set_error("pf_attractor: unknown flags %d", flags);
  const int kind_mean = flags & PF_ATTRACTOR_MEAN, type_exp = (flags & PF_ATTRACTOR_EXP) ? 1 : 0;
  long long warps_needed = static_cast<long long>(B) * H * W;
  const long long cap = 8LL * sm_count();   // eight 256-thread blocks per SM, grid-stride beyond
  unsigned blocks = static_cast<unsigned>(warps_needed < cap * 8 ? (warps_needed + 7) / 8 : cap);
  attractor_kernel<<<blocks, 256, 0, ST>>>(A, A_ld, nA, b_prev, PH, PW, B, H, W, nbins, kind_mean, type_exp,
                                           ac_scale(PH, H), ac_scale(PW, W), b_out);
  return check_launch("attractor_kernel");
}

int pf_attractor_normed(const float* A, int32_t A_ld, int32_t nA, const float* b_prev, int32_t PH, int32_t PW, int32_t B,
                        int32_t H, int32_t W, int32_t nbins, int32_t flags, float min_depth, float max_depth, float* b_out,
                        float* centers, void* stream) {
  if (nbins != 64 || nA > 32) return set_error("pf_attractor_normed: n_bins must be 64 and n_attractors <= 32");
  if (flags & ~3) return set_error("pf_attractor_normed: unknown flags %d", flags);
  if (!(max_depth > min_depth)) return set_error("pf_attractor_normed: max_depth must exceed min_depth");
  const int kind_mean = flags & PF_ATTRACTOR_MEAN, type_exp = (flags & PF_ATTRACTOR_EXP) ? 1 : 0;
  long long warps_needed = static_cast<long long>(B) * H * W;
  const long long cap = 8LL * sm_count();
  unsigned blocks = static_cast<unsigned>(warps_needed < cap * 8 ? (warps_needed + 7) / 8 : cap);
  attractor_normed_kernel<<<blocks, 256, 0, ST>>>(A, A_ld, nA, b_prev, PH, PW, B, H, W, nbins, kind_mean, type_exp,
                                                  ac_scale(PH, H), ac_scale(PW, W), b_out, min_depth, max_depth, centers);
  return check_launch("attractor_normed_kernel");
}

int pf_seed_bins(const float* S, int32_t S_ld, int64_t pixels, int32_t nbins, int32_t flags, float min_depth,
                 float max_depth, float* out, void* stream) {
  if (nbins != 64) return set_error("pf_seed_bins: n_bins must be 64");
  if (flags & ~3) return set_error("pf_seed_bins: unknown flags %d", flags);
  if (S_ld < 64) return set_error("pf_seed_bins: S_ld must be >= 64");
  if (!(max_depth > min_depth)) return set_error("pf_seed_bins: max_depth must exceed min_depth");
  const long long cap = 8LL * sm_count();
  unsigned blocks = static_cast<unsigned>(pixels < cap * 8 ? (pixels + 7) / 8 : cap);
  if (blocks == 0) return 0;
  seed_bins_kernel<<<blocks, 256, 0, ST>>>(S, S_ld, pixels, flags & PF_SEED_NORMED, (flags & PF_SEED_TO_UNIT) ? 1 : 0,
                                           min_depth, max_depth, out);
  return check_launch("seed_bins_kernel");
}

int pf_logbinom_depth(const float* pt, int32_t pt_ld, const float* b_centers, int32_t BH, int32_t BW, int32_t B,
                      int32_t H, int32_t W, int32_t nbins, float min_temp, float max_temp, float* depth, void* stream) {
  if (nbins != 64) return set_error("pf_logbinom_depth: n_bins must be 64");
  if (pt_ld % 4) return set_error("pf_logbinom_depth: pt_ld must be a multiple of 4");
  logbinom_depth_kernel<<<8 * sm_count(), 256, 0, ST>>>(pt, pt_ld, b_centers, BH, BW, B, H, W, nbins, min_temp, max_temp,
                                                 ac_scale(BH, H), ac_scale(BW, W), depth);
  return check_launch("logbinom_depth_kernel");
}

int pf_stitch_accumulate(float* num, float* den, int32_t CH, int32_t CW, const float* tiles, int32_t T, int32_t th,
                         int32_t tw, const int32_t* origins, const float* mask, int32_t up_h, int32_t up_w,
                         void* stream) {
  long long total = static_cast<long long>(T) * (up_h > 0 ? up_h : th) * (up_w > 0 ? up_w : tw);
  stitch_accumulate_kernel<<<nblocks(total, 256), 256, 0, ST>>>(num, den, CH, CW, tiles, T, th, tw, origins, mask, up_h,
                                                                 up_w);
  return check_launch("stitch_accumulate_kernel");
}

int pf_stitch_gather(const float* preds, const int32_t* tiles, int32_t n, int32_t th, int32_t tw, const float* mask,
                     int32_t up_h, int32_t up_w, const float* base_num, const float* base_den, int32_t CH, int32_t CW,
                     float* num_out, float* den_out, float* avg_out, void* stream) {
  if (n < 0 || n > 4096) return set_error("pf_stitch_gather: n %d out of range (0..4096)", n);
  if ((up_h > 0) != (up_w > 0)) return set_error("pf_stitch_gather: up_h/up_w must both be set or both be 0");
  dim3 block(32, 8), grid((CW + 31) / 32, (CH + 7) / 8);
  stitch_gather_kernel<<<grid, block, static_cast<size_t>(n) * 12, ST>>>(preds, tiles, n, th, tw, mask, up_h, up_w, base_num,
                                                                       base_den, CH, CW, num_out, den_out, avg_out);
  return check_launch("stitch_gather_kernel");
}

int pf_stitch_finalize(const float* num, const float* den, int64_t n, float* out, void* stream) {
  stitch_finalize_kernel<<<nblocks(n, 256), 256, 0, ST>>>(num, den, n, out);
  return check_launch("stitch_finalize_kernel");
}

int pf_stitch_reduce(float* stack, int32_t world, int64_t n, void* stream) {
  stitch_reduce_kernel<<<nblocks(2 * n, 256), 256, 0, ST>>>(stack, world, n);
  return check_launch("stitch_reduce_kernel");
}

int pf_stitch_resize(const float* num, const float* den, int32_t H, int32_t W, int32_t OH, int32_t OW, float* num_out,
                     float* den_out, void* stream) {
  stitch_resize_kernel<<<nblocks(static_cast<long long>(OH) * OW, 256), 256, 0, ST>>>(num, den, H, W, OH, OW, num_out,
                                                                                       den_out);
  return check_launch("stitch_resize_kernel");
}

}  // extern "C"
