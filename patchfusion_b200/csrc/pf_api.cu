// C-ABI glue: error reporting, TMA tensor-map construction (+cache), pf_gemm host wrapper, weight packing.
#include <cuda_bf16.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "pf_kernels.h"

namespace pf {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
// ---- per-launch profiler (bench.py's roofline pass): one CUDA event after every launch of this library on the
// profiled stream; the duration of launch i is event[i] - event[i-1] (launches are back to back on one stream).
struct ProfRec { const char* name; double flops; char label[80]; cudaEvent_t ev; };
static std::vector<ProfRec> g_prof;
static bool g_prof_on = false;
static cudaStream_t g_prof_stream = nullptr;
static cudaEvent_t g_prof_ev0 = nullptr;
static thread_local double g_next_flops = 0.0;
static thread_local char g_next_label[80] = "";

void note_work(double flops, const char* fmt, ...) {
  if (!g_prof_on) return;
  g_next_flops = flops;
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_next_label, sizeof(g_next_label), fmt, ap);
  va_end(ap);
}
void count_launch(const char* name) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (g_prof_on) {
    ProfRec r;
    r.name = name; r.flops = g_next_flops;
    snprintf(r.label, sizeof(r.label), "%s", g_next_label[0] ? g_next_label : name);
    cudaEventCreate(&r.ev);
    cudaEventRecord(r.ev, g_prof_stream);
    g_prof.push_back(r);
    g_next_flops = 0.0; g_next_label[0] = 0;
  }
}
// tuning switches: -1 = not read yet (first use reads the environment variable of the same name)
static std::atomic<int> g_opt[6] = {{-1}, {-1}, {-1}, {-1}, {-1}, {-1}};
int option(int which) {
  static const char* names[6] = {"PF_OPT_TMA_EPILOGUE", "PF_OPT_HALO_MULTICAST", "PF_OPT_GEMM_MULTICAST", "PF_OPT_FUSED_RESAMPLE", "PF_OPT_PDL", "PF_OPT_RESIZE_SEPARABLE"};
  static const int defaults[6] = {1, 1, 1, 0, 0, 0};
  if (which < 0 || which > 5) return 0;
  int v = g_opt[which].load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv(names[which]);
    if (!e && which == PF_OPT_PDL) e = getenv("PF_B200_PDL");
    v = e ? atoi(e) : defaults[which];
    g_opt[which].store(v, std::memory_order_relaxed);
  }
  return v;
}
bool pdl_enabled() {
  // opt-in (PF_OPT_PDL / legacy PF_B200_PDL=1): every GEMM kernel is a 1-CTA/SM persistent kernel, so a dependent
  // cannot become resident before its predecessor's CTAs retire
  return option(PF_OPT_PDL) != 0;
}
int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch: %s", what, cudaGetErrorString(e));
  count_launch(what);
  return 0;
}

// ---------------------------------------------------------------------------------------------- tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct MapKey {
  uint64_t v[12];
  bool operator==(const MapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (int i = 0; i < 12; ++i) { h ^= k.v[i]; h *= 1099511628211ull; }
    return static_cast<size_t>(h);
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static std::mutex g_maps_mu;

static int encode(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.v[0] = reinterpret_cast<uint64_t>(ptr);
  key.v[1] = static_cast<uint64_t>(rank) | (static_cast<uint64_t>(dt) << 8);
  for (int i = 0; i < rank; ++i) {
    key.v[2 + i] = dims[i];
    key.v[6 + i] = (i + 1 < rank ? strides_bytes[i] : 0) ^ (static_cast<uint64_t>(box[i]) << 48);
  }
  {
    std::lock_guard<std::mutex> g(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return 0; }
  }
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if (reinterpret_cast<uintptr_t>(ptr) & 15) return set_error("tensor map: base pointer not 16-byte aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] & 15) return set_error("tensor map: stride %d (%llu B) not a multiple of 16", i, (unsigned long long)gstr[i]);
  }
  // rows of 128 bytes: SWIZZLE_128B (every operand tile and most staging tiles); rows of 64 bytes (the 32-column bf16
  // staging tiles of the halo conv epilogue, the e4m3 operand tiles of its FP8 instantiation): SWIZZLE_64B.  The box is part of the cache key, so the mode is too.
  const uint32_t row_bytes = box[0] * (dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : (dt == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2));
  const CUtensorMapSwizzle swz = row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = fn(out, dt, rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u", (int)r, rank,
                     (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                     (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
                     rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
  }
  std::lock_guard<std::mutex> g(g_maps_mu);
  if (g_maps.size() > 65536) g_maps.clear();      // callers with ever-changing pointers: bound the cache
  g_maps.emplace(key, *out);
  return 0;
}

int tmap_2d_bf16(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_cols,
                 uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t str[1] = {ld * 2};
  uint32_t box[2] = {box_cols, box_rows};
  return encode(out, ptr, 2, dims, str, box);
}
int tmap_2d_f32(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_cols,
                uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t str[1] = {ld * 4};
  uint32_t box[2] = {box_cols, box_rows};
  return encode(out, ptr, 2, dims, str, box, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
}
int tmap_3d_bf16(CUtensorMap* out, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t ld1, uint64_t ld2,
                 uint32_t b0, uint32_t b1, uint32_t b2) {
  uint64_t dims[3] = {d0, d1, d2};
  uint64_t str[2] = {ld1 * 2, ld2 * 2};
  uint32_t box[3] = {b0, b1, b2};
  return encode(out, ptr, 3, dims, str, box);
}
int tmap_4d_nhwc_bf16(CUtensorMap* out, const void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint64_t ld,
                      uint32_t box_c, uint32_t box_w, uint32_t box_h) {
  uint64_t dims[4] = {C, W, H, N};
  uint64_t str[3] = {ld * 2, ld * 2 * W, ld * 2 * W * H};
  uint32_t box[4] = {box_c, box_w, box_h, 1};
  return encode(out, ptr, 4, dims, str, box);
}

int tmap_2d_u8(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_cols,
               uint32_t box_rows) {
  uint64_t dims[2] = {cols, rows};
  uint64_t str[1] = {ld};
  uint32_t box[2] = {box_cols, box_rows};
  return encode(out, ptr, 2, dims, str, box, CU_TENSOR_MAP_DATA_TYPE_UINT8);
}
int tmap_4d_nhwc_u8(CUtensorMap* out, const void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint64_t ld,
                    uint32_t box_c, uint32_t box_w, uint32_t box_h) {
  uint64_t dims[4] = {C, W, H, N};
  uint64_t str[3] = {ld, ld * W, ld * W * H};
  uint32_t box[4] = {box_c, box_w, box_h, 1};
  return encode(out, ptr, 4, dims, str, box, CU_TENSOR_MAP_DATA_TYPE_UINT8);
}

// ---------------------------------------------------------------------------------------------- weight packing
__global__ void pack_weight_kernel(const float* __restrict__ w, int N, int N_pad, int num_src, int c0, int c1, int c2,
                                   int taps, const float* __restrict__ scale, __nv_bfloat16* __restrict__ dst,
                                   int Ktot) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  long long total = static_cast<long long>(N_pad) * Ktot;
  if (idx >= total) return;
  int n = static_cast<int>(idx / Ktot);
  int k = static_cast<int>(idx - static_cast<long long>(n) * Ktot);
  int cs[3] = {c0, c1, c2};
  int ctot = c0 + (num_src > 1 ? c1 : 0) + (num_src > 2 ? c2 : 0);
  float v = 0.0f;
  int cbase = 0, kbase = 0;
  for (int s = 0; s < num_src; ++s) {
    int cp = (cs[s] + 63) / 64 * 64;
    int seg = taps * cp;
    if (k < kbase + seg) {
      int kk = k - kbase;
      int tap = kk / cp, c = kk - tap * cp;
      if (n < N && c < cs[s]) {
        // PyTorch layout [N][Ctot][kh][kw], tap = ky*3+kx
        v = w[(static_cast<long long>(n) * ctot + cbase + c) * taps + tap];
        if (scale) v *= scale[n];
      }
      break;
    }
    kbase += seg;
    cbase += cs[s];
  }
  dst[idx] = __float2bfloat16(v);
}

__global__ void pack_convT_kernel(const float* __restrict__ w, int Cin, int Cout, int k, __nv_bfloat16* __restrict__ dst,
                                  int Kp) {
  long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  int Cp = (Cout + 31) / 32 * 32;
  long long total = static_cast<long long>(k) * k * Cp * Kp;
  if (idx >= total) return;
  int row = static_cast<int>(idx / Kp);
  int ci = static_cast<int>(idx - static_cast<long long>(row) * Kp);
  int tap = row / Cp, co = row - tap * Cp;
  float v = 0.0f;
  if (ci < Cin && co < Cout) v = w[(static_cast<long long>(ci) * Cout + co) * k * k + tap];   // [Cin][Cout][ky][kx]
  dst[idx] = __float2bfloat16(v);
}

// ---------------------------------------------------------------------------------------------- E4M3 quantization
// The arithmetic pf_pack_weight_e4m3 / pf_quantize_e4m3_tiles document in pf_b200.h, in IEEE fp32 with no contraction.
// e4m3_rn: cvt.rn.satfinite (round to nearest even; |v| <= 448 by construction, NaN -> NaN)
__device__ __forceinline__ uint32_t e4m3x2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// max of |x| that propagates NaN (fmaxf would drop it)
__device__ __forceinline__ float nanmax(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }
__device__ __forceinline__ float e4m3_ratio(float amax) { return amax == 0.f ? 0.f : __fdiv_rn(448.f, amax); }

__device__ __forceinline__ float block_nanmax(float m) {
  __shared__ float red[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = nanmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = nanmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) red[0] = m;
  }
  __syncthreads();
  m = red[0];
  __syncthreads();
  return m;
}

// one block per panel row: amax of the BN-folded fp32 row, then the row's Ktot bytes in pack_weight_kernel's K order
__global__ void pack_weight_e4m3_kernel(const float* __restrict__ w, int N, int num_src, int c0, int c1, int c2, int taps,
                                        const float* __restrict__ scale, uint8_t* __restrict__ dst, float* __restrict__ s_w,
                                        int Ktot) {
  const int n = blockIdx.x;
  const int cs[3] = {c0, c1, c2};
  const int ctot = c0 + (num_src > 1 ? c1 : 0) + (num_src > 2 ? c2 : 0);
  const long long row = static_cast<long long>(ctot) * taps;
  float m = 0.f;
  if (n < N) {
    const float sc = scale ? scale[n] : 1.f;
    for (long long i = threadIdx.x; i < row; i += blockDim.x) {
      const float v = scale ? __fmul_rn(w[n * row + i], sc) : w[n * row + i];
      m = nanmax(m, fabsf(v));
    }
  }
  const float amax = block_nanmax(m);
  const float r = e4m3_ratio(amax);
  if (n < N && threadIdx.x == 0) s_w[n] = __fdiv_rn(amax, 448.f);
  for (int k = 2 * threadIdx.x; k < Ktot; k += 2 * blockDim.x) {
    float v[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      int cbase = 0, kbase = 0;
      for (int s = 0; s < num_src; ++s) {
        const int cp = (cs[s] + 63) / 64 * 64, seg = taps * cp;
        if (k + e < kbase + seg) {
          const int kk = k + e - kbase, tap = kk / cp, c = kk - tap * cp;
          if (n < N && c < cs[s]) {
            float x = w[(static_cast<long long>(n) * ctot + cbase + c) * taps + tap];
            if (scale) x = __fmul_rn(x, scale[n]);
            v[e] = __fmul_rn(x, r);
          }
          break;
        }
        kbase += seg;
        cbase += cs[s];
      }
    }
    *reinterpret_cast<uint16_t*>(dst + static_cast<long long>(n) * Ktot + k) = static_cast<uint16_t>(e4m3x2(v[0], v[1]));
  }
}

// Activation sources of one conv: their bf16 maps, logical channels, row pitches, and where each 64-padded segment
// starts in the e4m3 map
struct QuantSrc {
  const __nv_bfloat16* p[3];
  int c[3], ld[3], koff[3];
  int ns, kc;        // sources, channels of the e4m3 map
};
constexpr int kQuantParts = PF_QUANT_PARTS;
static_assert(kQuantParts == 32, "quant_write_kernel reduces the partial maxima with one warp");

// launch 1: partial[t][b] = NaN-propagating max |x| over block b's share of tile t's pixels and logical channels
__global__ void quant_amax_kernel(QuantSrc q, long long hw, float* __restrict__ partial) {
  const int t = blockIdx.y;
  int gs[3], g = 0;                                        // 8-channel groups per pixel, per source and in all
  for (int s = 0; s < q.ns; ++s) { gs[s] = (q.c[s] + 7) / 8; g += gs[s]; }
  const long long items = hw * g;
  float m = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long px = i / g;
    int j = static_cast<int>(i - px * g), s = 0;
    while (j >= gs[s]) { j -= gs[s]; ++s; }
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(q.p[s] + (t * hw + px) * q.ld[s] + 8 * j));
    const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (8 * j + e < q.c[s]) {
        const float x = __uint_as_float(e & 1 ? (wv[e >> 1] & 0xffff0000u) : (wv[e >> 1] << 16));
        m = nanmax(m, fabsf(x));
      }
    }
  }
  m = block_nanmax(m);
  if (threadIdx.x == 0) partial[t * kQuantParts + blockIdx.x] = m;
}

// launch 2: amax_t from the partials (every block of the tile reduces the same values: identical result), s_a[t], and
// the e4m3 map [T, H, W, kc]: 8 output channels per thread, zeros in the pad channels of each segment
__global__ void quant_write_kernel(QuantSrc q, long long hw, const float* __restrict__ partial, uint8_t* __restrict__ out,
                                   float* __restrict__ s_a) {
  const int t = blockIdx.y;
  __shared__ float s_amax;
  if (threadIdx.x < 32) {
    float m = nanmax(partial[t * kQuantParts + threadIdx.x], 0.f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = nanmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) s_amax = m;
  }
  __syncthreads();
  const float amax = s_amax;
  const float r = e4m3_ratio(amax);
  if (blockIdx.x == 0 && threadIdx.x == 0) s_a[t] = __fdiv_rn(amax, 448.f);
  const int g = q.kc / 8;
  const long long items = hw * g;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long px = i / g;
    const int k = 8 * static_cast<int>(i - px * g);
    int s = q.ns - 1;
    while (s > 0 && k < q.koff[s]) --s;
    const int c = k - q.koff[s];
    uint32_t lo = 0, hi = 0;
    if (c < q.c[s]) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(q.p[s] + (t * hw + px) * q.ld[s] + c));
      const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float x = __uint_as_float(e & 1 ? (wv[e >> 1] & 0xffff0000u) : (wv[e >> 1] << 16));
        v[e] = c + e < q.c[s] ? __fmul_rn(x, r) : 0.f;
      }
      lo = e4m3x2(v[0], v[1]) | (e4m3x2(v[2], v[3]) << 16);
      hi = e4m3x2(v[4], v[5]) | (e4m3x2(v[6], v[7]) << 16);
    }
    *reinterpret_cast<uint2*>(out + (t * hw + px) * q.kc + k) = make_uint2(lo, hi);
  }
}

// pf_quantize_e4m3_static: quant_write_kernel's map at one ratio for every tile (e4m3x2's cvt.rn.satfinite saturates
// |v * r| > 448 to +-448); one pass over the sources, 8 output channels per thread
__global__ void quant_static_kernel(QuantSrc q, long long pixels, float r, uint8_t* __restrict__ out) {
  const int g = q.kc / 8;
  const long long items = pixels * g;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < items;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long px = i / g;
    const int k = 8 * static_cast<int>(i - px * g);
    int s = q.ns - 1;
    while (s > 0 && k < q.koff[s]) --s;
    const int c = k - q.koff[s];
    uint32_t lo = 0, hi = 0;
    if (c < q.c[s]) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(q.p[s] + px * q.ld[s] + c));
      const uint32_t wv[4] = {u.x, u.y, u.z, u.w};
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float x = __uint_as_float(e & 1 ? (wv[e >> 1] & 0xffff0000u) : (wv[e >> 1] << 16));
        v[e] = c + e < q.c[s] ? __fmul_rn(x, r) : 0.f;
      }
      lo = e4m3x2(v[0], v[1]) | (e4m3x2(v[2], v[3]) << 16);
      hi = e4m3x2(v[4], v[5]) | (e4m3x2(v[6], v[7]) << 16);
    }
    *reinterpret_cast<uint2*>(out + px * q.kc + k) = make_uint2(lo, hi);
  }
}

}  // namespace pf

using namespace pf;

extern "C" {

const char* pf_last_error(void) { return g_err; }
int pf_version(void) { return 100; }
long long pf_launch_count(void) { return g_launches.load(); }

int pf_set_option(int32_t which, int32_t value) {
  if (which < 0 || which > 5) return set_error("pf_set_option: unknown option %d", which);
  g_opt[which].store(value < 0 ? 0 : value, std::memory_order_relaxed);
  return 0;
}

int pf_profile_start(void* stream) {
  for (auto& r : g_prof) cudaEventDestroy(r.ev);
  g_prof.clear();
  if (g_prof_ev0) cudaEventDestroy(g_prof_ev0);
  g_prof_stream = static_cast<cudaStream_t>(stream);
  cudaEventCreate(&g_prof_ev0);
  cudaEventRecord(g_prof_ev0, g_prof_stream);
  g_prof_on = true;
  return 0;
}
int pf_profile_stop(void) {
  g_prof_on = false;
  if (!g_prof.empty()) cudaEventSynchronize(g_prof.back().ev);
  return static_cast<int>(g_prof.size());
}
int pf_profile_get(int32_t i, const char** name, const char** label, double* flops, float* ms) {
  if (i < 0 || i >= static_cast<int>(g_prof.size())) return set_error("pf_profile_get: index %d out of range", i);
  const ProfRec& r = g_prof[i];
  *name = r.name; *label = r.label; *flops = r.flops;
  cudaError_t e = cudaEventElapsedTime(ms, i == 0 ? g_prof_ev0 : g_prof[i - 1].ev, r.ev);
  if (e != cudaSuccess) return set_error("cudaEventElapsedTime: %s", cudaGetErrorString(e));
  return 0;
}

int pf_pack_weight(const float* w, int32_t N, int32_t N_pad, int32_t num_src, const int32_t* src_c, int32_t taps,
                   const float* scale, void* dst, void* stream) {
  if (num_src < 1 || num_src > 3 || (taps != 1 && taps != 9)) return set_error("pf_pack_weight: bad arguments");
  int c[3] = {src_c[0], num_src > 1 ? src_c[1] : 0, num_src > 2 ? src_c[2] : 0};
  int Ktot = 0;
  for (int s = 0; s < num_src; ++s) Ktot += taps * ((c[s] + 63) / 64 * 64);
  long long total = static_cast<long long>(N_pad) * Ktot;
  int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  pack_weight_kernel<<<static_cast<unsigned>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      w, N, N_pad, num_src, c[0], c[1], c[2], taps, scale, static_cast<__nv_bfloat16*>(dst), Ktot);
  return check_launch("pack_weight_kernel");
}

int pf_pack_weight_e4m3(const float* w, int32_t N, int32_t N_pad, int32_t num_src, const int32_t* src_c, int32_t taps,
                        const float* scale, void* dst, float* s_w, void* stream) {
  if (num_src < 1 || num_src > 3 || (taps != 1 && taps != 9) || N < 1 || N_pad < N || !w || !dst || !s_w)
    return set_error("pf_pack_weight_e4m3: bad arguments");
  int c[3] = {src_c[0], num_src > 1 ? src_c[1] : 0, num_src > 2 ? src_c[2] : 0};
  int Ktot = 0;
  for (int s = 0; s < num_src; ++s) Ktot += taps * ((c[s] + 63) / 64 * 64);
  pack_weight_e4m3_kernel<<<N_pad, 256, 0, static_cast<cudaStream_t>(stream)>>>(w, N, num_src, c[0], c[1], c[2], taps,
                                                                                 scale, static_cast<uint8_t*>(dst), s_w, Ktot);
  return check_launch("pack_weight_e4m3_kernel");
}

int pf_quantize_e4m3_tiles(int32_t num_src, const void* const* src, const int32_t* src_c, const int32_t* src_ld,
                           int32_t T, int32_t H, int32_t W, float* partial, void* out, float* s_a, void* stream) {
  if (num_src < 1 || num_src > 3 || !src || !src_c || !src_ld || T < 1 || H < 1 || W < 1 || !partial || !out || !s_a)
    return set_error("pf_quantize_e4m3_tiles: bad arguments");
  QuantSrc q;
  memset(&q, 0, sizeof(q));
  q.ns = num_src;
  for (int s = 0; s < num_src; ++s) {
    q.p[s] = static_cast<const __nv_bfloat16*>(src[s]);
    q.c[s] = src_c[s]; q.ld[s] = src_ld[s]; q.koff[s] = q.kc;
    if (!src[s] || src_c[s] < 1 || src_ld[s] < (src_c[s] + 7) / 8 * 8 || src_ld[s] % 8 || reinterpret_cast<uintptr_t>(src[s]) & 15)
      return set_error("pf_quantize_e4m3_tiles: source %d: channels %d, ld %d (a multiple of 8 covering them), 16-byte aligned",
                       s, src_c[s], src_ld[s]);
    q.kc += (src_c[s] + 63) / 64 * 64;
  }
  if (reinterpret_cast<uintptr_t>(out) & 7) return set_error("pf_quantize_e4m3_tiles: output not 8-byte aligned");
  const long long hw = static_cast<long long>(H) * W;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  note_work(0.0, "amax e4m3 T%d %dx%d K%d", T, H, W, q.kc);
  quant_amax_kernel<<<dim3(kQuantParts, T), 256, 0, st>>>(q, hw, partial);
  if (int rc = check_launch("quant_amax_kernel")) return rc;
  // enough blocks to fill the GPU whatever T is
  const long long items = hw * (q.kc / 8);
  long long bx = (items + 255) / 256;
  const long long cap = (4LL * sm_count() + T - 1) / T;
  if (bx > cap) bx = cap < 1 ? 1 : cap;
  note_work(0.0, "quantize e4m3 T%d %dx%d K%d", T, H, W, q.kc);
  quant_write_kernel<<<dim3(static_cast<unsigned>(bx), T), 256, 0, st>>>(q, hw, partial, static_cast<uint8_t*>(out), s_a);
  return check_launch("quant_write_kernel");
}

int pf_quantize_e4m3_static(int32_t num_src, const void* const* src, const int32_t* src_c, const int32_t* src_ld,
                            int32_t T, int32_t H, int32_t W, float ratio, void* out, void* stream) {
  if (num_src < 1 || num_src > 3 || !src || !src_c || !src_ld || T < 1 || H < 1 || W < 1 || !out || !(ratio >= 0.f))
    return set_error("pf_quantize_e4m3_static: bad arguments");
  QuantSrc q;
  memset(&q, 0, sizeof(q));
  q.ns = num_src;
  for (int s = 0; s < num_src; ++s) {
    q.p[s] = static_cast<const __nv_bfloat16*>(src[s]);
    q.c[s] = src_c[s]; q.ld[s] = src_ld[s]; q.koff[s] = q.kc;
    if (!src[s] || src_c[s] < 1 || src_ld[s] < (src_c[s] + 7) / 8 * 8 || src_ld[s] % 8 || reinterpret_cast<uintptr_t>(src[s]) & 15)
      return set_error("pf_quantize_e4m3_static: source %d: channels %d, ld %d (a multiple of 8 covering them), 16-byte aligned",
                       s, src_c[s], src_ld[s]);
    q.kc += (src_c[s] + 63) / 64 * 64;
  }
  if (reinterpret_cast<uintptr_t>(out) & 7) return set_error("pf_quantize_e4m3_static: output not 8-byte aligned");
  const long long pixels = static_cast<long long>(T) * H * W;
  const long long items = pixels * (q.kc / 8);
  long long bx = (items + 255) / 256;
  const long long cap = 8LL * sm_count();
  if (bx > cap) bx = cap;
  note_work(0.0, "quantize e4m3 static T%d %dx%d K%d", T, H, W, q.kc);
  quant_static_kernel<<<static_cast<unsigned>(bx), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      q, pixels, ratio, static_cast<uint8_t*>(out));
  return check_launch("quant_static_kernel");
}

int pf_pack_weight_convT(const float* w, int32_t Cin, int32_t Cout, int32_t k, void* dst, void* stream) {
  int Kp = (Cin + 63) / 64 * 64;
  long long total = static_cast<long long>(k) * k * ((Cout + 31) / 32 * 32) * Kp;
  int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  pack_convT_kernel<<<static_cast<unsigned>(blocks), threads, 0, static_cast<cudaStream_t>(stream)>>>(
      w, Cin, Cout, k, static_cast<__nv_bfloat16*>(dst), Kp);
  return check_launch("pack_convT_kernel");
}

static void choose_tile(int H, int W, int* bh, int* bw) {
  const int cand[6][2] = {{8, 16}, {4, 32}, {16, 8}, {2, 64}, {1, 128}, {32, 4}};
  long long best = -1;
  for (int i = 0; i < 6; ++i) {
    long long ty = (H + cand[i][0] - 1) / cand[i][0], tx = (W + cand[i][1] - 1) / cand[i][1];
    long long cost = ty * tx;
    if (best < 0 || cost < best) { best = cost; *bh = cand[i][0]; *bw = cand[i][1]; }
  }
}

int pf_gemm(pf_gemm_desc* u, void* stream) {
  if (!u) return set_error("pf_gemm: null descriptor");
  if (u->num_src < 1 || u->num_src > 3) return set_error("pf_gemm: num_src %d", u->num_src);
  if (u->taps != 1 && u->taps != 9) return set_error("pf_gemm: taps %d", u->taps);
  if (u->taps == 9 && u->a_mode != 1) return set_error("pf_gemm: 3x3 window needs a_mode 1");
  if (u->N <= 0) return set_error("pf_gemm: N %d", u->N);
  if (u->out_ld % 8 || u->out_col0 % 8) return set_error("pf_gemm: out_ld/out_col0 must be multiples of 8");
  const bool e4m3 = u->a_e4m3 != 0;
  const bool a_static = e4m3 && u->a_static != 0;
  // a linear layer on e4m3 operands (static scale): pf_gemm_pp_e4m3_kernel
  const bool lin8 = a_static && u->a_mode == 0 && u->taps == 1;
  if (lin8 && (u->num_src != 1 || u->N % 128 || u->a_c[0] % 128 || u->a_ld[0] % 16 || u->a_ld[0] < u->a_c[0] || !u->s_w ||
               u->ps > 1 || u->w2 || u->res1 || u->res2 || u->out2 ||
               (u->act != PF_ACT_NONE && u->act != PF_ACT_GELU && u->act != PF_ACT_RELU)))
    return set_error("pf_gemm: an e4m3 linear layer takes one e4m3 matrix source of K (a multiple of 128) <= a_ld "
                     "(a multiple of 16) byte rows, N a multiple of 128, s_w, and bias -> none / GELU / ReLU into one output");
  if (e4m3 && !lin8 && (u->a_mode != 1 || u->taps != 9 || u->bh != 0 || u->bw != 0 || getenv("PF_B200_NO_HALO") != nullptr ||
               u->rs_h[0] || u->rs_h[1] || u->rs_h[2] || (!u->s_a && !a_static) || !u->s_w))
    return set_error("pf_gemm: e4m3 operands take the 3x3 halo-tile conv with materialised sources and s_a / s_w");
  if ((u->a_static && !e4m3) || (u->out_e4m3 && !a_static))
    return set_error("pf_gemm: a static input scale needs e4m3 operands, an e4m3 output a static input scale");
  const bool out8 = u->out_e4m3 != 0;
  const int n_pad64 = (u->N + 63) / 64 * 64;
  if (out8 && (u->out_f32 || u->gamma || u->res1 || u->res2 || u->out2 || u->w2 || u->vt || u->ps > 1 || u->out_col0 ||
               u->out_ld % 16 || u->out_ld < n_pad64 || reinterpret_cast<uintptr_t>(u->out) % 16 || !(u->out_ratio >= 0.f)))
    return set_error("pf_gemm: an e4m3 output is a plain map / matrix of 64 ceil(N / 64) <= out_ld (a multiple of 16) "
                     "byte rows, 16-byte aligned, with out_ratio >= 0");
  // residuals and / or an e4m3 ReLU copy on a static-scale E4M3 conv: pf_conv3_halo_e4m3_res_kernel
  const bool copy8 = u->out2_e4m3 != 0;
  const bool res8 = a_static && !lin8 && (copy8 || u->res1 || u->res2);
  if (copy8 && !res8) return set_error("pf_gemm: an e4m3 ReLU copy (out2_e4m3) needs a static-scale E4M3 3x3 conv");
  if (res8 && (out8 || u->out_f32 || u->gamma || u->w2 || u->vt || u->ps > 1 || u->out_col0 || !u->out2 != !copy8 ||
               (u->block_n != 0 && u->block_n != 64 && u->block_n != 128) ||
               ((u->res1 || u->res2) && (u->res_ld % 2 || u->res_ld < u->N ||
                                         (reinterpret_cast<uintptr_t>(u->res1) | reinterpret_cast<uintptr_t>(u->res2)) % 4)) ||
               (copy8 && (u->out2_ld % 16 || u->out2_ld < n_pad64 || reinterpret_cast<uintptr_t>(u->out2) % 16 ||
                          !(u->out2_ratio >= 0.f)))))
    return set_error("pf_gemm: residuals / an e4m3 ReLU copy on an e4m3 conv take a bf16 output at column 0, block_n 0, "
                     "64 or 128, bf16 residuals of an even pitch >= N, and an e4m3 copy map of 64 ceil(N / 64) <= out2_ld "
                     "(a multiple of 16) byte rows, 16-byte aligned, with out2_ratio >= 0");
  GemmDesc d;
  memset(&d, 0, sizeof(d));
  d.num_src = u->num_src; d.a_mode = u->a_mode; d.taps = u->taps;
  int ksteps = 0;
  for (int s = 0; s < u->num_src; ++s) {
    d.chunks[s] = (u->a_c[s] + 63) / 64;
    d.k_true[s] = u->a_c[s];
    u->chunks[s] = d.chunks[s];
    ksteps += d.chunks[s] * u->taps;
    if (u->a_c[s] % 8 || u->a_ld[s] % 8) return set_error("pf_gemm: source %d channels/ld must be multiples of 8", s);
  }
  if (u->Ktot != ksteps * 64) return set_error("pf_gemm: Ktot %d != %d expected from sources", u->Ktot, ksteps * 64);
  // N tiling.  The packed weight panel has n_pad rows (ops.n_pad_for): N rounded up to 32 up to 256, above that to a
  // multiple of the width in [128, 256] that pads least.  Every n-tile width chosen below divides n_pad, so the last
  // n-tile reads zero-packed rows only.
  int n_pad = (u->N + 31) / 32 * 32;
  if (n_pad > 256) {
    int bestpad = 1 << 30, pw = 256;
    for (int c = 256; c >= 128; c -= 32) {
      int pad = (u->N + c - 1) / c * c - u->N;
      if (pad < bestpad) { bestpad = pad; pw = c; }
    }
    n_pad = (u->N + pw - 1) / pw * pw;
  }
  // 3x3 convs go through the halo-tile kernel (one A fetch per 64-channel chunk instead of nine) unless the caller
  // pins a tile shape or PF_B200_NO_HALO is set.
  static const bool no_halo = getenv("PF_B200_NO_HALO") != nullptr;
  const bool halo = u->a_mode == 1 && u->taps == 9 && u->bh == 0 && u->bw == 0 && !no_halo;
  d.M = u->M; d.NB = u->NB; d.H = u->H; d.W = u->W;
  CUtensorMap tmA[3], tmB;
  d.halo = halo ? 1 : 0;
  bool any_rs = false;
  for (int s = 0; s < u->num_src; ++s) {
    if (u->rs_h[s] < 0 || u->rs_w[s] < 0 || (u->rs_h[s] > 0) != (u->rs_w[s] > 0)) return set_error("pf_gemm: bad rs_h/rs_w of source %d", s);
    any_rs = any_rs || u->rs_h[s] > 0;
  }
  if (any_rs && !halo) return set_error("pf_gemm: resampled sources (rs_h > 0) need the 3x3 halo-tile path");
  if (halo) {
    d.bh = 16; d.bw = 8;
    d.tiles_y = (u->H + 15) / 16; d.tiles_x = (u->W + 7) / 8;
    d.m_tiles = u->NB * d.tiles_y * d.tiles_x;
    int first_plain = -1;
    for (int s = 0; s < u->num_src; ++s) {
      if (u->rs_h[s] > 0) {
        // read through a fused bilinear resample: no tensor map, the producer warps gather from the low-resolution map
        d.rs_ptr[s] = static_cast<const __nv_bfloat16*>(u->a_ptr[s]);
        d.rs_h[s] = u->rs_h[s]; d.rs_w[s] = u->rs_w[s]; d.rs_ld[s] = u->a_ld[s];
        d.rs_sy[s] = u->H > 1 ? static_cast<float>(u->rs_h[s] - 1) / static_cast<float>(u->H - 1) : 0.f;
        d.rs_sx[s] = u->W > 1 ? static_cast<float>(u->rs_w[s] - 1) / static_cast<float>(u->W - 1) : 0.f;
        d.rs_any = 1;
        if (reinterpret_cast<uintptr_t>(u->a_ptr[s]) & 15) return set_error("pf_gemm: resampled source %d not 16-byte aligned", s);
        continue;
      }
      if (e4m3) {
        // one e4m3 map holds every source, each padded to 64 channels (pf_quantize_e4m3_tiles); a_ld[0] in bytes
        int kc = 0;
        for (int j = 0; j < u->num_src; ++j) kc += d.chunks[j] * 64;
        if (u->a_ld[0] < kc || u->a_ld[0] % 16) return set_error("pf_gemm: e4m3 map pitch %d < %d channels", u->a_ld[0], kc);
        if (s == 0 && tmap_4d_nhwc_u8(&tmA[0], u->a_ptr[0], kc, u->W, u->H, u->NB, u->a_ld[0], 64, 10, 18)) return 1;
        tmA[s] = tmA[0];
      } else if (tmap_4d_nhwc_bf16(&tmA[s], u->a_ptr[s], u->a_c[s], u->W, u->H, u->NB, u->a_ld[s], 64, 10, 18)) {
        return 1;
      }
      if (first_plain < 0) first_plain = s;
    }
    for (int s = 0; s < u->num_src; ++s)       // placeholder maps for the resampled sources (never dereferenced)
      if (u->rs_h[s] > 0) {
        if (first_plain >= 0) tmA[s] = tmA[first_plain];
        else memset(&tmA[s], 0, sizeof(CUtensorMap));
      }
  } else if (u->a_mode == 1) {
    int bh = u->bh, bw = u->bw;
    if (bh == 0 || bw == 0) choose_tile(u->H, u->W, &bh, &bw);
    if (bh * bw != 128) return set_error("pf_gemm: bh*bw must be 128");
    d.bh = bh; d.bw = bw;
    d.tiles_y = (u->H + bh - 1) / bh; d.tiles_x = (u->W + bw - 1) / bw;
    d.m_tiles = u->NB * d.tiles_y * d.tiles_x;
    for (int s = 0; s < u->num_src; ++s)
      if (tmap_4d_nhwc_bf16(&tmA[s], u->a_ptr[s], u->a_c[s], u->W, u->H, u->NB, u->a_ld[s], 64, bw, bh)) return 1;
  } else if (lin8) {
    // 128-byte K blocks: {128 B, 128 rows} boxes of the e4m3 matrix [M, a_ld[0] bytes]
    d.m_tiles = (u->M + 127) / 128;
    if (tmap_2d_u8(&tmA[0], u->a_ptr[0], u->a_c[0], u->M, u->a_ld[0], 128, 128)) return 1;
  } else {
    d.m_tiles = (u->M + 127) / 128;
    for (int s = 0; s < u->num_src; ++s)
      if (tmap_2d_bf16(&tmA[s], u->a_ptr[s], u->a_c[s], u->M, u->a_ld[s], 64, 128)) return 1;
  }
  u->bh = d.bh; u->bw = d.bw; u->tiles_y = d.tiles_y; u->tiles_x = d.tiles_x; u->m_tiles = d.m_tiles;
  // Both kernels hold a warpgroup's 64 x block_n fp32 accumulator tile in registers and are compiled per width
  // (pf_gemm_kernel: kGemmWidths; halo kernel: 32, 64, 128 and 192).
  int bn = u->block_n;
  if (bn == 0) {
    if (halo) {
      // the widest halo width that divides the panel; a fused trailing layer wider than that is refused below
      bn = n_pad % 192 == 0 ? 192 : (n_pad % 128 == 0 ? 128 : (n_pad % 64 == 0 ? 64 : 32));
    } else if (u->ps > 1 || u->w2) {
      // pixel shuffle: an n-tile must not straddle two (ky,kx) taps (the widest width dividing the padded Cout); a
      // fused trailing layer needs the whole row in one n-tile
      const int span = u->ps > 1 ? (u->ps_cout + 31) / 32 * 32 : n_pad;
      for (int w : kGemmWidths)
        if (span % w == 0) bn = w;
      if (u->w2 && bn != n_pad) return set_error("pf_gemm: fused trailing layer needs the whole row in one N tile (N %d)", u->N);
    } else if (n_pad % 128 == 0) {
      // 128 or 256 columns: a 256-column tile reads less shared memory per MMA, but halves the tile count.  Take 256
      // unless it needs more waves of tiles over the SMs for the same columns (N = 1024 at 73 m-tiles: 584 tiles of 128
      // are 4.4 waves on 132 SMs, 292 tiles of 256 are 2.2 waves, so 128 finishes first).
      const long long t128 = static_cast<long long>(d.m_tiles) * (n_pad / 128), sms = sm_count();
      const long long waves128 = (t128 + sms - 1) / sms, waves256 = (t128 / 2 + sms - 1) / sms;
      bn = n_pad % 256 == 0 && 2 * waves256 <= waves128 ? 256 : 128;
    } else {
      for (int w : kGemmWidths)
        if (n_pad % w == 0) bn = w;
    }
  }
  // An e4m3 output is stored in 64-byte column groups: a 32-column n-tile would share its group with the next one.  So
  // such a conv takes 64-column n-tiles even where the panel's n_pad rows are a multiple of 32 only (N = 160 in the
  // vits U-Net): its weight maps then end at n_pad rows and the copy engine zero-fills the rows past them.
  uint64_t b_rows = 0;
  if (res8) {
    // the kernel's widths are 64 and 128; a last n-tile past the panel's n_pad rows reads the copy engine's zero fill
    if (u->block_n == 0) bn = n_pad % 128 == 0 ? 128 : 64;
    b_rows = static_cast<uint64_t>(n_pad);
  } else if (out8 && bn == 32 && u->N > 32) {
    if (u->block_n != 0) return set_error("pf_gemm: an e4m3 output needs block_n >= 64 when N > 32 (N %d)", u->N);
    bn = 64;
    b_rows = static_cast<uint64_t>(n_pad);
  }
  d.block_n = bn; d.N = u->N; d.n_tiles = (u->N + bn - 1) / bn;
  u->block_n = bn; u->n_tiles = d.n_tiles;
  if (b_rows == 0) b_rows = static_cast<uint64_t>(d.n_tiles) * bn;
  if (e4m3) {
    if (tmap_2d_u8(&tmB, u->w_ptr, u->Ktot, b_rows, u->Ktot, 64, bn)) return 1;
    d.a_e4m3 = 1; d.s_a = u->s_a; d.s_w = u->s_w;
    d.a_static = a_static ? 1 : 0; d.a_scale = u->a_scale;
    d.out_e4m3 = out8 ? 1 : 0; d.out_ratio = copy8 ? u->out2_ratio : u->out_ratio;
  } else if (tmap_2d_bf16(&tmB, u->w_ptr, u->Ktot, static_cast<uint64_t>(d.n_tiles) * bn, u->Ktot, 64, bn)) {
    return 1;
  }
  d.bias = u->bias; d.act = u->act;
  d.res1 = static_cast<const __nv_bfloat16*>(u->res1);
  d.res2 = static_cast<const __nv_bfloat16*>(u->res2);
  d.res_ld = u->res_ld;
  d.gamma = u->gamma;
  d.out = u->out; d.out_f32 = u->out_f32 || u->gamma != nullptr; d.out_ld = u->out_ld; d.out_col0 = u->out_col0;
  d.out2 = static_cast<__nv_bfloat16*>(u->out2); d.out2_ld = u->out2_ld;
  if ((u->out_f32 || u->gamma) && reinterpret_cast<uintptr_t>(u->out) % 32 != 0)
    return set_error("pf_gemm: fp32 outputs must be 32-byte aligned (256-bit epilogue stores)");
  // 256-bit epilogue accesses need 32-byte aligned rows: bf16 pitches / offsets in multiples of 16 elements
  d.wide = ((reinterpret_cast<uintptr_t>(u->out) | reinterpret_cast<uintptr_t>(u->out2) | reinterpret_cast<uintptr_t>(u->res1) |
             reinterpret_cast<uintptr_t>(u->res2)) % 32 == 0) &&
           u->out_col0 % 16 == 0 && (d.out_f32 || u->out_ld % 16 == 0) && (!u->out2 || u->out2_ld % 16 == 0) &&
           (!(u->res1 || u->res2) || u->res_ld % 16 == 0);
  d.ps = u->ps > 1 ? u->ps : 1;
  d.n_logical = u->N;
  if (d.ps > 1) {
    if (u->a_mode != 0) return set_error("pf_gemm: pixel shuffle needs a_mode 0");
    int cpad = (u->ps_cout + 31) / 32 * 32;           // per-tap column stride of pf_pack_weight_convT
    if (cpad % bn != 0) return set_error("pf_gemm: padded ps_cout %d must be a multiple of block_n %d", cpad, bn);
    if (u->N != d.ps * d.ps * cpad) return set_error("pf_gemm: pixel shuffle N %d != k*k*pad32(Cout) %d", u->N, d.ps * d.ps * cpad);
    d.ps_cout_pad = cpad;
    d.n_logical = u->ps_cout;
  }
  d.w2 = u->w2; d.b2 = u->b2; d.n2 = u->n2; d.act2 = u->act2; d.skip_main = u->skip_main;
  d.out3 = u->out3; d.out3_ld = u->out3_ld;
  if (d.w2) {
    if (d.n_tiles != 1) return set_error("pf_gemm: fused trailing layer needs the whole row in one N tile (N %d)", u->N);
    if (d.n2 < 1 || d.n2 > 16 || !d.out3) return set_error("pf_gemm: fused trailing layer n2 %d (1..16), out3 required", d.n2);
    if (u->N % 4) return set_error("pf_gemm: fused trailing layer needs N % 4 == 0");
  }
  d.vt = static_cast<__nv_bfloat16*>(u->vt);
  d.vt_col0 = u->vt_col0; d.vt_seq = u->vt_seq; d.vt_seq_pad = u->vt_seq_pad; d.vt_dim = u->vt_dim;
  if (d.vt && (d.vt_col0 % bn) != 0) return set_error("pf_gemm: vt_col0 must be a multiple of block_n");
  // Linear layers with several m-tiles per n-tile are L2 -> SM bandwidth bound: pairs of CTAs share the weight tile by
  // TMA multicast (PF_OPT_GEMM_MULTICAST / PF_OPT_HALO_MULTICAST).  Needs an even split of the n-tile into 1024-B aligned halves.
  // PF_OPT_HALO_MULTICAST: 0 off, 1 clusters of 2, 2 clusters of 4
  int cl = 1;
  if (d.m_tiles >= 4 && static_cast<long long>(d.m_tiles) * d.n_tiles >= sm_count()) {
    if (halo) cl = option(PF_OPT_HALO_MULTICAST) >= 2 ? 4 : (option(PF_OPT_HALO_MULTICAST) == 1 ? 2 : 1);
    else if (option(PF_OPT_GEMM_MULTICAST) != 0 && u->a_mode == 0 && d.ps == 1 && bn % 16 == 0) cl = 2;
  }
  d.halo_cl = halo ? cl : 1;
  const bool mc = cl > 1;
  CUtensorMap tmBh;
  if (mc && (e4m3 ? tmap_2d_u8(&tmBh, u->w_ptr, u->Ktot, b_rows, u->Ktot, 64, bn / cl)
                  : tmap_2d_bf16(&tmBh, u->w_ptr, u->Ktot, static_cast<uint64_t>(d.n_tiles) * bn, u->Ktot, 64, bn / cl)))
    return 1;
  // Epilogue through shared memory + TMA: plain bf16 outputs in 64-column groups (32-column groups in the halo kernel at
  // block_n 32), and, in pf_gemm_kernel only, fp32 outputs and the fp32 residual stream (x += gamma * v) in 32-column
  // chunks.  Halo convs reading a fused resample keep the direct stores.  PF_OPT_TMA_EPILOGUE = 0 keeps the direct
  // stores everywhere.
  const bool no_tma_epi = option(PF_OPT_TMA_EPILOGUE) == 0;
  CUtensorMap tmOut, tmOut2;
  d.tma_out = 0;
  // The copy clips columns >= out_col0 + N only at 16-byte granularity: a row that ends inside a 16-byte piece would get
  // the staged zeros of columns N .. written over what the caller keeps there, so such outputs take the direct stores.
  const uint64_t ocols = static_cast<uint64_t>(u->out_col0) + u->N;
  const bool ends16 = ocols % (d.out_f32 ? 4 : 8) == 0;
  if (res8) {
    // the bf16 output in {64 ch, 8 px, 2 rows} boxes as a plain halo conv's, the e4m3 copy as the q8 kernel's e4m3 map
    if (!no_tma_epi) {
      if (!ends16 || reinterpret_cast<uintptr_t>(u->out) % 16)
        return set_error("pf_gemm: an e4m3 conv with residuals / a ReLU copy needs a 16-byte aligned bf16 output whose rows end "
                         "on a 16-byte boundary");
      if (tmap_4d_nhwc_bf16(&tmOut, u->out, ocols, u->W, u->H, u->NB, u->out_ld, 64, 8, 2)) return 1;
      if (copy8 && tmap_4d_nhwc_u8(&tmOut2, u->out2, n_pad64, u->W, u->H, u->NB, u->out2_ld, 64, 8, 2)) return 1;
      d.tma_out = 1;
    }
  } else if (out8) {
    // the q8 kernel's e4m3 epilogue: {64 bytes, 8 px, 2 rows} boxes of a map N rounded up to 64 columns wide, so the
    // stores write the pad columns (as zero) too
    // ({64 bytes, 16 rows} boxes of the linear layer's [M, out_ld bytes] matrix)
    if (!no_tma_epi && (lin8 ? tmap_2d_u8(&tmOut, u->out, n_pad64, u->M, u->out_ld, 64, 16)
                             : tmap_4d_nhwc_u8(&tmOut, u->out, n_pad64, u->W, u->H, u->NB, u->out_ld, 64, 8, 2)))
      return 1;
    d.tma_out = no_tma_epi ? 0 : 1;
  } else if (!no_tma_epi && !(halo && any_rs) && d.ps == 1 && !d.w2 && !d.res1 && !d.res2 && !d.out2 && ends16) {
    // each consumer warp stores its 16 rows in whole column groups (bf16) / 32-column chunks (fp32)
    const uint32_t group = halo && bn == 32 ? 32 : 64;
    if (!d.out_f32 && bn % group == 0 && reinterpret_cast<uintptr_t>(u->out) % 16 == 0) {
      if (u->a_mode == 0) {
        if (tmap_2d_bf16(&tmOut, u->out, ocols, u->M, u->out_ld, 64, 16)) return 1;
      } else {
        // the halo kernel's 16 x 8 pixel tile: {group, 8, 2} boxes, one per consumer warp
        const uint32_t bwx = d.bw < 16 ? d.bw : 16;
        if (tmap_4d_nhwc_bf16(&tmOut, u->out, ocols, u->W, u->H, u->NB, u->out_ld, group, bwx, 16 / bwx)) return 1;
      }
      d.tma_out = 1;
    } else if (d.out_f32 && u->a_mode == 0 &&u->out_ld % 4 == 0 && reinterpret_cast<uintptr_t>(u->out) % 16 == 0) {
      if (tmap_2d_f32(&tmOut, u->out, ocols, u->M, u->out_ld, 32, 16)) return 1;
      d.tma_out = 2;
    }
  }
  // Plain linear layers run on pf_gemm_pp_kernel: each consumer warpgroup owns whole 128 x 128 tiles and one tile's
  // epilogue runs under the other warpgroup's MMAs.  It takes one source, N in whole 128-column tiles and the epilogues
  // it has: bias -> none / GELU / ReLU through the bf16 bulk store, the fp32 bulk store or gamma reduce-add, and a fused
  // qkv projection whose V^T third it stores from the fragment.  block_n stays the launch's work-item width (a 256 item
  // is two tiles).  The coarse image's linears (M = 1037, 9 m-tiles) take it too.  Measured on an H100 80GB HBM3 at
  // 700 W, vitl (before -> after, ms): qkv 0.034 -> 0.025, fc1 0.041 -> 0.037, fc2 0.029 -> 0.029, proj 0.013 -> 0.014.
  // proj's 72 tiles leave the second warpgroup of every CTA idle, but the loss is 1 us per launch, against 9 us gained
  // on qkv, so no separate rule keeps it on pf_gemm_kernel.
  const bool pp_act = u->act == PF_ACT_NONE || u->act == PF_ACT_GELU || u->act == PF_ACT_RELU;
  // its V^T store indexes the buffer with 32-bit offsets
  const bool pp_vt = !d.vt || (d.tma_out == 1 && d.vt_seq > 0 &&
                               static_cast<long long>((u->M + d.vt_seq - 1) / d.vt_seq + 1) * d.vt_dim * d.vt_seq_pad < (1ll << 31));
  if (u->a_mode == 0 && u->num_src == 1 && d.tma_out != 0 && u->N % kPpBN == 0 && bn % kPpBN == 0 && pp_act && pp_vt) {
    d.pp = 1;
    const uint64_t rows = static_cast<uint64_t>(d.n_tiles) * bn;
    if (lin8) {     // the e4m3 panel in 128-byte K blocks, like A
      if (tmap_2d_u8(&tmB, u->w_ptr, u->Ktot, rows, u->Ktot, 128, kPpBN)) return 1;
      if (mc && tmap_2d_u8(&tmBh, u->w_ptr, u->Ktot, rows, u->Ktot, 128, kPpBN / 2)) return 1;
    } else {
      if (tmap_2d_bf16(&tmB, u->w_ptr, u->Ktot, rows, u->Ktot, 64, kPpBN)) return 1;
      if (mc && tmap_2d_bf16(&tmBh, u->w_ptr, u->Ktot, rows, u->Ktot, 64, kPpBN / 2)) return 1;
    }
  }
  // the FP8 conv has only the plain-output fragment epilogue (bias + activation -> stmatrix -> bulk store); the e4m3
  // linear layer only the ping-pong kernel
  if (e4m3 && !lin8 && d.tma_out != 1)
    return set_error("pf_gemm: an e4m3 conv needs the bulk-store epilogue: a plain bf16 output, 16-byte aligned, and "
                     "PF_OPT_TMA_EPILOGUE on");
  if (lin8 && !d.pp)
    return set_error("pf_gemm: an e4m3 linear layer runs on the ping-pong kernel only: a bulk-store output (16-byte "
                     "aligned, rows ending on a 16-byte boundary, PF_OPT_TMA_EPILOGUE on)");
  return gemm_launch(d, tmA, tmB, mc ? &tmBh : nullptr, d.tma_out ? &tmOut : nullptr, static_cast<cudaStream_t>(stream),
                     res8 && copy8 && d.tma_out ? &tmOut2 : nullptr);
}

}  // extern "C"
