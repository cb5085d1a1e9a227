// Implicit-GEMM engine of the PatchFusion hot path (wgmma / TMA / mbarrier, sm_90a).
//
// One persistent, warp-specialised kernel serves every dense contraction of the path (the plain linear layers run on a
// ping-pong variant of it, pf_gemm_pp_kernel, further down):
//   * ViT / Swin linear layers            (`dinov2/layers/attention.py:51,60`, `mlp.py:36-39`, `swin_layers.py:140,162`)
//   * 1x1 convs (NHWC == plain GEMM)      (`depth_anything/dpt.py:30-38`, metric-head MLPs `localbins_layers.py:84-117`)
//   * 3x3 stride-1 pad-1 convs over a channel-concat of up to three NHWC sources
//                                          (`depth_anything/blocks.py:53-58`, `patchfusion.py:122-127,263-267`,
//                                           `guided_fusion_model.py:34-69,98-99,203`)
//   * ConvTranspose k==stride as GEMM + pixel-shuffle store (`depth_anything/dpt.py:40-53`)
//
// D[M,N] = sum_{src,tap,c} A_src[pixel(m)+tap, c] * Wp[n, k(src,tap,c)]   (bf16 x bf16 -> fp32 in registers)
//
// A tiles are fetched by TMA straight from the activation tensors: a 3x3 tap is just a (dx,dy) offset of the 4-D
// box {64ch, bw, bh, 1} and the hardware zero-fills out-of-image pixels (conv padding), out-of-range channels and
// rows, so there is no im2col buffer and no halo code.  Weights are pre-packed K-major [N, Ktot] with every
// (source, tap) segment padded to a multiple of 64 channels, matching the producer's enumeration order.
//
// Warp roles (pf_gemm_kernel): warps 0-7 = two consumer warpgroups.  Warpgroup h computes tile rows 64h .. 64h + 63
// against all BN columns of the n-tile, one wgmma.m64nBNk16 per k16 step with both operands read by the tensor core
// from the swizzled TMA tiles in shared memory (every A tile is 128 rows x 128 B in the canonical K-major layout, so
// the warpgroup's A operand is a descriptor at its 8 KB row offset).  Warp w owns tile rows 16w .. 16w + 15, so after
// the mainloop every accumulator row lives in one warp.  The same warps then run the epilogue.  Plain outputs (bias /
// activation / gamma) are finished in the accumulator's fragment layout, staged 16 rows x 128 B at a time in one of the
// warp's two swizzled staging tiles (stmatrix for bf16, 8-byte stores for fp32) and moved by a bulk tensor store, or a
// bulk reduce-add for the fp32 residual stream.  The variants that need a whole row per thread (residuals / fused tail /
// ReLU copy / pixel shuffle / the V^T third of a fused qkv projection) send a 16 x 32 fp32 block at a time through a per-warp
// swizzled shared-memory transpose so that a thread holds 16 columns of one accumulator row, and store directly.
// The last warp is the TMA producer; the halo kernel has two more warps before it, the operand producers of
// its optional fused bilinear resample (idle otherwise).  While the consumers drain a tile, the producer already fills
// the operand ring for the next one.
//
// BN is a template parameter of both kernels, so every wgmma has a fixed shape and none sits under a data-dependent
// branch: the last n-tile issues all BN columns (the packed weight rows beyond N are zero, the epilogue drops those
// columns) and the zero-padded last 64-channel chunk of a source issues all four k16 steps (its pad channels are TMA
// zero fill against zero-packed weights).
#include "pf_common.cuh"
#include "pf_kernels.h"

namespace pf {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KiB
constexpr int kEpiWarps = 8;                       // consumer warps: two warpgroups
// pf_gemm_kernel: consumers + one TMA producer warp; pf_conv3_halo_kernel: + two resample producer warps before it.
// A consumer thread holds BN / 2 fp32 accumulators (plus 32 A-fragment registers in the halo kernel): no idle warps,
// so that the per-thread register budget (65536 / threads, capped at 168) stays large.
constexpr int kGemmThreads = (kEpiWarps + 1) * 32;
constexpr int kHaloThreads = (kEpiWarps + 3) * 32;
constexpr int kRsWarp0 = kEpiWarps;                         // halo kernel: warps 8, 9 = resample producers
constexpr int kMaxSmem = 227 * 1024;
// per consumer warp: the 16 x 32 fp32 accumulator transpose of the row-per-thread epilogue.  Both kernels have two such
// blocks per warp, the staging tiles of the TMA-store epilogue (16 rows x 128 B, SWIZZLE_128B, or x 64 B, SWIZZLE_64B)
// used in turn; the first doubles as the transpose block
constexpr int kXposeWarp = 16 * 32 * 4;
constexpr int kStageWarp = 2 * kXposeWarp;
constexpr int kBarBytes = 512;

// pf_gemm_kernel operand ring: one stage = the 128-row A tile + BN weight rows of one 64-wide K block; as many stages
// as fit next to the transposes and barriers, at most eight
__host__ __device__ constexpr int gemm_stage_bytes(int bn) { return kATileBytes + bn * kBlockK * 2; }
__host__ __device__ constexpr int gemm_stages(int bn) {
  return (kMaxSmem - 1024 /*align*/ - kBarBytes - kEpiWarps * kStageWarp) / gemm_stage_bytes(bn) < 8
             ? (kMaxSmem - 1024 - kBarBytes - kEpiWarps * kStageWarp) / gemm_stage_bytes(bn)
             : 8;
}

struct GemmKernelParams {
  CUtensorMap tmA[3];
  CUtensorMap tmB;
  CUtensorMap tmBh;     // multicast variant: box of block_n / cl weight rows (each CTA of the cluster fetches one part)
  CUtensorMap tmOut;    // d.tma_out: output tensor (bf16 {64 cols, 16 rows} boxes, or fp32 {32 cols, 16 rows})
  GemmDesc d;
  int total_tiles;
  int k_steps;  // 64-wide K blocks per tile
  // pf_conv3_halo_e4m3_res_kernel: the e4m3 ReLU copy d.out2 ({64 B, 8 px, 2 rows} boxes).  Last, so that the other
  // kernels' parameter offsets are what they were.
  CUtensorMap tmOut2;
};


struct TileCoord {
  int n0;               // first output column
  int m0;               // linear: first row
  int img, y0, x0;      // conv: tile origin
};

__device__ __forceinline__ TileCoord decode_tile(const GemmDesc& d, int t) {
  TileCoord c;
  int nt = t % d.n_tiles;
  int mt = t / d.n_tiles;
  c.n0 = nt * d.block_n;
  c.m0 = mt * kBlockM;
  c.img = 0; c.y0 = 0; c.x0 = 0;
  if (d.a_mode == 1) {
    int per_img = d.tiles_y * d.tiles_x;
    c.img = mt / per_img;
    int r = mt - c.img * per_img;
    c.y0 = (r / d.tiles_x) * d.bh;
    c.x0 = (r % d.tiles_x) * d.bw;
  }
  return c;
}

// One W-column chunk of one accumulator row: bias -> activation -> residuals -> store.  FULL == all W columns exist
// (vector loads/stores, no predication); the tail variant predicates every column but keeps all indices static so
// f[] stays in registers.
constexpr int kMaxTail = 16;   // widest fused trailing 1x1 layer

// W = chunk width in accumulator columns; TAILN = compile-time bound on the fused trailing layer's outputs (0 = no
// trailing layer): keeps the executed code path short - the fully unrolled 16-output variant alone is ~3k
// instructions and thrashed the instruction cache.
template <bool FULL, int W, int TAILN>
__device__ __forceinline__ void epilogue_chunk(const GemmDesc& d, float (&f)[W], long long orow, int ncol, int lcol,
                                               int nvalid, float (&y2)[kMaxTail], uint32_t (&xv)[TAILN == 0 ? W / 8 : 1][8]) {
  if (d.bias != nullptr) {
    if (FULL) {
      const float4* bp = reinterpret_cast<const float4*>(d.bias + lcol);
#pragma unroll
      for (int j = 0; j < W / 4; ++j) {
        float4 b = __ldg(bp + j);
        f[4 * j] += b.x; f[4 * j + 1] += b.y; f[4 * j + 2] += b.z; f[4 * j + 3] += b.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) f[j] += __ldg(d.bias + lcol + j);
    }
  }
  if (d.act == PF_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < W; ++j) f[j] = fmaxf(f[j], 0.0f);
  } else if (d.act == PF_ACT_GELU) {
    if (FULL) {
#pragma unroll
      for (int j = 0; j < W; j += 2) gelu_erf2(f[j], f[j + 1]);
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) f[j] = gelu_erf(f[j]);
    }
  } else if (d.act == PF_ACT_SOFTPLUS) {
#pragma unroll
    for (int j = 0; j < W; ++j) if (FULL || j < nvalid) f[j] = softplus(f[j]);
  }
  // fused trailing 1x1 layer: y[i] += sum_j W2[i][lcol + j] * f[j]  (row-local: the thread owns the whole row)
  if (TAILN > 0) {
#pragma unroll
    for (int i = 0; i < TAILN; ++i) {
      if (i < d.n2) {
        const float* wp = d.w2 + static_cast<long long>(i) * d.n_logical + lcol;
        // four independent partial sums: a single accumulator is a 32-deep FFMA dependency chain (latency-bound)
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        if (FULL) {
#pragma unroll
          for (int j = 0; j < W / 4; ++j) {
            float4 w4 = __ldg(reinterpret_cast<const float4*>(wp) + j);
            a0 = fmaf(w4.x, f[4 * j], a0); a1 = fmaf(w4.y, f[4 * j + 1], a1);
            a2 = fmaf(w4.z, f[4 * j + 2], a2); a3 = fmaf(w4.w, f[4 * j + 3], a3);
          }
        } else {
#pragma unroll
          for (int j = 0; j < W; ++j) if (j < nvalid) a0 = fmaf(__ldg(wp + j), f[j], a0);
        }
        y2[i] += (a0 + a1) + (a2 + a3);
      }
    }
    if (d.skip_main) return;
  }
#pragma unroll
  for (int rsel = 0; rsel < 2; ++rsel) {
    const __nv_bfloat16* rbase = rsel == 0 ? d.res1 : d.res2;
    if (rbase == nullptr) continue;
    const __nv_bfloat16* rp = rbase + orow * d.res_ld + lcol;
    if (FULL && d.wide) {
#pragma unroll
      for (int j = 0; j < W / 16; ++j) {
        uint32_t u[8];
        ld_global_256(rp + 16 * j, u);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u[e]));
          f[16 * j + 2 * e] += t.x; f[16 * j + 2 * e + 1] += t.y;
        }
      }
    } else if (FULL) {
#pragma unroll
      for (int j = 0; j < W / 8; ++j) {
        uint4 u = __ldg(reinterpret_cast<const uint4*>(rp) + j);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 t = __bfloat1622float2(h[e]);
          f[8 * j + 2 * e] += t.x; f[8 * j + 2 * e + 1] += t.y;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) f[j] += __bfloat162float(rp[j]);
    }
  }
  const int oc = lcol + d.out_col0;      // physical output column
  if (d.vt != nullptr && ncol >= d.vt_col0) {
    // attention V written transposed: vt[(b*heads + h)*64 + dd][token]
    const int m = static_cast<int>(orow);
    const int b = m / d.vt_seq, tok = m - b * d.vt_seq;
    __nv_bfloat16* vp = d.vt + (static_cast<long long>(b) * d.vt_dim + (ncol - d.vt_col0)) * d.vt_seq_pad + tok;
#pragma unroll
    for (int j = 0; j < W; ++j)
      if (FULL || j < nvalid) vp[static_cast<long long>(j) * d.vt_seq_pad] = __float2bfloat16(f[j]);
  } else if (d.gamma != nullptr) {
    // x <- x + gamma * (acc + bias): fp32 residual stream updated in place
    float* xp = reinterpret_cast<float*>(d.out) + orow * d.out_ld + oc;
    if (FULL && TAILN == 0) {
      // one full 32-B sector per access; the residual-stream segment was fetched by epilogue_cols before the
      // accumulator wait (xv), so only the update + store remain here
#pragma unroll
      for (int j = 0; j < (TAILN == 0 ? W / 8 : 1); ++j) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(d.gamma + lcol + 8 * j));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(d.gamma + lcol + 8 * j + 4));
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) xv[j][e] = __float_as_uint(fmaf(gg[e], f[8 * j + e], __uint_as_float(xv[j][e])));
        st_global_256(xp + 8 * j, xv[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) xp[j] += __ldg(d.gamma + lcol + j) * f[j];
    }
  } else if (d.out_f32) {
    float* op = reinterpret_cast<float*>(d.out) + orow * d.out_ld + oc;
    if (FULL) {
#pragma unroll
      for (int j = 0; j < W; j += 8) {
        const uint32_t u[8] = {__float_as_uint(f[j]), __float_as_uint(f[j + 1]), __float_as_uint(f[j + 2]), __float_as_uint(f[j + 3]),
                               __float_as_uint(f[j + 4]), __float_as_uint(f[j + 5]), __float_as_uint(f[j + 6]), __float_as_uint(f[j + 7])};
        st_global_256(op + j, u);
      }
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) op[j] = f[j];
    }
  } else {
    __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(d.out) + orow * d.out_ld + oc;
    if (FULL && d.wide) {
#pragma unroll
      for (int j = 0; j < W; j += 16) {
        uint32_t u[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) u[e] = pack_bf16(f[j + 2 * e], f[j + 2 * e + 1]);
        st_global_256(op + j, u);
      }
    } else if (FULL) {
#pragma unroll
      for (int j = 0; j < W; j += 8)
        *reinterpret_cast<uint4*>(op + j) = make_uint4(pack_bf16(f[j], f[j + 1]), pack_bf16(f[j + 2], f[j + 3]),
                                                        pack_bf16(f[j + 4], f[j + 5]), pack_bf16(f[j + 6], f[j + 7]));
    } else {
#pragma unroll
      for (int j = 0; j < W; ++j) if (j < nvalid) op[j] = __float2bfloat16(f[j]);
    }
    if (d.out2 != nullptr) {
      __nv_bfloat16* o2 = d.out2 + orow * d.out2_ld + lcol;
      if (FULL && d.wide) {
#pragma unroll
        for (int j = 0; j < W; j += 16) {
          uint32_t u[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) u[e] = pack_bf16(fmaxf(f[j + 2 * e], 0.f), fmaxf(f[j + 2 * e + 1], 0.f));
          st_global_256(o2 + j, u);
        }
      } else if (FULL) {
#pragma unroll
        for (int j = 0; j < W; j += 8)
          *reinterpret_cast<uint4*>(o2 + j) =
              make_uint4(pack_bf16(fmaxf(f[j], 0.f), fmaxf(f[j + 1], 0.f)), pack_bf16(fmaxf(f[j + 2], 0.f), fmaxf(f[j + 3], 0.f)),
                         pack_bf16(fmaxf(f[j + 4], 0.f), fmaxf(f[j + 5], 0.f)), pack_bf16(fmaxf(f[j + 6], 0.f), fmaxf(f[j + 7], 0.f)));
      } else {
#pragma unroll
        for (int j = 0; j < W; ++j) if (j < nvalid) o2[j] = __float2bfloat16(fmaxf(f[j], 0.0f));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Accumulator fragment -> one row half per thread.  A warp holds rows 16w .. 16w + 15 of the tile in one m64nBN
// fragment: element 4j + e at (row lane/4, column 8j + 2(lane%4) + e), 4j + 2 + e at row lane/4 + 8.  acc_stage16<K>
// writes columns 32K .. 32K + 31 into the warp's 16 x 32 fp32 block; lane l then reads row l & 15, columns
// 16 (l >> 4) .. + 15.  Word (r, c) sits at r * 32 + (c ^ s(r)), s mapping row bits 0, 1, 2, 3 to bits 0, 3, 2 + 4, 1:
// the fragment writes (8 rows x 4 column pairs) and the row reads (16 rows x 2 halves) each touch 32 distinct banks.
__device__ __forceinline__ int xpose16_swz(int r) { return (r & 1) | ((r & 8) >> 2) | (r & 4) | ((r & 2) << 2) | ((r & 4) << 2); }
template <int K, int S>
__device__ __forceinline__ void acc_stage16(const float (&a)[S], float* buf, int lane) {
  const int r0 = lane >> 2, cl = 2 * (lane & 3);
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * K + jj;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int c = 8 * jj + cl + e;
      buf[r0 * 32 + (c ^ xpose16_swz(r0))] = a[4 * j + e];
      buf[(r0 + 8) * 32 + (c ^ xpose16_swz(r0 + 8))] = a[4 * j + 2 + e];
    }
  }
}
// runtime chunk index (uniform over the warp, k < S / 16); register indices stay compile-time
template <int S, int K = 0>
__device__ __forceinline__ void acc_stage16_k(int k, const float (&a)[S], float* buf, int lane) {
  if constexpr (K + 1 < S / 16) {
    if (k == K) acc_stage16<K>(a, buf, lane);
    else acc_stage16_k<S, K + 1>(k, a, buf, lane);
  } else {
    acc_stage16<K>(a, buf, lane);
  }
}
// word j of this thread's staged row: rowp[j ^ s] (rowp = the 32-word row, s = its swizzle)
template <int W>
__device__ __forceinline__ void acc_read_row(const float* rowp, int s, uint32_t (&v)[W]) {
#pragma unroll
  for (int j = 0; j < W; ++j) v[j] = __float_as_uint(rowp[j ^ s]);
}

// one W-column chunk starting at accumulator column cb of this thread's row (staged by the caller; read through
// acc_read_row(rowp, sw))
template <int W, int TAILN>
__device__ __forceinline__ void epilogue_cols(const GemmDesc& d, const float* rowp, int sw, int cb, const TileCoord& c,
                                              int ocol0, long long orow, bool row_ok, float (&y2)[kMaxTail]) {
  const int ncol = c.n0 + cb;            // global N index of v[0] (selects the V^T path)
  const int lcol = ocol0 + cb;           // logical output channel of v[0] (bias / gamma / residual index)
  const int nvalid = min(W, d.n_logical - lcol);   // columns of this chunk that exist
  if (!row_ok || nvalid <= 0) return;
  // x += gamma * v: fetch the fp32 residual-stream segment (one full sector per thread) before reading the
  // accumulator, so its L2 latency overlaps the shared-memory loads
  uint32_t xpre[TAILN == 0 ? W / 8 : 1][8];
  const bool pre = TAILN == 0 && d.gamma != nullptr && nvalid == W && !(d.vt != nullptr && ncol >= d.vt_col0);
  if (pre) {
    const float* xp = reinterpret_cast<const float*>(d.out) + orow * d.out_ld + lcol + d.out_col0;
#pragma unroll
    for (int j = 0; j < (TAILN == 0 ? W / 8 : 1); ++j) ld_global_256(xp + 8 * j, xpre[j]);
  }
  uint32_t v[W];
  acc_read_row<W>(rowp, sw, v);
  float f[W];
#pragma unroll
  for (int j = 0; j < W; ++j) f[j] = __uint_as_float(v[j]);
  if (nvalid == W) epilogue_chunk<true, W, TAILN>(d, f, orow, ncol, lcol, W, y2, xpre);
  else epilogue_chunk<false, W, TAILN>(d, f, orow, ncol, lcol, nvalid, y2, xpre);
}

// The 32-column blocks of the tile that hold columns < N; each thread takes 16 columns of its row per block.
template <int TAILN, int S>
__device__ __forceinline__ void epilogue_row(const GemmDesc& d, const float (&acc)[S], float* buf, int lane,
                                             const TileCoord& c, int ocol0, long long orow, bool row_ok,
                                             float (&y2)[kMaxTail]) {
  const int r = lane & 15;
  const float* rowp = buf + r * 32;
  const int sw = xpose16_swz(r) ^ (lane & 16);     // column 16 (lane >> 4) + j of row r is word j ^ sw of rowp
  for (int k = 0; 32 * k < 2 * S && c.n0 + 32 * k < d.N; ++k) {
    acc_stage16_k(k, acc, buf, lane);
    __syncwarp();
    epilogue_cols<16, TAILN>(d, rowp, sw, 32 * k + (lane & 16), c, ocol0, orow, row_ok, y2);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------------------
// Epilogue through shared memory + TMA (pf_gemm_kernel, d.tma_out != 0), in the accumulator's own layout.
// Bias, activation and the gamma scale are per-column vectors and per-element functions, so they are applied where the
// accumulator already is: a thread's fragment holds columns 8j + 2 (lane % 4) + {0, 1} of rows lane / 4 and lane / 4 + 8,
// and adds the bias as one float2 per j.  The warp's 16 rows then go into a swizzled 2 KB staging tile (stmatrix for
// bf16, 8-byte stores for fp32) and ONE elected lane moves the tile with a bulk tensor copy: 128-byte requests, no LSU
// work; the fp32 residual stream is updated by a bulk reduce-add (no read at all).  Each warp has two staging tiles
// and uses them in turn, so a copy reads one while the next block is computed into the other.

struct EpiTma {
  const CUtensorMap* tm;
  uint32_t stg;        // shared address of this warp's two staging tiles (1024-B aligned, kXposeWarp bytes each)
  uint8_t* stg_ptr;
  int cur;             // the tile the next block is staged in
};

// byte offset of the staging tile to fill next: the copy issued from it two blocks ago has finished reading it
__device__ __forceinline__ int epi_stage_acquire(EpiTma& e, int lane) {
  if (lane == 0) bulk_wait_read1();
  __syncwarp();
  const int off = e.cur * kXposeWarp;
  e.cur ^= 1;
  return off;
}

// v = this thread's 16 accumulators of columns 32k .. 32k + 31 (k uniform over the warp, k < S / 16); register indices
// stay compile-time
template <int S, int K = 0>
__device__ __forceinline__ void acc_chunk(int k, const float (&a)[S], float (&v)[16]) {
  if constexpr (K + 1 < S / 16) {
    if (k != K) { acc_chunk<S, K + 1>(k, a, v); return; }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = a[16 * K + i];
}

__device__ __forceinline__ void epi_act(const GemmDesc& d, float (&f)[16]) {
  if (d.act == PF_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 16; ++j) f[j] = fmaxf(f[j], 0.0f);
  } else if (d.act == PF_ACT_GELU) {
#pragma unroll
    for (int j = 0; j < 16; j += 2) gelu_erf2(f[j], f[j + 1]);
  } else if (d.act == PF_ACT_SOFTPLUS) {
#pragma unroll
    for (int j = 0; j < 16; ++j) f[j] = softplus(f[j]);
  }
}
// p[col], p[col + 1] of a per-column vector (col even); columns >= n_logical read nothing (TMA clips them)
__device__ __forceinline__ float2 epi_vec2(const float* p, int col, int n_logical) {
  if (col + 1 < n_logical) return __ldg(reinterpret_cast<const float2*>(p + col));
  return make_float2(col < n_logical ? __ldg(p + col) : 0.f, 0.f);
}
// One 32-column chunk in fragment layout, col = logical column of v[0]: v[4j + e] and v[4j + 2 + e] are column
// col + 8j + e of the thread's two rows.  (acc + bias) -> activation -> * gamma, element by element.
__device__ __forceinline__ void epi_frag(const GemmDesc& d, float (&v)[16], int col, bool scale) {
  if (d.bias != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 b = epi_vec2(d.bias, col + 8 * j, d.n_logical);
      v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.x; v[4 * j + 3] += b.y;
    }
  }
  epi_act(d, v);
  if (scale) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 g = epi_vec2(d.gamma, col + 8 * j, d.n_logical);
      v[4 * j] *= g.x; v[4 * j + 1] *= g.y; v[4 * j + 2] *= g.x; v[4 * j + 3] *= g.y;
    }
  }
}

// store this warp's 16 rows x 128 B (64 bf16 / 32 fp32 columns) starting at column col
__device__ __forceinline__ void epi_tma_store(const GemmDesc& d, const EpiTma& e, const uint8_t* tile, const TileCoord& c,
                                              int warp, int col) {
  if (d.a_mode == 1) {
    const int r0 = warp * 16;
    const int yy = r0 / d.bw, xx = r0 - yy * d.bw;
    tma_store_4d(e.tm, tile, col, c.x0 + xx, c.y0 + yy, c.img);
  } else {
    tma_store_2d(e.tm, tile, col, c.m0 + warp * 16);
  }
}
// bf16 output: groups of G = 64 columns (128-byte row segments, SWIZZLE_128B), or of G = 32 (64-byte row segments,
// SWIZZLE_64B: the halo kernel at BN = 32), G / 32 chunks of 32 columns each.  A chunk packed to bf16 is four 8 x 8
// matrices per 16 columns (column octet o, rows 0-7 / 8-15), written by stmatrix: lane l addresses row r = l & 15 of
// octet pair member l >> 4, 16-byte piece o ^ (r & 7) of the 128-byte row, or o ^ ((r >> 1) & 3) of the 64-byte row
// (the swizzle XORs address bits 4-6 with bits 7-9, or bits 4-5 with bits 7-8).
// SC (the FP8 halo conv): the accumulator is first multiplied by s_a[img] * s_w[column] (__fmul_rn each, so the bias add
// that follows is a separate rounding: v = fl(fl(acc * fl(s_a * s_w)) + bias)).
__device__ __forceinline__ void epi_dequant(const GemmDesc& d, float (&v)[16], int col, float sa) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 w = epi_vec2(d.s_w, col + 8 * j, d.n_logical);
    const float kx = __fmul_rn(sa, w.x), ky = __fmul_rn(sa, w.y);
    v[4 * j] = __fmul_rn(v[4 * j], kx); v[4 * j + 1] = __fmul_rn(v[4 * j + 1], ky);
    v[4 * j + 2] = __fmul_rn(v[4 * j + 2], kx); v[4 * j + 3] = __fmul_rn(v[4 * j + 3], ky);
  }
}
// SC = 2 (the static-scale instantiation): the one scale d.a_scale of the launch instead of s_a[img].
template <int G, int S, int SC = 0>
__device__ __forceinline__ void epilogue_tile_tma_bf16(const GemmDesc& d, EpiTma& e, const float (&acc)[S],
                                                       const TileCoord& c, int warp, int lane) {
  static_assert(G == 64 || G == 32, "group width");
  float sa = 0.f;
  if constexpr (SC == 1) sa = c.img < d.NB ? __ldg(d.s_a + c.img) : 0.f;   // img >= NB: a cluster's phantom tile
  if constexpr (SC == 2) sa = d.a_scale;
  const int oct = lane >> 4;
  const uint32_t lane_off = (lane & 15) * (2 * G);
  const int swz = G == 64 ? (lane & 7) : ((lane >> 1) & 3);
  for (int g = 0; G * g < 2 * S; ++g) {
    const int lcol = c.n0 + g * G;
    if (lcol >= d.n_logical) break;
    const int tile = epi_stage_acquire(e, lane);
#pragma unroll
    for (int h = 0; h < G / 32; ++h) {
      float v[16];
      acc_chunk(G / 32 * g + h, acc, v);
      if constexpr (SC != 0) epi_dequant(d, v, lcol + 32 * h + 2 * (lane & 3), sa);
      epi_frag(d, v, lcol + 32 * h + 2 * (lane & 3), false);
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int o = 4 * h + 2 * p;           // octets o (lanes 0-15) and o + 1 (lanes 16-31)
        const uint32_t addr = e.stg + tile + lane_off + (((o + oct) ^ swz) << 4);
        stmatrix_x4(addr, pack_bf16(v[8 * p], v[8 * p + 1]), pack_bf16(v[8 * p + 2], v[8 * p + 3]),
                        pack_bf16(v[8 * p + 4], v[8 * p + 5]), pack_bf16(v[8 * p + 6], v[8 * p + 7]));
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      epi_tma_store(d, e, e.stg_ptr + tile, c, warp, d.out_col0 + lcol);
      bulk_commit();
    }
  }
}

// e4m3 output (the static-scale halo conv and the E4M3 ping-pong GEMM with d.out_e4m3): the dequantized, biased and
// activated fp32 value v of each element is quantized straight to e4m3_rn(sat(v * out_ratio)), never through bf16, and
// stored as the operand of the next E4M3 conv or linear: groups of 64 columns = 64-byte row segments (SWIZZLE_64B:
// 16-byte piece j of row r at j ^ ((r >> 1) & 3)), one {64 B, 8 px, 2 rows} (conv) or {64 B, 16 rows} (linear) bulk
// store per warp and group.  A thread's fragment gives two adjacent
// columns per row and octet, so it writes them as one 16-bit e4m3x2 at byte 32h + 8j + 2 (lane % 4) of rows lane / 4
// and lane / 4 + 8: per store instruction the eight rows of a warp fall in distinct 16-byte pieces of distinct bank
// halves, no bank conflict (tests/test_fp8_static_host.py models the layout).  Columns N .. 64 ceil(N / 64) - 1 are
// written as 0 (the consumer reads whole 64-byte chunks, and a stale byte could be an e4m3 NaN), including the second
// half of the group at block_n 32 (the host allows that width for N <= 32 only).  FULL (the E4M3 ping-pong GEMM, N a
// multiple of its 128-column tile): every column of the tile exists, so the column guards go (and with them the
// registers the multicast instantiation would otherwise spill).
__device__ __forceinline__ uint32_t e4m3x2_rn(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
template <int S, bool FULL = false>
__device__ __forceinline__ void epilogue_tile_tma_e4m3(const GemmDesc& d, EpiTma& e, const float (&acc)[S],
                                                       const TileCoord& c, int warp, int lane) {
  constexpr int BN = 2 * S;
  const int n_pad = (d.n_logical + 63) & ~63;
  const int r0 = lane >> 2, q = lane & 3;
  const uint32_t swz = (r0 >> 1) & 3;          // rows r0 and r0 + 8 share it
  const float rn = d.out_ratio;
  for (int g = 0; 64 * g < (BN < 64 ? 64 : BN); ++g) {
    const int lcol = c.n0 + g * 64;
    if (!FULL && lcol >= n_pad) break;
    const int tile = epi_stage_acquire(e, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v[16];
      if (64 * g + 32 * h < BN) {
        acc_chunk(2 * g + h, acc, v);
        epi_dequant(d, v, lcol + 32 * h + 2 * q, d.a_scale);
        epi_frag(d, v, lcol + 32 * h + 2 * q, false);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = lcol + 32 * h + 8 * j + 2 * q;
        uint32_t lo = 0, hi = 0;
        if (FULL) {
          lo = e4m3x2_rn(__fmul_rn(v[4 * j], rn), __fmul_rn(v[4 * j + 1], rn));
          hi = e4m3x2_rn(__fmul_rn(v[4 * j + 2], rn), __fmul_rn(v[4 * j + 3], rn));
        } else if (64 * g + 32 * h < BN) {
          lo = e4m3x2_rn(col < d.n_logical ? __fmul_rn(v[4 * j], rn) : 0.f,
                         col + 1 < d.n_logical ? __fmul_rn(v[4 * j + 1], rn) : 0.f);
          hi = e4m3x2_rn(col < d.n_logical ? __fmul_rn(v[4 * j + 2], rn) : 0.f,
                         col + 1 < d.n_logical ? __fmul_rn(v[4 * j + 3], rn) : 0.f);
        }
        const int b = 32 * h + 8 * j + 2 * q;  // byte within the 64-byte row segment
        const uint32_t off = static_cast<uint32_t>((((b >> 4) ^ swz) << 4) | (b & 15));
        uint8_t* t = e.stg_ptr + tile;
        *reinterpret_cast<uint16_t*>(t + r0 * 64 + off) = static_cast<uint16_t>(lo);
        *reinterpret_cast<uint16_t*>(t + (r0 + 8) * 64 + off) = static_cast<uint16_t>(hi);
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      epi_tma_store(d, e, e.stg_ptr + tile, c, warp, lcol);
      bulk_commit();
    }
  }
}

// pf_conv3_halo_e4m3_res_kernel (the DPT decoder's convs under dpt_precision 'fp8_static'): the static-scale bf16
// epilogue of the q8 kernel, v = act(fl(acc * fl(a_scale * s_w[n])) + bias[n]), then + res1, then + res2 in fp32 (the
// order of the row-per-thread epilogue), stored as bf16 through stmatrix staging and {64 ch, 8 px, 2 rows} bulk stores.
// The residuals are read in the fragment layout straight from global memory: a thread's two adjacent columns of one
// pixel are one 4-byte bf16x2 load, and the four lanes of a pixel read 16 contiguous bytes.  Every residual element is
// read exactly once, so staging it through shared memory (a TMA load, then ldmatrix) would add a barrier round trip and
// a second pass over shared memory for no reuse; the loads of a 32-column chunk are all issued before the first add.
// Pixels past W / H (and a cluster's phantom tile) read nothing; the bulk store clips them.
// d.out2 != nullptr adds the e4m3 ReLU copy q = e4m3_rn(sat(max(bf16(v), 0) * d.out_ratio)): quantized from the
// bf16-ROUNDED value, so it equals pf_quantize_e4m3_static of the bf16 output's ReLU element for element.  It is the
// q8 kernel's e4m3 output (64-byte SWIZZLE_64B staging tile, e4m3x2 stores, pad columns up to 64 ceil(N / 64) zero)
// in the warp's second staging tile (the bf16 values go to the first), stored through P.tmOut2 after the group's bf16
// store.
__device__ __forceinline__ float2 res_pair(const __nv_bfloat16* row, int col, int n) {
  if (col + 1 < n) return __bfloat1622float2(__ldg(reinterpret_cast<const __nv_bfloat162*>(row + col)));
  return make_float2(col < n ? __bfloat162float(row[col]) : 0.f, 0.f);
}
template <int S>
__device__ __forceinline__ void epilogue_tile_tma_res(const GemmDesc& d, EpiTma& e, const CUtensorMap* tm2,
                                                      const float (&acc)[S], const TileCoord& c, int warp, int lane) {
  constexpr int BN = 2 * S;
  static_assert(BN % 64 == 0, "whole 64-column groups");
  const int r0 = lane >> 2, q = lane & 3;
  // this thread's pixels: tile rows 16 warp + r0 and + 8 of the 16 x 8 pixel tile = (y0 + 2 warp + i, x0 + r0)
  const __nv_bfloat16* rrow[2][2];          // [residual][pixel], nullptr: no such residual or pixel
  {
    const int x = c.x0 + r0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int y = c.y0 + 2 * warp + i;
      const bool ok = c.img < d.NB && y < d.H && x < d.W;
      const long long pix = (static_cast<long long>(c.img) * d.H + y) * d.W + x;
      rrow[0][i] = ok && d.res1 != nullptr ? d.res1 + pix * d.res_ld : nullptr;
      rrow[1][i] = ok && d.res2 != nullptr ? d.res2 + pix * d.res_ld : nullptr;
    }
  }
  const int oct = lane >> 4;
  const uint32_t lane_off = (lane & 15) * 128;
  const int swz = lane & 7;
  const uint32_t swz8 = (r0 >> 1) & 3;
  const float rn = d.out_ratio;
  const bool copy = d.out2 != nullptr;
  const int n = d.n_logical;
  const int n_pad = (n + 63) & ~63;
  for (int g = 0; 64 * g < BN; ++g) {
    const int lcol = c.n0 + g * 64;
    if (lcol >= n_pad) break;             // (lcol is a multiple of 64: lcol < n_pad means lcol < N)
    // with the copy, the group's bf16 tile and copy tile are both filled in one pass: wait until the bulk stores of
    // the previous group have read both (the copy's bytes are then written as they are made, not held in registers)
    int tile = 0;
    if (copy) {
      if (lane == 0) bulk_wait_read0();
      __syncwarp();
    } else {
      tile = epi_stage_acquire(e, lane);
    }
    uint8_t* t8 = e.stg_ptr + kXposeWarp;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int col0 = lcol + 32 * h + 2 * q;
      uint32_t rv[2][2][4];                 // the residuals' bf16x2 pairs
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 t = rrow[r][i] != nullptr ? res_pair(rrow[r][i], col0 + 8 * j, n) : make_float2(0.f, 0.f);
            rv[r][i][j] = pack_bf16(t.x, t.y);
          }
      float v[16];
      acc_chunk(2 * g + h, acc, v);
      epi_dequant(d, v, col0, d.a_scale);
      epi_frag(d, v, col0, false);
      uint32_t pk[4][2];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float lo = v[4 * j + 2 * i], hi = v[4 * j + 2 * i + 1];
#pragma unroll
          for (int r = 0; r < 2; ++r)
            if (rrow[r][i] != nullptr) {
              const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rv[r][i][j]));
              lo += t.x; hi += t.y;
            }
          pk[j][i] = pack_bf16(lo, hi);
          if (copy) {
            const int col = col0 + 8 * j;
            const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pk[j][i]));
            const int by = 32 * h + 8 * j + 2 * q;  // byte within the 64-byte row segment
            const uint32_t off = static_cast<uint32_t>((((by >> 4) ^ swz8) << 4) | (by & 15));
            *reinterpret_cast<uint16_t*>(t8 + (r0 + 8 * i) * 64 + off) = static_cast<uint16_t>(
                e4m3x2_rn(col < n ? __fmul_rn(fmaxf(b.x, 0.f), rn) : 0.f, col + 1 < n ? __fmul_rn(fmaxf(b.y, 0.f), rn) : 0.f));
          }
        }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int o = 4 * h + 2 * p;           // octets o (lanes 0-15) and o + 1 (lanes 16-31)
        const uint32_t addr = e.stg + tile + lane_off + (((o + oct) ^ swz) << 4);
        stmatrix_x4(addr, pk[2 * p][0], pk[2 * p][1], pk[2 * p + 1][0], pk[2 * p + 1][1]);
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      epi_tma_store(d, e, e.stg_ptr + tile, c, warp, d.out_col0 + lcol);
      bulk_commit();
    }
    if (copy && lane == 0) {
      tma_store_4d(tm2, t8, lcol, c.x0, c.y0 + 2 * warp, c.img);
      bulk_commit();
    }
  }
}

// fp32 output (a_mode 0): chunks of 32 columns (128-byte row segments).  A thread writes its column pairs as 8-byte
// stores: pair j of row r is half (lane & 1) of 16-byte piece (2j + (lane % 4) / 2) ^ (r & 7) (rows r and r + 8 share
// the swizzle; a half-warp's four rows meet in two pieces, a 2-way bank conflict on 8 stores per chunk).
// The residual-stream update x += gamma * (acc + bias) stages gamma * (acc + bias) and lets the copy engine ADD it into
// x (cp.reduce.async.bulk.tensor .add.f32, performed in the L2): the SM never reads x.  Each element is updated by
// exactly one tile: deterministic.  SC = 2 (the E4M3 ping-pong GEMM): the accumulator is dequantized first, as in
// epilogue_tile_tma_bf16.
template <int S, int SC = 0>
__device__ __forceinline__ void epilogue_tile_tma_f32(const GemmDesc& d, EpiTma& e, const float (&acc)[S],
                                                      const TileCoord& c, int warp, int lane) {
  const int r = lane >> 2, q = lane & 3;
  const uint32_t lane_off = r * 128 + (q & 1) * 8;
  for (int ch = 0; 32 * ch < 2 * S; ++ch) {
    const int lcol = c.n0 + ch * 32;
    if (lcol >= d.n_logical) break;
    const int tile = epi_stage_acquire(e, lane);
    float v[16];
    acc_chunk(ch, acc, v);
    if constexpr (SC != 0) epi_dequant(d, v, lcol + 2 * q, d.a_scale);
    epi_frag(d, v, lcol + 2 * q, d.gamma != nullptr);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t addr = e.stg + tile + lane_off + (((2 * j + (q >> 1)) ^ r) << 4);
      st_shared_v2f(addr, v[4 * j], v[4 * j + 1]);
      st_shared_v2f(addr + 8 * 128, v[4 * j + 2], v[4 * j + 3]);
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      if (d.gamma != nullptr) tma_reduce_add_2d(e.tm, e.stg_ptr + tile, d.out_col0 + lcol, c.m0 + warp * 16);
      else tma_store_2d(e.tm, e.stg_ptr + tile, d.out_col0 + lcol, c.m0 + warp * 16);
      bulk_commit();
    }
  }
}

// Tile schedule.  Plain: CTA b takes tiles b, b + grid, ...  Multicast pairs (MC): cluster c takes tile PAIRS c, c + clusters, ...
// where pair p = (m-tile pair p / n_tiles, n-tile p % n_tiles) and the CTA of cluster rank r owns m-tile 2 * mp + r
// (an odd last m-tile pairs with an all-out-of-range one: TMA zero-fills it, the epilogue drops its rows).
struct TileIter {
  int first, step, count, rank, n_tiles, cl;
  __device__ __forceinline__ int tile(int i) const {
    if (cl == 1) return i;
    const int nt = i % n_tiles, mp = i / n_tiles;
    return (cl * mp + rank) * n_tiles + nt;
  }
};
// cl = CTAs per cluster sharing the weight tiles (1 = plain schedule): cluster g takes work items g, g + clusters, ...
// where item p = (m-tile group p / n_tiles, n-tile p % n_tiles) and the CTA of cluster rank r owns m-tile cl * group + r.
__device__ __forceinline__ TileIter make_iter(const GemmDesc& d, int total_tiles, int cl) {
  TileIter it;
  it.cl = cl; it.n_tiles = d.n_tiles;
  if (cl == 1) { it.first = blockIdx.x; it.step = gridDim.x; it.count = total_tiles; it.rank = 0; }
  else { it.first = blockIdx.x / cl; it.step = gridDim.x / cl; it.count = ((d.m_tiles + cl - 1) / cl) * d.n_tiles; it.rank = cluster_ctarank(); }
  return it;
}

// fused trailing layer output of one row: fp32 [rows, out3_ld], bias + activation
__device__ __forceinline__ void tail_store(const GemmDesc& d, long long orow, const float (&y2)[kMaxTail]) {
  float* op = d.out3 + orow * d.out3_ld;
#pragma unroll
  for (int i = 0; i < kMaxTail; ++i) {
    if (i < d.n2) {
      float v2 = y2[i] + (d.b2 != nullptr ? __ldg(d.b2 + i) : 0.f);
      if (d.act2 == PF_ACT_RELU) v2 = fmaxf(v2, 0.f);
      else if (d.act2 == PF_ACT_SOFTPLUS) v2 = softplus(v2);
      else if (d.act2 == PF_ACT_GELU) v2 = gelu_erf(v2);
      op[i] = v2;
    }
  }
}

// Epilogue of one tile by consumer warp `warp`: tile rows 16 warp .. 16 warp + 15, all 2 S columns.  Lanes l and
// l ^ 16 share row l & 15.  et == nullptr (halo kernel): direct stores only.
template <int S>
__device__ __forceinline__ void epilogue_tile(const GemmDesc& d, const TileCoord& c, const float (&acc)[S], int warp,
                                              int lane, float* buf, EpiTma* et) {
  const int r = 16 * warp + (lane & 15);   // accumulator row of this thread
  // ---- row mapping
  bool row_ok;
  long long orow;       // output row (pixel / token) index
  if (d.a_mode == 1) {
    const int yy = r / d.bw, xx = r - yy * d.bw;
    const int y = c.y0 + yy, x = c.x0 + xx;
    row_ok = (y < d.H) && (x < d.W) && (c.img < d.NB);     // img >= NB: the phantom tile of a multicast cluster
    orow = (static_cast<long long>(c.img) * d.H + y) * d.W + x;
  } else {
    const int m = c.m0 + r;
    row_ok = m < d.M;
    orow = m;
  }
  int ocol0 = c.n0;     // output column of accumulator column 0
  if (d.ps > 1 && d.a_mode == 0) {
    // ConvTranspose k==s: columns are ordered (ky, kx, cout); this N tile belongs to one (ky,kx).
    const int tap = c.n0 / d.ps_cout_pad;
    ocol0 = c.n0 - tap * d.ps_cout_pad;
    const int ky = tap / d.ps, kx = tap - ky * d.ps;
    const int m = c.m0 + r;
    const int img = m / (d.H * d.W);
    const int rem = m - img * d.H * d.W;
    const int y = rem / d.W, x = rem - y * d.W;
    orow = (static_cast<long long>(img) * d.H * d.ps + y * d.ps + ky) * (d.W * d.ps) + x * d.ps + kx;
  }
  // TMA epilogue for this tile?  (the V^T tiles of the fused qkv projection keep the transposing direct store)
  if (et != nullptr && d.tma_out != 0 && !(d.vt != nullptr && c.n0 >= d.vt_col0)) {
    if (d.tma_out == 2) {
      epilogue_tile_tma_f32(d, *et, acc, c, warp, lane);
    } else if constexpr (S % 32 == 0) {     // the host selects tma_out 1 only for widths of whole 64-column groups
      epilogue_tile_tma_bf16<64>(d, *et, acc, c, warp, lane);
    }
    return;
  }
  // In pf_gemm_kernel `buf` is also this warp's first TMA staging tile: a direct-store tile (the V^T tiles of the fused
  // qkv projection) may follow a TMA tile whose bulk copy is still reading it.
  if (et != nullptr && d.tma_out != 0) {
    if (lane == 0) bulk_wait_read0();
    __syncwarp();
  }
  float y2[kMaxTail];
#pragma unroll
  for (int i = 0; i < kMaxTail; ++i) y2[i] = 0.f;
  if (d.w2 == nullptr) epilogue_row<0>(d, acc, buf, lane, c, ocol0, orow, row_ok, y2);
  else if (d.n2 <= 1) epilogue_row<1>(d, acc, buf, lane, c, ocol0, orow, row_ok, y2);
  else if (d.n2 <= 4) epilogue_row<4>(d, acc, buf, lane, c, ocol0, orow, row_ok, y2);
  else epilogue_row<kMaxTail>(d, acc, buf, lane, c, ocol0, orow, row_ok, y2);
  if (d.w2 != nullptr) {
    // lanes l and l ^ 16 hold the fused trailing layer's partial sums over alternate 16-column halves of one row
#pragma unroll
    for (int i = 0; i < kMaxTail; ++i)
      if (i < d.n2) y2[i] += __shfl_xor_sync(0xffffffffu, y2[i], 16);
    if (row_ok && lane < 16) tail_store(d, orow, y2);
  }
}

// consumer warp done with a shared-memory stage: one arrival per warp, in every CTA of the cluster when the stage
// was filled by multicast
template <int CL>
__device__ __forceinline__ void release_stage(uint64_t* bar, int lane) {
  __syncwarp();
  if (lane == 0) {
    if (CL > 1) {
#pragma unroll
      for (int r = 0; r < CL; ++r) mbar_arrive_cluster(bar, r);
    } else {
      mbar_arrive(bar);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// Phase timeline of pf_gemm_kernel, pf_gemm_pp_kernel and pf_conv3_halo_kernel (built only with -DPF_GEMM_TIMELINE;
// pf_gemm_timeline reads it).  One lane per role records clock64 intervals in registers and adds them to g_gemm_timeline when its CTA retires:
// the TMA producer (slots 0-2: tiles, cycles waiting for an empty stage - halo slot or weight stage in the halo kernel -,
// cycles in its loop) and lane 0 of each consumer warpgroup's first warp (slots 3-7: tiles, cycles waiting for a full
// stage / halo slot, mainloop cycles including those waits, epilogue cycles, cycles in its loop).  All kernels add to
// the same slots: a reader takes the sums around launches of one kernel and shape.  Every other build compiles the
// stamps to nothing.
#ifdef PF_GEMM_TIMELINE
constexpr int kTimelineSlots = 8;
__device__ unsigned long long g_gemm_timeline[kTimelineSlots];
struct GemmTimeline {
  long long v[5] = {0, 0, 0, 0, 0};
  __device__ __forceinline__ long long now() const { return clock64(); }
  __device__ __forceinline__ void add(int i, long long t0) { v[i] += clock64() - t0; }
  __device__ __forceinline__ void tile() { v[0] += 1; }
  __device__ __forceinline__ void flush(int slot0, int n) const {
    for (int i = 0; i < n; ++i) atomicAdd(&g_gemm_timeline[slot0 + i], static_cast<unsigned long long>(v[i]));
  }
};
#else
struct GemmTimeline {
  __device__ __forceinline__ long long now() const { return 0; }
  __device__ __forceinline__ void add(int, long long) {}
  __device__ __forceinline__ void tile() {}
  __device__ __forceinline__ void flush(int, int) const {}
};
#endif

// MC = true: launched as clusters of 2 CTAs that take two m-tiles of the SAME n-tile; each CTA fetches half of the
// weight tile and multicasts it into both CTAs' shared memory (halves the weight traffic of the linear layers).
template <bool MC, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1) pf_gemm_kernel(const __grid_constant__ GemmKernelParams P) {
  constexpr int CL = MC ? 2 : 1;
  constexpr int stage_bytes = gemm_stage_bytes(BN);
  constexpr int stages = gemm_stages(BN);
  extern __shared__ uint8_t smem_raw[];
  const GemmDesc& d = P.d;
  // 1024-B alignment is required by SWIZZLE_128B operand tiles.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xpose = smem + stages * stage_bytes;      // [kEpiWarps][2][2 KB], 1024-B aligned (stage sizes are 1 KB multiples)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(xpose + kEpiWarps * kStageWarp);
  uint64_t* empty_bar = full_bar + stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();          // persistent kernel, all CTAs resident: let the next kernel's prologue start

  constexpr int kTmaWarp = kEpiWarps;
  if (warp == kTmaWarp && lane == 0) {
    for (int s = 0; s < d.num_src; ++s) prefetch_tmap(&P.tmA[s]);
    prefetch_tmap(&P.tmB);
    // a stage is refilled only after every consumer warp of every CTA it was multicast to released it
    for (int s = 0; s < stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kEpiWarps * CL); }
    if (d.tma_out) prefetch_tmap(&P.tmOut);
    fence_barrier_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // the peer's barriers exist before anything is multicast into its shared memory
  const TileIter it = make_iter(d, P.total_tiles, CL);
  pdl_wait();                       // predecessor's results are visible from here on

  if (warp >= kEpiWarps) {
    if (warp == kTmaWarp) {
      // ===================== TMA producer =====================
      // whole warp in uniform control flow (coordinates and stage counters in uniform registers), one elected lane issues
      GemmTimeline tl;
      const long long tl_start = tl.now();
      int stage = 0; uint32_t phase = 0;
      for (int ti = it.first; ti < it.count; ti += it.step) {
        TileCoord c = decode_tile(d, it.tile(ti));
        tl.tile();
        int kb = 0;  // running 64-wide K block index into the packed weights
        for (int s = 0; s < d.num_src; ++s) {
          for (int tap = 0; tap < d.taps; ++tap) {
            int dy = d.taps == 9 ? tap / 3 - 1 : 0;
            int dx = d.taps == 9 ? tap % 3 - 1 : 0;
            for (int ch = 0; ch < d.chunks[s]; ++ch, ++kb) {
              const long long tl_w = tl.now();
              mbar_wait(&empty_bar[stage], phase ^ 1);
              tl.add(1, tl_w);
              uint8_t* sa = smem + stage * stage_bytes;
              uint8_t* sb = sa + kATileBytes;
              if (elect_one()) {
                mbar_expect_tx(&full_bar[stage], stage_bytes);
                if (d.a_mode == 0) tma_load_2d(sa, &P.tmA[s], &full_bar[stage], ch * kBlockK, c.m0);
                else tma_load_4d(sa, &P.tmA[s], &full_bar[stage], ch * kBlockK, c.x0 + dx, c.y0 + dy, c.img);
                if (MC) {
                  constexpr int half_rows = BN / 2;
                  tma_load_2d_mc(sb + it.rank * half_rows * 128, &P.tmBh, &full_bar[stage], kb * kBlockK,
                                 c.n0 + it.rank * half_rows, static_cast<uint16_t>(3));
                } else {
                  tma_load_2d(sb, &P.tmB, &full_bar[stage], kb * kBlockK, c.n0);
                }
              }
              if (++stage == stages) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
      tl.add(2, tl_start);
      if (lane == 0) tl.flush(0, 3);
    }
  } else {
    // ===================== consumers (warps 0..7): wgmma mainloop + epilogue =====================
    EpiTma et;
    et.tm = &P.tmOut; et.stg_ptr = xpose + warp * kStageWarp; et.stg = smem_u32(et.stg_ptr); et.cur = 0;
    float* buf = reinterpret_cast<float*>(et.stg_ptr);
    const uint32_t a_off = static_cast<uint32_t>((warp >> 2) * 64 * 128);   // this warpgroup's 64 rows of the A tile
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    int rs = 0;                                             // oldest stage not yet released
    GemmTimeline tl;
    const long long tl_start = tl.now();
    for (int ti = it.first; ti < it.count; ti += it.step) {
      const TileCoord c = decode_tile(d, it.tile(ti));
      tl.tile();
      const long long tl_main = tl.now();
      uint32_t accum = 0;
      for (int kb = 0; kb < P.k_steps; ++kb) {
        const long long tl_w = tl.now();
        mbar_wait(&full_bar[stage], phase);
        tl.add(1, tl_w);
        const uint32_t sa = smem_u32(smem + stage * stage_bytes);
        const uint64_t adesc = wgmma_desc_k128(sa + a_off);
        const uint64_t bdesc = wgmma_desc_k128(sa + kATileBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) Wgmma<BN>::ss(acc, adesc + 2 * k, bdesc + 2 * k, accum | k);
        wgmma_commit();
        accum = 1;
        wgmma_wait<1>();                                    // the group of block kb - 1 is done ...
        if (kb > 0) {                                       // ... and it was the last reader of its stage
          release_stage<CL>(&empty_bar[rs], lane);
          if (++rs == stages) rs = 0;
        }
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();                                      // the tile's last block is done: its stage is free
      release_stage<CL>(&empty_bar[rs], lane);
      if (++rs == stages) rs = 0;
      tl.add(2, tl_main);
      const long long tl_epi = tl.now();
      epilogue_tile(d, c, acc, warp, lane, buf, &et);
      __syncwarp();
      tl.add(3, tl_epi);
    }
    if (lane == 0) bulk_wait0();    // the staging tiles are read (and the writes performed) before the CTA retires
    tl.add(4, tl_start);
    if (lane == 0 && (warp & 3) == 0) tl.flush(3, 5);
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // no CTA exits while its peer may still multicast into it / arrive on its barriers
}

// ------------------------------------------------------------------------------------------------------------
// Ping-pong GEMM for the plain linear layers (pf_gemm_pp_kernel, d.pp): a_mode 0, one source, N a multiple of 128, and
// an epilogue of bias -> none / GELU / ReLU with a bf16 bulk store, an fp32 bulk store, the gamma residual reduce-add,
// or the V^T third of a fused qkv projection.
//
// In pf_gemm_kernel both warpgroups finish a tile's mainloop together and then run its epilogue together, so the tensor
// cores idle for the whole epilogue (about half of a tile's time on the ViT qkv and fc1 linears).  Here consumer
// warpgroup h owns WHOLE 128 x 128 tiles: tiles 0, 2, 4, ... of the CTA's sequence go to warpgroup 0 and 1, 3, 5, ... to
// warpgroup 1, and the producer loads their K blocks in that order.  Per k16 step a warpgroup issues two
// wgmma.m64n128k16 (A rows 0-63 and 64-127, both operands from shared memory), so each B tile is read by one warpgroup
// only.  Two named barriers hand the tensor cores from one warpgroup to the other: a warpgroup starts a tile's MMAs once
// the other has issued all of the previous tile's, and while one runs its epilogue the other runs its mainloop.
// A block_n = 256 work item (the width pf_gemm chooses for the launch) is two consecutive 128-column tiles.
// A warp's accumulator rows 16w .. 16w + 15 of each 64-row half go through the same fragment-layout epilogue as
// pf_gemm_kernel's, as "warp" w and w + 4 of a 128-row tile; the V^T tiles store straight from the fragment.
constexpr int kPpStageBytes = kATileBytes + kPpBN * kBlockK * 2;      // 32 KiB: A 128 x 64 + B 128 x 64
constexpr int kPpStages = (kMaxSmem - 1024 /*align*/ - kBarBytes - kEpiWarps * kStageWarp) / kPpStageBytes;
static_assert(kPpStages == 6, "pf_gemm_pp_kernel operand ring");
constexpr int kPpTurnBar = 1;        // named barriers 1 and 2: warpgroup 0's and warpgroup 1's turn to issue MMAs

// the two consumer warpgroups (256 threads) meet on named barrier ID: one waits, the other arrives
template <int ID>
__device__ __forceinline__ void named_bar_sync256() { asm volatile("bar.sync %0, 256;" ::"n"(ID) : "memory"); }
template <int ID>
__device__ __forceinline__ void named_bar_arrive256() { asm volatile("bar.arrive %0, 256;" ::"n"(ID) : "memory"); }

// V^T third of a fused qkv projection, stored from the accumulator fragment: vt[(b * heads + h) * 64 + dd][token].
// For one column the eight lanes 4i + q (i = 0..7) hold eight consecutive tokens, 16 contiguous bytes of a V^T row
// (split where the tokens cross an image boundary, m / vt_seq).  Same bias -> activation as the row path, so the same
// bits.  32-bit offsets keep the accumulators' neighbours in registers.  SC = 2: dequantized first (E4M3 operands).
template <int S, int SC = 0>
__device__ __forceinline__ void epilogue_tile_vt(const GemmDesc& d, const float (&acc)[S], const TileCoord& c, int warp,
                                                 int lane) {
  const int q = lane & 3;
  int ro[2];               // element offset of this thread's two tokens in V^T row 0 (-1: row past M); the host
                           // takes this path only when every V^T index fits in 31 bits
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = c.m0 + 16 * warp + (lane >> 2) + 8 * h;
    const int b = m / d.vt_seq, tok = m - b * d.vt_seq;
    ro[h] = m < d.M ? b * d.vt_dim * d.vt_seq_pad + tok : -1;
  }
  for (int ch = 0; 32 * ch < 2 * S; ++ch) {
    const int lcol = c.n0 + ch * 32;
    if (lcol >= d.n_logical) break;
    float v[16];
    acc_chunk(ch, acc, v);
    if constexpr (SC != 0) epi_dequant(d, v, lcol + 2 * q, d.a_scale);
    epi_frag(d, v, lcol + 2 * q, false);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = lcol + 8 * j + 2 * q + e;
        if (n >= d.n_logical) continue;
        __nv_bfloat16* vp = d.vt + (n - d.vt_col0) * d.vt_seq_pad;
        if (ro[0] >= 0) vp[ro[0]] = __float2bfloat16(v[4 * j + e]);
        if (ro[1] >= 0) vp[ro[1]] = __float2bfloat16(v[4 * j + 2 + e]);
      }
    }
  }
}

// 64 rows x 128 columns of a pf_gemm_pp_kernel tile: rows 16 warp .. 16 warp + 15 of this consumer warp.  F8 (the E4M3
// instantiation): every output kind first takes the static-scale dequantization act(fl(acc * fl(a_scale * s_w[n])) +
// bias[n]) of the q8 halo conv, and d.out_e4m3 adds the e4m3 output (the next linear's operand matrix, 64-byte
// column groups through a uint8 tensor map: epilogue_tile_tma_e4m3 with {64 B, 16 rows} boxes).
template <bool F8, int S>
__device__ __forceinline__ void epilogue_tile_pp(const GemmDesc& d, EpiTma& et, const float (&acc)[S], const TileCoord& c,
                                                 int warp, int lane) {
  constexpr int SC = F8 ? 2 : 0;
  if (d.vt != nullptr && c.n0 >= d.vt_col0) epilogue_tile_vt<S, SC>(d, acc, c, warp, lane);
  else if (d.tma_out == 2) epilogue_tile_tma_f32<S, SC>(d, et, acc, c, warp, lane);
  else {
    if constexpr (F8) {
      if (d.out_e4m3) {
        epilogue_tile_tma_e4m3<S, true>(d, et, acc, c, warp, lane);
        return;
      }
    }
    epilogue_tile_tma_bf16<64, S, SC>(d, et, acc, c, warp, lane);
  }
}

// F8: the E4M3 instantiation (pf_gemm_pp_e4m3_kernel, d.a_e4m3 with a static input scale).  A K block is 128 e4m3
// bytes, so the A and B tiles keep their 128-byte swizzled rows, the 32 KiB stage and the six-stage ring; its four k32
// steps issue two wgmma.m64n128k32.f32.e4m3.e4m3 each, at the same descriptor offsets as the bf16 k16 steps.
template <bool MC, bool F8>
__device__ __forceinline__ void gemm_pp_body(const GemmKernelParams& P) {
  constexpr int CL = MC ? 2 : 1;
  constexpr int kKBlock = F8 ? 2 * kBlockK : kBlockK;   // K elements of one 128-byte block
  extern __shared__ uint8_t smem_raw[];
  const GemmDesc& d = P.d;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + kPpStages * kPpStageBytes;   // [kEpiWarps][2][2 KB] staging tiles, 1024-B aligned
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg + kEpiWarps * kStageWarp);
  uint64_t* empty_bar = full_bar + kPpStages;

  // warp-uniform by construction, so the warpgroup / tile / ring state derived from it lives in uniform registers
  // and the 128 accumulators leave room for the epilogue
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();

  constexpr int kTmaWarp = kEpiWarps;
  if (warp == kTmaWarp && lane == 0) {
    prefetch_tmap(&P.tmA[0]);
    prefetch_tmap(MC ? &P.tmBh : &P.tmB);
    // a stage is read by ONE warpgroup: refilled after its 4 warps in every CTA it was multicast to released it
    for (int s = 0; s < kPpStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4 * CL); }
    prefetch_tmap(&P.tmOut);
    fence_barrier_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // the peer's barriers exist before anything is multicast into its shared memory
  const TileIter it = make_iter(d, P.total_tiles, CL);
  // this CTA's tile sequence: its work items in schedule order, each split into block_n / 128 tiles (both CTAs of a
  // cluster walk the same sequence, so their warpgroups stay aligned on the multicast stages)
  const int sub_log2 = d.block_n == 2 * kPpBN ? 1 : 0;
  const int items = it.first < it.count ? (it.count - 1 - it.first) / it.step + 1 : 0;
  const int tiles = items << sub_log2;
  pdl_wait();                       // predecessor's results are visible from here on

  if (warp >= kEpiWarps) {
    if (warp == kTmaWarp) {
      // ===================== TMA producer: the K blocks of tile 0, tile 1, ... =====================
      GemmTimeline tl;
      const long long tl_start = tl.now();
      int stage = 0; uint32_t phase = 0;
      for (int p = 0; p < tiles; ++p) {
        TileCoord c = decode_tile(d, it.tile(it.first + (p >> sub_log2) * it.step));
        c.n0 += (p & sub_log2) * kPpBN;
        tl.tile();
        for (int kb = 0; kb < P.k_steps; ++kb) {
          const long long tl_w = tl.now();
          mbar_wait(&empty_bar[stage], phase ^ 1);
          tl.add(1, tl_w);
          uint8_t* sa = smem + stage * kPpStageBytes;
          uint8_t* sb = sa + kATileBytes;
          if (elect_one()) {
            mbar_expect_tx(&full_bar[stage], kPpStageBytes);
            tma_load_2d(sa, &P.tmA[0], &full_bar[stage], kb * kKBlock, c.m0);
            if (MC) {
              constexpr int half_rows = kPpBN / 2;
              tma_load_2d_mc(sb + it.rank * half_rows * 128, &P.tmBh, &full_bar[stage], kb * kKBlock,
                             c.n0 + it.rank * half_rows, static_cast<uint16_t>(3));
            } else {
              tma_load_2d(sb, &P.tmB, &full_bar[stage], kb * kKBlock, c.n0);
            }
          }
          if (++stage == kPpStages) { stage = 0; phase ^= 1; }
        }
      }
      tl.add(2, tl_start);
      if (lane == 0) tl.flush(0, 3);
    }
  } else {
    // ===================== consumer warpgroups: every other tile each, mainloops in turn =====================
    const int wg = warp >> 2, w = warp & 3;
    EpiTma et;
    et.tm = &P.tmOut; et.stg_ptr = stg + warp * kStageWarp; et.stg = smem_u32(et.stg_ptr); et.cur = 0;
    int stage = 0; uint32_t phase = 0;
    // ring position of the next block this warpgroup reads: skip n blocks (the other warpgroup's tile)
    auto skip = [&](int n) {
      stage += n;
      while (stage >= kPpStages) { stage -= kPpStages; phase ^= 1; }
    };
    skip(wg * P.k_steps);
    GemmTimeline tl;
    const long long tl_start = tl.now();
    for (int p = wg; p < tiles; p += 2) {
      TileCoord c = decode_tile(d, it.tile(it.first + (p >> sub_log2) * it.step));
      c.n0 += (p & sub_log2) * kPpBN;
      tl.tile();
      if (p > 0) {                                          // the other warpgroup has issued tile p - 1's MMAs
        if (wg == 0) named_bar_sync256<kPpTurnBar>();
        else named_bar_sync256<kPpTurnBar + 1>();
      }
      const long long tl_main = tl.now();
      // tile rows 0-63 and 64-127, declared per tile: the previous tile's values are dead once its epilogue has read
      // them (the first wgmma ignores them, scale-d = 0)
      float acc0[kPpBN / 2], acc1[kPpBN / 2];
#pragma unroll
      for (int i = 0; i < kPpBN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
      uint32_t accum = 0;
      int prev = 0;                                         // stage of the previous K block
      for (int kb = 0; kb < P.k_steps; ++kb) {
        const long long tl_w = tl.now();
        mbar_wait(&full_bar[stage], phase);
        tl.add(1, tl_w);
        const uint32_t sa = smem_u32(smem + stage * kPpStageBytes);
        const uint64_t adesc = wgmma_desc_k128(sa);
        const uint64_t adesc1 = wgmma_desc_k128(sa + 64 * 128);
        const uint64_t bdesc = wgmma_desc_k128(sa + kATileBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {          // 32-byte K steps: k16 bf16 / k32 e4m3
          if constexpr (F8) {
            Wgmma8<kPpBN>::ss(acc0, adesc + 2 * k, bdesc + 2 * k, accum | k);
            Wgmma8<kPpBN>::ss(acc1, adesc1 + 2 * k, bdesc + 2 * k, accum | k);
          } else {
            Wgmma<kPpBN>::ss(acc0, adesc + 2 * k, bdesc + 2 * k, accum | k);
            Wgmma<kPpBN>::ss(acc1, adesc1 + 2 * k, bdesc + 2 * k, accum | k);
          }
        }
        wgmma_commit();
        accum = 1;
        wgmma_wait<1>();                                    // the group of block kb - 1 is done ...
        if (kb > 0) release_stage<CL>(&empty_bar[prev], lane);   // ... and it was the last reader of its stage
        prev = stage;
        skip(1);
      }
      if (p + 1 < tiles) {                                  // the other warpgroup's turn
        if (wg == 0) named_bar_arrive256<kPpTurnBar + 1>();
        else named_bar_arrive256<kPpTurnBar>();
      }
      wgmma_wait<0>();                                      // the tile's last block is done: its stage is free
      release_stage<CL>(&empty_bar[prev], lane);
      skip(P.k_steps);                                      // tile p + 1 is the other warpgroup's
      tl.add(2, tl_main);
      const long long tl_epi = tl.now();
      epilogue_tile_pp<F8>(d, et, acc0, c, w, lane);
      epilogue_tile_pp<F8>(d, et, acc1, c, w + 4, lane);
      __syncwarp();
      tl.add(3, tl_epi);
    }
    if (lane == 0) bulk_wait0();    // the staging tiles are read (and the writes performed) before the CTA retires
    tl.add(4, tl_start);
    if (lane == 0 && w == 0) tl.flush(3, 5);
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // no CTA exits while its peer may still multicast into it / arrive on its barriers
}

template <bool MC>
__global__ void __launch_bounds__(kGemmThreads, 1) pf_gemm_pp_kernel(const __grid_constant__ GemmKernelParams P) {
  gemm_pp_body<MC, false>(P);
}
template <bool MC>
__global__ void __launch_bounds__(kGemmThreads, 1) pf_gemm_pp_e4m3_kernel(const __grid_constant__ GemmKernelParams P) {
  gemm_pp_body<MC, true>(P);
}

// ------------------------------------------------------------------------------------------------------------
// 3x3 convolution with a shared-memory HALO tile (stride 1, zero pad 1).
//
// The generic kernel above fetches the A operand once per tap: 9 TMA boxes of 16 KB per 64-channel chunk, all hitting
// the same pixels.  Here one TMA box {64 ch, 10, 18, 1} brings the (16+2) x (8+2) pixel neighbourhood of a 16x8
// output tile (23 KB) and all nine taps are issued from it: for tap (dy,dx) accumulator row r = 8 yy + xx reads halo
// pixel (yy + dy) * 10 + xx + dx, so the consumers' ldmatrix row addresses simply shift per tap (the 128B-swizzle XOR
// is a function of the shared-memory address bits, so shifted rows of a TMA-written tile are read the same way).
// A traffic from L2 drops 6.3x; the weights stream per (chunk, tap) as before.
//
// Consumers split the tile by ROWS: warpgroup h owns tile rows 64h .. 64h + 63 (pixel rows 8h .. 8h + 7) and all BN
// columns, warp w rows 16w .. 16w + 15.  Each warp loads its A rows once per tap and each warpgroup issues one
// m64nBNk16 per k16 step.  BN is a template parameter, so every wgmma has a fixed shape and none sits under a
// data-dependent branch: the last n-tile issues all BN columns (the packed weight rows beyond N are zero) and the
// zero-padded last 64-channel chunk of a source issues all four k16 steps (its pad channels are TMA zero fill, or
// zeros written by the resample warps).  The mainloop keeps one tap's wgmma group in flight while the next tap's A
// fragments load.
constexpr int kHaloW = 10, kHaloH = 18;
constexpr int kHaloBytes = kHaloW * kHaloH * 128;          // 23040
constexpr int kHaloSlot = 24 * 1024;                        // 1024-B aligned slot
constexpr int kHaloSlots = 3;
// The FP8 instantiation (F8: e4m3 operands) keeps the 64-channel chunk, so a pixel of the halo is a 64-byte row
// (SWIZZLE_64B): 11520-byte halo tiles in 12 KB slots and BN x 64-byte weight tap tiles.  What it saves goes to the
// weight ring.  EB = bytes per element.
__host__ __device__ constexpr int halo_slot(bool f8) { return f8 ? 12 * 1024 : kHaloSlot; }
__host__ __device__ constexpr int halo_bytes(bool f8) { return f8 ? kHaloW * kHaloH * 64 : kHaloBytes; }
// shared memory left for the weight ring next to the halo slots, the epilogue staging tiles and barriers
__host__ __device__ constexpr int halo_bbytes(bool f8) {
  return kMaxSmem - 1024 /*align*/ - kBarBytes - kEpiWarps * kStageWarp - kHaloSlots * halo_slot(f8);
}
constexpr int kHaloBBytes = halo_bbytes(false);
// taps per weight stage: amortise the per-stage barrier round trip over several taps while two stages still fit
__host__ __device__ constexpr int halo_kc(int bn, bool f8 = false) {
  return 2 * 9 * bn * kBlockK * (f8 ? 1 : 2) <= halo_bbytes(f8) ? 9
                                                                 : (2 * 3 * bn * kBlockK * (f8 ? 1 : 2) <= halo_bbytes(f8) ? 3 : 1);
}
// weight ring depth: as many stages of halo_kc taps as fit (at least two by the choice of halo_kc), at most six
__host__ __device__ constexpr int halo_stages(int bn, bool f8 = false) {
  return halo_bbytes(f8) / (halo_kc(bn, f8) * bn * kBlockK * (f8 ? 1 : 2)) < 6
             ? halo_bbytes(f8) / (halo_kc(bn, f8) * bn * kBlockK * (f8 ? 1 : 2))
             : 6;
}
// The second staging tile per warp costs no weight stage and no taps per stage at any width
static_assert(halo_kc(32) == 9 && halo_stages(32) == 3 && halo_kc(64) == 3 && halo_stages(64) == 5 &&
                  halo_kc(128) == 3 && halo_stages(128) == 2 && halo_kc(192) == 1 && halo_stages(192) == 5,
              "halo weight ring");
static_assert(halo_kc(32, true) == 9 && halo_stages(32, true) == 6 && halo_kc(64, true) == 9 && halo_stages(64, true) == 4 &&
                  halo_kc(128, true) == 9 && halo_stages(128, true) == 2 && halo_kc(192, true) == 3 &&
                  halo_stages(192, true) == 4,
              "FP8 halo weight ring");


// ---- fused bilinear resample (align_corners=True) of a halo-kernel source -------------------------------------------
// F.interpolate(x, (H, W), mode='bilinear', align_corners=True) feeding a 3x3 conv (guided_fusion_model.py:98-99,
// 191-203) used to be materialised by resize_bilinear_tiled_kernel (5 % of the step, written once and read back by the
// conv).  Instead a producer warp builds the 18 x 10 pixel halo of one 64-channel chunk directly in the swizzled
// operand tile TMA would have written: lane -> (halo pixel, 8-channel piece), four 16-byte taps from the low-resolution
// map (L1/L2 resident: the taps of neighbouring pixels overlap), the same fp32 blend and bf16 rounding as the
// stand-alone kernel, zeros for the conv padding ring / pad channels.  Same source coordinate as ATen: scale * dst.
__device__ __forceinline__ void rs_coord(int dst, int in, float scale, int& lo, int& hi, float& frac) {
  const float src = scale * dst;
  lo = static_cast<int>(src);
  if (lo > in - 1) lo = in - 1;
  hi = lo + (lo < in - 1 ? 1 : 0);
  frac = src - lo;
}
__device__ __forceinline__ void halo_fill_bilinear(uint32_t slot, const GemmDesc& d, int s, int ch, const TileCoord& c, int lane) {
  const int ih = d.rs_h[s], iw = d.rs_w[s], ld = d.rs_ld[s];
  const __nv_bfloat16* src = d.rs_ptr[s] + static_cast<size_t>(c.img) * ih * iw * ld + ch * kBlockK;
  const int cvalid = d.k_true[s] - ch * kBlockK;            // channels of this chunk that exist (multiple of 8)
  const float sy = d.rs_sy[s], sx = d.rs_sx[s];
  const int j = lane & 7;                                    // 16-byte piece (8 channels) of the pixel's 128-byte row
  const bool jok = j * 8 < cvalid && c.img < d.NB;
#pragma unroll 5
  for (int p = lane >> 3; p < kHaloW * kHaloH; p += 4) {
    const int hy = p / kHaloW, hx = p - hy * kHaloW;
    const int Y = c.y0 - 1 + hy, X = c.x0 - 1 + hx;
    uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
    if (jok && Y >= 0 && Y < d.H && X >= 0 && X < d.W) {
      int y0, y1, x0, x1; float fy, fx;
      rs_coord(Y, ih, sy, y0, y1, fy);
      rs_coord(X, iw, sx, x0, x1, fx);
      const __nv_bfloat16* r0 = src + static_cast<size_t>(y0) * iw * ld + j * 8;
      const __nv_bfloat16* r1 = src + static_cast<size_t>(y1) * iw * ld + j * 8;
      const uint4 ua = __ldg(reinterpret_cast<const uint4*>(r0 + static_cast<size_t>(x0) * ld));
      const uint4 ub = __ldg(reinterpret_cast<const uint4*>(r0 + static_cast<size_t>(x1) * ld));
      const uint4 uc = __ldg(reinterpret_cast<const uint4*>(r1 + static_cast<size_t>(x0) * ld));
      const uint4 ud = __ldg(reinterpret_cast<const uint4*>(r1 + static_cast<size_t>(x1) * ld));
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
      o0 = ow[0]; o1 = ow[1]; o2 = ow[2]; o3 = ow[3];
    }
    st_shared_v4(slot + p * 128 + ((j ^ (p & 7)) << 4), o0, o1, o2, o3);
  }
}

// A fragments of one tap for this warp's 16 rows: lane l addresses its row (ra = the row's 128-byte halo pixel),
// 16-byte chunk 2k + (l >> 4) of k16 step k (SWIZZLE_128B: chunk j of the row at address a sits at j ^ ((a >> 7) & 7)).
__device__ __forceinline__ void halo_a_frags(uint32_t ra, int lane, uint32_t (&fa)[4][4]) {
  const uint32_t sw = (ra >> 7) & 7;
#pragma unroll
  for (int k = 0; k < kBlockK / 16; ++k) ldmatrix_x4(ra + (((2 * k + (lane >> 4)) ^ sw) << 4), fa[k]);
}
// FP8: the row is a 64-byte e4m3 halo pixel, k32 step k is 16-byte chunks 2k, 2k + 1 (SWIZZLE_64B: chunk j of the row at
// address a sits at j ^ ((a >> 7) & 3)).  The .b16 fragment of a 32-byte k slice is the k32 e4m3 A fragment (Wgmma8).
__device__ __forceinline__ void halo_a_frags(uint32_t ra, int lane, uint32_t (&fa)[2][4]) {
  const uint32_t sw = (ra >> 7) & 3;
#pragma unroll
  for (int k = 0; k < 2; ++k) ldmatrix_x4(ra + (((2 * k + (lane >> 4)) ^ sw) << 4), fa[k]);
}

// CL > 1: clusters of CL (2 or 4) CTAs take CL m-tiles (pixel tiles) of the SAME n-tile; each CTA fetches 1/CL of the rows
// of every weight tile and multicasts it into all of them.  The weights are ~90 % of this kernel's L2 -> SM traffic (one
// 23 KB halo against nine 4-24 KB tap tiles per 64-channel chunk).
//
// F8: the E4M3 instantiation (pf_conv3_halo_e4m3_kernel, d.a_e4m3).  The sources are 64-channel segments of one e4m3
// map, each k16 step becomes a k32 step (two per tap, wgmma.m64nBNk32.f32.e4m3.e4m3 with A from registers) and the
// plain-output epilogue multiplies the accumulator by s_a[image] * s_w[column] before the bias.
//
// Q8 (F8 only): the static-scale instantiation (pf_conv3_halo_e4m3_q8_kernel, d.a_static): one input scale d.a_scale
// for the launch, and either the bf16 output or (d.out_e4m3) the e4m3 operand map of the next conv.
// RES (Q8 only): pf_conv3_halo_e4m3_res_kernel, the bf16 output with residuals and the e4m3 ReLU copy
// (epilogue_tile_tma_res).
template <int CL, int BN, bool F8, bool Q8 = false, bool RES = false>
__device__ __forceinline__ void conv3_halo_body(const GemmKernelParams& P) {
  constexpr bool MC = CL > 1;
  constexpr uint16_t kMask = static_cast<uint16_t>((1u << CL) - 1);
  constexpr int EB = F8 ? 1 : 2;                            // bytes per operand element
  constexpr int kRow = kBlockK * EB;                        // bytes of one pixel / weight row of a 64-channel chunk
  constexpr int kc = halo_kc(BN, F8);                       // taps per B stage
  constexpr int b_tile_bytes = BN * kRow;
  constexpr int b_stage_bytes = kc * b_tile_bytes;
  constexpr int stages = halo_stages(BN, F8);               // B ring
  constexpr int kSlot = halo_slot(F8);
  constexpr int kKSteps = F8 ? 2 : kBlockK / 16;            // MMAs per tap
  extern __shared__ uint8_t smem_raw[];
  const GemmDesc& d = P.d;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_b = smem + kHaloSlots * kSlot;
  uint8_t* xpose = smem_b + stages * b_stage_bytes;         // [kEpiWarps][2][2 KB] staging tiles, 1024-B aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(xpose + kEpiWarps * kStageWarp);
  uint64_t* a_full = bars;                                  // [kHaloSlots]
  uint64_t* a_empty = a_full + kHaloSlots;
  uint64_t* b_full = a_empty + kHaloSlots;                  // [stages]
  uint64_t* b_empty = b_full + stages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  constexpr int kTmaWarp = kRsWarp0 + 2;
  if (warp == kTmaWarp && lane == 0) {
    for (int s = 0; s < d.num_src; ++s) if (d.rs_h[s] == 0) prefetch_tmap(&P.tmA[s]);
    prefetch_tmap(&P.tmB);
    for (int s = 0; s < kHaloSlots; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], kEpiWarps); }
    // a multicast weight stage is refilled only after the consumers of ALL CTAs of the cluster released it
    for (int s = 0; s < stages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], kEpiWarps * CL); }
    if (d.tma_out) prefetch_tmap(&P.tmOut);
    if (RES && d.out2 != nullptr) prefetch_tmap(&P.tmOut2);
    fence_barrier_init();
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // the peers' barriers exist before anything is multicast into their shared memory
  const TileIter it = make_iter(d, P.total_tiles, CL);
  pdl_wait();                       // predecessor's results are visible from here on

  if (warp >= kEpiWarps) {
    if (warp == kTmaWarp) {
      // whole warp in uniform control flow, one elected lane issues the copies
      GemmTimeline tl;
      const long long tl_start = tl.now();
      int as = 0; uint32_t aph = 0;
      int bs = 0; uint32_t bph = 0;
      for (int ti = it.first; ti < it.count; ti += it.step) {
        TileCoord c = decode_tile(d, it.tile(ti));
        tl.tile();
        int kbase = 0;                                       // first 64-wide K block of this source in the weights
        int cbase = 0;                                       // F8: first 64-channel chunk of this source in the map
        for (int s = 0; s < d.num_src; ++s) {
          const int nch = d.chunks[s];
          for (int ch = 0; ch < nch; ++ch) {
            if (d.rs_h[s] == 0) {                            // (resampled sources: the producer warps own the slot)
              const long long tl_w = tl.now();
              mbar_wait(&a_empty[as], aph ^ 1);
              tl.add(1, tl_w);
              if (elect_one()) {
                mbar_expect_tx(&a_full[as], halo_bytes(F8));
                tma_load_4d(smem + as * kSlot, &P.tmA[s], &a_full[as], (F8 ? cbase + ch : ch) * kBlockK, c.x0 - 1,
                            c.y0 - 1, c.img);
              }
            }
            if (++as == kHaloSlots) { as = 0; aph ^= 1; }
            for (int tap0 = 0; tap0 < 9; tap0 += kc) {
              const long long tl_w = tl.now();
              mbar_wait(&b_empty[bs], bph ^ 1);
              tl.add(1, tl_w);
              if (elect_one()) {
                mbar_expect_tx(&b_full[bs], b_stage_bytes);
                if (MC) {
                  constexpr int part_rows = BN / CL;
                  for (int j = 0; j < kc; ++j)
                    tma_load_2d_mc(smem_b + bs * b_stage_bytes + j * b_tile_bytes + it.rank * part_rows * kRow, &P.tmBh,
                                   &b_full[bs], (kbase + (tap0 + j) * nch + ch) * kBlockK, c.n0 + it.rank * part_rows,
                                   kMask);
                } else {
                  for (int j = 0; j < kc; ++j)
                    tma_load_2d(smem_b + bs * b_stage_bytes + j * b_tile_bytes, &P.tmB, &b_full[bs],
                                (kbase + (tap0 + j) * nch + ch) * kBlockK, c.n0);
                }
              }
              if (++bs == stages) { bs = 0; bph ^= 1; }
            }
          }
          kbase += 9 * nch;
          cbase += nch;
        }
      }
      tl.add(2, tl_start);
      if (lane == 0) tl.flush(0, 3);
    } else if (warp < kRsWarp0 + 2 && d.rs_any) {
      // ===================== resample producers: halo tiles of the sources read through a bilinear resample =====================
      int as = 0; uint32_t aph = 0;
      int turn = 0;                                          // the two warps take alternate resampled chunks
      for (int ti = it.first; ti < it.count; ti += it.step) {
        TileCoord c = decode_tile(d, it.tile(ti));
        for (int s = 0; s < d.num_src; ++s) {
          for (int ch = 0; ch < d.chunks[s]; ++ch) {
            if (d.rs_h[s] != 0) {
              if ((turn & 1) == warp - kRsWarp0) {
                mbar_wait(&a_empty[as], aph ^ 1);
                if constexpr (!F8) halo_fill_bilinear(smem_u32(smem + as * kSlot), d, s, ch, c, lane);
                __syncwarp();
                if (lane == 0) mbar_arrive(&a_full[as]);
              }
              ++turn;
            }
            if (++as == kHaloSlots) { as = 0; aph ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== consumers (warps 0..7): wgmma over the nine shifted views of each halo tile + epilogue =====
    EpiTma et;
    et.tm = &P.tmOut; et.stg_ptr = xpose + warp * kStageWarp; et.stg = smem_u32(et.stg_ptr); et.cur = 0;
    float* buf = reinterpret_cast<float*>(et.stg_ptr);
    const int arow = 16 * warp + (lane & 15);               // tile row this lane addresses for ldmatrix
    const uint32_t a_off = static_cast<uint32_t>(((arow >> 3) * kHaloW + (arow & 7)) * kRow);
    float acc[BN / 2];
    uint32_t fa[2][kKSteps][4];                             // A fragments of two taps: one loads while the other is read
    int as = 0; uint32_t aph = 0;
    int bs = 0; uint32_t bph = 0;
    int rbs = 0;                                            // oldest B stage not yet released
    GemmTimeline tl;
    const long long tl_start = tl.now();
    for (int ti = it.first; ti < it.count; ti += it.step) {
      const TileCoord c = decode_tile(d, it.tile(ti));
      tl.tile();
      const long long tl_main = tl.now();
      uint32_t accum = 0;
      for (int s = 0; s < d.num_src; ++s) {
        for (int ch = 0; ch < d.chunks[s]; ++ch) {
          long long tl_w = tl.now();
          mbar_wait(&a_full[as], aph);
          tl.add(1, tl_w);
          const uint32_t a_base = smem_u32(smem + as * kSlot) + a_off;
          uint32_t sb = 0;
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            if (tap % kc == 0) {
              tl_w = tl.now();
              mbar_wait(&b_full[bs], bph);
              tl.add(1, tl_w);
              sb = smem_u32(smem_b + bs * b_stage_bytes);
              if (++bs == stages) { bs = 0; bph ^= 1; }
            }
            // fa[tap & 1] was last read by the group of tap - 2, retired by the wait below at tap - 1
            halo_a_frags(a_base + static_cast<uint32_t>(((tap / 3) * kHaloW + tap % 3) * kRow), lane, fa[tap & 1]);
            const uint64_t bdesc = F8 ? wgmma_desc_k64(sb + (tap % kc) * b_tile_bytes)
                                      : wgmma_desc_k128(sb + (tap % kc) * b_tile_bytes);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kKSteps; ++k) {
              if constexpr (F8) Wgmma8<BN>::rs(acc, fa[tap & 1][k], bdesc + 2 * k, accum | k);
              else Wgmma<BN>::rs(acc, fa[tap & 1][k], bdesc + 2 * k, accum | k);
            }
            wgmma_commit();
            accum = 1;
            wgmma_wait<1>();                                 // the group of tap - 1 is done
            if (tap > 0 && tap % kc == 0) {                  // ... and it was the last reader of its B stage
              release_stage<CL>(&b_empty[rbs], lane);
              if (++rbs == stages) rbs = 0;
            }
          }
          wgmma_wait<0>();                                   // tap 8 is done: its B stage and the halo slot are free
          release_stage<CL>(&b_empty[rbs], lane);
          if (++rbs == stages) rbs = 0;
          release_stage<1>(&a_empty[as], lane);
          if (++as == kHaloSlots) { as = 0; aph ^= 1; }
        }
      }
      tl.add(2, tl_main);
      const long long tl_epi = tl.now();
      // plain bf16 outputs (the host sets tma_out for the whole launch): fragment layout, stmatrix staging, bulk
      // stores of {G ch, 8 px, 2 rows} boxes (TMA clips pixels past W / H, columns past the output and the phantom
      // img >= NB tile of a cluster); everything else row per thread
      if constexpr (RES) {
        epilogue_tile_tma_res(d, et, &P.tmOut2, acc, c, warp, lane);
      } else if constexpr (Q8) {
        if (d.out_e4m3) epilogue_tile_tma_e4m3(d, et, acc, c, warp, lane);
        else epilogue_tile_tma_bf16<BN == 32 ? 32 : 64, BN / 2, 2>(d, et, acc, c, warp, lane);
      } else if constexpr (F8) epilogue_tile_tma_bf16<BN == 32 ? 32 : 64, BN / 2, 1>(d, et, acc, c, warp, lane);
      else if (d.tma_out) epilogue_tile_tma_bf16<BN == 32 ? 32 : 64>(d, et, acc, c, warp, lane);
      else epilogue_tile(d, c, acc, warp, lane, buf, nullptr);
      __syncwarp();
      tl.add(3, tl_epi);
    }
    if (lane == 0) bulk_wait0();    // the staging tiles are read (and the writes performed) before the CTA retires
    tl.add(4, tl_start);
    if (lane == 0 && (warp & 3) == 0) tl.flush(3, 5);
  }
  __syncthreads();
  if (MC) cluster_sync_all();       // no CTA exits while its peer may still multicast into it / arrive on its barriers
}

template <int CL, int BN>
__global__ void __launch_bounds__(kHaloThreads, 1) pf_conv3_halo_kernel(const __grid_constant__ GemmKernelParams P) {
  conv3_halo_body<CL, BN, false>(P);
}
template <int CL, int BN>
__global__ void __launch_bounds__(kHaloThreads, 1) pf_conv3_halo_e4m3_kernel(const __grid_constant__ GemmKernelParams P) {
  conv3_halo_body<CL, BN, true>(P);
}
template <int CL, int BN>
__global__ void __launch_bounds__(kHaloThreads, 1) pf_conv3_halo_e4m3_q8_kernel(const __grid_constant__ GemmKernelParams P) {
  conv3_halo_body<CL, BN, true, true>(P);
}
template <int CL, int BN>
__global__ void __launch_bounds__(kHaloThreads, 1) pf_conv3_halo_e4m3_res_kernel(const __grid_constant__ GemmKernelParams P) {
  conv3_halo_body<CL, BN, true, true, true>(P);
}


// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
static int g_sm_counts[kMaxDevices] = {0};

using KernelFn = void (*)(GemmKernelParams);
// pf_conv3_halo_kernel<CL, bn>, nullptr for a width without an instantiation
template <int CL, bool F8>
static KernelFn halo_kernel_cl(int bn) {
  switch (bn) {
    case 32: return F8 ? pf_conv3_halo_e4m3_kernel<CL, 32> : pf_conv3_halo_kernel<CL, 32>;
    case 64: return F8 ? pf_conv3_halo_e4m3_kernel<CL, 64> : pf_conv3_halo_kernel<CL, 64>;
    case 128: return F8 ? pf_conv3_halo_e4m3_kernel<CL, 128> : pf_conv3_halo_kernel<CL, 128>;
    case 192: return F8 ? pf_conv3_halo_e4m3_kernel<CL, 192> : pf_conv3_halo_kernel<CL, 192>;
    default: return nullptr;
  }
}
template <int CL>
static KernelFn halo_q8_kernel_cl(int bn) {
  switch (bn) {
    case 32: return pf_conv3_halo_e4m3_q8_kernel<CL, 32>;
    case 64: return pf_conv3_halo_e4m3_q8_kernel<CL, 64>;
    case 128: return pf_conv3_halo_e4m3_q8_kernel<CL, 128>;
    case 192: return pf_conv3_halo_e4m3_q8_kernel<CL, 192>;
    default: return nullptr;
  }
}
// the DPT decoder's widths: N = C = 64 / 128 / 256 (two 128-column n-tiles) and output_conv1's C / 2 = 64 / 128
template <int CL>
static KernelFn halo_res_kernel_cl(int bn) {
  switch (bn) {
    case 64: return pf_conv3_halo_e4m3_res_kernel<CL, 64>;
    case 128: return pf_conv3_halo_e4m3_res_kernel<CL, 128>;
    default: return nullptr;
  }
}
template <bool F8>
static KernelFn halo_kernel_t(int cl, int bn) {
  return cl == 4 ? halo_kernel_cl<4, F8>(bn) : (cl == 2 ? halo_kernel_cl<2, F8>(bn) : halo_kernel_cl<1, F8>(bn));
}
// q8: pf_conv3_halo_e4m3_q8_kernel (static input scale), f8 must be set too; res: pf_conv3_halo_e4m3_res_kernel, q8 too
static KernelFn halo_kernel(int cl, int bn, bool f8 = false, bool q8 = false, bool res = false) {
  if (res) return cl == 4 ? halo_res_kernel_cl<4>(bn) : (cl == 2 ? halo_res_kernel_cl<2>(bn) : halo_res_kernel_cl<1>(bn));
  if (q8) return cl == 4 ? halo_q8_kernel_cl<4>(bn) : (cl == 2 ? halo_q8_kernel_cl<2>(bn) : halo_q8_kernel_cl<1>(bn));
  return f8 ? halo_kernel_t<true>(cl, bn) : halo_kernel_t<false>(cl, bn);
}
// pf_gemm_kernel<MC, bn> for the widths of kGemmWidths, nullptr otherwise
template <bool MC>
static KernelFn gemm_kernel_mc(int bn) {
  switch (bn) {
    case 32: return pf_gemm_kernel<MC, 32>;
    case 64: return pf_gemm_kernel<MC, 64>;
    case 96: return pf_gemm_kernel<MC, 96>;
    case 128: return pf_gemm_kernel<MC, 128>;
    case 192: return pf_gemm_kernel<MC, 192>;
    case 256: return pf_gemm_kernel<MC, 256>;
    default: return nullptr;
  }
}
static KernelFn gemm_kernel(bool mc, int bn) { return mc ? gemm_kernel_mc<true>(bn) : gemm_kernel_mc<false>(bn); }
static KernelFn gemm_pp_kernel(bool mc, bool f8 = false) {
  if (f8) return mc ? pf_gemm_pp_e4m3_kernel<true> : pf_gemm_pp_e4m3_kernel<false>;
  return mc ? pf_gemm_pp_kernel<true> : pf_gemm_pp_kernel<false>;
}

int gemm_launch(const GemmDesc& d, const CUtensorMap* tmA, const CUtensorMap& tmB, const CUtensorMap* tmBh,
                const CUtensorMap* tmOut, cudaStream_t stream, const CUtensorMap* tmOut2) {
  static bool attr_done[kMaxDevices] = {false};
  const int dev = current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaSuccess;
    for (bool mc : {false, true})
      for (int bn : kGemmWidths)
        if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_kernel(mc, bn), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    for (bool mc : {false, true})
      for (bool f8 : {false, true})
        if (e == cudaSuccess) e = cudaFuncSetAttribute(gemm_pp_kernel(mc, f8), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    for (int v = 0; v < 3; ++v)
      for (int cl : {1, 2, 4})
        for (int bn : {32, 64, 128, 192})
          if (e == cudaSuccess)
            e = cudaFuncSetAttribute(halo_kernel(cl, bn, v > 0, v > 1), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    for (int cl : {1, 2, 4})
      for (int bn : {64, 128})
        if (e == cudaSuccess)
          e = cudaFuncSetAttribute(halo_kernel(cl, bn, true, true, true), cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (e != cudaSuccess) return set_error("cudaFuncSetAttribute(gemm kernels): %s", cudaGetErrorString(e));
    cudaDeviceGetAttribute(&g_sm_counts[dev], cudaDevAttrMultiProcessorCount, dev);
    attr_done[dev] = true;
  }
  const int g_sm_count = g_sm_counts[dev];
  // the static-scale E4M3 conv with residuals or an e4m3 ReLU copy (pf_gemm sets out2 there only with out2_e4m3)
  const bool res8 = d.halo && d.a_e4m3 && d.a_static && (d.res1 != nullptr || d.res2 != nullptr || d.out2 != nullptr);
  {
    const long long rows = d.a_mode == 1 ? static_cast<long long>(d.NB) * d.H * d.W : d.M;
    int ktrue = 0;
    for (int s = 0; s < d.num_src; ++s) ktrue += d.k_true[s];
    const int n_true = d.ps > 1 ? d.n_logical * d.ps * d.ps : d.N;
    note_work(2.0 * rows * ktrue * d.taps * n_true, "%s rows%lld K%dx%d N%d%s%s%s", d.taps == 9 ? (d.a_e4m3 ? (d.a_static ? (d.out_e4m3 ? "conv3x3_e4m3_static_q8out" : (res8 ? "conv3x3_e4m3_static_res" : "conv3x3_e4m3_static")) : "conv3x3_e4m3") : "conv3x3") : (d.a_mode == 1 ? "conv1x1" : (d.ps > 1 ? "convT" : (d.a_e4m3 ? (d.out_e4m3 ? "linear_e4m3_q8out" : "linear_e4m3") : "linear"))),
              rows, d.taps, ktrue, n_true, d.act ? (d.act == PF_ACT_GELU ? " gelu" : (d.act == PF_ACT_RELU ? " relu" : " softplus")) : "",
              d.gamma ? " gamma" : (d.vt ? " vt" : ""), d.w2 ? " tail" : "");
  }
  GemmKernelParams P;
  for (int s = 0; s < d.num_src; ++s) P.tmA[s] = tmA[s];
  for (int s = d.num_src; s < 3; ++s) P.tmA[s] = tmA[0];
  P.tmB = tmB;
  P.tmBh = tmBh ? *tmBh : tmB;
  P.tmOut = tmOut ? *tmOut : tmB;
  P.tmOut2 = tmOut2 ? *tmOut2 : tmB;
  P.d = d;
  if (d.tma_out && !tmOut) return set_error("gemm: tma_out without an output tensor map");
  int ks = 0;
  for (int s = 0; s < d.num_src; ++s) ks += d.chunks[s] * d.taps;
  const bool pp8 = d.pp && d.a_e4m3;
  if (pp8) ks = d.k_true[0] / (2 * kBlockK);       // 128-byte K blocks of e4m3 (the host checks K % 128 == 0)
  P.k_steps = ks;
  P.total_tiles = d.m_tiles * d.n_tiles;
  if (P.total_tiles <= 0 || ks <= 0) return set_error("gemm: empty problem");
  int grid = P.total_tiles < g_sm_count ? P.total_tiles : g_sm_count;
  if (d.halo) {
    const bool f8 = d.a_e4m3 != 0, q8 = f8 && d.a_static != 0;
    const KernelFn hk = halo_kernel(d.halo_cl, d.block_n, f8, q8, res8);
    if (hk == nullptr)
      return set_error("conv3 halo: block_n %d (32, 64, 128 or 192; 64 or 128 with residuals or a ReLU copy)", d.block_n);
    const int b_bytes = halo_kc(d.block_n, f8) * d.block_n * kBlockK * (f8 ? 1 : 2);     // one weight stage
    const int hstages = halo_stages(d.block_n, f8);
    size_t hsmem = 1024 + static_cast<size_t>(kHaloSlots) * halo_slot(f8) + static_cast<size_t>(hstages) * b_bytes +
                   kEpiWarps * kStageWarp + kBarBytes;
    cudaError_t le;
    if (tmBh != nullptr) {
      // weight-multicast clusters of cl CTAs over (m-tile group, n-tile) work items.  Every CTA is persistent, so the grid
      // must not exceed what is co-resident: ask the driver how many clusters of this shape fit (GPC boundaries).
      const int cl = d.halo_cl;
      const int groups = ((d.m_tiles + cl - 1) / cl) * d.n_tiles;
      cudaLaunchConfig_t cfg = {};
      cfg.blockDim = dim3(kHaloThreads); cfg.dynamicSmemBytes = hsmem; cfg.stream = stream;
      cudaLaunchAttribute at[2];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[1].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      static int max_clusters[kMaxDevices][4][5] = {};
      int (&mcl)[5] = max_clusters[dev][res8 ? 3 : (q8 ? 2 : (f8 ? 1 : 0))];
      if (mcl[cl] == 0) {
        cfg.gridDim = dim3(cl * (g_sm_count / cl));
        int n = 0;
        cudaError_t qe = cudaOccupancyMaxActiveClusters(&n, hk, &cfg);
        if (qe != cudaSuccess || n < 1) { cudaGetLastError(); n = g_sm_count / cl; }
        mcl[cl] = n < g_sm_count / cl ? n : g_sm_count / cl;
      }
      const int clusters = groups < mcl[cl] ? groups : mcl[cl];
      cfg.gridDim = dim3(cl * clusters);
      cfg.numAttrs = pdl_enabled() ? 2 : 1;
      le = cudaLaunchKernelEx(&cfg, hk, P);
    } else {
      le = launch_pdl(hk, dim3(grid), dim3(kHaloThreads), hsmem, stream, P);
    }
    if (le != cudaSuccess)
      return set_error("%s launch: %s", res8 ? "pf_conv3_halo_e4m3_res_kernel" : (q8 ? "pf_conv3_halo_e4m3_q8_kernel" : (f8 ? "pf_conv3_halo_e4m3_kernel" : "pf_conv3_halo_kernel")),
                       cudaGetErrorString(le));
  } else {
    if (d.pp && (d.block_n % kPpBN != 0 || d.num_src != 1 || d.a_mode != 0 || !d.tma_out))
      return set_error("gemm: the ping-pong kernel takes plain linear layers at block_n 128 / 256 (block_n %d)", d.block_n);
    const KernelFn gk = d.pp ? gemm_pp_kernel(tmBh != nullptr, pp8) : gemm_kernel(tmBh != nullptr, d.block_n);
    if (gk == nullptr) return set_error("gemm: block_n %d (32, 64, 96, 128, 192 or 256)", d.block_n);
    const size_t smem = 1024 + (d.pp ? static_cast<size_t>(kPpStages) * kPpStageBytes
                                     : static_cast<size_t>(gemm_stages(d.block_n)) * gemm_stage_bytes(d.block_n)) +
                        kEpiWarps * kStageWarp + kBarBytes;
    cudaError_t le;
    if (tmBh != nullptr) {
      // weight-multicast pairs: clusters of 2 CTAs over (m-tile pair, n-tile) work items
      const int pairs = ((d.m_tiles + 1) / 2) * d.n_tiles;
      const int clusters = pairs < g_sm_count / 2 ? pairs : g_sm_count / 2;
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(2 * clusters); cfg.blockDim = dim3(kGemmThreads); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
      cudaLaunchAttribute at[2];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      at[1].val.programmaticStreamSerializationAllowed = 1;
      cfg.attrs = at;
      cfg.numAttrs = pdl_enabled() ? 2 : 1;
      le = cudaLaunchKernelEx(&cfg, gk, P);
    } else {
      le = launch_pdl(gk, dim3(grid), dim3(kGemmThreads), smem, stream, P);
    }
    if (le != cudaSuccess)
      return set_error("%s launch: %s", pp8 ? "pf_gemm_pp_e4m3_kernel" : (d.pp ? "pf_gemm_pp_kernel" : "pf_gemm_kernel"),
                       cudaGetErrorString(le));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("pf_gemm_kernel launch: %s", cudaGetErrorString(e));
  count_launch(d.halo ? (d.a_e4m3 ? (d.a_static ? (res8 ? "pf_conv3_halo_e4m3_res_kernel" : "pf_conv3_halo_e4m3_q8_kernel") : "pf_conv3_halo_e4m3_kernel") : "pf_conv3_halo_kernel")
                       : (pp8 ? "pf_gemm_pp_e4m3_kernel" : (d.pp ? "pf_gemm_pp_kernel" : "pf_gemm_kernel")));
  return 0;
}


}  // namespace pf

extern "C" int pf_gemm_timeline(unsigned long long* out, int32_t reset) {
#ifdef PF_GEMM_TIMELINE
  static_assert(pf::kTimelineSlots == PF_GEMM_TIMELINE_SLOTS, "timeline slots");
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess && out != nullptr)
    e = cudaMemcpyFromSymbol(out, pf::g_gemm_timeline, sizeof(unsigned long long) * pf::kTimelineSlots);
  if (e == cudaSuccess && reset) {
    const unsigned long long zero[pf::kTimelineSlots] = {};
    e = cudaMemcpyToSymbol(pf::g_gemm_timeline, zero, sizeof(zero));
  }
  if (e != cudaSuccess) return pf::set_error("pf_gemm_timeline: %s", cudaGetErrorString(e));
  return 0;
#else
  (void)out; (void)reset;
  return pf::set_error("pf_gemm_timeline: library built without -DPF_GEMM_TIMELINE");
#endif
}
