// Fused attention for the DINOv2 blocks: softmax(Q K^T * scale) V without materialising the (B,heads,N,N) score
// tensor the reference builds (`dinov2/layers/attention.py:53-59`).  head_dim = 64, no mask, N = 1037 tokens.
//
// One CTA per (image b, head h, 128-query tile): two consumer warpgroups of 64 query rows each and one TMA producer warp.
//   S[64x128] = Q[64x64] . K_j[128x64]^T    wgmma, Q fragments loaded once by ldmatrix, K_j from the swizzled TMA tile
//   O[64x64] += P[64x128] . V_j[128x64]     wgmma with P as the register A operand: the S accumulator fragment of a
//                                           16-key slice IS the A fragment of that k16 step once rounded to bf16, so P
//                                           never touches shared memory; V^T tiles come from the transposed copy the
//                                           qkv GEMM epilogue writes (K-major B).
// Online softmax (running maximum / sum per row, O rescaled when the maximum moves) in fp32 on the exp2 unit; each row
// is spread over the four lanes of a quad.  K_j / V_j stream through a TMA ring shared by both warpgroups.  Keys past
// `seq` (the last block holds 1037 - 8*128 = 13) are zero-filled by TMA and masked to -inf.
#include <stdlib.h>

#include "pf_common.cuh"
#include "pf_kernels.h"

namespace pf {

constexpr int kQTile = 128, kKTile = 128, kHd = 64;
constexpr int kAttnWG = 2;                                // consumer warpgroups (64 query rows each)
constexpr int kAttnThreads = kAttnWG * 128 + 32;          // + TMA producer warp
constexpr int kKVStages = 3;
constexpr int kTileBytes = 16384;
constexpr int kOffQ = 0;                                  // [128 q][64]
constexpr int kOffKV = kTileBytes;                        // kKVStages x { K [128 keys][64], V^T 2 x [64 d][64 keys] }
constexpr int kOffBar = kOffKV + kKVStages * 2 * kTileBytes;
constexpr int kAttnSmem = 1024 + kOffBar + 256;

struct AttnParams {
  CUtensorMap tmQK;   // 3-D {2*D, seq, B}, box {64, 128, 1}
  CUtensorMap tmVt;   // 2-D {seq, B*heads*64} (row pitch seq_pad), box {64, 64}
  int B, seq, heads, D;
  int n_qt;           // query tiles per (b, h)
  float scale_log2;   // scale * log2(e)
  __nv_bfloat16* out;
  int out_ld;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kAttnThreads, 1) pf_attention_kernel(const __grid_constant__ AttnParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                  // [kKVStages]
  uint64_t* kv_empty = kv_full + kKVStages;      // [kKVStages]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x % P.n_qt;
  const int bh = blockIdx.x / P.n_qt;
  const int b = bh / P.heads, head = bh - b * P.heads;
  const int n_kv = (P.seq + kKTile - 1) / kKTile;
  constexpr int kProducer = kAttnWG * 4;

  if (warp == kProducer && lane == 0) {
    prefetch_tmap(&P.tmQK);
    prefetch_tmap(&P.tmVt);
    mbar_init(q_full, 1);
    for (int s = 0; s < kKVStages; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], kAttnWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == kProducer) {
    if (elect_one()) {
      mbar_expect_tx(q_full, kTileBytes);
      tma_load_3d(smem + kOffQ, &P.tmQK, q_full, head * kHd, qt * kQTile, b);
      int st = 0; uint32_t ph = 0;
      for (int j = 0; j < n_kv; ++j) {
        mbar_wait(&kv_empty[st], ph ^ 1);
        uint8_t* sk = smem + kOffKV + st * 2 * kTileBytes;
        mbar_expect_tx(&kv_full[st], 2 * kTileBytes);
        tma_load_3d(sk, &P.tmQK, &kv_full[st], P.D + head * kHd, j * kKTile, b);
        const int vrow = (b * P.heads + head) * kHd;
        tma_load_2d(sk + kTileBytes, &P.tmVt, &kv_full[st], j * kKTile, vrow);
        tma_load_2d(sk + kTileBytes + 8192, &P.tmVt, &kv_full[st], j * kKTile + 64, vrow);
        if (++st == kKVStages) { st = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup g owns query rows 64 g .. 64 g + 63 of the tile =====================
  const int g = warp >> 2, wq = warp & 3;
  mbar_wait(q_full, 0);
  uint32_t qf[4][4];                              // Q fragments of the four k16 steps (head_dim 64)
  {
    const uint32_t base = smem_u32(smem + kOffQ);
    const int row = 64 * g + 16 * wq + (lane & 15);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      ldmatrix_x4(base + row * 128 + ((((2 * k) + (lane >> 4)) ^ (row & 7)) << 4), qf[k]);
  }
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 units) / sum of rows lane/4, lane/4 + 8
  const float sl2 = P.scale_log2;
  int st = 0; uint32_t ph = 0;
  for (int j = 0; j < n_kv; ++j) {
    mbar_wait(&kv_full[st], ph);
    const uint32_t sk = smem_u32(smem + kOffKV + st * 2 * kTileBytes);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) Wgmma<128>::rs(s, qf[k], wgmma_desc_k128(sk) + 2 * k, k);
    wgmma_commit();
    wgmma_wait<0>();
    // ---- online softmax over this block's 128 keys
    const int kv_left = P.seq - j * kKTile;
    if (kv_left < kKTile) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int key = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        if (key >= kv_left) s[i] = -INFINITY;
      }
    }
    float x0 = -INFINITY, x1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
      x0 = fmaxf(x0, fmaxf(s[i], s[i + 1]));
      x1 = fmaxf(x1, fmaxf(s[i + 2], s[i + 3]));
    }
#pragma unroll
    for (int d = 1; d < 4; d <<= 1) {
      x0 = fmaxf(x0, __shfl_xor_sync(0xffffffffu, x0, d));
      x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, d));
    }
    const float n0 = fmaxf(m0, x0 * sl2), n1 = fmaxf(m1, x1 * sl2);
    const float c0 = ex2_approx(m0 - n0), c1 = ex2_approx(m1 - n1);   // 0 on the first block (m = -inf)
    m0 = n0; m1 = n1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int i = 0; i < 64; i += 4) {
      s[i] = ex2_approx(fmaf(s[i], sl2, -n0));
      s[i + 1] = ex2_approx(fmaf(s[i + 1], sl2, -n0));
      s[i + 2] = ex2_approx(fmaf(s[i + 2], sl2, -n1));
      s[i + 3] = ex2_approx(fmaf(s[i + 3], sl2, -n1));
      r0 += s[i] + s[i + 1];
      r1 += s[i + 2] + s[i + 3];
    }
    l0 = l0 * c0 + r0;
    l1 = l1 * c1 + r1;
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      o[i] *= c0; o[i + 1] *= c0;
      o[i + 2] *= c1; o[i + 3] *= c1;
    }
    // ---- O += P V: the k16 step kk takes S fragment elements 8 kk .. 8 kk + 7 as its A fragment
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t pa[4] = {pack_bf16(s[8 * kk], s[8 * kk + 1]), pack_bf16(s[8 * kk + 2], s[8 * kk + 3]),
                              pack_bf16(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16(s[8 * kk + 6], s[8 * kk + 7])};
      Wgmma<64>::rs(o, pa, wgmma_desc_k128(sk + kTileBytes + (kk >> 2) * 8192) + 2 * (kk & 3), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);
    if (++st == kKVStages) { st = 0; ph ^= 1; }
  }
  // ---- normalise and store: row lane/4 (+8) of this warp's 16 rows, columns 8 jd + 2 (lane % 4)
#pragma unroll
  for (int d = 1; d < 4; d <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, d);
    l1 += __shfl_xor_sync(0xffffffffu, l1, d);
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int q0 = qt * kQTile + 64 * g + 16 * wq + (lane >> 2);
  __nv_bfloat16* ob = P.out + static_cast<size_t>(b) * P.seq * P.out_ld + head * kHd + 2 * (lane & 3);
#pragma unroll
  for (int jd = 0; jd < 8; ++jd) {
    if (q0 < P.seq)
      *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(q0) * P.out_ld + 8 * jd) = pack_bf16(o[4 * jd] * i0, o[4 * jd + 1] * i0);
    if (q0 + 8 < P.seq)
      *reinterpret_cast<uint32_t*>(ob + static_cast<size_t>(q0 + 8) * P.out_ld + 8 * jd) =
          pack_bf16(o[4 * jd + 2] * i1, o[4 * jd + 3] * i1);
  }
}

}  // namespace pf

using namespace pf;

extern "C" int pf_attention(const void* qk, int32_t qk_ld, const void* vt, int32_t B, int32_t seq, int32_t seq_pad,
                            int32_t heads, float scale, void* out, int32_t out_ld, void* stream) {
  static bool attr_done[kMaxDevices] = {false};
  const int dev = current_device();
  if (!attr_done[dev]) {
    cudaError_t e = cudaFuncSetAttribute(pf_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem);
    if (e != cudaSuccess) return set_error("cudaFuncSetAttribute(pf_attention_kernel): %s", cudaGetErrorString(e));
    attr_done[dev] = true;
  }
  const int D = heads * kHd;
  if (B < 1 || seq < 1 || heads < 1) return set_error("pf_attention: empty problem");
  if (qk_ld % 8 || seq_pad % 8 || out_ld % 8) return set_error("pf_attention: strides must be multiples of 8");
  if (seq_pad < seq) return set_error("pf_attention: seq_pad %d < seq %d", seq_pad, seq);
  AttnParams P;
  if (tmap_3d_bf16(&P.tmQK, qk, 2 * D, seq, B, qk_ld, static_cast<uint64_t>(seq) * qk_ld, 64, 128, 1)) return 1;
  // columns >= seq read as zeros: TMA zero-fills past the map's seq width, so the padding of V^T is never read
  // (tests/test_gpu_attn_parity.py::test_layout_contracts fills it with NaN)
  if (tmap_2d_bf16(&P.tmVt, vt, seq, static_cast<uint64_t>(B) * heads * kHd, seq_pad, 64, 64)) return 1;
  P.B = B; P.seq = seq; P.heads = heads; P.D = D;
  P.n_qt = (seq + kQTile - 1) / kQTile;
  P.scale_log2 = scale * 1.4426950408889634f;
  P.out = static_cast<__nv_bfloat16*>(out);
  P.out_ld = out_ld;
  note_work(4.0 * B * heads * static_cast<double>(seq) * seq * kHd, "attention B%d heads%d seq%d", B, heads, seq);
  cudaError_t le = launch_pdl(pf_attention_kernel, dim3(B * heads * P.n_qt), dim3(kAttnThreads), kAttnSmem,
                              static_cast<cudaStream_t>(stream), P);
  if (le != cudaSuccess) return set_error("pf_attention_kernel launch: %s", cudaGetErrorString(le));
  return check_launch("pf_attention_kernel");
}
