// wgmma attention kernels (sm_90a).
//
//  vit_attention_kernel           : CLIP ViT-L/14 self-attention (HF:modeling_clip.py:261-279, :300-336): 257 tokens,
//                                   16 heads x 64, no mask.  Q, K and V are read by TMA straight from the row-major QKV
//                                   buffer (no transpose pass).
//  llama_prefill_attention_kernel : causal attention with KV cache (HF:modeling_llama.py:199-222, :251-289), head_dim 128,
//                                   HF's 2-D attention_mask as one bit per cache position.
//
// Both are the same flash-attention loop, one warpgroup per 64-row query tile:
//   S = Q K^T        wgmma m64n64k16, Q and K K-major in shared memory (128-byte swizzle, TMA boxes of 64 rows x 64 columns)
//   online softmax   in registers: each query row is held by the 4 lanes of a quad, row max / sum by two shuffles
//   O += P V         wgmma m64n{HD}k16 with P as the REGISTER A operand (the S fragment layout is the A fragment layout) and
//                    V as a transposed (MN-major) shared-memory B operand -- V is used exactly as it is stored.
// K/V blocks of 64 keys are double-buffered: thread 0 issues the TMA loads of block j + 2 as soon as block j is consumed.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace vly {

struct VitAttnParams {
  int F;                    // frames
  int tokens;               // 257
  int heads;                // 16
  int D;                    // 1024
  __nv_bfloat16* ctx;       // [F*tokens, D]
  float scale_log2e;        // head_dim^-0.5 * log2(e)
};

struct PrefillAttnParams {
  int B, S, past, nH, H, Smax;
  __nv_bfloat16* ctx;   // [B*S, H]
  float scale_log2e;    // 128^-0.5 * log2(e)
  // HF's 2-D attention_mask (padding mask AND-ed into the causal mask, HF:masking_utils), one bit per cache position:
  // [B, mask_words] words, bit k of row b = key k may be attended.  NULL = no key is masked (the common case).
  const uint32_t* key_bits;
  int mask_words;
};

template <int HD>
struct FlashCfg {
  static constexpr int BOX = 64 * 128;                     // 64 rows x 64 bf16 (one TMA box, 128-byte swizzle)
  static constexpr int TILE = HD / 64 * BOX;               // 64 rows x HD
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE;                       // [2 stages]
  static constexpr int OFF_V = OFF_K + 2 * TILE;           // [2 stages]
  static constexpr int OFF_BAR = OFF_V + 2 * TILE;
  static constexpr int SMEM_BYTES = OFF_BAR + 64 + 1024;   // + alignment slack
  static constexpr int THREADS = 128;
};

// The shared loop.  load_kv(j, stage) issues the TMA loads of key block j (K and V, 2 * TILE bytes) on kv_full[stage];
// key_ok(row, key) says whether query row `row` (0..63 of the tile) may attend key `key`; finish(row, col, o0, o1) stores two
// adjacent output columns of a row (already divided by the row sum).
template <int HD, typename LoadKV, typename KeyOk, typename Finish>
VLY_DEVINL void flash_attention_tile(uint8_t* smem, uint32_t base_u32, uint64_t* q_full, uint64_t* kv_full, int nkv, float scale_log2e,
                                     LoadKV load_kv, KeyOk key_ok, Finish finish) {
  using C = FlashCfg<HD>;
  constexpr int OR = HD / 2;                               // O accumulator registers per thread
  const int t = threadIdx.x, w = t >> 5, l = t & 31;
  const int r_lo = w * 16 + (l >> 2), c_lo = (l & 3) * 2;  // fragment row (and r_lo + 8), first column of each 8-column group
  float o[OR];
#pragma unroll
  for (int i = 0; i < OR; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  const uint64_t desc_q = make_smem_desc_sw128(base_u32 + C::OFF_Q, 16, 1024);
  mbar_wait(q_full, 0);
  for (int j = 0; j < nkv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    // ---- S = Q K^T ----
    float s[32];
    const uint64_t desc_k = make_smem_desc_sw128(base_u32 + C::OFF_K + st * C::TILE, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint64_t off = uint64_t((kk >> 2) * (C::BOX / 16) + (kk & 3) * 2);
      wgmma_ss_n64(s, desc_q + off, desc_k + off, kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    // ---- mask + online softmax (scores in log2 units) ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int g = 0; g < 8; ++g)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int row = r_lo + 8 * (i >> 1), key = j * 64 + g * 8 + c_lo + (i & 1);
        const float v = key_ok(row, key) ? s[4 * g + i] * scale_log2e : -INFINITY;
        s[4 * g + i] = v;
        mx[i >> 1] = fmaxf(mx[i >> 1], v);
      }
    float alpha[2], mb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float mn = fmaxf(m[h], mx[h]);
      mb[h] = mn > -INFINITY ? mn : 0.f;                   // a row with nothing visible yet keeps p = 0 and no NaN
      alpha[h] = fast_exp2(m[h] - mb[h]);                  // m = -inf -> 0 (o and lsum are 0 then anyway)
      m[h] = mn;
      lsum[h] *= alpha[h];
    }
#pragma unroll
    for (int g = 0; g < OR / 4; ++g) {
      o[4 * g] *= alpha[0]; o[4 * g + 1] *= alpha[0];
      o[4 * g + 2] *= alpha[1]; o[4 * g + 3] *= alpha[1];
    }
    uint32_t pa[4][4];                                     // P as bf16 A fragments, one per 16 keys
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const float p0 = fast_exp2(s[4 * g] - mb[0]), p1 = fast_exp2(s[4 * g + 1] - mb[0]);
      const float p2 = fast_exp2(s[4 * g + 2] - mb[1]), p3 = fast_exp2(s[4 * g + 3] - mb[1]);
      lsum[0] += p0 + p1;
      lsum[1] += p2 + p3;
      pa[g >> 1][(g & 1) * 2] = pack_bf16x2(p0, p1);
      pa[g >> 1][(g & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    // ---- O += P V ----
    const uint64_t desc_v = make_smem_desc_sw128(base_u32 + C::OFF_V + st * C::TILE, C::BOX, 1024);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {                       // 16 keys = two 1024-byte atoms of V
      if constexpr (HD == 64) wgmma_rs_n64_tb(*reinterpret_cast<float(*)[32]>(o), pa[kk], desc_v + uint64_t(kk * 128), 1);
      else wgmma_rs_n128_tb(*reinterpret_cast<float(*)[64]>(o), pa[kk], desc_v + uint64_t(kk * 128), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncthreads();                                       // every warp is done with this stage
    if (t == 0 && j + 2 < nkv) load_kv(j + 2, st);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 1);
    lsum[h] += __shfl_xor_sync(0xffffffffu, lsum[h], 2);
  }
  const float inv0 = lsum[0] > 0.f ? __frcp_rn(lsum[0]) : 0.f;   // fully masked query row -> zeros (its output is never attended)
  const float inv1 = lsum[1] > 0.f ? __frcp_rn(lsum[1]) : 0.f;
#pragma unroll
  for (int g = 0; g < OR / 4; ++g) {
    finish(r_lo, g * 8 + c_lo, o[4 * g] * inv0, o[4 * g + 1] * inv0);
    finish(r_lo + 8, g * 8 + c_lo, o[4 * g + 2] * inv1, o[4 * g + 3] * inv1);
  }
}

VLY_DEVINL uint8_t* flash_smem(uint32_t* base_u32) {
  extern __shared__ uint8_t smem_raw[];
  *base_u32 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  return smem_raw + (*base_u32 - smem_u32(smem_raw));
}

// ============================================================================================
// ViT attention.  grid = F * heads * ceil(tokens / 64); tma_qkv: 2D map over qkv [F*tokens, 3*D], box {64, 64}.
// Rows of a box past the frame belong to the next frame (or are zero-filled past the tensor): their keys are masked, their
// query rows are not stored.
// ============================================================================================
__global__ void __launch_bounds__(128, 1)
vit_attention_kernel(const __grid_constant__ CUtensorMap tma_qkv, const VitAttnParams p) {
  using C = FlashCfg<64>;
  uint32_t base_u32;
  uint8_t* smem = flash_smem(&base_u32);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;   // [2]
  const int n_qt = (p.tokens + 63) / 64;
  const int qt = blockIdx.x % n_qt, item = blockIdx.x / n_qt;
  const int f = item / p.heads, h = item % p.heads;
  const int row0 = f * p.tokens;
  const int nkv = n_qt;
  auto load_kv = [&](int j, int st) {
    mbar_expect_tx(&kv_full[st], 2 * C::TILE);
    tma_load_2d(smem + C::OFF_K + st * C::TILE, &tma_qkv, &kv_full[st], p.D + h * 64, row0 + j * 64);
    tma_load_2d(smem + C::OFF_V + st * C::TILE, &tma_qkv, &kv_full[st], 2 * p.D + h * 64, row0 + j * 64);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_qkv);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    pdl_wait();                   // the QKV GEMM's output is read by the TMA loads below
    mbar_expect_tx(q_full, C::TILE);
    tma_load_2d(smem + C::OFF_Q, &tma_qkv, q_full, h * 64, row0 + qt * 64);
    load_kv(0, 0);
    if (nkv > 1) load_kv(1, 1);
  }
  const int tokens = p.tokens;
  flash_attention_tile<64>(
      smem, base_u32, q_full, kv_full, nkv, p.scale_log2e, load_kv, [&](int, int key) { return key < tokens; },
      [&](int r, int col, float o0, float o1) {
        const int q = qt * 64 + r;
        if (q < tokens)
          *reinterpret_cast<uint32_t*>(p.ctx + ((size_t)f * tokens + q) * p.D + h * 64 + col) = pack_bf16x2(o0, o1);
      });
}

// ============================================================================================
// LLaMA prefill attention (causal, head_dim 128, KV cache [B, nH, Smax, 128], q/k in the RoPE-interleaved column order
// written by the QKV epilogue -- the same permutation on both sides of the dot product; v and the output in natural order).
// grid = B * nH * ceil(S / 64).  tma_q: 2D over qbuf [B*S, H], box {64, 64};  tma_k / tma_v: 3D over the cache
// {128, Smax, B*nH}, box {64, 64, 1}.
// ============================================================================================
__global__ void __launch_bounds__(128, 1)
llama_prefill_attention_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                               const __grid_constant__ CUtensorMap tma_v, const PrefillAttnParams p) {
  using C = FlashCfg<128>;
  uint32_t base_u32;
  uint8_t* smem = flash_smem(&base_u32);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;   // [2]
  const int n_qt = (p.S + 63) / 64;
  const int qt = blockIdx.x % n_qt;
  const int bh = blockIdx.x / n_qt;          // b * nH + h
  const int b = bh / p.nH, h = bh % p.nH;
  const int kv_len = p.past + p.S;
  const int q_hi = min(p.S, (qt + 1) * 64);                  // one past the last query row of this tile
  const int nkv = (p.past + q_hi + 63) / 64;                 // key blocks any row of the tile can see
  auto load_kv = [&](int j, int st) {
    mbar_expect_tx(&kv_full[st], 2 * C::TILE);
    uint8_t* kd = smem + C::OFF_K + st * C::TILE;
    uint8_t* vd = smem + C::OFF_V + st * C::TILE;
    tma_load_3d(kd, &tma_k, &kv_full[st], 0, j * 64, bh);
    tma_load_3d(kd + C::BOX, &tma_k, &kv_full[st], 64, j * 64, bh);
    tma_load_3d(vd, &tma_v, &kv_full[st], 0, j * 64, bh);
    tma_load_3d(vd + C::BOX, &tma_v, &kv_full[st], 64, j * 64, bh);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_v);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    pdl_wait();                   // q and the appended K/V rows come from the QKV GEMM of this layer
    mbar_expect_tx(q_full, C::TILE);
    tma_load_2d(smem + C::OFF_Q, &tma_q, q_full, h * 128, b * p.S + qt * 64);
    tma_load_2d(smem + C::OFF_Q + C::BOX, &tma_q, q_full, h * 128 + 64, b * p.S + qt * 64);
    load_kv(0, 0);
    if (nkv > 1) load_kv(1, 1);
  }
  const uint32_t* kbits = p.key_bits ? p.key_bits + (size_t)b * p.mask_words : nullptr;
  const int q_pos0 = p.past + qt * 64;                       // absolute position of tile row 0
  flash_attention_tile<128>(
      smem, base_u32, q_full, kv_full, nkv, p.scale_log2e, load_kv,
      [&](int r, int key) {
        return key <= q_pos0 + r && key < kv_len && (kbits == nullptr || ((__ldg(kbits + (key >> 5)) >> (key & 31)) & 1u));
      },
      [&](int r, int col, float o0, float o1) {
        const int q = qt * 64 + r;
        if (q < p.S) *reinterpret_cast<uint32_t*>(p.ctx + ((size_t)b * p.S + q) * p.H + h * 128 + col) = pack_bf16x2(o0, o1);
      });
}

}  // namespace vly
