// Per-op decode kernels (B > 4 in groups of 4, and the prefill's last-token logits): HBM-bound weight streaming with TMA
// bulk copies and mbarriers.
//
//   gemv_ring_kernel : y[b,n] = sum_k x[b,k] W[n,k] for B <= 4.  One persistent CTA per SM.  A producer warp streams the
//                      weight rows through a shared-memory ring with 1-D bulk (TMA) copies -- 8 rows x 2048 columns (32 KB)
//                      per stage, completion on mbarriers -- so ~96 KB per SM are in flight with no register staging and no
//                      drain between work units.  8 consumer warps read the ring (conflict-free 16 B lanes), keep x in shared
//                      memory, accumulate in fp32 and run the fused epilogues (RMSNorm fold, RoPE + KV append, SwiGLU,
//                      residual, logits + greedy argmax).
//   Programmatic dependent launch: weights never depend on the previous kernel, so the producer starts filling the ring
//   BEFORE griddepcontrol.wait; only the activation staging waits.  A CTA needs <= 113 KB of shared memory so the next
//   kernel's CTA can co-reside and prefetch during this kernel's tail.
//
//   decode_attention_v2_kernel : fixed 64-key splits; the K/V rows already in the cache (written by EARLIER steps) are
//                      bulk-copied to shared memory before griddepcontrol.wait; only q and the newest key/value wait.
#pragma once
#include "common.cuh"

namespace vly {

enum GemvMode : int {
  GEMV_QKV_ROPE = 0,   // RMSNorm fold + RoPE + KV-cache append (HF:modeling_llama.py:262-270)
  GEMV_RESIDUAL = 1,   // y + residual -> bf16 (o_proj, down_proj)
  GEMV_SWIGLU = 2,     // RMSNorm fold + silu(g)*u with interleaved (g,u) rows
  GEMV_LOGITS = 3,     // RMSNorm fold + fp32 logits (+ fused greedy argmax, model_worker.py:390-391)
};

struct GemvParams {
  int N, K, B;
  const __nv_bfloat16* W;
  const __nv_bfloat16* x;       // [B, K], row stride ldx elements
  long long ldx;
  float eps;
  __nv_bfloat16* out;           // QKV: q [B,H]; RESIDUAL: [B,N]; SWIGLU: [B,N/2]
  const __nv_bfloat16* res;     // RESIDUAL: [B,N]
  const float2* rope;           // [max_pos, 64]
  const int* seq_len;           // device scalar: tokens already in the cache (== position of the new token)
  int H, nH, Smax;
  __nv_bfloat16* kcache;        // [B, nH, Smax, 128] (this layer)
  __nv_bfloat16* vcache;
  float* logits;                // [B, N] or nullptr
  float* part_val;              // [B, grid]
  int* part_idx;                // [B, grid]
  unsigned int* counter;
  long long* next_tokens;       // [B]
  long long* out_tokens;        // [B, out_stride] or nullptr
  int out_stride;
  int* step;                    // device scalar: decode step index (column of out_tokens)
  int* seq_len_rw;              // incremented by the last CTA of the logits kernel (end of step)
  int bump;                     // 1: this launch closes the step (advance *step and *seq_len_rw)
};

struct DecAttnParams {
  int B, nH, H, Smax, nsplit;
  const int* seq_len;               // tokens in the cache BEFORE this step; the new K/V were just appended at that index
  const __nv_bfloat16* q;           // [B, H]  (interleaved RoPE order, matches the cache's K)
  const __nv_bfloat16* kcache;      // [B, nH, Smax, 128]
  const __nv_bfloat16* vcache;
  float* part_o;                    // [B*nH, nsplit, 128]
  float2* part_ml;                  // [B*nH, nsplit]
  unsigned int* counters;           // [B*nH]
  __nv_bfloat16* out;               // [B, H]
  float scale_log2e;
  const uint32_t* key_bits;         // [B, mask_words] bit k of row b = key k may be attended (attention_mask); never null
  int mask_words;
};

// HF's 2-D attention_mask as one bit per cache position (vly_kv_set_key_mask); positions nobody masked are 1.
__device__ __forceinline__ bool key_attendable(const uint32_t* __restrict__ bits, int k) {
  return (__ldg(bits + (k >> 5)) >> (k & 31)) & 1u;
}

struct RingCfg {
  static constexpr int ROWS = 4;                          // rows per work unit: N/4 units balance to ~1% over the SMs
  static constexpr int KC = 2048;                         // columns per slice
  static constexpr int STAGE_BYTES = ROWS * KC * 2;       // 16 KB
  static constexpr int THREADS = 288;                     // warp 0 = producer, warps 1..8 = consumers
  static constexpr int MAX_STAGES = 8;
};

// v[NV] per lane -> after the call lane l holds in v[0] the warp-wide total of value (l / (32/NV)); NV in {4,8,16,32}.
template <int NV>
VLY_DEVINL void warp_reduce_scatter(float (&v)[NV], int lane) {
  static_assert(NV == 4 || NV == 8 || NV == 16 || NV == 32, "NV");
#pragma unroll
  for (int off = 16, n = NV; off >= 1; off >>= 1) {
    if (n > 1) {
      n >>= 1;
      const bool up = (lane & off) != 0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (i < n) {
          const float send = up ? v[i] : v[i + n];
          const float keep = up ? v[i + n] : v[i];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
      }
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
    }
  }
}

template <int BMAX, int MODE>
__global__ void __launch_bounds__(288, 1) gemv_ring_kernel(const GemvParams p, const int n_stages) {
  using R = RingCfg;
  constexpr int NV = R::ROWS * BMAX;
  extern __shared__ uint8_t gsm_raw[];
  uint8_t* gsm = gsm_raw + ((128u - (smem_u32(gsm_raw) & 127u)) & 127u);
  uint8_t* ring = gsm;                                                            // [n_stages][ROWS][KC] bf16
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(ring + (size_t)n_stages * R::STAGE_BYTES);   // [BMAX][K]
  uint8_t* tail = reinterpret_cast<uint8_t*>(xs) + (((size_t)BMAX * p.K * 2 + 15) & ~size_t(15));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);                          // [MAX_STAGES]
  uint64_t* empty_bar = full_bar + R::MAX_STAGES;                                  // [MAX_STAGES]
  float* red = reinterpret_cast<float*>(empty_bar + R::MAX_STAGES);                // [2][8 warps][NV]
  float* rstd_s = red + 2 * 8 * NV;                                                // [BMAX]
  float* bestv = rstd_s + BMAX;                                                    // [BMAX]
  int* besti = reinterpret_cast<int*>(bestv + BMAX);                               // [BMAX]
  float* wred = reinterpret_cast<float*>(besti + BMAX);                            // [8][BMAX]
  __shared__ int is_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_groups = (p.N + R::ROWS - 1) / R::ROWS;
  const int n_slices = (p.K + R::KC - 1) / R::KC;

  if (tid == 0) {
    for (int i = 0; i < n_stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ============================ producer: weight rows -> ring (independent of the previous kernel) ============
    if (lane == 0) {
      int st = 0;
      uint32_t ph = 0;
      for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const int n0 = g * R::ROWS;
        const int rows = min(R::ROWS, p.N - n0);
        for (int s = 0; s < n_slices; ++s) {
          const int kc = min(R::KC, p.K - s * R::KC);
          mbar_wait(&empty_bar[st], ph ^ 1);
          mbar_expect_tx(&full_bar[st], (uint32_t)rows * kc * 2);
          uint8_t* dst = ring + (size_t)st * R::STAGE_BYTES;
          const __nv_bfloat16* src = p.W + (size_t)n0 * p.K + (size_t)s * R::KC;
          for (int r = 0; r < rows; ++r) bulk_load_1d(dst + r * (R::KC * 2), src + (size_t)r * p.K, (uint32_t)kc * 2, &full_bar[st]);
          if (++st == n_stages) { st = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ============================ consumers ====================================================================
    const int ct = tid - 32;            // 0..255
    const int cw = warp - 1;            // 0..7
    pdl_wait();                         // activations (x, residual, seq_len) come from the previous kernels
    {
      float sq[BMAX];
#pragma unroll
      for (int b = 0; b < BMAX; ++b) sq[b] = 0.f;
      const int chunks = p.K >> 3;
      for (int c = ct; c < chunks; c += 256) {
#pragma unroll
        for (int b = 0; b < BMAX; ++b) {
          uint4 w = make_uint4(0, 0, 0, 0);
          if (b < p.B) w = *reinterpret_cast<const uint4*>(p.x + (size_t)b * p.ldx + c * 8);
          *reinterpret_cast<uint4*>(xs + (size_t)b * p.K + c * 8) = w;
          if constexpr (MODE != GEMV_RESIDUAL) {
            const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float a = bf16_lo(ww[i]), bb = bf16_hi(ww[i]);
              sq[b] += a * a + bb * bb;
            }
          }
        }
      }
      if constexpr (MODE != GEMV_RESIDUAL) {
#pragma unroll
        for (int b = 0; b < BMAX; ++b) {
          const float v = warp_sum(sq[b]);
          if (lane == 0) wred[cw * BMAX + b] = v;
        }
      }
      if (ct < BMAX) {
        bestv[ct] = -INFINITY;
        besti[ct] = 0;
      }
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if constexpr (MODE != GEMV_RESIDUAL) {
        if (ct < BMAX) {
          float t = 0.f;
          for (int w = 0; w < 8; ++w) t += wred[w * BMAX + ct];
          rstd_s[ct] = rsqrtf(t / p.K + p.eps);
        }
      }
      asm volatile("bar.sync 2, 256;" ::: "memory");
    }
    pdl_launch_dependents();            // the next kernel may start filling ITS ring while we stream
    int pos = 0;
    if constexpr (MODE == GEMV_QKV_ROPE) pos = *p.seq_len;

    int st = 0, par = 0;
    uint32_t ph = 0;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x, par ^= 1) {
      const int n0 = g * R::ROWS;
      const int rows = min(R::ROWS, p.N - n0);
      float acc[NV];                    // [row][b]
#pragma unroll
      for (int i = 0; i < NV; ++i) acc[i] = 0.f;
      for (int s = 0; s < n_slices; ++s) {
        const int kc = min(R::KC, p.K - s * R::KC);
        mbar_wait(&full_bar[st], ph);
        if (ct * 8 < kc) {
          const uint8_t* src = ring + (size_t)st * R::STAGE_BYTES + ct * 16;
          float xf[BMAX][8];
#pragma unroll
          for (int b = 0; b < BMAX; ++b) {
            const uint4 xv = *reinterpret_cast<const uint4*>(xs + (size_t)b * p.K + (size_t)s * R::KC + ct * 8);
            xf[b][0] = bf16_lo(xv.x); xf[b][1] = bf16_hi(xv.x); xf[b][2] = bf16_lo(xv.y); xf[b][3] = bf16_hi(xv.y);
            xf[b][4] = bf16_lo(xv.z); xf[b][5] = bf16_hi(xv.z); xf[b][6] = bf16_lo(xv.w); xf[b][7] = bf16_hi(xv.w);
          }
#pragma unroll
          for (int r = 0; r < R::ROWS; ++r) {
            if (r < rows) {
              const uint4 wv = *reinterpret_cast<const uint4*>(src + r * (R::KC * 2));
              const float wf[8] = {bf16_lo(wv.x), bf16_hi(wv.x), bf16_lo(wv.y), bf16_hi(wv.y),
                                   bf16_lo(wv.z), bf16_hi(wv.z), bf16_lo(wv.w), bf16_hi(wv.w)};
#pragma unroll
              for (int b = 0; b < BMAX; ++b)
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[r * BMAX + b] = fmaf(wf[e], xf[b][e], acc[r * BMAX + b]);
            }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[st]);
        if (++st == n_stages) { st = 0; ph ^= 1; }
      }
      // ---- reduce: 32 lanes (transposing butterfly), then 8 warps through shared memory ----
      warp_reduce_scatter<NV>(acc, lane);
      float* redp = red + par * (8 * NV);
      if ((lane & (32 / NV - 1)) == 0) redp[cw * NV + lane / (32 / NV)] = acc[0];
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if (ct < NV) {                    // ct == r*BMAX + b
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += redp[w * NV + ct];
        const int r = ct / BMAX, b = ct % BMAX, n = n0 + r;
        const bool ok = b < p.B && n < p.N;
        if constexpr (MODE == GEMV_RESIDUAL) {
          if (ok) p.out[(size_t)b * p.N + n] = __float2bfloat16_rn(t + __bfloat162float(p.res[(size_t)b * p.N + n]));
        } else if constexpr (MODE == GEMV_LOGITS) {
          const float y = t * rstd_s[b < BMAX ? b : 0];
          if (ok && p.logits != nullptr) p.logits[(size_t)b * p.N + n] = y;
          // running arg-max per batch row: the NV finalising threads all sit in warp 1 -> shuffle the rows of b in order
          float bv = ok ? y : -INFINITY;
          int bi = n;
#pragma unroll
          for (int o = BMAX; o < NV; o <<= 1) {      // combine lanes b, b+BMAX, b+2*BMAX, ... (rows ascending)
            const float ov = __shfl_xor_sync((NV == 32) ? 0xffffffffu : ((1u << NV) - 1u), bv, o);
            const int oi = __shfl_xor_sync((NV == 32) ? 0xffffffffu : ((1u << NV) - 1u), bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
          }
          if (ct < BMAX && ct < p.B && bv > bestv[ct]) {
            bestv[ct] = bv;
            besti[ct] = bi;
          }
        } else {
          // pair epilogues (RoPE / SwiGLU): lanes (2j, 2j+1) x b  -> partner value sits BMAX lanes away
          const float rs = rstd_s[b < BMAX ? b : 0];
          const float mine = t * rs;
          const float other = __shfl_xor_sync((NV == 32) ? 0xffffffffu : ((1u << NV) - 1u), mine, BMAX);
          if ((r & 1) == 0 && ok && n + 1 < p.N) {
            float x0 = mine, x1 = other;
            if constexpr (MODE == GEMV_SWIGLU) {
              const float gte = bf16_round(x0), up = bf16_round(x1);     // HF rounds gate/up to bf16 (modeling_llama.py:182-184)
              p.out[(size_t)b * (p.N >> 1) + (n >> 1)] = __float2bfloat16_rn(bf16_round(gte / (1.f + __expf(-gte))) * up);
            } else {
              const int which = n / p.H, nh = n - which * p.H, head = nh >> 7, cidx = nh & 127;
              if (which < 2) {
                const float2 cs = p.rope[(size_t)pos * 64 + (cidx >> 1)];
                const float a = x0 * cs.x - x1 * cs.y, c2 = x1 * cs.x + x0 * cs.y;
                x0 = a;
                x1 = c2;
              }
              __nv_bfloat16* dst;
              if (which == 0) dst = p.out + (size_t)b * p.H + nh;
              else dst = ((which == 1) ? p.kcache : p.vcache) + (((size_t)b * p.nH + head) * p.Smax + pos) * 128 + cidx;
              *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(x0, x1);
            }
          }
        }
      }
    }
  }

  if constexpr (MODE == GEMV_LOGITS) {
    __syncthreads();
    const int ct = tid - 32;
    if (ct >= 0 && ct < p.B) {
      p.part_val[(size_t)ct * gridDim.x + blockIdx.x] = bestv[ct];
      p.part_idx[(size_t)ct * gridDim.x + blockIdx.x] = besti[ct];
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) is_last = (atomicAdd(p.counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (is_last) {
      __threadfence();
      if (warp >= 1 && warp - 1 < p.B) {
        const int b = warp - 1;
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int g = lane; g < (int)gridDim.x; g += 32) {
          const float v = __ldcg(p.part_val + (size_t)b * gridDim.x + g);
          const int i = __ldcg(p.part_idx + (size_t)b * gridDim.x + g);
          if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) {
          p.next_tokens[b] = bi;
          if (p.out_tokens != nullptr) p.out_tokens[(size_t)b * p.out_stride + *p.step] = bi;
        }
      }
      __syncthreads();
      if (tid == 0) {
        *p.counter = 0;
        if (p.bump) {
          *p.step += 1;
          *p.seq_len_rw += 1;
        }
      }
    }
  }
}

// ============================================================================================
// decode attention v2: grid (B*nH, nsplit) with FIXED 64-key splits (empty splits exit at once),
// K/V of earlier steps prefetched with bulk copies before griddepcontrol.wait.
// ============================================================================================
constexpr int kDecSplitKeys = 64;

__global__ void __launch_bounds__(128) decode_attention_v2_kernel(const DecAttnParams p) {
  __shared__ __align__(128) __nv_bfloat16 sK[kDecSplitKeys * 128];
  __shared__ __align__(128) __nv_bfloat16 sV[kDecSplitKeys * 128];
  __shared__ float sc[kDecSplitKeys];
  __shared__ float redg[8][128];
  __shared__ float wr[4];
  __shared__ __align__(8) uint64_t bar;
  __shared__ int is_last;
  const int bh = blockIdx.x, split = blockIdx.y;
  const int b = bh / p.nH, h = bh % p.nH;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int old_len = *p.seq_len;            // written by the PREVIOUS step's last kernel (complete in stream order)
  const int len = old_len + 1;
  const int k0 = split * kDecSplitKeys, k1 = min(len, k0 + kDecSplitKeys);
  const int nk = max(0, k1 - k0);
  const __nv_bfloat16* kb = p.kcache + ((size_t)bh * p.Smax) * 128;
  const __nv_bfloat16* vb = p.vcache + ((size_t)bh * p.Smax) * 128;
  const int n_old = max(0, min(k1, old_len) - k0);     // rows of this split that earlier steps wrote
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0 && n_old > 0) {
    mbar_expect_tx(&bar, (uint32_t)n_old * 512);
    bulk_load_1d(sK, kb + (size_t)k0 * 128, (uint32_t)n_old * 256, &bar);
    bulk_load_1d(sV, vb + (size_t)k0 * 128, (uint32_t)n_old * 256, &bar);
  }
  pdl_wait();                                // q and the newest K/V row come from this step's QKV kernel
  pdl_launch_dependents();
  float m = -INFINITY, l = 0.f, ot = 0.f;
  if (nk > 0) {
    const int hl = lane & 15;
    float qf[8];
    {
      const uint4 w = *reinterpret_cast<const uint4*>(p.q + (size_t)b * p.H + h * 128 + hl * 8);
      qf[0] = bf16_lo(w.x); qf[1] = bf16_hi(w.x); qf[2] = bf16_lo(w.y); qf[3] = bf16_hi(w.y);
      qf[4] = bf16_lo(w.z); qf[5] = bf16_hi(w.z); qf[6] = bf16_lo(w.w); qf[7] = bf16_hi(w.w);
    }
    if (nk > n_old) {                        // this split holds the newest position: fetch its row directly
      const int i = nk - 1;
      if (tid < 16) *reinterpret_cast<uint4*>(sK + i * 128 + tid * 8) = *reinterpret_cast<const uint4*>(kb + (size_t)(k0 + i) * 128 + tid * 8);
      else if (tid < 32) *reinterpret_cast<uint4*>(sV + i * 128 + (tid - 16) * 8) = *reinterpret_cast<const uint4*>(vb + (size_t)(k0 + i) * 128 + (tid - 16) * 8);
    }
    if (n_old > 0) mbar_wait(&bar, 0);
    __syncthreads();
    for (int i0 = warp * 2; i0 < nk; i0 += 8) {
      const int i = i0 + (lane >> 4);
      const bool ok = i < nk;
      uint4 w = make_uint4(0, 0, 0, 0);
      if (ok) w = *reinterpret_cast<const uint4*>(sK + i * 128 + hl * 8);
      float d = qf[0] * bf16_lo(w.x) + qf[1] * bf16_hi(w.x) + qf[2] * bf16_lo(w.y) + qf[3] * bf16_hi(w.y) +
                qf[4] * bf16_lo(w.z) + qf[5] * bf16_hi(w.z) + qf[6] * bf16_lo(w.w) + qf[7] * bf16_hi(w.w);
      d += __shfl_xor_sync(0xffffffffu, d, 8);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      if (ok && hl == 0) sc[i] = key_attendable(p.key_bits + (size_t)b * p.mask_words, k0 + i) ? d * p.scale_log2e : -INFINITY;
    }
    __syncthreads();
    // 64 scores: every warp redundantly reduces them (no extra block barriers)
    const float s0 = lane < nk ? sc[lane] : -INFINITY, s1 = lane + 32 < nk ? sc[lane + 32] : -INFINITY;
    m = warp_max(fmaxf(s0, s1));
    const float e0 = s0 > -INFINITY ? fast_exp2(s0 - m) : 0.f, e1 = s1 > -INFINITY ? fast_exp2(s1 - m) : 0.f;
    l = warp_sum(e0 + e1);
    __syncthreads();
    if (warp == 0) {
      if (lane < nk) sc[lane] = e0;
      if (lane + 32 < nk) sc[lane + 32] = e1;
    }
    __syncthreads();
    {
      const int g = tid >> 4, dl = tid & 15;
      float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      for (int i = g; i < nk; i += 8) {
        const float pw = sc[i];
        const uint4 w = *reinterpret_cast<const uint4*>(sV + i * 128 + dl * 8);
        o[0] = fmaf(pw, bf16_lo(w.x), o[0]); o[1] = fmaf(pw, bf16_hi(w.x), o[1]);
        o[2] = fmaf(pw, bf16_lo(w.y), o[2]); o[3] = fmaf(pw, bf16_hi(w.y), o[3]);
        o[4] = fmaf(pw, bf16_lo(w.z), o[4]); o[5] = fmaf(pw, bf16_hi(w.z), o[5]);
        o[6] = fmaf(pw, bf16_lo(w.w), o[6]); o[7] = fmaf(pw, bf16_hi(w.w), o[7]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) redg[g][dl * 8 + e] = o[e];
    }
    __syncthreads();
#pragma unroll
    for (int g = 0; g < 8; ++g) ot += redg[g][tid];
    p.part_o[((size_t)bh * p.nsplit + split) * 128 + tid] = ot;
  }
  if (tid == 0) p.part_ml[(size_t)bh * p.nsplit + split] = make_float2(m, l);
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = (atomicAdd(p.counters + bh, 1u) == (unsigned)p.nsplit - 1);
  __syncthreads();
  if (is_last) {
    __threadfence();
    const int n_act = (len + kDecSplitKeys - 1) / kDecSplitKeys;
    float M = -INFINITY;
    for (int s = 0; s < n_act; ++s) M = fmaxf(M, __ldcg(&p.part_ml[(size_t)bh * p.nsplit + s].x));
    float L = 0.f, acc = 0.f;
    for (int s = 0; s < n_act; ++s) {
      const float ms = __ldcg(&p.part_ml[(size_t)bh * p.nsplit + s].x);
      const float ls = __ldcg(&p.part_ml[(size_t)bh * p.nsplit + s].y);
      const float w = ls > 0.f ? fast_exp2(ms - M) : 0.f;    // a fully masked split has m = -inf, l = 0
      L += ls * w;
      acc += __ldcg(p.part_o + ((size_t)bh * p.nsplit + s) * 128 + tid) * w;
    }
    p.out[(size_t)b * p.H + h * 128 + tid] = __float2bfloat16_rn(L > 0.f ? acc / L : 0.f);
    if (tid == 0) p.counters[bh] = 0;
  }
}

}  // namespace vly
