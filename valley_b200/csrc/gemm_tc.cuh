// Warp-specialised Hopper GEMM:  D[M,N] = A[M,K] * B[N,K]^T   (bf16 in, fp32 accumulate in registers)
//
//   warpgroup 0    : TMA producer (one thread): A tile 128x64, B tile BNx64 per stage, 128B swizzle, mbarrier complete_tx
//   warpgroups 1-2 : consumers -- each owns 64 rows of the 128-row tile and issues wgmma.mma_async m64n128k16 (BN / 128 per
//                    k-step) straight from the shared-memory ring; one wgmma group stays in flight while the previous stage
//                    is handed back to the producer.
//   epilogue       : the accumulators go through shared memory (the ring is free once the main loop has drained) so that
//                    every thread owns 32-column chunks of ONE output row -- the row statistics, RoPE pairs and SwiGLU pairs
//                    below are row-local -- then the fused epilogue is applied and the row is stored.
//   One 128 x BN tile per CTA: the grid covers the tiles.
//
// Both operands are K-major, i.e. A is a row-major activation matrix and B is an nn.Linear weight
// [out_features, in_features] exactly as HuggingFace stores it.
//
// Fused epilogues (what the reference runs as separate ATen kernels):
//   LayerNorm / RMSNorm *prologue*:  LN(x) W^T = rstd * (x W'^T - mean * colsum(W')) + (b + W beta),
//     W' = W * gamma folded at load time, so the GEMM runs on the raw residual stream and the row
//     statistics (mean, rstd) are applied here.  The statistics arrive as per-row partial (sum, sumsq)
//     pairs written by the epilogue of the GEMM that produced x (deterministic, no atomics).
//   bias, quick_gelu, residual add, SwiGLU (gate/up rows interleaved), RoPE + KV-cache append.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace vly {

enum EpiMode : int {
  EPI_BIAS = 0,           // out = acc (+ bias)                                    -> bf16
  EPI_LN_BIAS = 1,        // out = rstd*(acc - mean*colsum) + bias                 -> bf16   (ViT QKV)
  EPI_LN_BIAS_GELU = 2,   // quick_gelu(rstd*(acc - mean*colsum) + bias)           -> bf16   (ViT fc1)
  EPI_BIAS_RES_STATS = 3, // out = acc (+ bias) + residual; partial (sum,sumsq)    -> bf16   (ViT out_proj/fc2, LLaMA o/down)
  EPI_RMS_QKV_ROPE = 4,   // v = rstd*acc; RoPE on q,k; q -> qbuf, k,v -> KV cache -> bf16   (LLaMA prefill QKV)
  EPI_RMS_SWIGLU = 5,     // silu(rstd*acc[2j]) * (rstd*acc[2j+1])                 -> bf16   (LLaMA gate/up)
  EPI_RMS_F32 = 6,        // out = rstd*acc                                        -> fp32   (lm_head logits)
};

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles;
  void* out;
  long long ldo;                  // output row stride in elements
  const float* bias;              // [N] fp32 or nullptr
  const float* colsum;            // [N] fp32 (LN fold)
  const float2* stats_in;         // [M, stats_in_nt] partial (sum, sumsq) of the A rows
  int stats_in_nt;
  float inv_dim;                  // 1 / K_logical (row length the statistics are over)
  float eps;
  float2* stats_out;              // [M, num_n_tiles] partial (sum, sumsq) of the bf16-rounded output rows
  const __nv_bfloat16* residual;  // [M, ldr]
  long long ldr;
  // EPI_RMS_QKV_ROPE
  const float2* rope;             // [max_pos, 64] (cos, sin), bf16-rounded values
  int S, past, H, nH, Smax;       // row m -> (b = m / S, s = m % S), position = past + s
  __nv_bfloat16* kcache;          // [B, nH, Smax, 128] for this layer
  __nv_bfloat16* vcache;
  // EPI_BIAS_RES_STATS, fused all-gather: besides `out`, every finished row is stored into the gather buffer of every
  // rank (peer-mapped device pointers, NVLink P2P stores).  Local row m = (local frame f, token t) with f = m / peer_tokens
  // goes to gather row ((peer_frame_off + f * peer_frame_stride) * peer_tokens + t): stride 1 = this rank owns a contiguous
  // block of frames, stride = world size = frames dealt round-robin over the ranks
  __nv_bfloat16* peer_out[8];
  int n_peers;
  int peer_tokens, peer_frame_stride;
  long long peer_frame_off;
};

// x*sigmoid(1.702x) and x*sigmoid(x) on the fast MUFU path
// sigmoid(y) = 0.5 + 0.5 tanh(y / 2): ONE MUFU op (tanh.approx.f32) instead of two (ex2 + rcp).  tanh.approx has a relative
// error of about 2^-11 (PTX ISA); the 0.5 + 0.5 tanh turns it into an ABSOLUTE error of ~2^-12 on sigmoid, so v * sigmoid(.) is
// off by up to ~|v| 2^-12.  That is below the bf16 rounding of the result for v >~ 0 but exceeds it where the result is tiny:
// quick-GELU arguments below about -1.6, SiLU arguments below about -2.7 (tests/test_gpu_prefill_per_op.py bounds it).  A 128 x 256 fc1 tile has 32768 activations per CTA: at 16 MUFU ops per clock per SM the
// exp + reciprocal form alone took 4096 cycles -- the whole main loop of a K = 1024 tile.
VLY_DEVINL float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
VLY_DEVINL float quick_gelu_f(float v) {   // v * sigmoid(1.702 v)
  const float h = 0.5f * v;
  return fmaf(h, tanh_approx(0.851f * v), h);
}
VLY_DEVINL float silu_f(float v) {         // v * sigmoid(v)
  const float h = 0.5f * v;
  return fmaf(h, tanh_approx(h), h);
}

template <int BN>
struct GemmCfg {
  static_assert(BN == 128 || BN == 256, "tile width");
  static constexpr int BM = 128, BK = 64;
  static constexpr int STAGES = (BN == 256) ? 4 : 6;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;               // 192 KB
  static constexpr int ACC_LD = BN + 4;                                 // fp32 staging row pitch (floats)
  static_assert(BM * ACC_LD * 4 <= RING_BYTES, "accumulator staging must fit in the drained ring");
  static constexpr int VEC_BYTES = 2 /*bias, colsum*/ * BN * 4;
  static constexpr int SMEM_BYTES = RING_BYTES + 1024 /*align slack*/ + 256 /*barriers*/ + VEC_BYTES;
  static constexpr int THREADS = 384;
};

template <int BN, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int BM = Cfg::BM, BK = Cfg::BK, STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base_u32 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (base_u32 - smem_u32(smem_raw));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::RING_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  float* sbias = reinterpret_cast<float*>(smem + Cfg::RING_BYTES + 256);   // [BN]
  float* scol = sbias + BN;                                                  // [BN]

  const int wg = threadIdx.x >> 7;
  const int num_kb = (p.K + BK - 1) / BK;
  const int m_blk = (int)blockIdx.x / p.num_n_tiles, n_blk = (int)blockIdx.x % p.num_n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);                             // every consumer thread releases the stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: the prologue above touches nothing the previous kernel of the stream produces, so under the
  // programmatic-serialisation attribute it overlaps that kernel's tail; the threads that read its data wait for it first.
  pdl_launch_dependents();

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    if (threadIdx.x == 0) {
      pdl_wait();
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
        tma_load_2d(sA + stage * Cfg::A_BYTES, &tma_a, &full_bar[stage], kb * BK, m_blk * BM);
        tma_load_2d(sB + stage * Cfg::B_BYTES, &tma_b, &full_bar[stage], kb * BK, n_blk * BN);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================================== consumers =========================================
  const int ct = threadIdx.x - 128;                    // 0..255 over both consumer warpgroups
  const int t = threadIdx.x & 127;                     // thread within this warpgroup
  const int row0 = (wg - 1) * 64;                      // first tile row of this warpgroup
  constexpr int NB = BN / 128;                         // m64n128 accumulators per thread
  float acc[NB][64];
#pragma unroll
  for (int nb = 0; nb < NB; ++nb)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[nb][i] = 0.f;
  {
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t da = make_smem_desc_sw128(base_u32 + stage * Cfg::A_BYTES + row0 * 128, 16, 1024);
      const uint64_t db = make_smem_desc_sw128(base_u32 + STAGES * Cfg::A_BYTES + stage * Cfg::B_BYTES, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)    // 128 rows of B = 16 KB further on: +1024 in the 16-byte address field
          wgmma_ss_n128(acc[nb], da + 2 * k, db + 2 * k + nb * 1024, (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                      // the group of the previous stage has retired: hand that stage back
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int nb = 0; nb < NB; ++nb) wgmma_fence_regs(acc[nb]);
  }

  pdl_wait();                                          // residual rows / row statistics of the previous kernel are read below
  // per-column vectors of this tile -> smem once (instead of per-element global loads in every thread)
  constexpr bool kHasVec = (EPI == EPI_BIAS || EPI == EPI_BIAS_RES_STATS || EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU);
  if constexpr (kHasVec) {
    for (int i = ct; i < BN; i += 256) {
      const int n = n_blk * BN + i;
      sbias[i] = (p.bias != nullptr && n < p.N) ? __ldg(p.bias + n) : 0.f;
      if constexpr (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU) scol[i] = (n < p.N) ? __ldg(p.colsum + n) : 0.f;
    }
  }
  // every consumer has finished reading the ring (both warpgroups' wgmma retired): it becomes the fp32 staging tile
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* stg = reinterpret_cast<float*>(smem);
  {
    const int w = t >> 5, l = t & 31;
    const int r = row0 + w * 16 + (l >> 2), c0 = (l & 3) * 2;
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = nb * 128 + j * 8 + c0;
        *reinterpret_cast<float2*>(stg + (size_t)r * Cfg::ACC_LD + col) = make_float2(acc[nb][4 * j], acc[nb][4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (size_t)(r + 8) * Cfg::ACC_LD + col) = make_float2(acc[nb][4 * j + 2], acc[nb][4 * j + 3]);
      }
  }
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // this warpgroup's 64 rows are staged

  // ===================================== epilogue =========================================
  // two threads per row (adjacent lanes): half hf owns the 32-column chunks [hf * BN / 64, (hf + 1) * BN / 64)
  const int r_in_tile = row0 + (t >> 1);
  const int hf = t & 1;
  const int row = m_blk * BM + r_in_tile;
  const bool row_ok = row < p.M;

  float mean = 0.f, rstd = 1.f;
  if constexpr (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU || EPI == EPI_RMS_QKV_ROPE || EPI == EPI_RMS_SWIGLU ||
                EPI == EPI_RMS_F32) {
    if (row_ok) {
      float s = 0.f, ss = 0.f;
      const float2* st = p.stats_in + (size_t)row * p.stats_in_nt;
      for (int i = 0; i < p.stats_in_nt; ++i) {
        const float2 v = st[i];
        s += v.x;
        ss += v.y;
      }
      if constexpr (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU) {
        mean = s * p.inv_dim;
        const float var = fmaxf(ss * p.inv_dim - mean * mean, 0.f);
        rstd = rsqrtf(var + p.eps);
      } else {
        rstd = rsqrtf(ss * p.inv_dim + p.eps);
      }
    }
  }
  int b_idx = 0, pos = 0;
  if constexpr (EPI == EPI_RMS_QKV_ROPE) {
    if (row_ok) {
      b_idx = row / p.S;
      pos = p.past + (row % p.S);
    }
  }
  float st_sum = 0.f, st_sq = 0.f;
  long long peer_row = 0;
  if constexpr (EPI == EPI_BIAS_RES_STATS) {
    if (p.n_peers > 0) {
      const int f = row / p.peer_tokens;
      peer_row = (p.peer_frame_off + (long long)f * p.peer_frame_stride) * p.peer_tokens + (row - f * p.peer_tokens);
    }
  }
  const float* srow = stg + (size_t)r_in_tile * Cfg::ACC_LD;
  auto process_chunk = [&](const int c) {
    const int n0 = n_blk * BN + c * 32;
    if (row_ok && n0 < p.N) {
    float v[32];
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 a4 = *reinterpret_cast<const float4*>(srow + c * 32 + i);
      v[i] = a4.x; v[i + 1] = a4.y; v[i + 2] = a4.z; v[i + 3] = a4.w;
    }

    if constexpr (EPI == EPI_BIAS || EPI == EPI_BIAS_RES_STATS) {
      const float4* b4 = reinterpret_cast<const float4*>(sbias + c * 32);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 bb = b4[j];
        v[4 * j] += bb.x; v[4 * j + 1] += bb.y; v[4 * j + 2] += bb.z; v[4 * j + 3] += bb.w;
      }
    }
    if constexpr (EPI == EPI_LN_BIAS || EPI == EPI_LN_BIAS_GELU) {
      const float4* b4 = reinterpret_cast<const float4*>(sbias + c * 32);
      const float4* c4 = reinterpret_cast<const float4*>(scol + c * 32);
      const float nm = -mean * rstd;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 bb = b4[j], cc = c4[j];
        const float bq[4] = {bb.x, bb.y, bb.z, bb.w}, cq[4] = {cc.x, cc.y, cc.z, cc.w};
#pragma unroll
        for (int t4 = 0; t4 < 4; ++t4) {
          float t = fmaf(rstd, v[4 * j + t4], fmaf(nm, cq[t4], bq[t4]));   // rstd*(acc - mean*colsum) + bias
          if constexpr (EPI == EPI_LN_BIAS_GELU) t = quick_gelu_f(t);
          v[4 * j + t4] = t;
        }
      }
    }
    if constexpr (EPI == EPI_RMS_QKV_ROPE || EPI == EPI_RMS_SWIGLU || EPI == EPI_RMS_F32) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] *= rstd;
    }

    if constexpr (EPI == EPI_BIAS_RES_STATS) {
      // residual add, bf16 rounding, partial row statistics of the ROUNDED values
      uint4 o[4];
      const uint4* rp = reinterpret_cast<const uint4*>(p.residual + (size_t)row * p.ldr + n0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 rr = __ldg(rp + j);
        const uint32_t rw[4] = {rr.x, rr.y, rr.z, rr.w};
        uint32_t ow[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float a = v[j * 8 + t * 2] + bf16_lo(rw[t]);
          const float b = v[j * 8 + t * 2 + 1] + bf16_hi(rw[t]);
          ow[t] = pack_bf16x2(a, b);
          const float ar = bf16_lo(ow[t]), br = bf16_hi(ow[t]);
          st_sum += ar + br;
          st_sq += ar * ar + br * br;
        }
        o[j] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
      uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + n0);
#pragma unroll
      for (int j = 0; j < 4; ++j) op[j] = o[j];
      if (p.n_peers > 0) {          // compute + collective in one kernel: the tile is pushed to every rank as it retires
        for (int q = 0; q < p.n_peers; ++q) {
          uint4* pp = reinterpret_cast<uint4*>(p.peer_out[q] + (size_t)peer_row * p.ldo + n0);
#pragma unroll
          for (int j = 0; j < 4; ++j) pp[j] = o[j];
        }
      }
    } else if constexpr (EPI == EPI_RMS_SWIGLU) {
      uint32_t ow[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float a = silu_f(v[4 * j]) * v[4 * j + 1];
        const float b = silu_f(v[4 * j + 2]) * v[4 * j + 3];
        ow[j] = pack_bf16x2(a, b);
      }
      uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + (n0 >> 1));
      op[0] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      op[1] = make_uint4(ow[4], ow[5], ow[6], ow[7]);
    } else if constexpr (EPI == EPI_RMS_F32) {
      float* op = reinterpret_cast<float*>(p.out) + (size_t)row * p.ldo + n0;
      if (n0 + 32 <= p.N && (p.ldo & 3) == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          reinterpret_cast<float4*>(op)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (n0 + i < p.N) op[i] = v[i];
      }
    } else if constexpr (EPI == EPI_RMS_QKV_ROPE) {
      const int which = n0 / p.H;            // 0 q, 1 k, 2 v (uniform over the chunk: H % 32 == 0)
      const int nh = n0 - which * p.H;
      const int head = nh >> 7, cidx = nh & 127;
      if (which < 2) {
        // interleaved layout: columns (2j, 2j+1) hold original dims (j, j+64) of the head
        const float2* cs = p.rope + (size_t)pos * 64 + (cidx >> 1);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 c_s = __ldg(cs + j);
          const float x0 = v[2 * j], x1 = v[2 * j + 1];
          v[2 * j] = x0 * c_s.x - x1 * c_s.y;
          v[2 * j + 1] = x1 * c_s.x + x0 * c_s.y;
        }
      }
      __nv_bfloat16* dst;
      if (which == 0) {
        dst = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + nh;
      } else {
        __nv_bfloat16* cache = (which == 1) ? p.kcache : p.vcache;
        dst = cache + (((size_t)b_idx * p.nH + head) * p.Smax + pos) * 128 + cidx;
      }
      uint4* op = reinterpret_cast<uint4*>(dst);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        op[j] = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                           pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
    } else {
      // EPI_BIAS / EPI_LN_BIAS / EPI_LN_BIAS_GELU -> bf16 rows
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + n0;
      if (n0 + 32 <= p.N && (p.ldo & 7) == 0) {
        uint4* op = reinterpret_cast<uint4*>(dst);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          op[j] = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]), pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                             pack_bf16x2(v[8 * j + 4], v[8 * j + 5]), pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (n0 + i < p.N) dst[i] = __float2bfloat16_rn(v[i]);
      }
    }
    }  // row_ok && n0 < N
  };
  constexpr int CPT = BN / 64;                          // chunks per thread
#pragma unroll
  for (int cc = 0; cc < CPT; ++cc) process_chunk(hf * CPT + cc);
  if constexpr (EPI == EPI_BIAS_RES_STATS) {
    st_sum += __shfl_xor_sync(0xffffffffu, st_sum, 1);
    st_sq += __shfl_xor_sync(0xffffffffu, st_sq, 1);
    if (hf == 0 && row_ok && p.stats_out != nullptr) p.stats_out[(size_t)row * p.num_n_tiles + n_blk] = make_float2(st_sum, st_sq);
  }
}

}  // namespace vly
