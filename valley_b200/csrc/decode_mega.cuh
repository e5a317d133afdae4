// One persistent cooperative kernel per decode step ("mega-kernel").
//
// Decode at B <= 4 is pure weight streaming (13.2 GB / step at 7B, 25.7 GB at 13B).  Launching 5 kernels per layer leaves the
// HBM idle at every kernel boundary (launch gap, activation staging, first-load latency, tail imbalance: ~5 us x 160 per step).
// Here ONE kernel runs the whole step on one CTA per SM:
//   warp 0 (1 thread) : producer -- walks the step's weight matrices in execution order (QKV, o_proj, gate/up, down of
//                       every layer, then lm_head) and streams this CTA's rows through a shared-memory ring with 1-D bulk
//                       (TMA) copies, mbarrier complete_tx.  It never waits for a phase boundary -- weights do not depend on
//                       activations -- so while the consumers sit in a grid barrier the ring fills with the NEXT phase's
//                       weights and HBM keeps streaming.  The ring geometry is PER PHASE (PhaseDesc::rows, ::kc, chosen on the
//                       host per matrix shape): K is cut into equal stages (no short tail stage: 5120 = 2 x 2560, not
//                       2048 + 2048 + 1024) and the rows per work unit are picked so the units balance over the SMs
//                       (on 132 SMs: 5120 rows = 640 units of 8 = 4.8 per SM -> 5 rounds at 97 %; 1280 units of 4 -> 10 rounds at 97 %).
//   warps 1..16       : compute -- per phase: the activation rows arrive in shared memory by bulk copy (RMSNorm statistics
//                       where a norm is folded), multiply the ring stages (fp32 accumulate), warp-reduce, and hand the 16
//                       per-warp partials of a work unit to the finalize warp through a 4-slot mbarrier handoff -- there is NO
//                       blocking barrier inside the streaming loop.  The attention phase runs warp-per-item (32 keys of one
//                       (sequence, head) per item, online softmax in registers, last-arriver merge): no block-level barrier.
//                       Phases are separated by a grid-wide barrier.
//   warp 17           : finalize -- sums the partials and runs the fused epilogue (RoPE + KV append, SwiGLU, residual,
//                       logits + running arg-max); its global operands are prefetched while the unit is being computed.
// Cross-CTA activations are read through L2 (bulk copies / ld.global.cg) -- the L1 of an SM is not coherent with other SMs' writes.
#pragma once
#include "common.cuh"
#include "simt_kernels.cuh"
#include "decode_kernels.cuh"
#include "sampling.cuh"

namespace vly {

enum PhaseType : int { PH_QKV = 0, PH_ATTN = 1, PH_OPROJ = 2, PH_GATEUP = 3, PH_DOWN = 4, PH_LOGITS = 5 };

struct PhaseDesc {
  int type, N, K, layer;
  int rows, kc;                 // ring geometry of this phase: weight rows per work unit, columns per ring stage
  int inflight;                 // stages of THIS phase's size kept in flight (~100 KB of bulk copies outstanding per SM)
  const __nv_bfloat16* W;       // [N, K] (nullptr for PH_ATTN)
  const __nv_bfloat16* x_in;    // activation rows [B, K]
  __nv_bfloat16* out;           // QKV: q [B,H]; OPROJ/DOWN: x [B,H] (in place, also the residual); GATEUP: hb [B,I]
  __nv_bfloat16* kcache;        // [B, nH, Smax, 128] of this layer
  __nv_bfloat16* vcache;
};

struct StepParams {
  const PhaseDesc* phases;
  int n_phases;
  int B, H, nH, Smax, V, Kmax;
  float eps, scale_log2e;
  const float2* rope;
  int* seq_len;                 // tokens in the cache before this step (== position of the new token); bumped at the end
  int* step;                    // column of out_tokens; bumped at the end
  const __nv_bfloat16* embed;
  const long long* tokens_in;   // [B]
  __nv_bfloat16* x;             // [B, H] residual stream
  const __nv_bfloat16* q;       // [B, H]
  __nv_bfloat16* attn;          // [B, H]
  float* part_o;                // [B*nH, nsplit, 128]
  float2* part_ml;              // [B*nH, nsplit]
  unsigned int* attn_counters;  // [B*nH]
  int nsplit;                   // capacity of the split dimension (Smax / ATTN_KEYS_MIN)
  const uint32_t* key_bits;     // [B, mask_words] attention_mask, one bit per cache position (1 = attend)
  int mask_words;
  float* logits;                // [B, V]
  float* part_val;              // [B, grid]
  int* part_idx;
  long long* next_tokens;       // [B]
  long long* out_tokens;        // [B, out_stride]
  int out_stride;
  SampleState* sample;          // token selection state (greedy / temperature sampling, eos bookkeeping); sampling.cuh
  unsigned int* grid_counter;   // monotonically increasing arrival counter of the grid barrier (never reset: no memset node per step)
  unsigned int* grid_epoch;     // launches that ran to completion; barrier k of a launch waits for (epoch * n_grid_syncs + k) * gridDim
  int n_grid_syncs;             // grid barriers one launch executes (one per grid-synchronised phase + the embedding phase)
  int attn_ikeys;               // 0: pick 16 / 32 keys per attention item by shape; else forced (VLY_ATTN_IKEYS, A/B measurements)
  int n_stages;
  int stage_bytes;              // ring slot size: max over the phases of rows * (kc * 2 + row pad)
  int n_inflight;               // global cap on the stages in flight (PhaseDesc::inflight is the per-phase value; the ring may be deeper)
  int l2_hint;                  // 1: the weight copies into the ring carry L2::evict_first; 0: no cache hint
  long long* dbg;               // optional [gridDim][32] cycle counters: [0..3] sync, stage-x, weight loop, attention totals;
                                // [8 + 3*type + {0,1,2}] = stage-x, loop, trailing grid sync of every phase of that PhaseType;
                                // [26 + type] = cycles the producer waited for a free ring slot while filling that PhaseType
  int select;                   // 1: the last phase selects the tokens; 0: it writes the logits and a provisional arg-max, and
                                // sample_filter_kernel selects after the step (a top-k / top-p request)
};

struct MegaCfg {
  static constexpr int ROWS = 4;                         // CUDA-core path (B = 1): at most 4 weight rows per work unit
  static constexpr int ROWS_TC = 8;                      // tensor-core path (B = 2..4): at most 8 (the N of an m16n8k16 MMA)
  static constexpr int PAD_TC = 64;                      // tensor-core path: rows of a ring stage / of the activation block are
                                                         // 64 bytes apart modulo 128, so the 16-byte fragment loads of a
                                                         // quarter-warp never share a bank
  static constexpr int CONSUMERS = 512, THREADS = 576;   // producer warp + 16 compute warps + 1 finalize warp
  static constexpr int RED_SLOTS = 4;
  static constexpr int MAX_STAGES = 8;
  static constexpr int ATTN_KEYS_MIN = 16;               // keys per attention work item: 16 (one pass) while every item finds a
                                                         // free warp, else 32 (two passes); the split buffers hold Smax / 16
};

VLY_DEVINL uint4 ldcg_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];\n" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
VLY_DEVINL float ldcg_bf16(const __nv_bfloat16* p) {
  unsigned short v;
  asm volatile("ld.global.cg.u16 %0, [%1];\n" : "=h"(v) : "l"(p) : "memory");
  return __uint_as_float((uint32_t)v << 16);
}
// D[16x8] += A[16x16] * B[16x8], bf16 inputs, fp32 accumulate (legacy tensor path: plenty for an HBM-bound consumer)
VLY_DEVINL void mma_m16n8k16_bf16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

VLY_DEVINL uint32_t ld_acquire_u32(const unsigned int* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// generic-proxy writes (other CTAs', made visible by the grid barrier) -> async-proxy (bulk copy) reads of global memory
VLY_DEVINL void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }

// consumers-only grid barrier (512 threads per CTA take part; the producer warp streams on)
VLY_DEVINL void grid_sync_consumers(unsigned int* counter, unsigned int target, int ct) {
  asm volatile("bar.sync 2, 544;" ::: "memory");          // every write of this CTA happens-before thread 0's release
  if (ct == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;\n" ::"l"(counter) : "memory");
    while ((int)(ld_acquire_u32(counter) - target) < 0) {     // wrap-safe
    }
  }
  asm volatile("bar.sync 2, 544;" ::: "memory");
}

// ------------------------------ attention phase ------------------------------
// Runs on the 16 compute warps (cw = 0..15); no block-level barrier inside.
// (A CTA-per-(sequence, head) variant with a shared-memory merge was measured at 13B, B = 4: slower -- one SM cannot keep enough
//  K/V loads in flight from registers; spreading every head over all SMs wins despite the global-memory merge.)
VLY_DEVINL void mega_attention_phase(const StepParams& p, const PhaseDesc& d, const int cw, const int lane, const int pos) {
  // ------------------------------ attention: one warp per (sequence, head, key split) ------------------------------
  // A half-warp covers one key row (16 lanes x 16 bytes = 128 head dims); a pass handles 16 keys (8 per half-warp): all 8 K
  // and 8 V rows of a lane are requested up front (one L2 / HBM round trip), scores are reduced with a transposing shuffle
  // tree (8 instead of 32 shuffles), softmax runs online in registers across the passes of an item, P.V accumulates per
  // lane over its 8 head dims.  Items are dealt warp-major over the SMs so one layer's K/V is pulled by every SM at once.
  const int len = pos + 1;
  // Item size = a multiple of 16 keys (one 16-key pass per 16).  What costs is the NUMBER of items -- every item ends in a
  // publish (partial stores, fence, atomic) and is one more partial for the merge -- while a pass only lengthens a warp's serial
  // chain.  So: 16 keys if every 16-key item finds its own warp (B = 1), else the smallest multiple of 16 >= 32 whose item count fits the
  // warps (5 % overflow into a second, nearly empty round costs less than a third pass for everybody).
  const int n_warps = 16 * (int)gridDim.x;
  int ikeys = p.attn_ikeys;
  if (ikeys == 0) {
    if (p.B * p.nH * ((len + 15) >> 4) <= n_warps) ikeys = 16;
    else
      for (ikeys = 32; ikeys < 256; ikeys += 16)
        if (p.B * p.nH * ((len + ikeys - 1) / ikeys) <= n_warps + n_warps / 20) break;
  }
  const int n_act = (len + ikeys - 1) / ikeys;
  const int items = p.B * p.nH * n_act;
  const int hl = lane & 15, hw = lane >> 4;
  for (int it = cw * gridDim.x + blockIdx.x; it < items; it += gridDim.x * 16) {
    const int split = it % n_act, bh = it / n_act;
    const int b = bh / p.nH, h = bh - b * p.nH;
    const int k0 = split * ikeys, nk = min(len - k0, ikeys);
    const __nv_bfloat16* kb = d.kcache + ((size_t)bh * p.Smax + k0) * 128 + hl * 8;
    const __nv_bfloat16* vb = d.vcache + ((size_t)bh * p.Smax + k0) * 128 + hl * 8;
    const uint32_t* kbw = p.key_bits + (size_t)b * p.mask_words;                                  // one mask bit per cache position
    float qf[8];
    {
      const uint4 w = ldcg_v4(p.q + (size_t)b * p.H + h * 128 + hl * 8);
      qf[0] = bf16_lo(w.x); qf[1] = bf16_hi(w.x); qf[2] = bf16_lo(w.y); qf[3] = bf16_hi(w.y);
      qf[4] = bf16_lo(w.z); qf[5] = bf16_hi(w.z); qf[6] = bf16_lo(w.w); qf[7] = bf16_hi(w.w);
    }
    float m_run = -INFINITY, l_run = 0.f;
    float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int kk0 = 0; kk0 < nk; kk0 += 16) {
      const uint32_t kbits = __ldg(kbw + ((k0 + kk0) >> 5)) >> ((k0 + kk0) & 31);                // the 16 mask bits of this pass
      uint4 kw[8], vw[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = kk0 + 2 * j + hw;
        const bool ok = key < nk;
        kw[j] = ok ? ldcg_v4(kb + (size_t)key * 128) : make_uint4(0, 0, 0, 0);
        vw[j] = ok ? ldcg_v4(vb + (size_t)key * 128) : make_uint4(0, 0, 0, 0);
      }
      float sc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint4 w = kw[j];
        sc[j] = qf[0] * bf16_lo(w.x) + qf[1] * bf16_hi(w.x) + qf[2] * bf16_lo(w.y) + qf[3] * bf16_hi(w.y) +
                qf[4] * bf16_lo(w.z) + qf[5] * bf16_hi(w.z) + qf[6] * bf16_lo(w.w) + qf[7] * bf16_hi(w.w);
      }

      // transposing reduction over the 16 lanes of the half-warp: afterwards sc[0] = the full dot product of key
      // kk0 + 2 * (hl >> 1) + hw (held twice: lanes hl and hl ^ 1)
#pragma unroll
      for (int off = 8, n = 4; off >= 2; off >>= 1, n >>= 1) {
        const bool up = (hl & off) != 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i < n) {
            const float send = up ? sc[i] : sc[i + n];
            const float keep = up ? sc[i + n] : sc[i];
            sc[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
          }
        }
      }
      sc[0] += __shfl_xor_sync(0xffffffffu, sc[0], 1);
      const int my_key = kk0 + 2 * (hl >> 1) + hw;
      const bool valid = my_key < nk && ((kbits >> (my_key - kk0)) & 1u);
      const float s_my = valid ? sc[0] * p.scale_log2e : -INFINITY;
      float mx = s_my;
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 8));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 16));
      const float m_new = fmaxf(m_run, mx);
      const float pm = valid ? fast_exp2(s_my - m_new) : 0.f;              // (valid => m_new is finite)
      const float corr = (m_run > -INFINITY) ? fast_exp2(m_run - m_new) : 0.f;
      float ls = pm;                                                         // every key is held by a lane pair: skip xor 1
      ls += __shfl_xor_sync(0xffffffffu, ls, 2);
      ls += __shfl_xor_sync(0xffffffffu, ls, 4);
      ls += __shfl_xor_sync(0xffffffffu, ls, 8);
      ls += __shfl_xor_sync(0xffffffffu, ls, 16);
      l_run = l_run * corr + ls;
      m_run = m_new;
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] *= corr;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float pj = __shfl_sync(0xffffffffu, pm, (lane & 16) + 2 * j);  // weight of key kk0 + 2j + hw
        const uint4 w = vw[j];
        o[0] = fmaf(pj, bf16_lo(w.x), o[0]); o[1] = fmaf(pj, bf16_hi(w.x), o[1]);
        o[2] = fmaf(pj, bf16_lo(w.y), o[2]); o[3] = fmaf(pj, bf16_hi(w.y), o[3]);
        o[4] = fmaf(pj, bf16_lo(w.z), o[4]); o[5] = fmaf(pj, bf16_hi(w.z), o[5]);
        o[6] = fmaf(pj, bf16_lo(w.w), o[6]); o[7] = fmaf(pj, bf16_hi(w.w), o[7]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] += __shfl_xor_sync(0xffffffffu, o[e], 16);   // even + odd keys
    if (n_act == 1) {
      // the whole (sequence, head) fitted one item: no partials, no merge
      if (hw == 0) {
        const float inv = l_run > 0.f ? 1.f / l_run : 0.f;
        *reinterpret_cast<uint4*>(p.attn + (size_t)b * p.H + h * 128 + hl * 8) =
            make_uint4(pack_bf16x2(o[0] * inv, o[1] * inv), pack_bf16x2(o[2] * inv, o[3] * inv),
                       pack_bf16x2(o[4] * inv, o[5] * inv), pack_bf16x2(o[6] * inv, o[7] * inv));
      }
      continue;
    }
    float* po = p.part_o + ((size_t)bh * p.nsplit + split) * 128 + hl * 8;
    if (hw == 0) {
      *reinterpret_cast<float4*>(po) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(po + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
    if (lane == 0) p.part_ml[(size_t)bh * p.nsplit + split] = make_float2(m_run, l_run);
    // publish: every lane's partial stores, then ONE acq_rel atomic by lane 0 (release orders the warp's stores -- made
    // cumulative by the __syncwarp -- before the count; acquire orders the merger's loads after it).  A separate membar.gl in
    // every lane plus a relaxed atomic cost an extra L2 round trip on the phase's critical path.
    __syncwarp();
    int last = 0;
    if (lane == 0) {
      unsigned int old;
      asm volatile("fence.acq_rel.gpu;\n\tatom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(p.attn_counters + bh) : "memory");
      last = (old == (unsigned)n_act - 1);
    }
    last = __shfl_sync(0xffffffffu, last, 0);
    if (last) {
      // ---- merge of the n_act (<= 128) partials by the warp that arrived last: lane s holds (max, sum) of splits s + 32 i.
      // The first batch of partial outputs is requested together with the (max, sum) pairs: one L2 round trip, not two.
      const float* pb = p.part_o + (size_t)bh * p.nsplit * 128 + lane * 4;
      float4 v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j)
        v[j] = (j < n_act) ? __ldcg(reinterpret_cast<const float4*>(pb + (size_t)j * 128)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float mv[4], lv[4], wv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        mv[i] = -INFINITY;
        lv[i] = 0.f;
        if (lane + 32 * i < n_act) {
          const float2 ml = __ldcg(&p.part_ml[(size_t)bh * p.nsplit + lane + 32 * i]);
          mv[i] = ml.x;
          lv[i] = ml.y;
        }
      }
      const float Mx = warp_max(fmaxf(fmaxf(mv[0], mv[1]), fmaxf(mv[2], mv[3])));
      float lw = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        wv[i] = lv[i] > 0.f ? fast_exp2(mv[i] - Mx) : 0.f;                  // a fully masked split has m = -inf, l = 0
        lw += lv[i] * wv[i];
      }
      const float L = warp_sum(lw);
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int s0 = 0; s0 < n_act; s0 += 8) {
        const int gi = s0 >> 5;
        const float wsel = gi == 0 ? wv[0] : (gi == 1 ? wv[1] : (gi == 2 ? wv[2] : wv[3]));
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float w = __shfl_sync(0xffffffffu, wsel, (s0 + j) & 31);
          acc.x = fmaf(v[j].x, w, acc.x); acc.y = fmaf(v[j].y, w, acc.y);
          acc.z = fmaf(v[j].z, w, acc.z); acc.w = fmaf(v[j].w, w, acc.w);
        }
        if (s0 + 8 < n_act) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            v[j] = (s0 + 8 + j < n_act) ? __ldcg(reinterpret_cast<const float4*>(pb + (size_t)(s0 + 8 + j) * 128)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      const float inv = L > 0.f ? 1.f / L : 0.f;
      *reinterpret_cast<uint2*>(p.attn + (size_t)b * p.H + h * 128 + lane * 4) =
          make_uint2(pack_bf16x2(acc.x * inv, acc.y * inv), pack_bf16x2(acc.z * inv, acc.w * inv));
      if (lane == 0) p.attn_counters[bh] = 0;
    }
  }
}

// operands of the epilogue that do not depend on the unit's result: fetched while the unit is still being computed
VLY_DEVINL void mega_epilogue_prefetch(const StepParams& p, const PhaseDesc& d, const bool ok, const int b, const int n, const int pos,
                                       float& pre0, float& pre1) {
  if (ok) {
    if (d.type == PH_OPROJ || d.type == PH_DOWN) pre0 = ldcg_bf16(d.out + (size_t)b * d.N + n);
    else if (d.type == PH_QKV && n < 2 * p.H) {
      const float2 cs = __ldg(p.rope + (size_t)pos * 64 + ((n & 127) >> 1));
      pre0 = cs.x;
      pre1 = cs.y;
    }
  }
}

// ------------------------------ fused epilogue of one work unit ------------------------------
// Executed by the lanes < NV of the epilogue warp: lane = r * BMAX + b holds t = the finished dot product of weight row n = n0 + r
// and batch row b.  pre0 / pre1: the operand prefetched before the unit completed (residual, or RoPE cos / sin).
template <int BMAX, int NV>
VLY_DEVINL void mega_unit_epilogue(const StepParams& p, const PhaseDesc& d, const int lane, const float t, const bool ok, const int r,
                                   const int b, const int n, const float pre0, const float pre1, const int pos, const float* rstd_s,
                                   float* bestv, int* besti, const bool samp_on, const float samp_it, const uint32_t samp_k0,
                                   const uint32_t samp_k1) {
  constexpr unsigned kMask = (NV == 32) ? 0xffffffffu : ((1u << NV) - 1u);
  if (d.type == PH_OPROJ || d.type == PH_DOWN) {
    if (ok) d.out[(size_t)b * d.N + n] = __float2bfloat16_rn(t + pre0);
  } else if (d.type == PH_LOGITS) {
    const float y = t * rstd_s[b];
    if (ok && p.logits != nullptr) p.logits[(size_t)b * d.N + n] = y;
    // greedy: the logit itself; sampling: logit / T + Gumbel noise (arg-max == multinomial(softmax(logits / T)))
    float bv = ok ? (samp_on ? sample_score(y, samp_it, samp_k0, samp_k1, n, b, pos) : y) : -INFINITY;
    int bi = n;
#pragma unroll
    for (int o = BMAX; o < NV; o <<= 1) {
      const float ov = __shfl_xor_sync(kMask, bv, o);
      const int oi = __shfl_xor_sync(kMask, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane < BMAX && lane < p.B && bv > bestv[lane]) {
      bestv[lane] = bv;
      besti[lane] = bi;
    }
  } else {
    const float mine = t * rstd_s[b];
    const float other = __shfl_xor_sync(kMask, mine, BMAX);
    if ((r & 1) == 0 && ok && n + 1 < d.N) {
      float x0 = mine, x1 = other;
      if (d.type == PH_GATEUP) {
        const float gte = bf16_round(x0), up = bf16_round(x1);      // HF:modeling_llama.py:182-184 rounds both
        d.out[(size_t)b * (d.N >> 1) + (n >> 1)] = __float2bfloat16_rn(bf16_round(gte / (1.f + __expf(-gte))) * up);
      } else {
        const int which = n / p.H, nh = n - which * p.H, head = nh >> 7, cidx = nh & 127;
        if (which < 2) {
          const float a = x0 * pre0 - x1 * pre1, c2 = x1 * pre0 + x0 * pre1;   // (cos, sin) prefetched
          x0 = a;
          x1 = c2;
        }
        __nv_bfloat16* dst;
        if (which == 0) dst = d.out + (size_t)b * p.H + nh;
        else dst = ((which == 1) ? d.kcache : d.vcache) + (((size_t)b * p.nH + head) * p.Smax + pos) * 128 + cidx;
        *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(x0, x1);
      }
    }
  }
}

// ---- arg-max over the per-CTA partials (lowest index on ties, like torch.argmax); advance the counters.
// Executed by the 16 compute warps of CTA 0 after the last grid barrier of the step. ----
VLY_DEVINL void mega_finish_step(const StepParams& p, const int cw, const int lane, const int ct) {
  if (cw < p.B) {
    const int b = cw;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int g = lane; g < (int)gridDim.x; g += 32) {
      const float v = __ldcg(p.part_val + (size_t)b * gridDim.x + g);
      const int i = __ldcg(p.part_idx + (size_t)b * gridDim.x + g);
      if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    warp_argmax(bv, bi);
    if (lane == 0) {
      const long long tok = p.select ? sample_finish_row(p.sample, b, bi) : bi;
      p.next_tokens[b] = tok;
      if (p.out_tokens != nullptr) p.out_tokens[(size_t)b * p.out_stride + *p.step] = tok;
    }
  }
  asm volatile("bar.sync 7, 512;" ::: "memory");
  if (ct == 0) {
    *p.step += 1;
    *p.seq_len += 1;
    *p.grid_epoch += 1;          // every CTA has passed the last barrier of this launch (they read the epoch at their start)
    if (p.select) sample_close_step(p.sample, p.B, true);
    else p.sample->steps_valid += 1;   // (sample_filter_kernel keeps done / all_done)
  }
}

template <int BMAX>
__global__ void __launch_bounds__(576, 1) decode_step_kernel(const StepParams p) {
  using M = MegaCfg;
  constexpr bool kTC = BMAX > 1;                                                         // tensor-core consumers
  constexpr int ROWS = kTC ? M::ROWS_TC : M::ROWS;                                       // max weight rows per work unit
  constexpr int NV = ROWS * BMAX;
  constexpr int PAD = kTC ? M::PAD_TC : 0;                                               // bytes appended to every ring / activation row
  extern __shared__ uint8_t msm_raw[];
  uint8_t* msm = msm_raw + ((128u - (smem_u32(msm_raw) & 127u)) & 127u);
  uint8_t* ring = msm;                                                                   // [n_stages][stage_bytes]
  __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(ring + (size_t)p.n_stages * p.stage_bytes);   // [BMAX][xs_stride]
  // activation rows: stride == Kmax for the CUDA-core path; == 64 bytes modulo 128 for the tensor-core path
  const int xs_stride = kTC ? (((p.Kmax * 2 + 127) & ~127) + PAD) / 2 : p.Kmax;
  const size_t xs_bytes = ((size_t)BMAX * xs_stride * 2 + 127) & ~size_t(127);
  uint8_t* tail = reinterpret_cast<uint8_t*>(xs) + xs_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty_bar = full_bar + M::MAX_STAGES;
  uint64_t* red_full = empty_bar + M::MAX_STAGES;                                        // [RED_SLOTS]
  uint64_t* red_empty = red_full + M::RED_SLOTS;                                         // [RED_SLOTS]
  uint64_t* x_bar = red_empty + M::RED_SLOTS;                                            // activation block landed
  float* red = reinterpret_cast<float*>(x_bar + 2);                                      // [RED_SLOTS][16][NV]
  float* rstd_s = red + M::RED_SLOTS * 16 * NV;                                          // [BMAX]
  float* bestv = rstd_s + BMAX;                                                          // [BMAX]
  int* besti = reinterpret_cast<int*>(bestv + BMAX);                                     // [BMAX]
  float* wred = reinterpret_cast<float*>(besti + BMAX);                                  // [16][BMAX]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (p.sample->all_done) return;       // every sequence has produced its stop token: the remaining replays are no-ops
  if (tid == 0) {
    for (int i = 0; i < p.n_stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 16);
    }
    for (int i = 0; i < M::RED_SLOTS; ++i) {
      mbar_init(&red_full[i], 16);
      mbar_init(&red_empty[i], 1);
    }
    mbar_init(x_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ======================================= producer =======================================
    if (lane == 0) {
      int st = 0;
      uint32_t ph = 0;
      // The ring may be deeper than the number of copies kept in flight: what streams fastest is a bounded number of bytes
      // outstanding per SM, but while the consumers sit in a grid barrier / stage activations the extra
      // slots keep HBM busy.
      int wst = 0, issued = 0, confirmed = 0;
      uint32_t wph = 0;
      long long* dbg_p = p.dbg != nullptr ? p.dbg + (size_t)blockIdx.x * 32 : nullptr;
      if (dbg_p != nullptr)
        for (int i = 26; i < 32; ++i) dbg_p[i] = 0;
      // The weights are read once per step (25.7 GB at 13B, 500x the L2): their copies carry L2::evict_first, so the stream
      // does not push out what the latency-bound parts of the step wait on -- the grid-barrier counter, the activation rows,
      // the attention partials and the KV cache.
      const bool hint = p.l2_hint != 0;
      const uint64_t pol_stream = l2_policy_evict_first();
      for (int pi = 0; pi < p.n_phases; ++pi) {
        // by value: a reference would be re-read from global memory after every mbarrier asm ("memory" clobber), and the time the
        // producer needs to re-arm a freed slot comes straight out of the bytes in flight
        const PhaseDesc d = p.phases[pi];
        if (d.type == PH_ATTN) continue;
        const int rows_u = d.rows, KCp = d.kc;
        const int row_stride = KCp * 2 + PAD;
        const int n_groups = (d.N + rows_u - 1) / rows_u;
        const int n_slices = (d.K + KCp - 1) / KCp;
        const int infl = min(d.inflight, p.n_inflight);
        long long t_blocked = 0;
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x) {
          const int n0 = g * rows_u;
          const int rows = min(rows_u, d.N - n0);
          for (int s = 0; s < n_slices; ++s) {
            const int kc = min(KCp, d.K - s * KCp);
            const long long t_w = dbg_p != nullptr ? clock64() : 0;
            mbar_wait(&empty_bar[st], ph ^ 1);
            while (issued - confirmed >= infl) {          // at most `infl` copies outstanding: the oldest must have landed
              mbar_wait(&full_bar[wst], wph);
              if (++wst == p.n_stages) { wst = 0; wph ^= 1; }
              ++confirmed;
            }
            if (dbg_p != nullptr) t_blocked += clock64() - t_w;
            ++issued;
            mbar_expect_tx(&full_bar[st], (uint32_t)rows * kc * 2);
            uint8_t* dst = ring + (size_t)st * p.stage_bytes;
            const __nv_bfloat16* src = d.W + (size_t)n0 * d.K + (size_t)s * KCp;
            if (PAD == 0 && kc == d.K) {                  // whole rows, unpadded: the unit is ONE contiguous block
              if (hint) bulk_load_1d_hint(dst, src, (uint32_t)rows * kc * 2, &full_bar[st], pol_stream);
              else bulk_load_1d(dst, src, (uint32_t)rows * kc * 2, &full_bar[st]);
            } else if (hint) {
              for (int r = 0; r < rows; ++r)
                bulk_load_1d_hint(dst + r * row_stride, src + (size_t)r * d.K, (uint32_t)kc * 2, &full_bar[st], pol_stream);
            } else {
              for (int r = 0; r < rows; ++r) bulk_load_1d(dst + r * row_stride, src + (size_t)r * d.K, (uint32_t)kc * 2, &full_bar[st]);
            }
            if (++st == p.n_stages) { st = 0; ph ^= 1; }
          }
        }
        // (the phase being filled, not the one being computed: the producer runs up to a ring ahead of the consumers)
        if (dbg_p != nullptr) dbg_p[26 + d.type] += t_blocked;
      }
    }
    return;
  }

  // ================================ compute warps (1..16) and finalize warp (17) ================================
  const bool is_fin = (warp == 17);
  const int ct = tid - 32;            // compute thread 0..511 (finalize warp: 512..543)
  const int cw = warp - 1;            // compute warp 0..15
  const int pos = *p.seq_len;
  const bool samp_on = p.select && p.sample->enabled != 0;
  const float samp_it = p.sample->inv_temp;
  const uint32_t samp_k0 = p.sample->seed_lo, samp_k1 = p.sample->seed_hi;
  unsigned int sync_no = 0;
  // written by block 0 at the very end of the previous completed launch (stream order): the same value in every CTA
  const unsigned int sync_base = *p.grid_epoch * (unsigned int)p.n_grid_syncs * gridDim.x;
  long long t_sync = 0, t_stage = 0, t_loop = 0, t_attn = 0, t0 = clock64();
  long long* dbg_o = (p.dbg != nullptr && ct == 0) ? p.dbg + (size_t)blockIdx.x * 32 : nullptr;
  if (dbg_o != nullptr)
    for (int i = 8; i < 26; ++i) dbg_o[i] = 0;       // [26, 32) belong to the producer
  // ---- phase -1: x = embed[token] (decode input) ----
  {
    if (!is_fin) {
      const int chunks = p.B * (p.H >> 3);
      for (int i = blockIdx.x * M::CONSUMERS + ct; i < chunks; i += gridDim.x * M::CONSUMERS) {
        const int b = i / (p.H >> 3), c = i % (p.H >> 3);
        long long id = p.tokens_in[b];
        id = id < 0 ? 0 : (id >= p.V ? p.V - 1 : id);
        *reinterpret_cast<uint4*>(p.x + (size_t)b * p.H + c * 8) = *reinterpret_cast<const uint4*>(p.embed + (size_t)id * p.H + c * 8);
      }
    } else if (lane < BMAX) {
      bestv[lane] = -INFINITY;
      besti[lane] = 0;
    }
    grid_sync_consumers(p.grid_counter, sync_base + (++sync_no) * gridDim.x, ct);
    t_sync += clock64() - t0;
  }

  int st = 0;
  uint32_t ph = 0, xph = 0;
  unsigned int unit_no = 0;           // running work-unit counter of this CTA: selects the handoff slot
  for (int pi = 0; pi < p.n_phases; ++pi) {
    const PhaseDesc d = p.phases[pi];
    // (an L1 prefetch of the next descriptor was tried here: it made every grid barrier ~1 us SLOWER -- bisected on the GPU)
    t0 = clock64();
    if (d.type == PH_ATTN) {
      if (!is_fin) mega_attention_phase(p, d, cw, lane, pos);
      t_attn += clock64() - t0;
      if (dbg_o != nullptr) dbg_o[8 + 3 * PH_ATTN + 1] += clock64() - t0;
    } else {
      // ------------------------------ weight phase ------------------------------
      const bool norm = (d.type == PH_QKV || d.type == PH_GATEUP || d.type == PH_LOGITS);
      const int rows_u = d.rows, KCp = d.kc;
      const int row_stride = KCp * 2 + PAD;
      if (!is_fin) {
        // the activation rows [B, K] (written by other CTAs before the grid barrier) arrive by bulk copy: one thread issues B
        // copies, everybody waits on the mbarrier -- one L2 round trip whatever K is, no per-thread load loop
        if (ct == 0) {
          fence_proxy_async_global();
          mbar_expect_tx(x_bar, (uint32_t)p.B * d.K * 2);
          for (int b = 0; b < p.B; ++b) bulk_load_1d(xs + (size_t)b * xs_stride, d.x_in + (size_t)b * d.K, (uint32_t)d.K * 2, x_bar);
        }
        mbar_wait(x_bar, xph);
        if (norm) {
          float sq[BMAX];
#pragma unroll
          for (int b = 0; b < BMAX; ++b) sq[b] = 0.f;
          const int chunks = d.K >> 3;
          for (int c = ct; c < chunks; c += M::CONSUMERS) {
#pragma unroll
            for (int b = 0; b < BMAX; ++b) {
              if (b < p.B) {
                const uint4 w = *reinterpret_cast<const uint4*>(xs + (size_t)b * xs_stride + c * 8);
                const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const float a = bf16_lo(ww[i]), bb = bf16_hi(ww[i]);
                  sq[b] += a * a + bb * bb;
                }
              }
            }
          }
#pragma unroll
          for (int b = 0; b < BMAX; ++b) {
            const float v = warp_sum(sq[b]);
            if (lane == 0) wred[cw * BMAX + b] = v;
          }
        }
      }
      xph ^= 1;
      if (norm) {
        asm volatile("bar.sync 2, 544;" ::: "memory");
        if (!is_fin && ct < BMAX) {
          float t = 0.f;
          for (int w = 0; w < 16; ++w) t += wred[w * BMAX + ct];
          rstd_s[ct] = rsqrtf(t / d.K + p.eps);
        }
        asm volatile("bar.sync 2, 544;" ::: "memory");
      }
      t_stage += clock64() - t0;
      if (dbg_o != nullptr) dbg_o[8 + 3 * d.type] += clock64() - t0;
      t0 = clock64();
      const int n_groups = (d.N + rows_u - 1) / rows_u;
      const int n_slices = (d.K + KCp - 1) / KCp;
      if (!is_fin) {
        // ===== compute warps: ring stage x activation rows -> per-warp partials -> handoff slot =====
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++unit_no) {
          const int n0 = g * rows_u;
          const int rows = min(rows_u, d.N - n0);
          const int slot = unit_no & (M::RED_SLOTS - 1);
          const uint32_t round = (unit_no / M::RED_SLOTS) & 1;
          if constexpr (kTC) {
            // ---- tensor-core consumer (B = 2..4): mma.sync m16n8k16 with A = activation rows (batch on M, rows >= B zero)
            // and B = up to 8 weight rows (N).  Lane (g = lane/4, t = lane%4) loads 16 contiguous bytes x[g][k..k+7] and
            // W[g][k..k+7]; both operands use the same k permutation, so two MMAs consume them.  The 32-wide k blocks of a
            // stage are dealt round-robin to the 16 warps.
            const int gq = lane >> 2, tq = lane & 3;
            // (two accumulators keep the pair of MMAs of a k block independent: the MMA latency, not the issue rate, would
            //  otherwise bound the consumers)
            float dacc[4] = {0.f, 0.f, 0.f, 0.f}, dacc1[4] = {0.f, 0.f, 0.f, 0.f};
            const bool w_ok = gq < rows, x_ok = gq < p.B;
            for (int s = 0; s < n_slices; ++s) {
              const int kc = min(KCp, d.K - s * KCp);
              mbar_wait(&full_bar[st], ph);
              const uint8_t* wrow = ring + (size_t)st * p.stage_bytes + gq * row_stride;
              const __nv_bfloat16* xrow = xs + (size_t)gq * xs_stride + (size_t)s * KCp;
              // the 32-column k blocks of the stage are dealt to the 16 warps in contiguous runs
              const int nblk = kc >> 5, bpw = (nblk + 15) >> 4;
              const int kb0 = cw * bpw, kb1 = min(kb0 + bpw, nblk);
#pragma unroll 4
              for (int kb = kb0; kb < kb1; ++kb) {
                const int k = kb << 5;
                uint4 wb = make_uint4(0, 0, 0, 0), xa = make_uint4(0, 0, 0, 0);
                if (w_ok) wb = *reinterpret_cast<const uint4*>(wrow + (k + tq * 8) * 2);
                if (x_ok) xa = *reinterpret_cast<const uint4*>(xrow + k + tq * 8);
                mma_m16n8k16_bf16(dacc, xa.x, 0u, xa.y, 0u, wb.x, wb.y);
                mma_m16n8k16_bf16(dacc1, xa.z, 0u, xa.w, 0u, wb.z, wb.w);
              }
              __syncwarp();
              if (lane == 0) mbar_arrive(&empty_bar[st]);
              if (++st == p.n_stages) { st = 0; ph ^= 1; }
            }
            dacc[0] += dacc1[0];
            dacc[1] += dacc1[1];
            // lane (g < B, t) holds D[batch g][weight rows 2t, 2t+1] summed over this warp's k range
            mbar_wait(&red_empty[slot], round ^ 1);
            if (gq < BMAX) {
              float* rp = red + (slot * 16 + cw) * NV;
              rp[(2 * tq) * BMAX + gq] = dacc[0];
              rp[(2 * tq + 1) * BMAX + gq] = dacc[1];
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&red_full[slot]);
            continue;
          }
          float acc[NV];
#pragma unroll
          for (int i = 0; i < NV; ++i) acc[i] = 0.f;
          for (int s = 0; s < n_slices; ++s) {
            const int kc = min(KCp, d.K - s * KCp);
            mbar_wait(&full_bar[st], ph);
            for (int c8 = ct * 8; c8 < kc; c8 += M::CONSUMERS * 8) {
              const uint8_t* src = ring + (size_t)st * p.stage_bytes + c8 * 2;
              float xf[BMAX][8];
#pragma unroll
              for (int b = 0; b < BMAX; ++b) {
                const uint4 xv = *reinterpret_cast<const uint4*>(xs + (size_t)b * xs_stride + (size_t)s * KCp + c8);
                xf[b][0] = bf16_lo(xv.x); xf[b][1] = bf16_hi(xv.x); xf[b][2] = bf16_lo(xv.y); xf[b][3] = bf16_hi(xv.y);
                xf[b][4] = bf16_lo(xv.z); xf[b][5] = bf16_hi(xv.z); xf[b][6] = bf16_lo(xv.w); xf[b][7] = bf16_hi(xv.w);
              }
#pragma unroll
              for (int r = 0; r < ROWS; ++r) {
                if (r < rows) {
                  const uint4 wv = *reinterpret_cast<const uint4*>(src + r * row_stride);
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
            if (++st == p.n_stages) { st = 0; ph ^= 1; }
          }
          warp_reduce_scatter<NV>(acc, lane);
          mbar_wait(&red_empty[slot], round ^ 1);           // the finalize warp has drained this slot (4 units ago)
          if ((lane & (32 / NV - 1)) == 0) red[(slot * 16 + cw) * NV + lane / (32 / NV)] = acc[0];
          __syncwarp();
          if (lane == 0) mbar_arrive(&red_full[slot]);
        }
      } else {
        // ===== finalize warp: sum the 16 partials of each unit, fused epilogue =====
        for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++unit_no) {
          const int n0 = g * rows_u;
          const int slot = unit_no & (M::RED_SLOTS - 1);
          const uint32_t round = (unit_no / M::RED_SLOTS) & 1;
          const int r = lane / BMAX, b = lane % BMAX, n = n0 + r;
          const bool ok = lane < NV && r < rows_u && b < p.B && n < d.N;
          // operands of the epilogue are fetched while the compute warps are still busy with this unit
          float pre0 = 0.f, pre1 = 0.f;
          mega_epilogue_prefetch(p, d, ok, b, n, pos, pre0, pre1);
          mbar_wait(&red_full[slot], round);
          float t = 0.f;
          if (lane < NV) {
#pragma unroll
            for (int w = 0; w < 16; ++w) t += red[(slot * 16 + w) * NV + lane];
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&red_empty[slot]);
          if (lane < NV)
            mega_unit_epilogue<BMAX, NV>(p, d, lane, t, ok, r, b, n, pre0, pre1, pos, rstd_s, bestv, besti, samp_on, samp_it, samp_k0, samp_k1);
        }
      }
      t_loop += clock64() - t0;
      if (dbg_o != nullptr) dbg_o[8 + 3 * d.type + 1] += clock64() - t0;
    }
    t0 = clock64();
    if (pi == p.n_phases - 1 && is_fin && lane < p.B) {
      p.part_val[(size_t)lane * gridDim.x + blockIdx.x] = bestv[lane];
      p.part_idx[(size_t)lane * gridDim.x + blockIdx.x] = besti[lane];
    }
    grid_sync_consumers(p.grid_counter, sync_base + (++sync_no) * gridDim.x, ct);
    t_sync += clock64() - t0;
    if (dbg_o != nullptr) dbg_o[8 + 3 * d.type + 2] += clock64() - t0;
  }
  if (dbg_o != nullptr) {
    dbg_o[0] = t_sync; dbg_o[1] = t_stage; dbg_o[2] = t_loop; dbg_o[3] = t_attn; dbg_o[4] = 0;
  }

  if (blockIdx.x == 0 && !is_fin) mega_finish_step(p, cw, lane, ct);
}

}  // namespace vly
