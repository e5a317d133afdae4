// On-device token selection for the decode loop (SURVEY 8 f-1).
//
// Reference semantics (valley/serve/model_worker.py:388-397, and HF generate as called at valley_model.py:432):
//   temperature < 1e-4 : token = argmax(last_token_logits)                         (:390-391)
//   otherwise          : probs = softmax(last_token_logits / temperature); token = multinomial(probs, 1)   (:392-395)
//   token == eos       : the sequence stops (:396-397); HF pads finished rows of a batch with pad_token_id and stops
//                        when every row has finished.
//
// multinomial(softmax(z)) is drawn with the Gumbel-max identity: argmax_n(z_n + G_n), G_n i.i.d. standard Gumbel, has exactly
// that distribution -- so sampling is the SAME fused arg-max epilogue the greedy path already runs, with a counter-based noise
// term and no softmax pass, no prefix sum and no host round trip.  The noise is Philox4x32-10 keyed by the request seed with the
// counter (vocabulary index, batch row, position of the query token): every path (the persistent decode kernel's epilogue, the
// stand-alone kernel below) computes bit-identical scores for the same logits, which is what the tests check, next to a
// goodness-of-fit test of the drawn distribution against softmax(logits / T).  (The stream differs from torch's Philox offsets,
// so ids are not comparable draw-by-draw with torch.multinomial -- no sampler on different hardware is.)
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace vly {

constexpr int kMaxSampleRows = 64;

// A request with a top-k / top-p filter (HF's TopKLogitsWarper / TopPLogitsWarper).  Such a request is selected by
// sample_filter_kernel after the decode step, not in the step's arg-max epilogue: the step then sees the plain-greedy state
// (enabled 0, no stop ids), and this block holds the request.  Written by the host (set_sampling).
struct SampleFilter {
  float temperature;          // s = logits / temperature, an IEEE fp32 division as in HF's TemperatureLogitsWarper
  float inv_temp;             // the draw: sample_score(logit, inv_temp, ...), the same Gumbel-max as the unfiltered sampler
  int top_k;                  // <= 0: off; >= V keeps every token
  float top_p;                // off unless 0 < top_p < 1
  uint32_t seed_lo, seed_hi;
  long long eos, pad, stop2;  // < 0: none (as in SampleState)
};

struct SampleState {          // lives in device memory next to the KV cache; read by every decode step
  float inv_temp;             // 1 / temperature
  int enabled;                // 0 = greedy (scores are the raw logits: bit-identical to the plain arg-max)
  uint32_t seed_lo, seed_hi;
  long long eos, pad;         // eos < 0: no stop token
  long long stop2;            // second stop id (the worker's single-token stop string, model_worker.py:355-360); < 0: none
  int all_done;               // every row has produced eos: further steps exit at once
  int steps_valid;            // decode steps executed before all_done was raised (the one that raised it included)
  int done[kMaxSampleRows];
  // (appended: the fields above keep their offsets, so the decode kernels that read them are unchanged)
  SampleFilter filt;          // the filtered request (sample_filter_kernel)
  unsigned int filt_arrive;   // CTAs of the running sample_filter_kernel that have finished their row; 0 between launches
};

__device__ __forceinline__ uint32_t philox4x32_10_first(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// score whose arg-max over n is the selected token
__device__ __forceinline__ float sample_score(float logit, float inv_temp, uint32_t seed_lo, uint32_t seed_hi, int n, int b, int pos) {
  const uint32_t x = philox4x32_10_first((uint32_t)n, (uint32_t)b, (uint32_t)pos, 0x56414c59u, seed_lo, seed_hi);
  const float u = ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f);      // (0, 1), 24 bits
  return fmaf(logit, inv_temp, -logf(-logf(u)));
}

// eos / pad bookkeeping for one row's freshly selected token; returns the token to emit
__device__ __forceinline__ long long sample_finish_row(SampleState* s, int b, long long tok) {
  if (s->eos < 0 && s->stop2 < 0) return tok;
  if (s->done[b]) return s->pad;
  if (tok == s->eos || tok == s->stop2) s->done[b] = 1;     // (ids are >= 0, an unset -1 never matches)
  return tok;
}

// Stand-alone selection over a [B, V] fp32 logits block: the first token after a prefill (reset = 1), and the post-step
// selection of the per-op decode paths (B > 4).  One CTA; rows are handled one after the other.
//   pos = *seq_len - 1 : position of the query token that produced these logits
__global__ void __launch_bounds__(1024) sample_rows_kernel(const float* __restrict__ logits, int B, int V, SampleState* s,
                                                           const int* seq_len, const int* step, long long* next_tokens,
                                                           long long* out_tokens, int out_stride, int reset) {
  __shared__ float sv[32];
  __shared__ int si[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (reset) {
    if (tid < kMaxSampleRows) s->done[tid] = 0;
    if (tid == 0) { s->all_done = 0; s->steps_valid = 0; }
    __syncthreads();
  } else {
    if (!s->enabled && s->eos < 0 && s->stop2 < 0) return;   // plain greedy: the arg-max epilogue already wrote the token
    if (s->all_done) {                              // every row finished earlier: keep emitting pad
      if (tid < B) {
        next_tokens[tid] = s->pad;
        if (out_tokens) out_tokens[(size_t)tid * out_stride + (*step - 1)] = s->pad;
      }
      return;
    }
  }
  const int pos = *seq_len - 1;
  const bool on = s->enabled != 0;
  const float it = s->inv_temp;
  const uint32_t k0 = s->seed_lo, k1 = s->seed_hi;
  for (int b = 0; b < B; ++b) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int n = tid; n < V; n += 1024) {
      const float y = logits[(size_t)b * V + n];
      const float v = on ? sample_score(y, it, k0, k1, n, b, pos) : y;
      if (v > bv) { bv = v; bi = n; }               // ascending n per thread: first maximum kept
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      bv = sv[lane];
      bi = si[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) {
        const long long tok = sample_finish_row(s, b, bi);
        next_tokens[b] = tok;
        if (out_tokens) out_tokens[(size_t)b * out_stride + (*step - 1)] = tok;
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    if (!reset) s->steps_valid += 1;
    if (s->eos >= 0 || s->stop2 >= 0) {
      int all = 1;
      for (int b = 0; b < B; ++b) all &= s->done[b];
      s->all_done = all;
    }
  }
}

// ---- top-k / top-p (nucleus) filtering, then the Gumbel-max draw over the kept tokens ----
// For one row, with z the fp32 logits and T the temperature:
//   s_n = z_n / T.
//   top_k: keep n iff s_n >= the k-th largest s, duplicates counted (HF removes scores < topk(scores, k)[-1]; ties are kept).
//   top_p: among the tokens top_k kept, with w_n = exp(s_n - s_max) and W = sum w, keep the tokens of score v iff the mass
//          strictly above v is < top_p * W.  This is HF's "ascending cumsum <= 1 - top_p is removed" written from the top: it
//          is stable for a small top_p and always keeps the maximum.  A tie group that straddles the cut is kept whole.
//   draw:  arg-max over the kept tokens of sample_score(z_n, 1/T, seed, n, b, pos), lowest index on ties.  A filter that keeps
//          everything therefore draws the token the unfiltered sampler draws.
// Both thresholds come from a radix select over order-preserving uint32 keys of s, 4 bits per level from the top: first the
// exact k-th key by counts, then the top-p cut by w-mass among the kept keys.  Each thread accumulates 16 private bins over a
// fixed strided subset of the row, and the bins are reduced in a fixed order; there are no floating-point atomics.  So the kept
// set and the token are a deterministic function of (logits, T, top_k, top_p, seed, row, position).
// One CTA per row.  The row's scores are staged in shared memory (V * 4 bytes of dynamic shared memory) when they fit;
// otherwise every pass recomputes them from the logits in global memory.
constexpr int kFilterThreads = 1024;
constexpr int kFilterStageMaxBytes = 200 * 1024;     // rows of up to 51200 scores are staged
enum { FILTER_FIRST = 0, FILTER_AFTER_MEGA = 1, FILTER_AFTER_PEROP = 2 };

__device__ __forceinline__ uint32_t score_key(float s) {   // unsigned order of the keys == order of the (finite) scores
  uint32_t u = __float_as_uint(s);
  if (u == 0x80000000u) u = 0u;                            // -0 == +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// mode FILTER_FIRST: the first token after a prefill (set_sampling has cleared the flags).
// FILTER_AFTER_MEGA / FILTER_AFTER_PEROP: after a decode step that wrote `logits` and a provisional arg-max.  Overwrites
//   next_tokens and out_tokens[:, *step - 1] and keeps done / all_done.  After the per-op kernels it also counts the step in
//   steps_valid; the persistent kernel counts its own steps.
// keep_out != nullptr (vly_test_sample_filter): writes the kept mask [B, V] and nothing else.
__global__ void __launch_bounds__(kFilterThreads) sample_filter_kernel(const float* __restrict__ logits, int V, SampleState* s,
                                                                       const int* seq_len, const int* step, long long* next_tokens,
                                                                       long long* out_tokens, int out_stride, int mode,
                                                                       uint8_t* keep_out) {
  extern __shared__ float srow[];                   // [V] scores, when staged
  __shared__ int cnt_w[32][16];
  __shared__ float mass_w[32][16];
  __shared__ int cnt_d[16];
  __shared__ float mass_d[16];
  __shared__ uint32_t max_w[32];
  __shared__ float bv_w[32];
  __shared__ int bi_w[32];
  __shared__ uint32_t sh_prefix;
  __shared__ int sh_krem, sh_stop;
  __shared__ float sh_above;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.x;
  const bool select = keep_out == nullptr;
  if (select && mode != FILTER_FIRST && s->all_done) {
    if (mode == FILTER_AFTER_PEROP && tid == 0) {   // the per-op kernels keep stepping: emit pad, as sample_rows_kernel does
      next_tokens[b] = s->filt.pad;
      if (out_tokens) out_tokens[(size_t)b * out_stride + (*step - 1)] = s->filt.pad;
    }
    return;                                         // (the persistent kernel skipped the step: nothing to select)
  }
  const SampleFilter f = s->filt;
  const float* z = logits + (size_t)b * V;
  const bool staged = (size_t)V * 4 <= (size_t)kFilterStageMaxBytes;
  auto score = [&](int n) { return staged ? srow[n] : z[n] / f.temperature; };

  uint32_t kmax = 0;
  for (int n = tid; n < V; n += kFilterThreads) {
    const float sc = z[n] / f.temperature;
    if (staged) srow[n] = sc;
    kmax = max(kmax, score_key(sc));
  }
  kmax = __reduce_max_sync(0xffffffffu, kmax);
  if (lane == 0) max_w[warp] = kmax;
  __syncthreads();
#pragma unroll 1
  for (int w = 0; w < 32; ++w) kmax = max(kmax, max_w[w]);

  uint32_t cut = 0;                                 // keep n iff score_key(s_n) >= cut
  if (f.top_k > 0 && f.top_k < V) {
    uint32_t prefix = 0, pmask = 0;
    int krem = f.top_k;                             // rank, from the top, of the wanted key among the keys under the prefix
#pragma unroll 1
    for (int shift = 28; shift >= 0; shift -= 4) {
      int c[16];
#pragma unroll
      for (int d = 0; d < 16; ++d) c[d] = 0;
      for (int n = tid; n < V; n += kFilterThreads) {
        const uint32_t k = score_key(score(n));
        if ((k & pmask) == prefix) {
          const int dg = (k >> shift) & 15;
#pragma unroll
          for (int d = 0; d < 16; ++d) c[d] += dg == d;
        }
      }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        const int t = __reduce_add_sync(0xffffffffu, c[d]);
        if (lane == 0) cnt_w[warp][d] = t;
      }
      __syncthreads();
      if (warp == 0) {
        if (lane < 16) {
          int t = 0;
          for (int w = 0; w < 32; ++w) t += cnt_w[w][lane];
          cnt_d[lane] = t;
        }
        __syncwarp();
        if (lane == 0) {
          int above = 0, d = 15;
          for (; d > 0; --d) {
            if (above + cnt_d[d] >= krem) break;
            above += cnt_d[d];
          }
          sh_krem = krem - above;
          sh_prefix = prefix | ((uint32_t)d << shift);
        }
      }
      __syncthreads();
      krem = sh_krem;
      prefix = sh_prefix;
      pmask |= 15u << shift;
    }
    cut = prefix;                                   // the k-th largest key
  }

  if (f.top_p > 0.f && f.top_p < 1.f) {
    const float smax = key_score(kmax);
    uint32_t prefix = 0, pmask = 0;
    float above = 0.f, target = 0.f;                // mass above the prefix's range; top_p * W (thread 0)
#pragma unroll 1
    for (int shift = 28; shift >= 0; shift -= 4) {
      float m[16];
#pragma unroll
      for (int d = 0; d < 16; ++d) m[d] = 0.f;
      for (int n = tid; n < V; n += kFilterThreads) {
        const float sc = score(n);
        const uint32_t k = score_key(sc);
        if (k >= cut && (k & pmask) == prefix) {
          const float w = expf(sc - smax);
          const int dg = (k >> shift) & 15;
#pragma unroll
          for (int d = 0; d < 16; ++d) m[d] += dg == d ? w : 0.f;
        }
      }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        float t = m[d];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
        if (lane == 0) mass_w[warp][d] = t;
      }
      __syncthreads();
      if (warp == 0) {
        if (lane < 16) {
          float t = 0.f;
          for (int w = 0; w < 32; ++w) t += mass_w[w][lane];
          mass_d[lane] = t;
        }
        __syncwarp();
        if (lane == 0) {
          if (shift == 28) {                        // every kept token is under the empty prefix: W
            float W = 0.f;
            for (int d = 15; d >= 0; --d) W += mass_d[d];
            target = f.top_p * W;
          }
          // the digit whose range holds the largest key v with (mass of the keys >= v) >= target: v is the last kept group
          float run = above;
          int d = 15;
          for (; d >= 0; --d) {
            if (run + mass_d[d] >= target) break;
            run += mass_d[d];
          }
          sh_stop = d < 0;                          // fp32 bin sums fell short of the target: keep the whole remaining range
          if (d >= 0) {
            sh_above = run;
            sh_prefix = prefix | ((uint32_t)d << shift);
          }
        }
      }
      __syncthreads();
      if (sh_stop) break;
      above = sh_above;
      prefix = sh_prefix;
      pmask |= 15u << shift;
    }
    cut = max(cut, prefix);
  }

  const int pos = select ? *seq_len - 1 : 0;
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int n = tid; n < V; n += kFilterThreads) {
    const bool keep = score_key(score(n)) >= cut;
    if (!select) {
      keep_out[(size_t)b * V + n] = keep;
    } else if (keep) {
      const float v = sample_score(z[n], f.inv_temp, f.seed_lo, f.seed_hi, n, b, pos);
      if (v > bv) { bv = v; bi = n; }               // ascending n per thread: first maximum kept
    }
  }
  if (!select) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane == 0) { bv_w[warp] = bv; bi_w[warp] = bi; }
  __syncthreads();
  if (warp != 0) return;
  bv = bv_w[lane];
  bi = bi_w[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  if (lane != 0) return;
  const bool stops = f.eos >= 0 || f.stop2 >= 0;
  long long tok = bi;
  if (stops) {                                      // sample_finish_row with the request's ids
    if (s->done[b]) tok = f.pad;
    else if (tok == f.eos || tok == f.stop2) s->done[b] = 1;
  }
  next_tokens[b] = tok;
  if (mode != FILTER_FIRST && out_tokens) out_tokens[(size_t)b * out_stride + (*step - 1)] = tok;
  __threadfence();
  if (atomicAdd(&s->filt_arrive, 1u) == gridDim.x - 1) {   // the last row to finish: every done flag is visible
    __threadfence();
    s->filt_arrive = 0;
    if (mode == FILTER_AFTER_PEROP) s->steps_valid += 1;
    if (stops) {
      const volatile int* done = s->done;
      int all = 1;
      for (int r = 0; r < (int)gridDim.x; ++r) all &= done[r];
      s->all_done = all;
    }
  }
}

}  // namespace vly
