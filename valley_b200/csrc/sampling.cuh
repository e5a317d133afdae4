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
#include "common.cuh"

namespace vly {

constexpr int kMaxSampleRows = 64;
constexpr int kMaxStopStrings = 8;       // stop strings matched on the device per request
constexpr int kMaxStopChars = 64;        // characters per device stop string: the width of the uint64 masks
constexpr int kStopRing = 64;            // tokens of history kept per row: a match spans at most kMaxStopChars tokens

struct SampleState {          // lives in device memory next to the KV cache; read by every decode step
  // the request, written by the host (set_sampling); the defaults are plain greedy with no stop token
  float temperature = 1.f;    // filtered scores are logits / temperature, an IEEE fp32 division as in HF's TemperatureLogitsWarper
  float inv_temp = 1.f;       // 1 / temperature: the draw, sample_score(logit, inv_temp, ...)
  int enabled = 0;            // 0 = greedy (scores are the raw logits: bit-identical to the plain arg-max)
  int filter = 0;             // the request has a top-k / top-p filter (applied only by a launch that passes filter = 1)
  int top_k = 0;              // top-k filter: <= 0 off; >= V keeps every token
  float top_p = 1.f;          // top-p filter: off unless 0 < top_p < 1
  uint32_t seed_lo = 0, seed_hi = 0;
  long long eos = -1, pad = 0;  // eos < 0: no stop token
  long long stop2 = -1;       // second stop id (the worker's single-token stop string, model_worker.py:355-360); < 0: none
  // stop strings (HF's StopStringCriteria over the tables of valley_b200/stop_strings.py); n_stop == 0: none.  A row whose
  // text ends with one, or that emits a token of the pause set, is finished; it emits pad afterwards only when eos / stop2
  // is set (HF pads only with an eos criterion).
  int n_stop = 0;
  int stop_walk = 0;          // tokens a match may span, the newest included: the longest stop string (HF's maximum_token_len)
  int stop_len[kMaxStopStrings] = {};
  const ulonglong2* stop_masks = nullptr;  // [n_stop][V]: x bit L-1: the token can end the string with its last L characters
                                           //             y bit p: the token fits with its end p characters before the string's end
  const uint8_t* tok_len = nullptr;        // [V] clean-string length of each token, capped at 255
  const uint32_t* pause = nullptr;         // [ceil(V / 32)] bits, or null: emitting one of these tokens finishes the row
  int* ring = nullptr;                     // [kMaxSampleRows][kStopRing]: each row's latest tokens, the next at ring_n % kStopRing
  int ring_n[kMaxSampleRows] = {};
  // recording (vly_sampling::scores_out / logits_out): caller buffers [slots][B][V] fp32, or null.  sample_filter_kernel writes
  // slot *step - 1 (slot 0 for the first token, launched without a step counter): the score it selects from, logits / rec_temp
  // or -inf where the filter removed the token, and the raw logit.
  float* rec_scores = nullptr;
  float* rec_logits = nullptr;
  float rec_temp = 1.f;
  // logits processors (HF's RepetitionPenalty / NoRepeatNGram / MinLength, in that order, before the temperature and the
  // filters): procs == 0: none.  hist [B][hist_stride] int32 is each row's input_ids as HF holds them -- the prompt, seeded
  // by set_sampling, then every token sample_filter_kernel emits (pad in a finished row), written at pos + 1.
  int procs = 0;
  float penalty = 1.f;        // 1: off
  int ngram = 0;              // 0: off
  int min_length = 0;         // eos is banned while the row is shorter; 0: off
  int* hist = nullptr;
  int hist_stride = 0;
  // the generation's progress
  int all_done = 0;           // every row has produced eos: further steps exit at once
  int steps_valid = 0;        // decode steps executed before all_done was raised (the one that raised it included)
  unsigned int arrive = 0;    // CTAs of the running sample_filter_kernel that have finished their row; 0 between launches
  int done[kMaxSampleRows] = {};
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

// once every row of the step has passed sample_finish_row: count the step (count_step) and raise all_done when every row stopped
__device__ __forceinline__ void sample_close_step(SampleState* s, int B, bool count_step) {
  if (count_step) s->steps_valid += 1;
  if (s->eos >= 0 || s->stop2 >= 0 || s->n_stop > 0) {
    const volatile int* done = s->done;             // (written by other CTAs in sample_filter_kernel)
    int all = 1;
    for (int b = 0; b < B; ++b) all &= done[b];
    s->all_done = all;
  }
}

// ---- stop strings: HF's StopStringCriteria for one row, over bit masks ----
// The row's text is the concatenation of its tokens' clean strings (valley_b200/stop_strings.py).  With t_0 the newest token
// and t_1, t_2, ... the ones before it, the row matches stop string i when, for some L with bit L-1 of end(i, t_0) set, the
// walk pos = L; for j = 1, 2, ...: require bit pos of posm(i, t_j), pos += len(t_j), reaches len(i) within stop_walk tokens.
// One warp: lane l follows the walks of L = l + 1 and l + 33.  ring: the row's latest kStopRing tokens, t_j at
// (n - 1 - j) % kStopRing, n = tokens pushed (t_0 included).  A token id outside [0, V) fits nowhere (HF clamps it to an
// all-empty row).  Returns the same value in every lane.
__device__ bool stop_match_warp(const SampleState& s, int V, const int* ring, int n, long long tok, int lane) {
  __shared__ unsigned long long pm[kStopRing];
  __shared__ int tl[kStopRing];
  const int walk = min(n, s.stop_walk);
  bool loaded = false, hit = false;
  for (int i = 0; i < s.n_stop && !hit; ++i) {
    const ulonglong2* m = s.stop_masks + (size_t)i * V;
    const unsigned long long end = (unsigned long long)tok < (unsigned long long)V ? m[tok].x : 0ull;
    if (end == 0ull) continue;                     // (warp-uniform)
    __syncwarp();
    for (int j = 1 + lane; j < walk; j += 32) {
      const int t = ring[(n - 1 - j) & (kStopRing - 1)];
      const bool in = (unsigned)t < (unsigned)V;
      pm[j] = in ? m[t].y : 0ull;
      if (!loaded) tl[j] = in ? s.tok_len[t] : 0;
    }
    loaded = true;
    __syncwarp();
    const int len = s.stop_len[i];
    bool mine = false;
    for (int L = lane + 1; L <= kMaxStopChars; L += 32) {
      if (!((end >> (L - 1)) & 1ull)) continue;
      int pos = L;
      for (int j = 1; pos < len && j < walk; ++j) {
        if (!((pm[j] >> pos) & 1ull)) break;
        pos += tl[j];
      }
      mine |= pos >= len;
    }
    hit = __any_sync(0xffffffffu, mine);
  }
  return hit;
}

// vly_test_stop_strings: one warp per row of tokens [B, n], read as a row whose newest token is the last: out[b] = match
__global__ void stop_match_test_kernel(const SampleState s, int V, const long long* tokens, int n, int* ring, uint8_t* out) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const long long* row = tokens + (size_t)b * n;
  int* r = ring + (size_t)b * kStopRing;
  for (int j = max(0, n - kStopRing) + lane; j < n; j += 32) r[j & (kStopRing - 1)] = (int)row[j];
  __syncwarp();
  const bool hit = stop_match_warp(s, V, r, n, row[n - 1], lane);
  if (lane == 0) out[b] = hit;
}

// ---- logits processors: HF's RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor ----
// For one row with input_ids ids[0..L) (cur_len = L) and raw scores z:
//   penalty: every id in ids (once, however often it occurs) scores z * penalty if z < 0, else z / penalty (IEEE fp32);
//   ngram n: for every start j <= L - n whose ids[j .. j+n-2] equal the row's last n - 1 ids, ids[j+n-1] scores -inf
//            (nothing when L + 1 < n: no start exists; n = 1 bans every id of the row);
//   min_length: eos scores -inf while L < min_length.
// -inf wins over the penalty in any order, so proc_score applies all three at once.  The CTA first marks the ids in two
// bitmaps in shared memory, `seen` (penalty) and `banned` (n-gram), with integer atomics: the maps -- and so the scores -- are
// a deterministic function of the row.  Ids outside [0, V) mark nothing.
struct ProcMaps {
  uint32_t* seen;
  uint32_t* banned;
  float penalty;
  long long eos_ban;          // the eos id while it is banned, else -1
};

template <typename Id>
__device__ void proc_build_maps(const Id* ids, int L, int V, float penalty, int ngram, int min_length, long long eos,
                                ProcMaps& m, int tid, int nthreads) {
  const int words = (V + 31) >> 5;
  for (int w = tid; w < words; w += nthreads) { m.seen[w] = 0u; m.banned[w] = 0u; }
  __syncthreads();
  if (penalty != 1.f)
    for (int j = tid; j < L; j += nthreads) {
      const long long t = (long long)ids[j];
      if (t >= 0 && t < V) atomicOr(&m.seen[t >> 5], 1u << (t & 31));
    }
  if (ngram > 0) {
    const Id* tail = ids + (L - ngram + 1);         // the row's last n - 1 ids
    for (int j = tid; j + ngram <= L; j += nthreads) {
      bool match = true;
      for (int k = 0; k < ngram - 1 && match; ++k) match = ids[j + k] == tail[k];
      const long long t = (long long)ids[j + ngram - 1];
      if (match && t >= 0 && t < V) atomicOr(&m.banned[t >> 5], 1u << (t & 31));
    }
  }
  __syncthreads();
  m.penalty = penalty;
  m.eos_ban = eos >= 0 && L < min_length ? eos : -1;
}

__device__ __forceinline__ float proc_score(const ProcMaps& m, int n, float z) {
  const uint32_t bit = 1u << (n & 31);
  if ((m.banned[n >> 5] & bit) || n == m.eos_ban) return -INFINITY;
  if (m.seen[n >> 5] & bit) return z < 0.f ? z * m.penalty : z / m.penalty;
  return z;
}

// vly_test_logits_process: one CTA per row of logits [B, V] with input_ids [B, L]: out = the processed scores
__global__ void __launch_bounds__(1024) logits_process_test_kernel(const float* logits, int V, const long long* ids, int L,
                                                                   float penalty, int ngram, int min_length, long long eos,
                                                                   float* out) {
  extern __shared__ uint32_t maps[];                // [2][ceil(V / 32)]
  const int b = blockIdx.x;
  ProcMaps m = {maps, maps + ((V + 31) >> 5), 1.f, -1};
  proc_build_maps(ids + (size_t)b * L, L, V, penalty, ngram, min_length, eos, m, threadIdx.x, blockDim.x);
  for (int n = threadIdx.x; n < V; n += blockDim.x) out[(size_t)b * V + n] = proc_score(m, n, logits[(size_t)b * V + n]);
}

// set_sampling, a request with processors that starts: hist[b][0..S) = prompt ids [B, S]
__global__ void hist_seed_kernel(int* hist, int stride, const long long* ids, int S) {
  const int b = blockIdx.x;
  for (int j = threadIdx.x; j < S; j += blockDim.x) hist[(size_t)b * stride + j] = (int)ids[(size_t)b * S + j];
}

// ---- stand-alone token selection: optional top-k / top-p (nucleus) filtering, then the Gumbel-max draw ----
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
// One CTA per row.  With a filter, the row's scores are staged in shared memory (V * 4 bytes of dynamic shared memory) when
// they fit; otherwise every pass recomputes them from the logits in global memory.  Without one (filter = 0) the kernel draws
// straight from the logits (the raw logit when greedy) and is launched without dynamic shared memory.  A launch with
// filter = 1 filters only when the request has a filter (SampleState::filter), so stop-string requests share its graphs.
// With stop strings, warp 0 then pushes the row's token into its ring and runs stop_match_warp (sample_filter_kernel is the
// step's selection whenever a request has stop strings).
// With logits processors (SampleState::procs; launched with filter = 1), the CTA first builds the row's ProcMaps from
// hist[b][0..pos], and every use of z_n as a score -- the staged scores, the draw, the recorded score -- becomes
// proc_score(z_n); the recorded logit stays z_n.  The emitted token is written to hist[b][pos + 1].
// Dynamic shared memory of a filter = 1 launch: the staged scores (when they fit), then the two maps.
constexpr int kFilterThreads = 1024;
constexpr int kFilterStageMaxBytes = 200 * 1024;     // rows of up to 51200 scores are staged
__host__ __device__ constexpr size_t filter_stage_bytes(int V) {
  return (size_t)V * 4 <= (size_t)kFilterStageMaxBytes ? (size_t)V * 4 : 0;
}
__host__ __device__ constexpr size_t proc_map_bytes(int V) { return (size_t)2 * ((V + 31) / 32) * 4; }

__device__ __forceinline__ uint32_t score_key(float s) {   // unsigned order of the keys == order of the (finite) scores
  uint32_t u = __float_as_uint(s);
  if (u == 0x80000000u) u = 0u;                            // -0 == +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_score(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Selects the first token after a prefill (set_sampling has cleared the flags), and the token after a decode step that wrote
// `logits` and a provisional arg-max: it then overwrites next_tokens and out_tokens[:, *step - 1].  It keeps done / all_done.
//   per_op: after the per-op decode kernels, which step on once all_done is raised and do not count steps: a plain greedy
//     request keeps the step's own arg-max, every row emits pad once all_done is raised, and the step is counted in
//     steps_valid.  After the persistent kernel (which counts its own steps and skips once all_done is raised) and for the
//     first token, none of these.
// keep_out != nullptr (vly_test_sample_filter): writes the kept mask [B, V] and nothing else.
// A recording request (SampleState::rec_scores / rec_logits) writes its slot in the final pass over the row, where `keep` is
// decided: the recorded -inf are exactly the tokens the draw excludes.  Nothing is recorded once all_done is raised.
__global__ void __launch_bounds__(kFilterThreads) sample_filter_kernel(const float* __restrict__ logits, int V, SampleState* s,
                                                                       const int* seq_len, const int* step, long long* next_tokens,
                                                                       long long* out_tokens, int out_stride, int filter,
                                                                       int per_op, uint8_t* keep_out) {
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
  if (select && per_op && !s->enabled && s->eos < 0 && s->stop2 < 0 && s->n_stop == 0 && !s->rec_scores && !s->rec_logits &&
      !s->procs)
    return;                                         // plain greedy: the step's arg-max is the token
  if (select && s->all_done) {
    if (per_op && tid == 0) {                       // the per-op kernels keep stepping: emit pad
      next_tokens[b] = s->pad;
      if (out_tokens) out_tokens[(size_t)b * out_stride + (*step - 1)] = s->pad;
    }
    return;                                         // (the persistent kernel skipped the step: nothing to select)
  }
  const float temperature = s->temperature, top_p = s->top_p;
  const int top_k = s->top_k;
  const float* z = logits + (size_t)b * V;
  const int pos = select ? *seq_len - 1 : 0;
  const bool procs = select && filter && s->procs;
  ProcMaps pm = {reinterpret_cast<uint32_t*>(srow + (filter ? filter_stage_bytes(V) / 4 : 0)), nullptr, 1.f, -1};
  pm.banned = pm.seen + (V + 31) / 32;
  if (procs)
    proc_build_maps(s->hist + (size_t)b * s->hist_stride, pos + 1, V, s->penalty, s->ngram, s->min_length, s->eos, pm, tid,
                    kFilterThreads);
  auto zp = [&](int n) { return procs ? proc_score(pm, n, z[n]) : z[n]; };   // the processed score of token n
  filter = filter && (s->filter || !select);
  const bool staged = filter && filter_stage_bytes(V) > 0;
  auto score = [&](int n) { return staged ? srow[n] : zp(n) / temperature; };

  uint32_t kmax = 0;
  if (filter) {
    for (int n = tid; n < V; n += kFilterThreads) {
      const float sc = zp(n) / temperature;
      if (staged) srow[n] = sc;
      kmax = max(kmax, score_key(sc));
    }
    kmax = __reduce_max_sync(0xffffffffu, kmax);
    if (lane == 0) max_w[warp] = kmax;
    __syncthreads();
#pragma unroll 1
    for (int w = 0; w < 32; ++w) kmax = max(kmax, max_w[w]);
  }

  uint32_t cut = 0;                                 // keep n iff score_key(s_n) >= cut
  if (filter && top_k > 0 && top_k < V) {
    uint32_t prefix = 0, pmask = 0;
    int krem = top_k;                               // rank, from the top, of the wanted key among the keys under the prefix
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

  if (filter && top_p > 0.f && top_p < 1.f) {
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
            target = top_p * W;
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

  const bool on = s->enabled != 0;
  const float inv_temp = s->inv_temp;
  const uint32_t k0 = s->seed_lo, k1 = s->seed_hi;
  float* rec_s = nullptr;
  float* rec_l = nullptr;
  const float rec_temp = s->rec_temp;
  if (select && (s->rec_scores || s->rec_logits)) {
    const size_t row = ((size_t)(step ? *step - 1 : 0) * gridDim.x + b) * V;
    if (s->rec_scores) rec_s = s->rec_scores + row;
    if (s->rec_logits) rec_l = s->rec_logits + row;
  }
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int n = tid; n < V; n += kFilterThreads) {
    const bool keep = !filter || score_key(score(n)) >= cut;
    if (!select) {
      keep_out[(size_t)b * V + n] = keep;
      continue;
    }
    const float zn = zp(n);
    if (rec_s) rec_s[n] = keep ? zn / rec_temp : -INFINITY;
    if (rec_l) rec_l[n] = z[n];
    if (keep) {
      const float v = on ? sample_score(zn, inv_temp, k0, k1, n, b, pos) : zn;
      if (v > bv) { bv = v; bi = n; }               // ascending n per thread: first maximum kept
    }
  }
  if (!select) return;
  warp_argmax(bv, bi);
  if (lane == 0) { bv_w[warp] = bv; bi_w[warp] = bi; }
  __syncthreads();
  if (warp != 0) return;
  bv = bv_w[lane];
  bi = bi_w[lane];
  warp_argmax(bv, bi);
  if (procs && bi == 0x7fffffff) bi = 0;            // the processors left every score -inf: torch's argmax takes 0
  long long tok = bi;
  if (s->n_stop > 0) {
    const int was_done = s->done[b];
    __syncwarp();
    if (lane == 0) tok = sample_finish_row(s, b, bi);
    tok = __shfl_sync(0xffffffffu, tok, 0);
    if (!was_done) {
      int* ring = s->ring + (size_t)b * kStopRing;
      const int n = s->ring_n[b] + 1;
      __syncwarp();
      if (lane == 0) { ring[(n - 1) & (kStopRing - 1)] = (int)tok; s->ring_n[b] = n; }
      bool hit = s->pause != nullptr && (unsigned long long)tok < (unsigned long long)V && ((s->pause[tok >> 5] >> (tok & 31)) & 1u);
      if (!hit) hit = stop_match_warp(*s, V, ring, n, tok, lane);
      if (hit && lane == 0) s->done[b] = 1;
    }
    if (lane != 0) return;
  } else {
    if (lane != 0) return;
    tok = sample_finish_row(s, b, bi);
  }
  if (procs && pos + 1 < s->hist_stride) s->hist[(size_t)b * s->hist_stride + pos + 1] = (int)tok;
  next_tokens[b] = tok;
  if (out_tokens) out_tokens[(size_t)b * out_stride + (*step - 1)] = tok;
  __threadfence();
  if (atomicAdd(&s->arrive, 1u) == gridDim.x - 1) {   // the last row to finish: every done flag is visible
    __threadfence();
    s->arrive = 0;
    sample_close_step(s, gridDim.x, per_op);
  }
}

}  // namespace vly
