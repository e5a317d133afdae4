// Beam search on the device: the selection step and the KV-cache reorder of HF generate's beam search (num_beams > 1, no
// sampling), so that a beam request keeps the decode loop's no-host-sync-per-token property.
//
// Semantics: transformers 5.5 GenerationMixin._beam_search, non-sampling branch, one step per decode step.  With nb beams,
// K = 2 * nb candidates (HF's beams_to_keep = max(2, 1 + n_eos) * nb with at most one eos id), t the tokens generated so far:
//   1. per beam row: log_softmax(logits) + running_beam_scores (initially 0 for beam 0, -1e9 for the others);
//   2. the top K accumulated scores over the flattened nb * V candidates (parent = index / V, token = index % V);
//   3. a candidate hits the stopping criteria if its token is eos, or at the last allowed step (MaxLengthCriteria);
//   4. the next running beams: the top nb candidates after adding -1e9 to those that hit;
//   5. the finished hypotheses: the old ones merged with those of the top nb candidates that just hit, each scored
//      score / generated_len ** length_penalty, with HF's early_stopping masks (_update_finished_beams); the best nb stay;
//   6. the search ends when _beam_search_has_unfinished_sequences is false (over the whole batch).
// Every "top" is descending with ties broken by the lowest index, which is what the torch restatement (valley_b200/beam.py)
// does with a stable sort.  log_softmax is z - lse with lse = max + log(sum exp(z - max)) summed in float64, so the result is
// the same whatever the summation order: the device and the torch restatement agree bit for bit (it differs from an fp32
// log_softmax by at most an ulp).  No floating-point atomics; every reduction runs in a fixed order.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "common.cuh"
#include "sampling.cuh"

namespace vly {

constexpr int kMaxBeams = 8;                  // K = 2 * nb candidates <= 16
constexpr int kBeamCands = 2 * kMaxBeams;
constexpr int kBeamThreads = 1024;
constexpr float kBeamNeg = -1.0e9f;          // HF's "very large negative value"

struct BeamState {            // device memory, one per KV cache that ran a beam request
  // the request (beam_init_kernel)
  int nb = 0, K = 0, n_steps = 0, prompt_len = 0;
  int early_stopping = 0;     // 0: False, 1: True, 2: "never"
  int lp_positive = 0;        // length_penalty > 0 (the "never" heuristic then assumes the maximum length)
  long long eos = -1;
  // progress
  int step = 0;               // tokens selected so far
  int done = 0;               // the search has ended: later steps exit at once
  unsigned int arrive = 0;    // CTAs of the running beam_step_kernel that have finished their item
  int heur[kMaxSampleRows];   // per item: HF's is_early_stop_heuristic_unsatisfied
  int open[kMaxSampleRows];   // per item: some candidate of the last step did not hit the stopping criteria
  float run_score[kMaxSampleRows];   // per row: running_beam_scores
  float fin_score[kMaxSampleRows];   // per row: beam_scores of the finished hypotheses
  int fin_flag[kMaxSampleRows];      // per row: is_sent_finished
  int fin_len[kMaxSampleRows];       // per row: generated length of the finished hypothesis
  int parent[kMaxSampleRows];        // per row: the cache row the running beam continues (the reorder's source)
  // recording (vly_beam's output pointers, caller buffers, or null): slot `step` of rec_scores / rec_logits [n_steps][rows][V]
  // gets each beam row's log-probabilities / raw logits; with bidx_out the step also keeps the beam-index rows
  float* rec_scores;
  float* rec_logits;
  long long* bidx_out;
  int* steps_out;
};

// Starts a request: rows = items * nb.  lp_div[L - 1] = (float)pow(L, length_penalty), L = 1 .. n_steps (Python's int ** float).
__global__ void beam_init_kernel(BeamState* s, int rows, int nb, int n_steps, int prompt_len, int early_stopping,
                                 float length_penalty, long long eos, float* lp_div, float* rec_scores, float* rec_logits,
                                 long long* bidx_out, int* steps_out) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    s->nb = nb; s->K = 2 * nb; s->n_steps = n_steps; s->prompt_len = prompt_len; s->early_stopping = early_stopping;
    s->lp_positive = length_penalty > 0.f; s->eos = eos; s->step = 0; s->done = 0; s->arrive = 0;
    s->rec_scores = rec_scores; s->rec_logits = rec_logits; s->bidx_out = bidx_out; s->steps_out = steps_out;
  }
  for (int r = tid; r < kMaxSampleRows; r += blockDim.x) {
    s->heur[r] = 1; s->open[r] = 1;
    s->run_score[r] = (r % nb == 0) ? 0.f : kBeamNeg;
    s->fin_score[r] = kBeamNeg; s->fin_flag[r] = 0; s->fin_len[r] = 0; s->parent[r] = r;
  }
  for (int l = tid; l < n_steps; l += blockDim.x) lp_div[l] = (float)pow((double)(l + 1), (double)length_penalty);
}

// (value, index) a beats b: larger value, lower index among equal values
__device__ __forceinline__ bool beam_better(float av, int ai, float bv, int bi) { return av > bv || (av == bv && ai < bi); }

// One beam-search step for item blockIdx.x (rows [g * nb, g * nb + nb)): reads the step's logits [rows, V], selects, writes the
// running and finished token rows of the next step (double-buffered by the parity of the step: buffer p of run_tok / fin_tok is
// [rows][stride]), the next input tokens and the parent rows.  A request that records beam indices keeps a beam-index row
// next to every token row the same way (run_bi / fin_bi, int32: entry p is the cache row the token at p was appended to).  The last CTA to finish decides whether the search goes on and
// raises SampleState::all_done when it ends, so that the remaining decode steps exit at once.
__global__ void __launch_bounds__(kBeamThreads) beam_step_kernel(const float* __restrict__ logits, int V, BeamState* s,
                                                                 long long* run_tok, long long* fin_tok, int* run_bi, int* fin_bi,
                                                                 int stride, const float* __restrict__ lp_div, long long* cur_tokens,
                                                                 SampleState* ss) {
  __shared__ float red_f[32];
  __shared__ double red_d[32];
  __shared__ double lse[kMaxBeams];
  __shared__ float wv[32][kBeamCands];
  __shared__ int wi[32][kBeamCands];
  __shared__ float cand_v[kBeamCands];
  __shared__ int cand_i[kBeamCands];
  __shared__ int run_src[kMaxBeams];          // new running beam j continues local beam run_src[j] ...
  __shared__ long long run_new[kMaxBeams];    // ... with this token
  __shared__ int fin_src[kMaxBeams];          // new finished slot j: candidate k (>= 0) or old finished slot -1 - q
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = blockIdx.x;
  if (s->done) return;                        // (the per-op decode kernels keep stepping after the search ended)
  const int nb = s->nb, K = s->K, t = s->step, r0 = g * nb, rows = gridDim.x * nb;

  // 1. lse of every beam row
  for (int j = 0; j < nb; ++j) {
    const float* z = logits + (size_t)(r0 + j) * V;
    float m = -INFINITY;
    for (int n = tid; n < V; n += kBeamThreads) m = fmaxf(m, z[n]);
    m = warp_max(m);
    if (lane == 0) red_f[warp] = m;
    __syncthreads();
    m = red_f[0];
    for (int w = 1; w < 32; ++w) m = fmaxf(m, red_f[w]);
    double sum = 0.0;
    for (int n = tid; n < V; n += kBeamThreads) sum += (double)expf(z[n] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) red_d[warp] = sum;
    __syncthreads();
    if (tid == 0) {
      double tot = 0.0;
      for (int w = 0; w < 32; ++w) tot += red_d[w];
      lse[j] = (double)m + log(tot);
    }
    __syncthreads();
  }

  // 2. top 16 accumulated scores of this thread's candidates (flat index f = j * V + n), sorted
  float lv[kBeamCands];
  int li[kBeamCands];
#pragma unroll
  for (int q = 0; q < kBeamCands; ++q) { lv[q] = -INFINITY; li[q] = 0x7fffffff; }
  for (int j = 0; j < nb; ++j) {
    const float* z = logits + (size_t)(r0 + j) * V;
    const double l = lse[j];
    const float rs = s->run_score[r0 + j];
    const size_t rec = ((size_t)t * rows + r0 + j) * V;         // the row's slot in the recorded [step][row][V] buffers
    float* rec_s = s->rec_scores ? s->rec_scores + rec : nullptr;
    float* rec_l = s->rec_logits ? s->rec_logits + rec : nullptr;
    for (int n = tid; n < V; n += kBeamThreads) {
      const float lp = (float)((double)z[n] - l);
      if (rec_s) rec_s[n] = lp;
      if (rec_l) rec_l[n] = z[n];
      float v = lp + rs;
      int i = j * V + n;
      if (!beam_better(v, i, lv[kBeamCands - 1], li[kBeamCands - 1])) continue;
#pragma unroll
      for (int q = 0; q < kBeamCands; ++q) {
        if (beam_better(v, i, lv[q], li[q])) {
          const float tv = lv[q]; const int ti = li[q];
          lv[q] = v; li[q] = i; v = tv; i = ti;
        }
      }
    }
  }
  // 3. merge: per warp, then over the warps; kBeamCands rounds of arg-max over the lists' heads
  for (int round = 0; round < kBeamCands; ++round) {
    float v = lv[0];
    int i = li[0];
    warp_argmax(v, i);
    if (li[0] == i) {                         // (flat indices are unique: exactly one lane pops its head)
#pragma unroll
      for (int q = 0; q < kBeamCands - 1; ++q) { lv[q] = lv[q + 1]; li[q] = li[q + 1]; }
      lv[kBeamCands - 1] = -INFINITY; li[kBeamCands - 1] = 0x7fffffff;
    }
    if (lane == 0) { wv[warp][round] = v; wi[warp][round] = i; }
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < kBeamCands; ++q) { lv[q] = wv[lane][q]; li[q] = wi[lane][q]; }
    for (int round = 0; round < kBeamCands; ++round) {
      float v = lv[0];
      int i = li[0];
      warp_argmax(v, i);
      if (li[0] == i) {
#pragma unroll
        for (int q = 0; q < kBeamCands - 1; ++q) { lv[q] = lv[q + 1]; li[q] = li[q + 1]; }
        lv[kBeamCands - 1] = -INFINITY; li[kBeamCands - 1] = 0x7fffffff;
      }
      if (lane == 0) { cand_v[round] = v; cand_i[round] = i; }
    }
  }
  __syncthreads();

  // 4. the bookkeeping of steps 3-6 for this item (at most 16 candidates: one thread)
  if (tid == 0) {
    const bool last = t + 1 >= s->n_steps;
    bool hit[kBeamCands];
    float adj[kBeamCands];
    int open = 0;
    for (int k = 0; k < K; ++k) {
      hit[k] = last || (long long)(cand_i[k] % V) == s->eos;
      adj[k] = hit[k] ? cand_v[k] + kBeamNeg : cand_v[k];
      open |= !hit[k];
    }
    // next running beams: top nb of adj
    float new_run[kMaxBeams];
    unsigned used = 0;
    for (int j = 0; j < nb; ++j) {
      int best = -1;
      for (int k = 0; k < K; ++k)
        if (!(used >> k & 1) && (best < 0 || adj[k] > adj[best])) best = k;
      used |= 1u << best;
      run_src[j] = cand_i[best] / V;
      run_new[j] = cand_i[best] % V;
      new_run[j] = adj[best];
    }
    // finished hypotheses: merge [old nb | K candidates], keep the top nb
    bool full = s->early_stopping == 1;
    for (int j = 0; j < nb; ++j) full = full && s->fin_flag[r0 + j];
    const bool heur = s->heur[g] != 0;
    const float div = lp_div[t];
    float ms[kMaxBeams + kBeamCands];
    int mf[kMaxBeams + kBeamCands], ml[kMaxBeams + kBeamCands];
    for (int j = 0; j < nb; ++j) { ms[j] = s->fin_score[r0 + j]; mf[j] = s->fin_flag[r0 + j]; ml[j] = s->fin_len[r0 + j]; }
    for (int k = 0; k < K; ++k) {
      const bool just = k < nb && hit[k];
      float v = __fdiv_rn(cand_v[k], div);
      if (full) v += kBeamNeg;
      if (!heur) v += kBeamNeg;
      if (!just) v += kBeamNeg;
      ms[nb + k] = v; mf[nb + k] = just; ml[nb + k] = t + 1;
    }
    used = 0;
    float fmin = INFINITY;
    int nf[kMaxBeams];
    for (int j = 0; j < nb; ++j) {
      int best = -1;
      for (int m = 0; m < nb + K; ++m)
        if (!(used >> m & 1) && (best < 0 || ms[m] > ms[best])) best = m;
      used |= 1u << best;
      fin_src[j] = best >= nb ? best - nb : -1 - best;
      nf[j] = mf[best];
      s->fin_score[r0 + j] = ms[best];
      s->fin_len[r0 + j] = ml[best];
      fmin = fminf(fmin, ms[best]);
    }
    for (int j = 0; j < nb; ++j) {
      s->fin_flag[r0 + j] = nf[j];
      s->run_score[r0 + j] = new_run[j];
      s->parent[r0 + j] = r0 + run_src[j];
    }
    // early-stop heuristic, at the new length t + 1
    const int best_len = (s->early_stopping == 2 && s->lp_positive) ? s->n_steps : t + 1;
    const float best_possible = __fdiv_rn(new_run[0], lp_div[best_len - 1]);
    int any = 0;
    for (int j = 0; j < nb; ++j) any |= best_possible > (nf[j] ? fmin : kBeamNeg);
    s->heur[g] = heur && any;
    s->open[g] = open;
  }
  __syncthreads();

  // 5. token rows of the next step: a candidate is its parent's running row + its token
  const long long* run_old = run_tok + (size_t)(t & 1) * rows * stride;
  long long* run_nxt = run_tok + (size_t)((t + 1) & 1) * rows * stride;
  const long long* fin_old = fin_tok + (size_t)(t & 1) * rows * stride;
  long long* fin_nxt = fin_tok + (size_t)((t + 1) & 1) * rows * stride;
  const bool track = s->bidx_out != nullptr;
  const int* run_bi_old = run_bi + (size_t)(t & 1) * rows * stride;
  int* run_bi_nxt = run_bi + (size_t)((t + 1) & 1) * rows * stride;
  const int* fin_bi_old = fin_bi + (size_t)(t & 1) * rows * stride;
  int* fin_bi_nxt = fin_bi + (size_t)((t + 1) & 1) * rows * stride;
  for (int e = tid; e < 2 * nb * (t + 1); e += kBeamThreads) {
    const int which = e / (nb * (t + 1)), r = e - which * nb * (t + 1), j = r / (t + 1), p = r - j * (t + 1);
    long long v;
    if (which == 0) {
      const int parent = r0 + run_src[j];
      v = p == t ? run_new[j] : run_old[(size_t)parent * stride + p];
      run_nxt[(size_t)(r0 + j) * stride + p] = v;
      if (track) run_bi_nxt[(size_t)(r0 + j) * stride + p] = p == t ? parent : run_bi_old[(size_t)parent * stride + p];
    } else {
      const int src = fin_src[j];
      int bi;
      if (src >= 0) {
        const int parent = r0 + cand_i[src] / V;
        v = p == t ? (long long)(cand_i[src] % V) : run_old[(size_t)parent * stride + p];
        bi = p == t ? parent : (track ? run_bi_old[(size_t)parent * stride + p] : 0);
      } else {
        v = fin_old[(size_t)(r0 - 1 - src) * stride + p];
        bi = track ? fin_bi_old[(size_t)(r0 - 1 - src) * stride + p] : 0;
      }
      fin_nxt[(size_t)(r0 + j) * stride + p] = v;
      if (track) fin_bi_nxt[(size_t)(r0 + j) * stride + p] = bi;
    }
  }
  if (tid < nb) cur_tokens[r0 + tid] = run_new[tid];

  // 6. the last item to finish decides whether the search goes on (HF's _beam_search_has_unfinished_sequences)
  __syncthreads();
  if (tid != 0) return;
  __threadfence();
  if (atomicAdd(&s->arrive, 1u) != gridDim.x - 1) return;
  __threadfence();
  const volatile BeamState* vs = s;
  int improvement = 0, all_fin = 1, valid = 0;
  for (int i = 0; i < (int)gridDim.x; ++i) { improvement |= vs->heur[i]; valid |= vs->open[i]; }
  for (int r = 0; r < rows; ++r) all_fin &= vs->fin_flag[r];
  const bool go_on = improvement && !(all_fin && s->early_stopping == 1) && valid;
  s->arrive = 0;
  s->step = t + 1;
  if (!go_on) {
    s->done = 1;
    ss->all_done = 1;
  }
}

// Results: for item g and j < nrs, output row g * nrs + j = finished slot j: seq_out [., n_cols] (fill beyond its length),
// scores_out, len_out; when recording, s->bidx_out [., n_cols] (-1 beyond its length) and *s->steps_out.
__global__ void beam_output_kernel(const BeamState* s, const long long* fin_tok, const int* fin_bi, int stride, int rows, int nrs,
                                   int n_cols, long long fill, long long* seq_out, float* scores_out, int* len_out) {
  const int o = blockIdx.x, g = o / nrs, j = o - g * nrs, r = g * s->nb + j;
  const size_t at = (size_t)(s->step & 1) * rows * stride + (size_t)r * stride;
  const long long* src = fin_tok + at;
  const int len = s->fin_len[r];
  for (int p = threadIdx.x; p < n_cols; p += blockDim.x) seq_out[(size_t)o * n_cols + p] = p < len ? src[p] : fill;
  if (s->bidx_out)
    for (int p = threadIdx.x; p < n_cols; p += blockDim.x) s->bidx_out[(size_t)o * n_cols + p] = p < len ? (long long)fin_bi[at + p] : -1;
  if (threadIdx.x == 0) {
    scores_out[o] = s->fin_score[r];
    len_out[o] = len;
    if (o == 0 && s->steps_out) *s->steps_out = s->step;
  }
}

// ---- KV-cache reorder (HF Cache.reorder_cache(beam_idx)) ----
// Row r of every layer's K and V takes row parent[r], for positions [*from_pos, *len) only (the prompt rows of the beams of
// one item are identical).  Rows are reordered within groups of `group` consecutive rows (a beam request's items; one group
// for the stand-alone call); a parent outside the row's group leaves the row as it is.  One CTA per (layer, K/V, group, head)
// walks the positions in blocks: it reads every source chunk the block needs into shared memory once, then writes the rows
// whose parent differs -- in place and race-free, since no other CTA touches these rows.  A group whose permutation is the
// identity exits at once; so does everything once *skip is set (the search has ended).
constexpr int kReorderThreads = 256;
constexpr int kReorderSmemBytes = 32 * 1024;
__host__ __device__ inline int reorder_block_positions(int group) {   // positions per block: group rows x 256 bytes each
  const int p = kReorderSmemBytes / (group * 256);
  return p > 0 ? p : 1;
}

__global__ void __launch_bounds__(kReorderThreads) kv_beam_reorder_kernel(__nv_bfloat16* cache, int B, int nH, int Smax, int group,
                                                                           const int* parent, const int* from_pos, const int* len,
                                                                           const int* skip) {
  extern __shared__ int4 chunk[];             // [group][P positions][16 x 16 bytes]
  if (skip && *skip) return;
  int c = blockIdx.x;
  const int h = c % nH;
  c /= nH;
  const int groups = B / group, g = c % groups, lw = c / groups;     // lw = layer * 2 + (0: K, 1: V)
  const int r0 = g * group;
  uint64_t changed = 0, needed = 0;
  for (int j = 0; j < group; ++j) {
    const int p = parent[r0 + j] - r0;
    if (p != j && p >= 0 && p < group) { changed |= 1ull << j; needed |= 1ull << p; }
  }
  if (!changed) return;
  const int P = reorder_block_positions(group), from = *from_pos, end = *len;
  auto row = [&](int j) { return reinterpret_cast<int4*>(cache + (((size_t)lw * B + r0 + j) * nH + h) * (size_t)Smax * 128); };
  for (int p0 = from; p0 < end; p0 += P) {
    const int n = (min(P, end - p0)) * 16;
    for (int j = 0; j < group; ++j) {
      if (!(needed >> j & 1)) continue;
      const int4* src = row(j) + (size_t)p0 * 16;
      for (int i = threadIdx.x; i < n; i += kReorderThreads) chunk[j * P * 16 + i] = src[i];
    }
    __syncthreads();
    for (int j = 0; j < group; ++j) {
      if (!(changed >> j & 1)) continue;
      const int4* src = chunk + (parent[r0 + j] - r0) * P * 16;
      int4* dst = row(j) + (size_t)p0 * 16;
      for (int i = threadIdx.x; i < n; i += kReorderThreads) dst[i] = src[i];
    }
    __syncthreads();
  }
}

}  // namespace vly
