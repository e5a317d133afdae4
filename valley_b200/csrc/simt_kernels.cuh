// SIMT kernels: layout / gather kernels around the tensor-core path, the per-op decode path's embedding
// gather, cross-entropy and weight-upload conversions.
#pragma once
#include "common.cuh"

namespace vly {

// ============================================================================================
// ViT front end
// ============================================================================================
// pixels [F,3,IMG,IMG] (fp32 / fp16 / bf16) -> patch matrix [F*G*G, KPAD] bf16, k = c*P*P + ky*P + kx
// (the flattening of conv weight [D,3,P,P]; HF:modeling_clip.py:208-210 casts pixels to the weight dtype).
template <typename T>
__global__ void im2col_kernel(const T* __restrict__ px, __nv_bfloat16* __restrict__ out, int F, int IMG, int P, int KPAD) {
  const int G = IMG / P, KK = 3 * P * P;
  const int chunks = KPAD / 8;
  const long long total = (long long)F * G * G * chunks;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = int(i % chunks);
    const long long row = i / chunks;
    const int pxi = int(row % G), pyi = int((row / G) % G), f = int(row / (G * G));
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = ch * 8 + e;
      if (k < KK) {
        const int c = k / (P * P), rem = k % (P * P), ky = rem / P, kx = rem % P;
        v[e] = float(px[(((long long)f * 3 + c) * IMG + (pyi * P + ky)) * IMG + (pxi * P + kx)]);
      } else {
        v[e] = 0.f;
      }
    }
    *reinterpret_cast<uint4*>(out + row * KPAD + ch * 8) =
        make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
}

VLY_DEVINL float block_sum_128(float v, float* red) {  // blockDim.x == 128
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return red[0] + red[1] + red[2] + red[3];
}

// CLS concat + position embedding + pre-LayerNorm (HF:modeling_clip.py:212-219, :677), one CTA per token row.
// Writes hidden_states[0] and its row statistics (for layer 0's LN1 fold).  D == 1024, 128 threads x 8.
__global__ void __launch_bounds__(128) vit_embed_ln_kernel(const __nv_bfloat16* __restrict__ patch_out,  // [F*NP, D]
                                                           const float* __restrict__ cls, const float* __restrict__ pos,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           __nv_bfloat16* __restrict__ x, float2* __restrict__ stats,
                                                           int stats_nt, int tokens, int D, float eps) {
  __shared__ float red[4];
  const int row = blockIdx.x, f = row / tokens, t = row % tokens;
  const int c0 = threadIdx.x * 8;
  float e[8];
  if (t == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) e[i] = bf16_round(cls[c0 + i] + pos[c0 + i]);
  } else {
    const uint4 pv = *reinterpret_cast<const uint4*>(patch_out + ((size_t)f * (tokens - 1) + (t - 1)) * D + c0);
    const uint32_t w[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      e[2 * i] = bf16_round(bf16_lo(w[i]) + pos[(size_t)t * D + c0 + 2 * i]);
      e[2 * i + 1] = bf16_round(bf16_hi(w[i]) + pos[(size_t)t * D + c0 + 2 * i + 1]);
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += e[i];
  const float mean = block_sum_128(s, red) / D;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += (e[i] - mean) * (e[i] - mean);
  const float rstd = rsqrtf(block_sum_128(ss, red) / D + eps);
  uint32_t o[4];
  float so = 0.f, sq = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = (e[2 * i] - mean) * rstd * gamma[c0 + 2 * i] + beta[c0 + 2 * i];
    const float b = (e[2 * i + 1] - mean) * rstd * gamma[c0 + 2 * i + 1] + beta[c0 + 2 * i + 1];
    o[i] = pack_bf16x2(a, b);
    const float ar = bf16_lo(o[i]), br = bf16_hi(o[i]);
    so += ar + br;
    sq += ar * ar + br * br;
  }
  *reinterpret_cast<uint4*>(x + (size_t)row * D + c0) = make_uint4(o[0], o[1], o[2], o[3]);
  so = block_sum_128(so, red);
  sq = block_sum_128(sq, red);
  if (threadIdx.x < stats_nt) stats[(size_t)row * stats_nt + threadIdx.x] = threadIdx.x == 0 ? make_float2(so, sq) : make_float2(0.f, 0.f);
}

// ============================================================================================
// temporal pool (valley_model.py:207, :215) -- pool BEFORE projecting (the projector is linear)
// feats [NV*T, tokens, D] -> vis_in [NV, (tokens-1)+T, D]: rows 0..tokens-2 = mean over T of patch rows,
// rows tokens-1.. = CLS row of each frame.
// ============================================================================================
__global__ void temporal_pool_kernel(const __nv_bfloat16* __restrict__ feats, __nv_bfloat16* __restrict__ out, int NV, int T,
                                     int tokens, int D) {
  const int rows_out = tokens - 1 + T;
  const int chunks = D / 8;
  const long long total = (long long)NV * rows_out * chunks;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = int(i % chunks);
    const long long ro = i / chunks;
    const int r = int(ro % rows_out), v = int(ro / rows_out);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (r < tokens - 1) {
      for (int t = 0; t < T; ++t) {
        const uint4 w = *reinterpret_cast<const uint4*>(feats + (((size_t)v * T + t) * tokens + (r + 1)) * D + ch * 8);
        acc[0] += bf16_lo(w.x); acc[1] += bf16_hi(w.x); acc[2] += bf16_lo(w.y); acc[3] += bf16_hi(w.y);
        acc[4] += bf16_lo(w.z); acc[5] += bf16_hi(w.z); acc[6] += bf16_lo(w.w); acc[7] += bf16_hi(w.w);
      }
      const float inv = 1.f / T;
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] *= inv;
    } else {
      const int t = r - (tokens - 1);
      const uint4 w = *reinterpret_cast<const uint4*>(feats + (((size_t)v * T + t) * tokens) * D + ch * 8);
      acc[0] = bf16_lo(w.x); acc[1] = bf16_hi(w.x); acc[2] = bf16_lo(w.y); acc[3] = bf16_hi(w.y);
      acc[4] = bf16_lo(w.z); acc[5] = bf16_hi(w.z); acc[6] = bf16_lo(w.w); acc[7] = bf16_hi(w.w);
    }
    *reinterpret_cast<uint4*>(out + ro * D + ch * 8) = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                                                                  pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
  }
}

// ============================================================================================
// embedding gather + visual splice (valley_model.py:160, :223-247): one CTA per sequence position.
// src_map[b,s] = -1 -> token embedding row; >= 0 -> row (img_idx[b]*rows_per_img + src) of the projected visual rows.
// Also emits the row sum-of-squares for the first RMSNorm fold.
// ============================================================================================
__global__ void __launch_bounds__(128) embed_splice_kernel(const long long* __restrict__ ids, const int* __restrict__ src_map,
                                                           const int* __restrict__ img_idx,
                                                           const __nv_bfloat16* __restrict__ embed,
                                                           const __nv_bfloat16* __restrict__ vis_rows, int rows_per_img,
                                                           __nv_bfloat16* __restrict__ out, float2* __restrict__ stats,
                                                           int stats_nt, int S, int H, int vocab) {
  __shared__ float red[4];
  const int row = blockIdx.x, b = row / S;
  const int src = src_map ? src_map[row] : -1;
  const __nv_bfloat16* sp;
  if (src < 0) {
    long long id = ids[row];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    sp = embed + (size_t)id * H;
  } else {
    sp = vis_rows + ((size_t)img_idx[b] * rows_per_img + src) * H;
  }
  float s = 0.f, sq = 0.f;
  for (int c = threadIdx.x * 8; c < H; c += 128 * 8) {
    const uint4 w = *reinterpret_cast<const uint4*>(sp + c);
    *reinterpret_cast<uint4*>(out + (size_t)row * H + c) = w;
    const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float a = bf16_lo(ww[i]), bb = bf16_hi(ww[i]);
      s += a + bb;
      sq += a * a + bb * bb;
    }
  }
  s = block_sum_128(s, red);
  sq = block_sum_128(sq, red);
  if (stats != nullptr && threadIdx.x < stats_nt)
    stats[(size_t)row * stats_nt + threadIdx.x] = threadIdx.x == 0 ? make_float2(s, sq) : make_float2(0.f, 0.f);
}

// decode: x[b,:] = embed[token[b],:]
__global__ void decode_embed_kernel(const long long* __restrict__ tokens, const __nv_bfloat16* __restrict__ embed,
                                    __nv_bfloat16* __restrict__ x, int H, int vocab) {
  const int b = blockIdx.x;
  long long id = tokens[b];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8)
    *reinterpret_cast<uint4*>(x + (size_t)b * H + c) = *reinterpret_cast<const uint4*>(embed + (size_t)id * H + c);
}

// ============================================================================================
// Shifted cross-entropy (valley_model.py:308-318): row r = (b, s) with s < S-1 scores logits[b, s, :] against labels[b, s+1];
// nll = logsumexp - logit[label]; labels == ignore_index are skipped; loss = mean over the counted rows.
// grid (B*(S-1)), 256 threads -> nll[r] (0 when ignored), cnt[r]; ce_mean_kernel folds them in a fixed order (deterministic).
// ============================================================================================
__global__ void __launch_bounds__(256) ce_rows_kernel(const float* __restrict__ logits, const long long* __restrict__ labels, int S, int V,
                                                      long long ignore_index, float* __restrict__ nll, int* __restrict__ cnt) {
  __shared__ float red[8];
  __shared__ float bc;
  const int r = blockIdx.x, b = r / (S - 1), s = r % (S - 1);
  const long long lab = labels[(size_t)b * S + s + 1];
  if (lab == ignore_index || lab < 0 || lab >= V) {
    if (threadIdx.x == 0) { nll[r] = 0.f; cnt[r] = 0; }
    return;
  }
  const float* x = logits + ((size_t)b * S + s) * V;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += 256) m = fmaxf(m, x[i]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int i = 1; i < 8; ++i) t = fmaxf(t, red[i]);
    bc = t;
  }
  __syncthreads();
  m = bc;
  float sum = 0.f;
  for (int i = threadIdx.x; i < V; i += 256) sum += expf(x[i] - m);
  sum = warp_sum(sum);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    nll[r] = m + logf(t) - x[lab];
    cnt[r] = 1;
  }
}

__global__ void __launch_bounds__(1024) ce_mean_kernel(const float* __restrict__ nll, const int* __restrict__ cnt, int rows, float* __restrict__ loss) {
  __shared__ double sv[32];
  __shared__ int sc[32];
  double a = 0.0;
  int c = 0;
  for (int i = threadIdx.x; i < rows; i += 1024) { a += nll[i]; c += cnt[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = a; sc[threadIdx.x >> 5] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    int n = 0;
    for (int i = 0; i < 32; ++i) { t += sv[i]; n += sc[i]; }
    *loss = n > 0 ? (float)(t / n) : __int_as_float(0x7fc00000);     // no counted label: nan, like torch
  }
}

// Generic dtype conversion to bf16 / fp32 staging (weights upload).
template <typename T>
__global__ void convert_to_bf16_kernel(const T* __restrict__ in, __nv_bfloat16* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(float(in[i]));
}
template <typename T>
__global__ void convert_to_f32_bf16rounded_kernel(const T* __restrict__ in, float* __restrict__ out, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = bf16_round(float(in[i]));
}

}  // namespace vly
