// libvalley_b200.so -- host side of the C ABI declared in include/valley_b200.h.
// Owns: packed weights, workspace, KV caches, CUDA graphs of the decode steps.  No torch, no CPU fallback.
#include <cuda_runtime.h>
#include <cuda.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/valley_b200.h"
#include "attention_tc.cuh"
#include "common.cuh"
#include "gemm_tc.cuh"
#include "simt_kernels.cuh"
#include "decode_kernels.cuh"
#include "decode_mega.cuh"
#include "preprocess.cuh"
#include "pooling_kernels.cuh"
#include "beam.cuh"

using namespace vly;
typedef __nv_bfloat16 bf16;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
extern "C" void vly_set_error_(const char* m) { snprintf(g_err, sizeof(g_err), "%s", m); }
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
extern "C" const char* vly_last_error(void) { return g_err; }
extern "C" const char* vly_version(void) { return "valley_b200 0.1 (sm_90a)"; }

#define CK(expr)                                                                                       \
  do {                                                                                                 \
    cudaError_t e_ = (expr);                                                                           \
    if (e_ != cudaSuccess) return fail(VLY_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
  } while (0)
#define TRY(expr)              \
  do {                         \
    int r_ = (expr);           \
    if (r_ != VLY_OK) return r_; \
  } while (0)

// ------------------------------------------------------------------------------------------------
// data structures
// ------------------------------------------------------------------------------------------------
// Bytes held by all live Mem objects of the process: [0] device memory, [1] pinned host memory (vly_held_bytes).
static std::atomic<int64_t> g_held_bytes[2];

// One allocation of the library: device memory, or pinned host memory (which the device can address too).  Move-only; the
// memory is freed when its owner is destroyed.  Its constructor and destructor are the only code that updates g_held_bytes.
struct Mem {
  void* p = nullptr;
  size_t bytes = 0;
  bool pinned = false;
  Mem() = default;
  Mem(void* q, size_t n, bool host) : p(q), bytes(n), pinned(host) { g_held_bytes[pinned] += (int64_t)bytes; }
  Mem(Mem&& o) noexcept { swap(o); }
  Mem& operator=(Mem&& o) noexcept {
    Mem t(std::move(o));
    swap(t);  // t leaves with what this held
    return *this;
  }
  ~Mem() {
    if (!p) return;
    if (pinned) cudaFreeHost(p);
    else cudaFree(p);
    g_held_bytes[pinned] -= (int64_t)bytes;
  }
  void swap(Mem& o) noexcept {
    std::swap(p, o.p);
    std::swap(bytes, o.bytes);
    std::swap(pinned, o.pinned);
  }
  // replaces what this holds by n new bytes; the old allocation is freed first
  int alloc(size_t n, bool host = false) {
    *this = Mem();
    void* q = nullptr;
    if (host) CK(cudaHostAlloc(&q, n, cudaHostAllocMapped));
    else CK(cudaMalloc(&q, n));
    *this = Mem(q, n, host);
    return VLY_OK;
  }
};
// a Mem that reads as a T*
template <typename T>
struct Owned : Mem {
  operator T*() const { return static_cast<T*>(p); }
  T* operator->() const { return static_cast<T*>(p); }
};

// grow-only workspace
static int ensure(Mem& b, size_t bytes) { return b.bytes >= bytes ? VLY_OK : b.alloc(bytes); }

struct Staged {
  std::vector<int64_t> shape;
  Mem mem;
  bool is_f32 = false;  // vectors are kept as fp32 holding bf16-rounded values; matrices as bf16
  int64_t numel = 0;
};

struct VitLayerW {
  Owned<bf16> wqkv, wo, w1, w2;
  Owned<float> qkv_cs, qkv_b, bo, c1, b1, b2;
};
struct LlamaLayerW {
  Owned<bf16> wqkv, wo, wgu, wdown;
};

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct vly_ctx {
  vly_config cfg;
  int num_sms = 0;
  PFN_encodeTiled encode = nullptr;
  std::mutex mu;
  std::map<std::string, Staged> staged;
  bool finalized = false;
  bool has_vit = false, has_llm = false;
  // ViT
  int kpad = 0;
  Owned<bf16> patch_w;
  Owned<float> cls, pos, pre_g, pre_b;
  std::vector<VitLayerW> vit;
  Owned<bf16> proj_w;
  Owned<float> proj_b;
  // LLaMA
  Owned<bf16> embed;
  std::vector<LlamaLayerW> layers;
  Owned<bf16> lm_head;
  Owned<float2> rope;
  // workspace
  Mem w_col, w_patch, w_qkv, w_ctx, w_h, w_stats, w_pool, w_x, w_q, w_attn, w_hb, w_pstats;
  cudaStream_t cap_stream = nullptr;
  int64_t launches = 0;           // kernels launched (and replayed in graphs) so far: counted by launch() only
  // fused all-gather state
  Owned<bf16> g_buf;              // [g_rows, vit_hidden] + flags
  int64_t g_rows = 0;
  int* g_flags = nullptr;
  bf16* g_peer_buf[8] = {};       // g_buf for this rank, CUDA IPC mappings of the other ranks' buffers
  int* g_peer_flags[8] = {};
  int g_world = 0, g_rank = 0, g_epoch = 0;
  Owned<int> g_timeout;           // pinned + mapped: set by gather_wait_kernel when a peer never signalled; read by the host
  Mem w_xlocal;
  // pooling variants (valley_model.py:40-52, :205-213)
  Owned<float> pool_U;                         // temporal_importance: W_proj^T w_pool, [256, vit_hidden] fp32
  struct DeltaW {                              // temporal_transformer: one post-LN nn.TransformerEncoderLayer + position_matrix
    Owned<bf16> in_w, out_w, l1_w, l2_w, pos;
    Owned<float> in_b, out_b, l1_b, l2_b, n1_g, n1_b, n2_g, n2_b;
    int ffn = 0, max_pos = 0;
  } delta;
  Mem w_score, w_pall, w_xp, w_dkv, w_dq, w_datt, w_dx1, w_df1, w_dx2;
  // frame preprocessing: strip + coefficient tables of the last geometry seen
  Mem w_strip, w_tables;
  int pre_H = 0, pre_W = 0;
  PreprocParams pre = {};
  // per-kernel test hooks: device scalars, work counters and partials of vly_test_gemv / vly_test_decode_attention; the packed
  // key bits of vly_test_prefill_attention
  Mem w_tgemv, w_tattn, w_tprefill;

  // (runs before the members above are freed)
  ~vly_ctx() {
    for (bf16* b : g_peer_buf)
      if (b && b != g_buf) cudaIpcCloseMemHandle(b);
    if (cap_stream) cudaStreamDestroy(cap_stream);
  }
};

// What a decode step ends with: the token selected by the persistent kernel or the per-op path's selection kernel, a filtered
// token (sample_filter_kernel after the step), or a beam search step (beam_step_kernel + kv_beam_reorder_kernel)
enum StepKind { STEP_TOKEN, STEP_FILTERED, STEP_BEAM, kStepKinds };

// The decode steps of one kind as CUDA graphs: one step, and kGraphSteps steps in one graph (fewer graph launches,
// kernel->kernel edges inside).  Captured on first use, and again for another beam count; the only owner of graph execs.
struct StepGraphs {
  cudaGraphExec_t one = nullptr, many = nullptr;
  int nodes = 0;                      // kernel launches per step
  int nb = 0;                         // beams per item the beam steps were captured for
  void reset() {
    if (one) cudaGraphExecDestroy(one);
    if (many) cudaGraphExecDestroy(many);
    one = many = nullptr;
  }
  ~StepGraphs() { reset(); }
};

struct vly_kv;
static int sync_len(vly_kv* kv);
struct vly_kv {
  vly_ctx* ctx;
  int B, Smax;
  Owned<bf16> cache;  // [L][2][B][nH][Smax][128]
  int host_len = 0;
  bool len_dirty = false;   // a stop token may have ended vly_generate early: host_len is re-read from the device on next use
  Owned<int> h_len;         // pinned: d_len is copied here on the generating stream, len_event marks the copy
  cudaEvent_t len_event = nullptr;
  Owned<int> d_len;       // device scalar
  int* d_step = nullptr;
  // decode workspace
  Owned<bf16> x, q, attn, hb;
  Owned<float> part_o;
  Owned<float2> part_ml;
  Owned<unsigned int> counters;       // [B*nH] + 1 (argmax)
  Owned<float> part_val;              // [B, SMs]: per-CTA arg-max partials
  Owned<int> part_idx;
  Owned<float> logits;                // [B, V]
  Owned<long long> cur_tokens;        // [B]
  Owned<long long> gen_tokens;        // [B, Smax]
  int nsplit = 1;
  // persistent decode kernel (B <= 4): the whole launch, fixed by vly_kv_create
  Owned<PhaseDesc> d_phases;
  StepParams mega = {};
  size_t mega_smem = 0;
  Owned<long long> dbg;               // [SMs][32] cycle counters (StepParams::dbg); allocated only with VLY_MEGA_DBG
  Owned<SampleState> d_sample;        // token selection state read by every decode step (sampling.cuh)
  bool sample_dirty = false;          // device state is not the plain-greedy default
  bool filtered = false;              // the last sampling set has a top-k / top-p filter: sample_filter_kernel selects
  bool recording = false;             // the last sampling set records scores or logits: sample_filter_kernel selects
  Owned<uint32_t> key_bits;           // [B, Smax/32] attention_mask bits (1 = attend); all ones unless vly_kv_set_key_mask
  bool masked = false;
  int mask_words() const { return Smax / 32; }
  // beam search (vly_beam_search), allocated on the cache's first beam request: the state, the running and finished token
  // rows [2 parities][2][B][Smax], their beam-index rows (same layout, int32; written only by requests that record beam
  // indices) and the length-penalty divisors [Smax]
  Owned<BeamState> d_beam;
  Owned<long long> beam_tok;
  Owned<int> beam_bidx;
  Owned<float> beam_div;
  Owned<int> beam_from;               // vly_kv_beam_reorder's first position
  // stop strings (set_sampling), allocated on the cache's first stop-string request: the tables and the per-row token rings
  // on the device (stop_layout), and the pinned copy they are uploaded from (stop_event: the last upload has read it)
  Owned<uint8_t> stop_buf, stop_stage;
  cudaEvent_t stop_event = nullptr;
  bool stop_ready = false;            // the running request has stop strings, and its tables and rings are on the device
  // logits processors (set_sampling), allocated on the cache's first processor request: every row's token history
  // [B][Smax] int32 (SampleState::hist)
  Owned<int> hist;
  bool procs_ready = false;           // the running request has processors, and its rows' histories are on the device
  StepGraphs graphs[kStepKinds];      // (declared after the buffers they refer to: destroyed before them)
  size_t layer_stride() const { return (size_t)2 * B * ctx->cfg.num_attention_heads * Smax * 128; }
  bf16* k_layer(int l) const { return cache + (size_t)l * layer_stride(); }
  bf16* v_layer(int l) const { return k_layer(l) + layer_stride() / 2; }

  ~vly_kv() {
    if (len_event) cudaEventDestroy(len_event);
    if (stop_event) cudaEventDestroy(stop_event);
  }
};

// after an eos-terminated vly_generate only the device knows how many steps ran (one blocking 4-byte read, off the hot path)
// (the copy was enqueued on the stream that ran the generation -- torch streams are non-blocking, so a legacy-stream
//  cudaMemcpy here would not be ordered after it)
static int sync_len(vly_kv* kv) {
  if (!kv->len_dirty) return VLY_OK;
  CK(cudaSetDevice(kv->ctx->cfg.device));
  CK(cudaEventSynchronize(kv->len_event));
  kv->host_len = *reinterpret_cast<volatile int*>(kv->h_len.p);
  kv->len_dirty = false;
  return VLY_OK;
}

static inline int cdiv(long long a, long long b) { return int((a + b - 1) / b); }

// cudaFuncSetAttribute is per DEVICE: a second vly_ctx on another GPU of the same process must opt in again, so what has been
// set is tracked per (device, kernel) -- not in function-local statics.
static std::mutex g_attr_mu;
static std::map<std::pair<int, const void*>, size_t> g_attr_set;
template <typename Kern>
static int ensure_smem_attr(int device, Kern kern, size_t bytes, bool max_carveout) {
  std::lock_guard<std::mutex> lk(g_attr_mu);
  size_t& have = g_attr_set[std::make_pair(device, (const void*)kern)];
  if (bytes > have || (have == 0 && max_carveout)) {
    if (bytes > 0) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    if (max_carveout) CK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    have = bytes > 0 ? bytes : 1;
  }
  return VLY_OK;
}

// ------------------------------------------------------------------------------------------------
// TMA descriptors
// ------------------------------------------------------------------------------------------------
static int make_tmap_2d(vly_ctx* c, CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t rows, uint64_t row_stride_bytes,
                        uint32_t box_inner, uint32_t box_rows, bool swizzle128 = true) {
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = c->encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(VLY_ERR_CUDA, "cuTensorMapEncodeTiled(2d) failed: %d (ptr=%p inner=%llu rows=%llu stride=%llu box=%u,%u)", (int)r, ptr,
                (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)row_stride_bytes, box_inner, box_rows);
  return VLY_OK;
}
static int make_tmap_3d(vly_ctx* c, CUtensorMap* m, const void* ptr, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1, uint64_t s2,
                        uint32_t b0, uint32_t b1) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {s1, s2};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = c->encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VLY_ERR_CUDA, "cuTensorMapEncodeTiled(3d) failed: %d", (int)r);
  return VLY_OK;
}

// ------------------------------------------------------------------------------------------------
// kernel launches
// ------------------------------------------------------------------------------------------------
static bool pdl_enabled() {
  static const bool on = getenv("VLY_NO_PDL") == nullptr;
  return on;
}
struct LaunchCfg {
  dim3 grid, block;
  size_t smem = 0;              // dynamic shared memory
  cudaStream_t st = 0;
  // programmatic dependent launch: the kernel's prologue overlaps the previous kernel's tail.  Only for kernels that call
  // griddepcontrol.wait before they touch the previous kernel's data.  VLY_NO_PDL=1 disables it.
  bool pdl = false;
  bool carveout = false;        // maximum shared-memory carve-out, so the NEXT kernel's CTA can co-reside (PDL overlap)
  bool cooperative = false;     // every CTA resident at once (grid barriers)
};
// Every kernel of the library is launched here, and this is the only code that counts launches (vly_kernel_launch_count;
// capture_steps derives StepGraphs::nodes from the count).  cudaLaunchKernelEx converts each argument to the kernel's
// parameter type, as <<<>>> does.
template <typename... KArgs, typename... Args>
static int launch(vly_ctx* c, void (*kern)(KArgs...), const LaunchCfg& l, Args&&... args) {
  if (l.smem > 0 || l.carveout) TRY(ensure_smem_attr(c->cfg.device, kern, l.smem, l.carveout));
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (l.pdl && pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (l.cooperative) {
    attr[n].id = cudaLaunchAttributeCooperative;
    attr[n++].val.cooperative = 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = l.grid;
  cfg.blockDim = l.block;
  cfg.dynamicSmemBytes = l.smem;
  cfg.stream = l.st;
  cfg.attrs = attr;
  cfg.numAttrs = n;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
  c->launches++;
  if (e != cudaSuccess) {
    cudaGetLastError();         // the failure is reported here; it must not surface in the caller's next error check
    const char* name = "kernel";
    cudaFuncGetName(&name, (const void*)kern);
    return fail(VLY_ERR_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(e));
  }
  return VLY_OK;
}

// The decode kernels are compiled for 1, 2 or 4 batch rows: f(std::integral_constant<int, rows for B>).
static inline int bmax_of(int B) { return B <= 1 ? 1 : (B <= 2 ? 2 : 4); }
template <typename F>
static int with_bmax(int B, F&& f) {
  if (bmax_of(B) == 1) return f(std::integral_constant<int, 1>());
  if (bmax_of(B) == 2) return f(std::integral_constant<int, 2>());
  return f(std::integral_constant<int, 4>());
}
// VLY_F32 / VLY_BF16 / VLY_F16 -> f(Type<float | bf16 | __half>)
template <typename T>
struct Type { using type = T; };
template <typename F>
static int with_dtype(int dtype, F&& f) {
  if (dtype == VLY_F32) return f(Type<float>());
  if (dtype == VLY_BF16) return f(Type<bf16>());
  if (dtype == VLY_F16) return f(Type<__half>());
  return fail(VLY_ERR_INVALID, "unknown dtype %d", dtype);
}

// ------------------------------------------------------------------------------------------------
// GEMM launcher
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI>
static int launch_gemm_t(vly_ctx* c, const bf16* A, long long lda, const bf16* W, long long ldw, GemmParams p, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  CUtensorMap ta, tb;
  TRY(make_tmap_2d(c, &ta, A, p.K, p.M, lda * 2, 64, 128));
  TRY(make_tmap_2d(c, &tb, W, p.K, p.N, ldw * 2, 64, BN));
  p.num_m_tiles = cdiv(p.M, 128);
  p.num_n_tiles = cdiv(p.N, BN);
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  return launch(c, gemm_tc_kernel<BN, EPI>, {dim3(tiles), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, st, true}, ta, tb, p);
}
template <int EPI>
static int launch_gemm(vly_ctx* c, int bn, const bf16* A, long long lda, const bf16* W, long long ldw, const GemmParams& p,
                       cudaStream_t st) {
  if (bn == 256) return launch_gemm_t<256, EPI>(c, A, lda, W, ldw, p, st);
  return launch_gemm_t<128, EPI>(c, A, lda, W, ldw, p, st);
}
static inline int pick_bn(int N) { return (N % 256 == 0) ? 256 : 128; }
// Tile width by wave efficiency: one CTA per SM at a time, so a launch runs ceil(tiles / SMs) rounds and what counts is how full
// the last round is.  M = 2056 (8 frames), N = 3072 on 132 SMs: 128 x 256 tiles -> 204 tiles = 2 rounds at 77 %; 128 x 128 -> 408
// tiles = 4 half-size rounds at 77 %.  256-wide tiles are kept unless the narrow ones fill the rounds > 5 % better (256 columns
// halve the A traffic per output).  M-dependent, so callers that exchange row statistics compute it ONCE per (N, M) and pass it
// around.  VLY_GEMM_BN=128|256 forces a width.
static inline int pick_bn_m(const vly_ctx* c, int N, int M) {
  if (N % 256 != 0) return 128;
  static const int env_bn = getenv("VLY_GEMM_BN") ? atoi(getenv("VLY_GEMM_BN")) : 0;
  if (env_bn == 128 || env_bn == 256) return env_bn;
  const long long t256 = (long long)cdiv(M, 128) * (N / 256), t128 = 2 * t256;
  if (t256 >= 3LL * c->num_sms) return 256;            // many rounds: the last one matters little, operand reuse matters more
  const double e256 = (double)t256 / ((double)cdiv(t256, c->num_sms) * c->num_sms);
  const double e128 = (double)t128 / ((double)cdiv(t128, c->num_sms) * c->num_sms);
  return (e128 > e256 * 1.05) ? 128 : 256;
}

// ------------------------------------------------------------------------------------------------
// weight packing kernels
// ------------------------------------------------------------------------------------------------
// One CTA per SOURCE row r.  dst row: mode 0 -> off + r; mode 1 (RoPE pair interleave inside 128-wide heads) ->
// off + h*128 + (d < 64 ? 2d : 2(d-64)+1); mode 2 (gate/up interleave) -> 2r + off.
__global__ void pack_rows_kernel(const bf16* __restrict__ src, int K, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ bias_in, bf16* __restrict__ dst, int Kdst, int mode, int off,
                                 float* __restrict__ colsum, float* __restrict__ bias_out) {
  __shared__ float r1[8], r2[8];
  const int r = blockIdx.x;
  int dr;
  if (mode == 0) dr = off + r;
  else if (mode == 1) {
    const int h = r >> 7, d = r & 127;
    dr = off + h * 128 + (d < 64 ? 2 * d : 2 * (d - 64) + 1);
  } else dr = 2 * r + off;
  float cs = 0.f, bb = 0.f;
  for (int k = threadIdx.x; k < Kdst; k += blockDim.x) {
    float wf = 0.f;
    if (k < K) {
      const float w = __bfloat162float(src[(size_t)r * K + k]);
      wf = gamma ? bf16_round(w * gamma[k]) : w;
      if (beta) bb += w * beta[k];
    }
    dst[(size_t)dr * Kdst + k] = __float2bfloat16_rn(wf);
    cs += wf;
  }
  cs = warp_sum(cs);
  bb = warp_sum(bb);
  if ((threadIdx.x & 31) == 0) {
    r1[threadIdx.x >> 5] = cs;
    r2[threadIdx.x >> 5] = bb;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
      a += r1[i];
      b += r2[i];
    }
    if (colsum) colsum[dr] = a;
    if (bias_out) bias_out[dr] = (bias_in ? bias_in[r] : 0.f) + b;
  }
}

// rope[pos, j] = (cos, sin) of pos * theta^(-2j/128), computed in fp32 like HF (modeling_llama.py:124-135) and rounded
// to bf16 (cos.to(x.dtype)).
__global__ void rope_table_kernel(float2* rope, int max_pos, float theta, int head_dim) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half = head_dim / 2;
  if (i >= max_pos * half) return;
  const int pos = i / half, j = i % half;
  const float inv = 1.0f / powf(theta, float(2 * j) / float(head_dim));
  const float fr = float(pos) * inv;
  rope[i] = make_float2(bf16_round(cosf(fr)), bf16_round(sinf(fr)));
}

__global__ void set_int_kernel(int* p, int v) { *p = v; }

// inputs_embeds -> x (copy) + row statistics
__global__ void __launch_bounds__(128) copy_rows_stats_kernel(const bf16* __restrict__ in, bf16* __restrict__ out,
                                                              float2* __restrict__ stats, int stats_nt, int H) {
  __shared__ float red[4];
  const int row = blockIdx.x;
  float s = 0.f, sq = 0.f;
  for (int c = threadIdx.x * 8; c < H; c += 128 * 8) {
    const uint4 w = *reinterpret_cast<const uint4*>(in + (size_t)row * H + c);
    *reinterpret_cast<uint4*>(out + (size_t)row * H + c) = w;
    const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float a = bf16_lo(ww[i]), b = bf16_hi(ww[i]);
      s += a + b;
      sq += a * a + b * b;
    }
  }
  s = block_sum_128(s, red);
  sq = block_sum_128(sq, red);
  if (threadIdx.x < stats_nt) stats[(size_t)row * stats_nt + threadIdx.x] = threadIdx.x == 0 ? make_float2(s, sq) : make_float2(0.f, 0.f);
}

// cache [B,nH,Smax,128] -> HF layout [B,nH,len,128]; K is stored RoPE-pair-interleaved and is de-interleaved here.
__global__ void kv_export_kernel(const bf16* __restrict__ cache, bf16* __restrict__ out, int Smax, int len, int deinterleave) {
  const int bh = blockIdx.y, s = blockIdx.x, c = threadIdx.x;  // 128 threads
  const int d = deinterleave ? ((c & 1) ? 64 + (c >> 1) : (c >> 1)) : c;
  out[((size_t)bh * len + s) * 128 + d] = cache[((size_t)bh * Smax + s) * 128 + c];
}

// ------------------------------------------------------------------------------------------------
// lifetime
// ------------------------------------------------------------------------------------------------
extern "C" int vly_create(const vly_config* cfg, vly_ctx** out) {
  if (!cfg || !out) return fail(VLY_ERR_INVALID, "vly_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(VLY_ERR_CUDA, "vly_create: no CUDA device visible -- this library has no CPU fallback");
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) return fail(VLY_ERR_CUDA, "vly_create: device is sm_%d%d; this library is built for sm_90a only", prop.major, prop.minor);
  if (cfg->hidden_size % 128 || cfg->hidden_size / cfg->num_attention_heads != 128)
    return fail(VLY_ERR_INVALID, "vly_create: head_dim must be 128 (hidden %d, heads %d)", cfg->hidden_size, cfg->num_attention_heads);
  if (cfg->intermediate_size % 64) return fail(VLY_ERR_INVALID, "vly_create: intermediate_size must be a multiple of 64");
  if (cfg->vit_hidden != 1024 || cfg->vit_hidden / cfg->vit_heads != 64 || cfg->vit_mlp % 256)
    return fail(VLY_ERR_INVALID, "vly_create: vision tower must be ViT-L width (1024, head_dim 64); the reference hard-codes 1024 (valley_model.py:192)");
  auto c = std::make_unique<vly_ctx>();
  c->cfg = *cfg;
  c->num_sms = prop.multiProcessorCount;
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || fn == nullptr)
    return fail(VLY_ERR_CUDA, "vly_create: cuTensorMapEncodeTiled entry point not found");
  c->encode = (PFN_encodeTiled)fn;
  if (cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking) != cudaSuccess)
    return fail(VLY_ERR_CUDA, "vly_create: cudaStreamCreate failed");
  *out = c.release();
  return VLY_OK;
}

extern "C" void vly_destroy(vly_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->cfg.device);
  delete c;
}

extern "C" int vly_num_sms(vly_ctx* c, int* out) {
  if (!c || !out) return fail(VLY_ERR_INVALID, "null");
  *out = c->num_sms;
  return VLY_OK;
}
extern "C" int vly_kernel_launch_count(vly_ctx* c, int64_t* out) {
  if (!c || !out) return fail(VLY_ERR_INVALID, "null");
  std::lock_guard<std::mutex> lk(c->mu);
  *out = c->launches;
  return VLY_OK;
}
extern "C" int vly_held_bytes(int64_t* device_bytes, int64_t* pinned_bytes) {
  if (!device_bytes || !pinned_bytes) return fail(VLY_ERR_INVALID, "null");
  *device_bytes = g_held_bytes[0];
  *pinned_bytes = g_held_bytes[1];
  return VLY_OK;
}

// ------------------------------------------------------------------------------------------------
// weights
// ------------------------------------------------------------------------------------------------
static bool ends_with(const std::string& s, const char* suf) {
  const size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}

extern "C" int vly_load_weight(vly_ctx* c, const char* name, const void* dev_ptr, int dtype, const int64_t* shape, int ndim) {
  if (!c || !name || !dev_ptr || !shape || ndim < 1 || ndim > 4) return fail(VLY_ERR_INVALID, "vly_load_weight: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->finalized) return fail(VLY_ERR_STATE, "vly_load_weight(%s): weights already finalised", name);
  if (dtype != VLY_F32 && dtype != VLY_BF16 && dtype != VLY_F16)
    return fail(VLY_ERR_INVALID, "vly_load_weight(%s): unknown dtype %d", name, dtype);
  CK(cudaSetDevice(c->cfg.device));
  Staged s;
  s.numel = 1;
  for (int i = 0; i < ndim; ++i) {
    s.shape.push_back(shape[i]);
    s.numel *= shape[i];
  }
  const std::string nm(name);
  s.is_f32 = (ndim == 1) || ends_with(nm, "position_embedding.weight");
  c->staged.erase(nm);
  TRY(s.mem.alloc((size_t)s.numel * (s.is_f32 ? 4 : 2)));
  const LaunchCfg l = {dim3((unsigned)std::min<long long>((s.numel + 255) / 256, 4096)), dim3(256)};
  TRY(with_dtype(dtype, [&](auto t) -> int {
    using E = typename decltype(t)::type;
    if (s.is_f32) return launch(c, convert_to_f32_bf16rounded_kernel<E>, l, (const E*)dev_ptr, (float*)s.mem.p, s.numel);
    if constexpr (std::is_same<E, bf16>::value) {         // a bf16 matrix is already in its staged format
      CK(cudaMemcpyAsync(s.mem.p, dev_ptr, (size_t)s.numel * 2, cudaMemcpyDeviceToDevice, 0));
      return VLY_OK;
    } else {
      return launch(c, convert_to_bf16_kernel<E>, l, (const E*)dev_ptr, (bf16*)s.mem.p, s.numel);
    }
  }));
  CK(cudaStreamSynchronize(0));  // the caller may free its tensor right after we return
  c->staged[nm] = std::move(s);
  return VLY_OK;
}

static int get_staged(vly_ctx* c, const std::string& name, bool f32, int64_t numel, void** out) {
  auto it = c->staged.find(name);
  if (it == c->staged.end()) return fail(VLY_ERR_STATE, "vly_finalize_weights: missing tensor '%s'", name.c_str());
  if (it->second.is_f32 != f32 || it->second.numel != numel)
    return fail(VLY_ERR_INVALID, "vly_finalize_weights: tensor '%s' has %lld elements (expected %lld)", name.c_str(),
                (long long)it->second.numel, (long long)numel);
  *out = it->second.mem.p;
  return VLY_OK;
}
// A tensor that needs no packing is staged in its final format: its staging allocation becomes the packed weight.
static int take(vly_ctx* c, const std::string& name, bool f32, int64_t numel, Mem* dst) {
  void* p;
  TRY(get_staged(c, name, f32, numel, &p));
  auto it = c->staged.find(name);
  *dst = std::move(it->second.mem);
  c->staged.erase(it);
  return VLY_OK;
}
static void drop_staged(vly_ctx* c, const std::string& name) { c->staged.erase(name); }

extern "C" int vly_finalize_weights(vly_ctx* c) {
  if (!c) return fail(VLY_ERR_INVALID, "null ctx");
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->finalized) return VLY_OK;
  CK(cudaSetDevice(c->cfg.device));
  const vly_config& g = c->cfg;
  const std::string vp = "model.vision_tower.vision_model.";
  c->has_vit = c->staged.count(vp + "embeddings.patch_embedding.weight") > 0;
  c->has_llm = c->staged.count("model.embed_tokens.weight") > 0;
  if (!c->has_vit && !c->has_llm) return fail(VLY_ERR_STATE, "vly_finalize_weights: no weights loaded");

  if (c->has_vit) {
    const int D = g.vit_hidden, M = g.vit_mlp, P = g.vit_patch, KK = 3 * P * P;
    c->kpad = ((KK + 63) / 64) * 64;
    const int tokens = (g.vit_image / P) * (g.vit_image / P) + 1;
    void* pw;
    TRY(get_staged(c, vp + "embeddings.patch_embedding.weight", false, (int64_t)D * KK, &pw));
    TRY(take(c, vp + "embeddings.class_embedding", true, D, &c->cls));
    TRY(take(c, vp + "embeddings.position_embedding.weight", true, (int64_t)tokens * D, &c->pos));
    TRY(take(c, vp + "pre_layrnorm.weight", true, D, &c->pre_g));
    TRY(take(c, vp + "pre_layrnorm.bias", true, D, &c->pre_b));
    TRY(c->patch_w.alloc((size_t)D * c->kpad * 2));
    TRY(launch(c, pack_rows_kernel, {dim3(D), dim3(256)}, (bf16*)pw, KK, nullptr, nullptr, nullptr, c->patch_w, c->kpad, 0, 0, nullptr,
               nullptr));
    CK(cudaDeviceSynchronize());
    drop_staged(c, vp + "embeddings.patch_embedding.weight");
    c->vit.resize(g.vit_layers);
    for (int l = 0; l < g.vit_layers; ++l) {
      const std::string q = vp + "encoder.layers." + std::to_string(l) + ".";
      VitLayerW& w = c->vit[l];
      void *g1, *b1n, *g2, *b2n;
      TRY(get_staged(c, q + "layer_norm1.weight", true, D, &g1));
      TRY(get_staged(c, q + "layer_norm1.bias", true, D, &b1n));
      TRY(get_staged(c, q + "layer_norm2.weight", true, D, &g2));
      TRY(get_staged(c, q + "layer_norm2.bias", true, D, &b2n));
      TRY(w.wqkv.alloc((size_t)3 * D * D * 2));
      TRY(w.qkv_cs.alloc(3 * D * 4));
      TRY(w.qkv_b.alloc(3 * D * 4));
      const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
      for (int i = 0; i < 3; ++i) {
        void *ww, *bb;
        TRY(get_staged(c, q + "self_attn." + nm[i] + ".weight", false, (int64_t)D * D, &ww));
        TRY(get_staged(c, q + "self_attn." + nm[i] + ".bias", true, D, &bb));
        TRY(launch(c, pack_rows_kernel, {dim3(D), dim3(256)}, (bf16*)ww, D, (float*)g1, (float*)b1n, (float*)bb, w.wqkv, D, 0, i * D,
                   w.qkv_cs, w.qkv_b));
        CK(cudaDeviceSynchronize());
        drop_staged(c, q + "self_attn." + nm[i] + ".weight");
      }
      void *w1, *b1;
      TRY(take(c, q + "self_attn.out_proj.weight", false, (int64_t)D * D, &w.wo));
      TRY(take(c, q + "self_attn.out_proj.bias", true, D, &w.bo));
      TRY(get_staged(c, q + "mlp.fc1.weight", false, (int64_t)M * D, &w1));
      TRY(get_staged(c, q + "mlp.fc1.bias", true, M, &b1));
      TRY(take(c, q + "mlp.fc2.weight", false, (int64_t)D * M, &w.w2));
      TRY(take(c, q + "mlp.fc2.bias", true, D, &w.b2));
      TRY(w.w1.alloc((size_t)M * D * 2));
      TRY(w.c1.alloc(M * 4));
      TRY(w.b1.alloc(M * 4));
      TRY(launch(c, pack_rows_kernel, {dim3(M), dim3(256)}, (bf16*)w1, D, (float*)g2, (float*)b2n, (float*)b1, w.w1, D, 0, 0, w.c1, w.b1));
      CK(cudaDeviceSynchronize());
      drop_staged(c, q + "mlp.fc1.weight");
    }
    if (c->staged.count("model.mm_projector.weight")) {
      TRY(take(c, "model.mm_projector.weight", false, (int64_t)g.hidden_size * D, &c->proj_w));
      TRY(take(c, "model.mm_projector.bias", true, g.hidden_size, &c->proj_b));
      const int H = g.hidden_size, NP = (g.vit_image / g.vit_patch) * (g.vit_image / g.vit_patch);
      if (g.patch_pooling_method == VLY_POOL_TEMPORAL_IMPORTANCE) {       // valley_model.py:40-43
        void* pw;
        TRY(get_staged(c, "model.pooling_layer.weight", false, (int64_t)NP * H, &pw));
        TRY(c->pool_U.alloc((size_t)NP * D * 4));
        TRY(launch(c, fold_importance_kernel, {dim3(NP), dim3(256)}, (const bf16*)pw, c->proj_w, c->pool_U, H, D));  // the bias cancels in the softmax
        CK(cudaDeviceSynchronize());
        drop_staged(c, "model.pooling_layer.weight");
      } else if (g.patch_pooling_method == VLY_POOL_TEMPORAL_TRANSFORMER) {   // valley_model.py:45-52
        const std::string q = "model.transformer_delta_encoder.layers.0.";
        vly_ctx::DeltaW& w = c->delta;
        auto it = c->staged.find(q + "linear1.weight");
        if (it == c->staged.end()) return fail(VLY_ERR_STATE, "vly_finalize_weights: missing tensor '%slinear1.weight'", q.c_str());
        w.ffn = (int)(it->second.numel / H);
        auto ip = c->staged.find("model.position_matrix");
        if (ip == c->staged.end()) return fail(VLY_ERR_STATE, "vly_finalize_weights: missing tensor 'model.position_matrix'");
        w.max_pos = (int)(ip->second.numel / H);
        struct { const char* name; bool f32; int64_t n; Mem* dst; } items[] = {
            {"self_attn.in_proj_weight", false, (int64_t)3 * H * H, &w.in_w}, {"self_attn.in_proj_bias", true, 3 * H, &w.in_b},
            {"self_attn.out_proj.weight", false, (int64_t)H * H, &w.out_w},   {"self_attn.out_proj.bias", true, H, &w.out_b},
            {"linear1.weight", false, (int64_t)w.ffn * H, &w.l1_w},           {"linear1.bias", true, w.ffn, &w.l1_b},
            {"linear2.weight", false, (int64_t)H * w.ffn, &w.l2_w},           {"linear2.bias", true, H, &w.l2_b},
            {"norm1.weight", true, H, &w.n1_g}, {"norm1.bias", true, H, &w.n1_b},
            {"norm2.weight", true, H, &w.n2_g}, {"norm2.bias", true, H, &w.n2_b}};
        for (auto& it2 : items) TRY(take(c, q + it2.name, it2.f32, it2.n, it2.dst));
        TRY(take(c, "model.position_matrix", false, (int64_t)w.max_pos * H, &w.pos));
      }
    }
  }

  if (c->has_llm) {
    const int H = g.hidden_size, I = g.intermediate_size, V = g.vocab_size, L = g.num_hidden_layers;
    TRY(take(c, "model.embed_tokens.weight", false, (int64_t)V * H, &c->embed));
    c->layers.resize(L);
    for (int l = 0; l < L; ++l) {
      const std::string q = "model.layers." + std::to_string(l) + ".";
      LlamaLayerW& w = c->layers[l];
      void *g1, *g2;
      TRY(get_staged(c, q + "input_layernorm.weight", true, H, &g1));
      TRY(get_staged(c, q + "post_attention_layernorm.weight", true, H, &g2));
      TRY(w.wqkv.alloc((size_t)3 * H * H * 2));
      const char* nm[3] = {"q_proj", "k_proj", "v_proj"};
      for (int i = 0; i < 3; ++i) {
        void* ww;
        TRY(get_staged(c, q + "self_attn." + nm[i] + ".weight", false, (int64_t)H * H, &ww));
        TRY(launch(c, pack_rows_kernel, {dim3(H), dim3(256)}, (bf16*)ww, H, (float*)g1, nullptr, nullptr, w.wqkv, H, i < 2 ? 1 : 0, i * H,
                   nullptr, nullptr));
        CK(cudaDeviceSynchronize());
        drop_staged(c, q + "self_attn." + nm[i] + ".weight");
      }
      void *wg, *wu;
      TRY(take(c, q + "self_attn.o_proj.weight", false, (int64_t)H * H, &w.wo));
      TRY(get_staged(c, q + "mlp.gate_proj.weight", false, (int64_t)I * H, &wg));
      TRY(get_staged(c, q + "mlp.up_proj.weight", false, (int64_t)I * H, &wu));
      TRY(take(c, q + "mlp.down_proj.weight", false, (int64_t)H * I, &w.wdown));
      TRY(w.wgu.alloc((size_t)2 * I * H * 2));
      TRY(launch(c, pack_rows_kernel, {dim3(I), dim3(256)}, (bf16*)wg, H, (float*)g2, nullptr, nullptr, w.wgu, H, 2, 0, nullptr, nullptr));
      TRY(launch(c, pack_rows_kernel, {dim3(I), dim3(256)}, (bf16*)wu, H, (float*)g2, nullptr, nullptr, w.wgu, H, 2, 1, nullptr, nullptr));
      CK(cudaDeviceSynchronize());
      drop_staged(c, q + "mlp.gate_proj.weight");
      drop_staged(c, q + "mlp.up_proj.weight");
    }
    void *nf, *lm;
    TRY(get_staged(c, "model.norm.weight", true, H, &nf));
    TRY(get_staged(c, "lm_head.weight", false, (int64_t)V * H, &lm));
    TRY(c->lm_head.alloc((size_t)V * H * 2));
    TRY(launch(c, pack_rows_kernel, {dim3(V), dim3(256)}, (bf16*)lm, H, (float*)nf, nullptr, nullptr, c->lm_head, H, 0, 0, nullptr, nullptr));
    CK(cudaDeviceSynchronize());
    drop_staged(c, "lm_head.weight");
    TRY(c->rope.alloc((size_t)g.max_position_embeddings * 64 * sizeof(float2)));
    TRY(launch(c, rope_table_kernel, {dim3(cdiv((long long)g.max_position_embeddings * 64, 256)), dim3(256)}, c->rope,
               g.max_position_embeddings, g.rope_theta, 128));
  }
  CK(cudaDeviceSynchronize());
  c->staged.clear();
  c->finalized = true;
  return VLY_OK;
}

// ------------------------------------------------------------------------------------------------
// ViT encode
// ------------------------------------------------------------------------------------------------
static int launch_vit_attention(vly_ctx* c, const bf16* qkv, int F, bf16* out, cudaStream_t st) {
  const vly_config& g = c->cfg;
  const int D = g.vit_hidden, tokens = (g.vit_image / g.vit_patch) * (g.vit_image / g.vit_patch) + 1;
  using C = FlashCfg<64>;
  CUtensorMap tq;
  TRY(make_tmap_2d(c, &tq, qkv, 3 * D, (uint64_t)F * tokens, (uint64_t)3 * D * 2, 64, 64));
  VitAttnParams p;
  p.F = F;
  p.tokens = tokens;
  p.heads = g.vit_heads;
  p.D = D;
  p.ctx = out;
  p.scale_log2e = 0.125f * 1.4426950408889634f;
  const int grid = F * g.vit_heads * cdiv(tokens, 64);
  return launch(c, vit_attention_kernel, {dim3(grid), dim3(C::THREADS), C::SMEM_BYTES, st, true}, tq, p);
}

static int vit_layers_needed(const vly_config& g, int select_layer, int* out) {
  const int idx = select_layer >= 0 ? select_layer : g.vit_layers + 1 + select_layer;
  if (idx < 0 || idx > g.vit_layers) return fail(VLY_ERR_INVALID, "select_layer %d out of range for %d layers", select_layer, g.vit_layers);
  *out = idx;
  return VLY_OK;
}

static int vit_encode_impl(vly_ctx* c, const void* pixels, int pixel_dtype, int F, int select_layer, void* out_dev, void* stream,
                           bool gather, long long gather_frame_off, int gather_frame_stride);

extern "C" int vly_vit_encode(vly_ctx* c, const void* pixels, int pixel_dtype, int F, int select_layer, void* out_dev, void* stream) {
  if (!c || !pixels || !out_dev || F <= 0) return fail(VLY_ERR_INVALID, "vly_vit_encode: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  return vit_encode_impl(c, pixels, pixel_dtype, F, select_layer, out_dev, stream, false, 0, 1);
}

static int vit_encode_impl(vly_ctx* c, const void* pixels, int pixel_dtype, int F, int select_layer, void* out_dev, void* stream,
                           bool gather, long long gather_frame_off, int gather_frame_stride) {
  if (!c->finalized || !c->has_vit) return fail(VLY_ERR_STATE, "vly_vit_encode: vision weights not loaded/finalised");
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const vly_config& g = c->cfg;
  const int D = g.vit_hidden, MLP = g.vit_mlp, P = g.vit_patch, IMG = g.vit_image;
  const int NP = (IMG / P) * (IMG / P), tokens = NP + 1;
  int n_layers;
  TRY(vit_layers_needed(g, select_layer, &n_layers));
  if (pixel_dtype != VLY_F32 && pixel_dtype != VLY_BF16 && pixel_dtype != VLY_F16)
    return fail(VLY_ERR_INVALID, "vly_vit_encode: unknown pixel dtype %d", pixel_dtype);
  const int CH = 256;  // frames per chunk: bounds the workspace (qkv 405 MB, mlp 540 MB) and keeps tiles plentiful
  const int fc_max = F < CH ? F : CH;
  const size_t Mmax = (size_t)fc_max * tokens;
  TRY(ensure(c->w_col, (size_t)fc_max * NP * c->kpad * 2));
  TRY(ensure(c->w_patch, (size_t)fc_max * NP * D * 2));
  TRY(ensure(c->w_qkv, Mmax * 3 * D * 2));
  TRY(ensure(c->w_ctx, Mmax * D * 2));
  TRY(ensure(c->w_h, Mmax * MLP * 2));
  const int nt_max = cdiv(D, 128);
  TRY(ensure(c->w_stats, Mmax * nt_max * sizeof(float2)));
  const size_t px_elem = pixel_dtype == VLY_F32 ? 4 : 2;
  for (int f0 = 0; f0 < F; f0 += CH) {
    const int fc = (F - f0) < CH ? (F - f0) : CH;
    const int M = fc * tokens;
    const int bn_d = pick_bn_m(c, D, M), nt = cdiv(D, bn_d);       // every N = D GEMM of this chunk (they exchange row statistics)
    const char* px = (const char*)pixels + (size_t)f0 * 3 * IMG * IMG * px_elem;
    bf16* x = (bf16*)out_dev + (size_t)f0 * tokens * D;
    bf16* col = (bf16*)c->w_col.p;
    TRY(with_dtype(pixel_dtype, [&](auto t) {
      using E = typename decltype(t)::type;
      return launch(c, im2col_kernel<E>, {dim3(c->num_sms * 8), dim3(256), 0, st}, (const E*)px, col, fc, IMG, P, c->kpad);
    }));
    {  // patch embedding GEMM (conv2d stride=kernel=14, no bias)
      GemmParams p = {};
      p.M = fc * NP; p.N = D; p.K = c->kpad;
      p.out = c->w_patch.p; p.ldo = D;
      TRY(launch_gemm<EPI_BIAS>(c, pick_bn_m(c, D, fc * NP), col, c->kpad, c->patch_w, c->kpad, p, st));
    }
    float2* stats = (float2*)c->w_stats.p;
    TRY(launch(c, vit_embed_ln_kernel, {dim3(M), dim3(128), 0, st}, (bf16*)c->w_patch.p, c->cls, c->pos, c->pre_g, c->pre_b, x, stats, nt,
               tokens, D, g.vit_eps));
    for (int l = 0; l < n_layers; ++l) {
      const VitLayerW& w = c->vit[l];
      {  // LN1 -> q,k,v
        GemmParams p = {};
        p.M = M; p.N = 3 * D; p.K = D;
        p.out = c->w_qkv.p; p.ldo = 3 * D;
        p.bias = w.qkv_b; p.colsum = w.qkv_cs;
        p.stats_in = stats; p.stats_in_nt = nt; p.inv_dim = 1.f / D; p.eps = g.vit_eps;
        TRY(launch_gemm<EPI_LN_BIAS>(c, pick_bn_m(c, 3 * D, M), x, D, w.wqkv, D, p, st));
      }
      TRY(launch_vit_attention(c, (bf16*)c->w_qkv.p, fc, (bf16*)c->w_ctx.p, st));
      {  // out_proj + residual
        GemmParams p = {};
        p.M = M; p.N = D; p.K = D;
        p.out = x; p.ldo = D; p.bias = w.bo; p.residual = x; p.ldr = D; p.stats_out = stats;
        TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, bn_d, (bf16*)c->w_ctx.p, D, w.wo, D, p, st));
      }
      {  // LN2 -> fc1 -> quick_gelu
        GemmParams p = {};
        p.M = M; p.N = MLP; p.K = D;
        p.out = c->w_h.p; p.ldo = MLP; p.bias = w.b1; p.colsum = w.c1;
        p.stats_in = stats; p.stats_in_nt = nt; p.inv_dim = 1.f / D; p.eps = g.vit_eps;
        TRY(launch_gemm<EPI_LN_BIAS_GELU>(c, pick_bn_m(c, MLP, M), x, D, w.w1, D, p, st));
      }
      {  // fc2 + residual (+ on the last layer of a sharded encode: push every tile to all ranks' gather buffers)
        GemmParams p = {};
        p.M = M; p.N = D; p.K = MLP;
        p.out = x; p.ldo = D; p.bias = w.b2; p.residual = x; p.ldr = D; p.stats_out = stats;
        if (gather && l == n_layers - 1) {
          p.n_peers = c->g_world;
          for (int q = 0; q < c->g_world; ++q) p.peer_out[q] = c->g_peer_buf[q];
          p.peer_tokens = tokens;
          p.peer_frame_stride = gather_frame_stride;
          p.peer_frame_off = gather_frame_off + (long long)f0 * gather_frame_stride;
        }
        TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, bn_d, (bf16*)c->w_h.p, MLP, w.w2, MLP, p, st));
      }
    }
    if (gather && n_layers == 0) return fail(VLY_ERR_INVALID, "vly_vit_encode_gather needs at least one encoder layer (select_layer != 0)");
  }
  return VLY_OK;
}

// ---- fused all-gather plumbing ----
struct PeerFlags { int* p[8]; };
__global__ void gather_signal_kernel(PeerFlags pf, int world, int rank, int epoch) {
  if ((int)threadIdx.x < world) {
    __threadfence_system();                                   // this GPU's peer stores (previous kernels) are performed
    *reinterpret_cast<volatile int*>(pf.p[threadIdx.x] + rank) = epoch;
  }
}
__global__ void gather_wait_kernel(volatile int* flags, int world, int epoch, int* timeout_flag) {
  if ((int)threadIdx.x < world) {
    const long long t0 = clock64();
    while (flags[threadIdx.x] < epoch) {
      if (clock64() - t0 > 20000000000LL) {                               // ~10 s: a peer died
        *reinterpret_cast<volatile int*>(timeout_flag) = 1;                // pinned host memory: the host sees it (gather_check_timeout)
        break;
      }
    }
    __threadfence_system();
  }
}

// A peer that never signals (dead / wedged rank) makes gather_wait_kernel give up after ~10 s and raise the context's pinned
// timeout flag.  The gather buffer then holds partially written or previous-epoch rows, so every later gather call -- and
// vly_gather_status, which callers poll after their next synchronisation -- fails loudly instead of decoding stale features.
static int gather_check_timeout(vly_ctx* c, const char* who) {
  if (c->g_timeout && *reinterpret_cast<volatile int*>(c->g_timeout.p) != 0)
    return fail(VLY_ERR_STATE, "%s: a peer rank never signalled its frame features (fused all-gather timed out); the gather "
                "buffer is stale -- the process group must be torn down", who);
  return VLY_OK;
}

extern "C" int vly_gather_status(vly_ctx* c, int* timed_out) {
  if (!c || !timed_out) return fail(VLY_ERR_INVALID, "vly_gather_status: null argument");
  *timed_out = (c->g_timeout && *reinterpret_cast<volatile int*>(c->g_timeout.p) != 0) ? 1 : 0;
  return *timed_out ? gather_check_timeout(c, "vly_gather_status") : VLY_OK;
}

extern "C" int vly_gather_create(vly_ctx* c, int64_t rows_total, void** local_buf, void* handle_out) {
  if (!c || rows_total <= 0 || !local_buf || !handle_out) return fail(VLY_ERR_INVALID, "vly_gather_create: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  if (c->g_buf) return fail(VLY_ERR_STATE, "vly_gather_create: a gather buffer already exists for this context");
  const size_t data = (((size_t)rows_total * c->cfg.vit_hidden * 2) + 255) & ~size_t(255);
  Owned<bf16> buf;
  TRY(buf.alloc(data + 256));
  CK(cudaMemset(buf, 0, data + 256));
  if (!c->g_timeout) {
    TRY(c->g_timeout.alloc(sizeof(int), true));
    *c->g_timeout = 0;
  }
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, buf));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  memcpy(handle_out, &h, 64);
  *local_buf = buf;
  c->g_buf = std::move(buf);
  c->g_rows = rows_total;
  c->g_flags = (int*)((char*)c->g_buf.p + data);
  return VLY_OK;
}

extern "C" int vly_gather_open_peers(vly_ctx* c, const void* handles, int world, int rank) {
  if (!c || !handles || world < 1 || world > 8 || rank < 0 || rank >= world) return fail(VLY_ERR_INVALID, "vly_gather_open_peers: bad argument (world <= 8)");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->g_buf) return fail(VLY_ERR_STATE, "vly_gather_open_peers: call vly_gather_create first");
  CK(cudaSetDevice(c->cfg.device));
  const size_t data = (((size_t)c->g_rows * c->cfg.vit_hidden * 2) + 255) & ~size_t(255);
  for (int q = 0; q < world; ++q) {
    void* base = nullptr;
    if (q == rank) base = c->g_buf;
    else {
      cudaIpcMemHandle_t h;
      memcpy(&h, (const char*)handles + (size_t)q * 64, 64);
      CK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    }
    c->g_peer_buf[q] = (bf16*)base;
    c->g_peer_flags[q] = (int*)((char*)base + data);
  }
  c->g_world = world;
  c->g_rank = rank;
  return VLY_OK;
}

// Tell every rank that this rank has finished reading the current epoch's gather buffer (enqueue after the consumer kernels).
extern "C" int vly_gather_release(vly_ctx* c, void* stream) {
  if (!c) return fail(VLY_ERR_INVALID, "null");
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->g_world == 0) return fail(VLY_ERR_STATE, "vly_gather_release: no gather group");
  TRY(gather_check_timeout(c, "vly_gather_release"));
  CK(cudaSetDevice(c->cfg.device));
  PeerFlags pf;
  for (int q = 0; q < 8; ++q) pf.p[q] = c->g_peer_flags[q] ? c->g_peer_flags[q] + 8 : nullptr;
  return launch(c, gather_signal_kernel, {dim3(1), dim3(32), 0, (cudaStream_t)stream}, pf, c->g_world, c->g_rank, c->g_epoch);
}

extern "C" int vly_vit_encode_gather(vly_ctx* c, const void* pixels, int pixel_dtype, int F, int frame_offset, int select_layer, void* stream) {
  return vly_vit_encode_gather_strided(c, pixels, pixel_dtype, F, frame_offset, 1, select_layer, stream);
}

extern "C" int vly_vit_encode_gather_strided(vly_ctx* c, const void* pixels, int pixel_dtype, int F, int frame_offset, int frame_stride,
                                             int select_layer, void* stream) {
  if (!c || F < 0 || frame_offset < 0 || frame_stride < 1 || (F > 0 && !pixels)) return fail(VLY_ERR_INVALID, "vly_vit_encode_gather: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->finalized || !c->has_vit) return fail(VLY_ERR_STATE, "vly_vit_encode_gather: vision weights not loaded/finalised");
  if (c->g_world == 0) return fail(VLY_ERR_STATE, "vly_vit_encode_gather: call vly_gather_create / vly_gather_open_peers first");
  const int tokens = (c->cfg.vit_image / c->cfg.vit_patch) * (c->cfg.vit_image / c->cfg.vit_patch) + 1;
  if (F > 0 && ((long long)frame_offset + (long long)(F - 1) * frame_stride + 1) * tokens > c->g_rows)
    return fail(VLY_ERR_INVALID, "vly_vit_encode_gather: frames %d + i*%d, i < %d exceed the gather buffer", frame_offset, frame_stride, F);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  TRY(gather_check_timeout(c, "vly_vit_encode_gather"));
  int* timeout_flag = c->g_timeout;
  if (c->g_epoch > 0) {   // every rank must have finished READING the previous epoch before anyone overwrites its buffer
    TRY(launch(c, gather_wait_kernel, {dim3(1), dim3(32), 0, st}, c->g_flags + 8, c->g_world, c->g_epoch, timeout_flag));
  }
  if (F > 0) {
    TRY(ensure(c->w_xlocal, (size_t)F * tokens * c->cfg.vit_hidden * 2));       // local residual stream (scratch)
    TRY(vit_encode_impl(c, pixels, pixel_dtype, F, select_layer, c->w_xlocal.p, stream, true, frame_offset, frame_stride));
  }
  // flag exchange: every rank tells every rank "my rows are in your buffer", then waits for all of them
  const int epoch = ++c->g_epoch;
  PeerFlags pf;
  for (int q = 0; q < 8; ++q) pf.p[q] = c->g_peer_flags[q];
  TRY(launch(c, gather_signal_kernel, {dim3(1), dim3(32), 0, st}, pf, c->g_world, c->g_rank, epoch));
  return launch(c, gather_wait_kernel, {dim3(1), dim3(32), 0, st}, c->g_flags, c->g_world, epoch, timeout_flag);
}

extern "C" int vly_project(vly_ctx* c, const void* feats, int64_t rows, void* out, void* stream) {
  if (!c || !feats || !out || rows <= 0) return fail(VLY_ERR_INVALID, "vly_project: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->finalized || !c->proj_w) return fail(VLY_ERR_STATE, "vly_project: mm_projector not loaded");
  CK(cudaSetDevice(c->cfg.device));
  GemmParams p = {};
  p.M = (int)rows; p.N = c->cfg.hidden_size; p.K = c->cfg.vit_hidden;
  p.out = out; p.ldo = c->cfg.hidden_size; p.bias = c->proj_b;
  return launch_gemm<EPI_BIAS>(c, pick_bn(p.N), (const bf16*)feats, p.K, c->proj_w, p.K, p, (cudaStream_t)stream);
}

// 'max' and 'temporal_transformer' act on the PROJECTED tokens (they do not commute with the projector): project all
// T*257 rows of one video at a time, then pool.  valley_model.py:208-209, :123-133.
static int pool_project_after(vly_ctx* c, const bf16* feats, int n_videos, int T, bf16* vis_rows, cudaStream_t st) {
  const vly_config& g = c->cfg;
  const int D = g.vit_hidden, H = g.hidden_size, tokens = (g.vit_image / g.vit_patch) * (g.vit_image / g.vit_patch) + 1;
  const int NP = tokens - 1, rows_out = NP + T, nhead = 8;
  const vly_ctx::DeltaW& w = c->delta;
  const bool tr = g.patch_pooling_method == VLY_POOL_TEMPORAL_TRANSFORMER;
  if (tr) {
    if (!w.in_w) return fail(VLY_ERR_STATE, "vly_pool_project: transformer_delta_encoder weights not loaded");
    if (T > 64 || T > w.max_pos) return fail(VLY_ERR_INVALID, "vly_pool_project: temporal transformer supports at most %d frames (got %d)", w.max_pos < 64 ? w.max_pos : 64, T);
    if ((H / nhead) % 64) return fail(VLY_ERR_INVALID, "vly_pool_project: hidden_size / 8 must be a multiple of 64");
  }
  TRY(ensure(c->w_pall, (size_t)T * tokens * H * 2));
  if (tr) {
    TRY(ensure(c->w_xp, (size_t)T * NP * H * 2));
    TRY(ensure(c->w_dkv, (size_t)T * NP * 2 * H * 2));
    TRY(ensure(c->w_dq, (size_t)NP * H * 2));
    TRY(ensure(c->w_datt, (size_t)NP * H * 2));
    TRY(ensure(c->w_dx1, (size_t)NP * H * 2));
    TRY(ensure(c->w_df1, (size_t)NP * w.ffn * 2));
    TRY(ensure(c->w_dx2, (size_t)NP * H * 2));
  }
  bf16* P = (bf16*)c->w_pall.p;
  for (int v = 0; v < n_videos; ++v) {
    bf16* vis = vis_rows + (size_t)v * rows_out * H;
    {  // mm_projector over every token of the video (valley_model.py:187-190)
      GemmParams p = {};
      p.M = T * tokens; p.N = H; p.K = D; p.out = P; p.ldo = H; p.bias = c->proj_b;
      TRY(launch_gemm<EPI_BIAS>(c, pick_bn_m(c, H, p.M), feats + (size_t)v * T * tokens * D, D, c->proj_w, D, p, st));
    }
    const LaunchCfg two_per_sm = {dim3(c->num_sms * 2), dim3(256), 0, st};
    if (!tr) {
      TRY(launch(c, temporal_max_kernel, two_per_sm, P, vis, T, tokens, H));
      continue;
    }
    bf16 *Xp = (bf16*)c->w_xp.p, *KV = (bf16*)c->w_dkv.p, *Q = (bf16*)c->w_dq.p, *att = (bf16*)c->w_datt.p;
    bf16 *X1 = (bf16*)c->w_dx1.p, *F1 = (bf16*)c->w_df1.p, *X2 = (bf16*)c->w_dx2.p;
    const bf16* Xlast = Xp + (size_t)(T - 1) * NP * H;          // rows of the last frame: the only queries that are used (:130)
    TRY(launch(c, delta_add_pos_kernel, two_per_sm, P, w.pos, Xp, T, tokens, H));
    GemmParams p = {};
    p.M = T * NP; p.N = 2 * H; p.K = H; p.out = KV; p.ldo = 2 * H; p.bias = w.in_b + H;          // k | v rows of in_proj
    TRY(launch_gemm<EPI_BIAS>(c, pick_bn_m(c, p.N, p.M), Xp, H, w.in_w + (size_t)H * H, H, p, st));
    p = {};
    p.M = NP; p.N = H; p.K = H; p.out = Q; p.ldo = H; p.bias = w.in_b;
    TRY(launch_gemm<EPI_BIAS>(c, pick_bn_m(c, p.N, p.M), Xlast, H, w.in_w, H, p, st));
    TRY(launch(c, delta_attention_kernel, {dim3(NP), dim3(nhead * 32), 0, st}, Q, KV, att, T, NP, H, nhead));
    p = {};
    p.M = NP; p.N = H; p.K = H; p.out = X1; p.ldo = H; p.bias = w.out_b; p.residual = Xlast; p.ldr = H;
    TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, pick_bn_m(c, p.N, p.M), att, H, w.out_w, H, p, st));
    TRY(launch(c, layernorm_rows_kernel, {dim3(NP), dim3(256), 0, st}, X1, w.n1_g, w.n1_b, X1, H, 1e-5f));
    p = {};
    p.M = NP; p.N = w.ffn; p.K = H; p.out = F1; p.ldo = w.ffn; p.bias = w.l1_b;
    TRY(launch_gemm<EPI_BIAS>(c, pick_bn_m(c, p.N, p.M), X1, H, w.l1_w, H, p, st));
    TRY(launch(c, relu_inplace_kernel, {dim3(c->num_sms), dim3(256), 0, st}, F1, (long long)NP * w.ffn / 8));
    p = {};
    p.M = NP; p.N = H; p.K = w.ffn; p.out = X2; p.ldo = H; p.bias = w.l2_b; p.residual = X1; p.ldr = H;
    TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, pick_bn_m(c, p.N, p.M), F1, w.ffn, w.l2_w, w.ffn, p, st));
    TRY(launch(c, layernorm_rows_kernel, {dim3(NP), dim3(256), 0, st}, X2, w.n2_g, w.n2_b, X2, H, 1e-5f));
    TRY(launch(c, delta_finish_kernel, two_per_sm, P, X2, vis, T, tokens, H));
  }
  return VLY_OK;
}

extern "C" int vly_pool_project(vly_ctx* c, const void* feats, int n_videos, int T, void* vis_rows, void* stream) {
  if (!c || !feats || !vis_rows || n_videos <= 0 || T <= 0) return fail(VLY_ERR_INVALID, "vly_pool_project: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->finalized || !c->proj_w) return fail(VLY_ERR_STATE, "vly_pool_project: mm_projector not loaded");
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const vly_config& g = c->cfg;
  const int D = g.vit_hidden, tokens = (g.vit_image / g.vit_patch) * (g.vit_image / g.vit_patch) + 1;
  const int rows = tokens - 1 + T;
  if (g.patch_pooling_method == VLY_POOL_MAX || g.patch_pooling_method == VLY_POOL_TEMPORAL_TRANSFORMER)
    return pool_project_after(c, (const bf16*)feats, n_videos, T, (bf16*)vis_rows, st);
  TRY(ensure(c->w_pool, (size_t)n_videos * rows * D * 2));
  if (g.patch_pooling_method == VLY_POOL_TEMPORAL_IMPORTANCE) {
    // softmax_t(w . flatten(proj(x_t))) weights: scores straight from the ViT features through the folded U (pooling_kernels.cuh)
    if (!c->pool_U) return fail(VLY_ERR_STATE, "vly_pool_project: model.pooling_layer.weight not loaded");
    TRY(ensure(c->w_score, (size_t)n_videos * T * 4));
    TRY(launch(c, importance_score_kernel, {dim3(T, n_videos), dim3(256), 0, st}, (const bf16*)feats, c->pool_U, (float*)c->w_score.p, T,
               tokens, D));
    TRY(launch(c, weighted_pool_kernel, {dim3(c->num_sms * 4), dim3(256), 0, st}, (const bf16*)feats, (const float*)c->w_score.p,
               (bf16*)c->w_pool.p, n_videos, T, tokens, D));
  } else {
    TRY(launch(c, temporal_pool_kernel, {dim3(c->num_sms * 4), dim3(256), 0, st}, (const bf16*)feats, (bf16*)c->w_pool.p, n_videos, T,
               tokens, D));
  }
  GemmParams p = {};
  p.M = n_videos * rows; p.N = g.hidden_size; p.K = D;
  p.out = vis_rows; p.ldo = g.hidden_size; p.bias = c->proj_b;
  return launch_gemm<EPI_BIAS>(c, pick_bn(p.N), (bf16*)c->w_pool.p, D, c->proj_w, D, p, st);
}

extern "C" int vly_embed_splice(vly_ctx* c, const int64_t* ids, const int32_t* src_map, const int32_t* img_idx, const void* vis_rows,
                                int rows_per_img, int B, int S, void* out, void* stream) {
  if (!c || !ids || !out || B <= 0 || S <= 0) return fail(VLY_ERR_INVALID, "vly_embed_splice: bad argument");
  if (src_map && (!img_idx || !vis_rows)) return fail(VLY_ERR_INVALID, "vly_embed_splice: src_map given without img_idx / vis_rows");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->finalized || !c->has_llm) return fail(VLY_ERR_STATE, "vly_embed_splice: LLM weights not loaded");
  CK(cudaSetDevice(c->cfg.device));
  return launch(c, embed_splice_kernel, {dim3(B * S), dim3(128), 0, (cudaStream_t)stream}, (const long long*)ids, src_map, img_idx, c->embed,
                (const bf16*)vis_rows, rows_per_img, (bf16*)out, nullptr, 0, S, c->cfg.hidden_size, c->cfg.vocab_size);
}

// ------------------------------------------------------------------------------------------------
// KV cache
// ------------------------------------------------------------------------------------------------
// Shared-memory budget of the persistent decode kernel (decode_mega.cuh): activation block + barriers / handoff slots, the
// rest is the weight ring.
static void mega_smem_layout(const vly_config& g, int bmax, size_t* x_bytes, size_t* misc) {
  const bool tc = bmax > 1;
  const int kmax = g.intermediate_size > g.hidden_size ? g.intermediate_size : g.hidden_size;
  const size_t xs_stride_b = tc ? (size_t)(((kmax * 2 + 127) & ~127) + MegaCfg::PAD_TC) : (size_t)kmax * 2;
  *x_bytes = ((size_t)bmax * xs_stride_b + 127) & ~size_t(127);
  const int nv = (tc ? MegaCfg::ROWS_TC : MegaCfg::ROWS) * bmax;
  *misc = (2 * MegaCfg::MAX_STAGES + 2 * MegaCfg::RED_SLOTS + 2) * 8 + (size_t)MegaCfg::RED_SLOTS * 16 * nv * 4 + (3 + 16) * bmax * 4 + 256;
}
static const size_t kMegaSmem = 226 * 1024;
static const int kMegaDbgCounters = 1024 * 8;    // capacity of vly_kv::dbg: 32 per CTA

// Overrides of the persistent decode kernel's launch plan, for tuning it on the GPU at hand (tools/bench_decode.py --configs).
// They are read from the environment by read_decode_settings() and nowhere else, once per KV cache when vly_kv_create
// builds the plan: a cache keeps the settings it was created with, whatever the environment says later.  Unset (0) keeps
// the library's choice.
struct DecodeSettings {
  int stage_kb = 0;         // VLY_MEGA_STAGE_KB: target ring stage size in KB (pick_phase_geometry)
  int rows = 0;             // VLY_MEGA_ROWS: weight rows per work unit (pick_phase_geometry)
  int inflight_kb = 100;    // VLY_MEGA_INFLIGHT_KB: KB of bulk copies kept in flight per SM, per phase (PhaseDesc::inflight)
  int stages = 0;           // VLY_MEGA_STAGES: ring depth cap (default 4); below 2 no cache can be created
  int inflight = 0;         // VLY_MEGA_INFLIGHT: cap on the stages in flight over all phases (default: the ring depth)
  int attn_ikeys = 0;       // VLY_ATTN_IKEYS: keys per attention work item, 16..256 in steps of 16 (default: by shape)
  int l2_hint = 1;          // VLY_MEGA_L2_HINT=0: the weight copies carry no L2::evict_first policy
  bool dbg = false;         // VLY_MEGA_DBG (any value): the kernel fills per-CTA cycle counters (vly_kv_debug_counters)
};
static DecodeSettings read_decode_settings() {
  auto num = [](const char* name, int unset) {
    const char* v = getenv(name);
    return v ? atoi(v) : unset;
  };
  DecodeSettings s;
  s.stage_kb = num("VLY_MEGA_STAGE_KB", 0);
  s.rows = num("VLY_MEGA_ROWS", 0);
  s.inflight_kb = num("VLY_MEGA_INFLIGHT_KB", 100);
  s.stages = num("VLY_MEGA_STAGES", 0);
  s.inflight = num("VLY_MEGA_INFLIGHT", 0);
  const int ik = num("VLY_ATTN_IKEYS", 0);
  s.attn_ikeys = (ik >= 16 && ik <= 256 && ik % 16 == 0) ? ik : 0;
  const char* hint = getenv("VLY_MEGA_L2_HINT");
  s.l2_hint = (hint && *hint) ? atoi(hint) != 0 : 1;
  s.dbg = getenv("VLY_MEGA_DBG") != nullptr;
  return s;
}

// Ring geometry of one weight phase of the persistent decode kernel: rows per work unit and columns per stage.  The rules:
//   * HBM streams best with a bounded number of bytes of bulk copies outstanding per SM (~100 KB): fewer leave it idle, more
//     only lengthen the queues;
//   * a bulk copy should be a few KB (>= 3-4 KB): many small row copies stream slower than fewer large ones;
//   * the consumers need a few hundred cycles to hand a landed stage back, which takes that stage out of flight: a ring of 3
//     large stages loses more to this than one of 5 smaller stages, so the target is a stage of 1/5 of the ring budget
//     (but 16-48 KB), cut so that K divides into EQUAL stages (no short tail stage);
//   * rows: the candidate (max, max / 2) that satisfies the copy-size rule, then the one whose work units balance better over
//     the SMs -- the phase lasts as long as its most loaded CTA: N = 5120 is 5 rounds of 8 rows (40) but 9 rounds of 4 (36).
// DecodeSettings::stage_kb / ::rows override.
static void pick_phase_geometry(const DecodeSettings& s, int bmax, size_t ring_budget, int N, int K, int num_sms, int* rows_out,
                                int* kc_out) {
  const bool tc = bmax > 1;
  const int max_rows = tc ? MegaCfg::ROWS_TC : MegaCfg::ROWS;
  const int pad = tc ? MegaCfg::PAD_TC : 0, gran = tc ? 64 : 8;
  // stage size: CUDA-core path 4 slots of ~41 KB (fewer, larger slots put more bytes in flight; more slots make the grid barriers
  // queue behind the extra prefetch traffic); tensor-core path 8 rows x ~2048 columns
  size_t target = s.stage_kb > 0 ? (size_t)s.stage_kb * 1024 : (tc ? 33 * 1024 + 512 : 41 * 1024);
  if (target > ring_budget / 2) target = ring_budget / 2;
  if (target < 8 * 1024) target = 8 * 1024;
  auto kc_for = [&](int rows) {
    const int cap = (int)((target / rows - pad) / 2);
    const int ns = cdiv(K, cap > gran ? cap : gran);
    int kc = cdiv(cdiv(K, ns), gran) * gran;
    return kc > K ? cdiv(K, gran) * gran : kc;
  };
  int rows = max_rows;
  if (s.rows > 0) rows = s.rows > max_rows ? max_rows : s.rows;
  else {
    if (kc_for(rows) * 2 < 3072 && K * 2 >= 3072) rows = max_rows / 2;            // keep every bulk copy >= 3 KB
    if (rows == max_rows && !tc) {        // (tensor-core path: half-filled HMMAs cost more than the imbalance they would remove)
      const long long load_full = (long long)cdiv(cdiv(N, max_rows), num_sms) * max_rows;
      const long long load_half = (long long)cdiv(cdiv(N, max_rows / 2), num_sms) * (max_rows / 2);
      if (load_half * 100 < load_full * 97) rows = max_rows / 2;                  // at least 3 % shorter critical path
    }
  }
  *rows_out = rows;
  *kc_out = kc_for(rows);
}

// The complete launch of the persistent decode-step kernel for kv (B <= 4): phase table, ring geometry and depth, shared memory
// and StepParams.  Everything it depends on -- shapes, weight and cache pointers, settings -- is fixed once the cache exists.
static int plan_decode_mega(vly_ctx* c, vly_kv* kv, const DecodeSettings& s) {
  const vly_config& g = c->cfg;
  const int B = kv->B, H = g.hidden_size, nH = g.num_attention_heads, I = g.intermediate_size, V = g.vocab_size;
  const int bmax = bmax_of(B);
  const int pad = bmax > 1 ? MegaCfg::PAD_TC : 0;
  size_t x_bytes, misc;
  mega_smem_layout(g, bmax, &x_bytes, &misc);
  const size_t ring_budget = kMegaSmem > x_bytes + misc ? kMegaSmem - x_bytes - misc : 0;
  // phase table: execution order of one step
  std::vector<PhaseDesc> ph;
  int stage_bytes = 0;
  auto add = [&](PhaseDesc d) {
    d.rows = d.kc = 0;
    if (d.type != PH_ATTN) {
      pick_phase_geometry(s, bmax, ring_budget, d.N, d.K, c->num_sms, &d.rows, &d.kc);
      const int sb = d.rows * (d.kc * 2 + pad);
      if (sb > stage_bytes) stage_bytes = sb;
    }
    ph.push_back(d);
  };
  for (int l = 0; l < g.num_hidden_layers; ++l) {
    const LlamaLayerW& w = c->layers[l];
    PhaseDesc d = {};
    d.layer = l; d.kcache = kv->k_layer(l); d.vcache = kv->v_layer(l);
    d.type = PH_QKV; d.N = 3 * H; d.K = H; d.W = w.wqkv; d.x_in = kv->x; d.out = kv->q; add(d);
    d.type = PH_ATTN; d.N = 0; d.K = 0; d.W = nullptr; d.x_in = nullptr; d.out = kv->attn; add(d);
    d.type = PH_OPROJ; d.N = H; d.K = H; d.W = w.wo; d.x_in = kv->attn; d.out = kv->x; add(d);
    d.type = PH_GATEUP; d.N = 2 * I; d.K = H; d.W = w.wgu; d.x_in = kv->x; d.out = kv->hb; add(d);
    d.type = PH_DOWN; d.N = H; d.K = I; d.W = w.wdown; d.x_in = kv->hb; d.out = kv->x; add(d);
  }
  {
    PhaseDesc d = {};
    d.type = PH_LOGITS; d.N = V; d.K = H; d.W = c->lm_head; d.x_in = kv->x; d.out = nullptr; add(d);
  }
  stage_bytes = (stage_bytes + 127) & ~127;
  // Stages of this phase's size kept in flight: ~100 KB of bulk copies outstanding per SM saturate HBM; every byte beyond
  // that only lengthens the queues the latency-critical traffic (grid barrier, activation staging, attention) waits in --
  // measured: 128 KB in flight made every barrier ~1 us slower at an unchanged streaming rate.  (On the H100, 400 W, 13B at
  // B = 4: an L2 prefetch running 64-192 KB per SM ahead of the ring made the step 0.7-1.5 ms slower.)  The ring may hold more slots
  // than are in flight: they absorb the consumers' hand-back latency.
  for (PhaseDesc& q : ph) {
    if (q.type == PH_ATTN) continue;
    const int sb = q.rows * (q.kc * 2 + pad);
    q.inflight = (s.inflight_kb * 1024 + sb / 2) / sb;
    if (q.inflight < 2) q.inflight = 2;
  }
  // depth of the ring: what fits next to the activation block, at most 4 (deeper rings made every grid barrier slower, see
  // pick_phase_geometry)
  int n_stages = (int)(((long long)kMegaSmem - (long long)x_bytes - (long long)misc) / (long long)stage_bytes);
  if (n_stages > MegaCfg::MAX_STAGES) n_stages = MegaCfg::MAX_STAGES;
  const int cap = s.stages > 0 ? s.stages : 4;
  if (n_stages > cap) n_stages = cap;
  if (n_stages < 2)
    return fail(VLY_ERR_INVALID, "vly_kv_create: activations (B=%d, K=%d) leave no room for the weight ring (%d stages, at least 2 needed)",
                B, std::max(I, H), n_stages);
  if (s.dbg) {
    fprintf(stderr, "[vly] decode ring: B=%d x=%zu B, ring budget %zu B, slot %d B, %d slots fit, %d used;", B, x_bytes, ring_budget,
            stage_bytes, (int)(ring_budget / stage_bytes), n_stages);
    for (int i = 0; i < 5 && i < (int)ph.size(); ++i)
      if (ph[i].type != PH_ATTN) fprintf(stderr, " type%d N=%d K=%d rows=%d kc=%d inflight=%d;", ph[i].type, ph[i].N, ph[i].K, ph[i].rows, ph[i].kc, ph[i].inflight);
    fprintf(stderr, " logits rows=%d kc=%d\n", ph.back().rows, ph.back().kc);
    TRY(kv->dbg.alloc(kMegaDbgCounters * sizeof(long long)));
  }
  TRY(kv->d_phases.alloc(ph.size() * sizeof(PhaseDesc)));
  CK(cudaMemcpy(kv->d_phases, ph.data(), ph.size() * sizeof(PhaseDesc), cudaMemcpyHostToDevice));

  StepParams& p = kv->mega;
  p = {};
  p.phases = kv->d_phases; p.n_phases = (int)ph.size();
  p.B = B; p.H = H; p.nH = nH; p.Smax = kv->Smax; p.V = V;
  p.Kmax = std::max(I, H);
  p.eps = g.rms_norm_eps; p.scale_log2e = 0.08838834764831845f * 1.4426950408889634f;
  p.rope = c->rope; p.seq_len = kv->d_len; p.step = kv->d_step; p.embed = c->embed; p.tokens_in = kv->cur_tokens;
  p.x = kv->x; p.q = kv->q; p.attn = kv->attn;
  p.part_o = kv->part_o; p.part_ml = kv->part_ml; p.attn_counters = kv->counters; p.nsplit = kv->nsplit;
  p.key_bits = kv->key_bits; p.mask_words = kv->mask_words();
  p.logits = kv->logits; p.part_val = kv->part_val; p.part_idx = kv->part_idx;
  p.next_tokens = kv->cur_tokens; p.out_tokens = kv->gen_tokens; p.out_stride = kv->Smax;
  p.sample = kv->d_sample;
  p.grid_counter = kv->counters + (size_t)B * nH + 1;
  p.grid_epoch = p.grid_counter + 1;
  p.n_grid_syncs = p.n_phases + 1;               // one per phase + the embedding phase
  p.attn_ikeys = s.attn_ikeys;
  p.n_stages = n_stages;
  p.stage_bytes = stage_bytes;
  p.n_inflight = s.inflight > 0 ? s.inflight : n_stages;      // (PhaseDesc::inflight is the per-phase value)
  if (p.n_inflight > n_stages) p.n_inflight = n_stages;
  p.l2_hint = s.l2_hint;
  p.dbg = kv->dbg;
  kv->mega_smem = (size_t)n_stages * stage_bytes + x_bytes + misc;
  return VLY_OK;
}

extern "C" int vly_kv_create(vly_ctx* c, int batch, int max_seq, vly_kv** out) {
  if (!c || !out || batch <= 0 || max_seq <= 0) return fail(VLY_ERR_INVALID, "vly_kv_create: bad argument");
  if (!c->finalized || !c->has_llm) return fail(VLY_ERR_STATE, "vly_kv_create: LLM weights not finalised");
  if (max_seq > c->cfg.max_position_embeddings) return fail(VLY_ERR_INVALID, "vly_kv_create: max_seq %d > max_position_embeddings %d", max_seq, c->cfg.max_position_embeddings);
  CK(cudaSetDevice(c->cfg.device));
  const vly_config& g = c->cfg;
  auto kv = std::make_unique<vly_kv>();
  kv->ctx = c;
  kv->B = batch;
  kv->Smax = (max_seq + 127) / 128 * 128;   // whole 128-key TMA tiles
  const int H = g.hidden_size, nH = g.num_attention_heads, I = g.intermediate_size, V = g.vocab_size, L = g.num_hidden_layers;
  const size_t cache_elems = (size_t)L * kv->layer_stride();
  TRY(kv->cache.alloc(cache_elems * 2));
  CK(cudaMemset(kv->cache, 0, cache_elems * 2));   // padded keys must be finite: P(=0) * V(pad) must stay 0
  kv->nsplit = kv->Smax / MegaCfg::ATTN_KEYS_MIN;   // capacity of the split dimension: the persistent kernel uses 16/32-key items,
                                                    // the per-op kernel fixed 64-key splits (it only touches the first Smax / 64 slots)
  TRY(kv->d_len.alloc(8));
  TRY(kv->h_len.alloc(sizeof(int), true));
  CK(cudaEventCreateWithFlags(&kv->len_event, cudaEventDisableTiming));
  kv->d_step = kv->d_len + 1;
  CK(cudaMemset(kv->d_len, 0, 8));
  // (at least 8 rows, rows >= batch stay zero)
  const size_t act_rows = batch < 8 ? 8 : batch;
  TRY(kv->x.alloc(act_rows * H * 2));
  TRY(kv->q.alloc(act_rows * H * 2));
  TRY(kv->attn.alloc(act_rows * H * 2));
  TRY(kv->hb.alloc(act_rows * I * 2));
  CK(cudaMemset(kv->x, 0, act_rows * H * 2));
  CK(cudaMemset(kv->attn, 0, act_rows * H * 2));
  CK(cudaMemset(kv->hb, 0, act_rows * I * 2));
  TRY(kv->part_o.alloc((size_t)batch * nH * kv->nsplit * 128 * 4));
  TRY(kv->part_ml.alloc((size_t)batch * nH * kv->nsplit * sizeof(float2)));
  TRY(kv->counters.alloc(((size_t)batch * nH + 4) * 4));
  CK(cudaMemset(kv->counters, 0, ((size_t)batch * nH + 4) * 4));
  TRY(kv->part_val.alloc((size_t)batch * c->num_sms * 4));   // every arg-max kernel runs at most one CTA per SM
  TRY(kv->part_idx.alloc((size_t)batch * c->num_sms * 4));
  TRY(kv->logits.alloc((size_t)batch * V * 4));
  TRY(kv->cur_tokens.alloc((size_t)batch * 8));
  TRY(kv->gen_tokens.alloc((size_t)batch * kv->Smax * 8));
  TRY(kv->d_sample.alloc(sizeof(SampleState)));
  {
    const SampleState s0 = {};
    CK(cudaMemcpy(kv->d_sample, &s0, sizeof(s0), cudaMemcpyHostToDevice));
  }
  TRY(kv->key_bits.alloc((size_t)batch * kv->mask_words() * 4));
  CK(cudaMemset(kv->key_bits, 0xff, (size_t)batch * kv->mask_words() * 4));
  if (batch <= 4) TRY(plan_decode_mega(c, kv.get(), read_decode_settings()));
  *out = kv.release();
  return VLY_OK;
}

extern "C" int vly_kv_decode_kernel(vly_kv* kv, char* name, int cap) {
  if (!kv || !name || cap <= 0) return fail(VLY_ERR_INVALID, "vly_kv_decode_kernel: bad argument");
  if (kv->B <= 4) snprintf(name, (size_t)cap, "decode_step_kernel<%d>", bmax_of(kv->B));
  else snprintf(name, (size_t)cap, "per-op TMA-ring decode kernels");
  return VLY_OK;
}

extern "C" void vly_kv_destroy(vly_kv* kv) {
  if (!kv) return;
  cudaSetDevice(kv->ctx->cfg.device);
  delete kv;
}

extern "C" int vly_kv_seq_len(vly_kv* kv, int* out) {
  if (!kv || !out) return fail(VLY_ERR_INVALID, "null");
  TRY(sync_len(kv));
  *out = kv->host_len;
  return VLY_OK;
}

extern "C" int vly_kv_reset(vly_kv* kv, void* stream) {
  if (!kv) return fail(VLY_ERR_INVALID, "null");
  CK(cudaSetDevice(kv->ctx->cfg.device));
  kv->host_len = 0;
  kv->len_dirty = false;
  CK(cudaMemsetAsync(kv->d_len, 0, 8, (cudaStream_t)stream));
  if (kv->masked) {
    CK(cudaMemsetAsync(kv->key_bits, 0xff, (size_t)kv->B * kv->mask_words() * 4, (cudaStream_t)stream));
    kv->masked = false;
  }
  return VLY_OK;
}

// one thread per 32-key word: bit i = mask[b, 32w+i] != 0; positions >= len stay attendable
__global__ void pack_key_mask_kernel(const uint8_t* __restrict__ mask, int len, int words, uint32_t* __restrict__ bits) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (w >= words) return;
  uint32_t v = 0;
  for (int i = 0; i < 32; ++i) {
    const int k = w * 32 + i;
    v |= uint32_t(k >= len || mask[(size_t)b * len + k] != 0) << i;
  }
  bits[(size_t)b * words + w] = v;
}

extern "C" int vly_kv_set_key_mask(vly_kv* kv, const uint8_t* mask_dev, int len, void* stream) {
  if (!kv || len < 0 || len > kv->Smax || (len > 0 && !mask_dev)) return fail(VLY_ERR_INVALID, "vly_kv_set_key_mask: bad argument (len %d, capacity %d)", len, kv ? kv->Smax : 0);
  std::lock_guard<std::mutex> lk(kv->ctx->mu);
  CK(cudaSetDevice(kv->ctx->cfg.device));
  const int words = kv->mask_words();
  if (len == 0) {
    CK(cudaMemsetAsync(kv->key_bits, 0xff, (size_t)kv->B * words * 4, (cudaStream_t)stream));
    kv->masked = false;
    return VLY_OK;
  }
  TRY(launch(kv->ctx, pack_key_mask_kernel, {dim3(cdiv(words, 128), kv->B), dim3(128), 0, (cudaStream_t)stream}, mask_dev, len, words,
             kv->key_bits));
  kv->masked = true;
  return VLY_OK;
}

extern "C" int vly_kv_export(vly_ctx* c, vly_kv* kv, int layer, int which, void* out, void* stream) {
  if (!c || !kv || !out || layer < 0 || layer >= c->cfg.num_hidden_layers || (which != 0 && which != 1)) return fail(VLY_ERR_INVALID, "vly_kv_export: bad argument");
  if (kv->ctx != c) return fail(VLY_ERR_INVALID, "vly_kv_export: the kv cache belongs to another context");
  TRY(sync_len(kv));     // (before the lock: it waits on this cache's last generate only)
  if (kv->host_len == 0) return VLY_OK;
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  return launch(c, kv_export_kernel, {dim3(kv->host_len, kv->B * c->cfg.num_attention_heads), dim3(128), 0, (cudaStream_t)stream},
                which ? kv->v_layer(layer) : kv->k_layer(layer), (bf16*)out, kv->Smax, kv->host_len, which == 0);
}

// ------------------------------------------------------------------------------------------------
// decode-side launchers
// ------------------------------------------------------------------------------------------------
// ---- per-op decode launchers (TMA ring + programmatic dependent launch) ----
template <int MODE>
static int launch_gemv_ring(vly_ctx* c, GemvParams p, bool pdl, cudaStream_t st) {
  const int bmax = bmax_of(p.B);
  if (p.B > 4) return fail(VLY_ERR_INVALID, "gemv: batch %d > 4 per call (callers split the batch)", p.B);
  if (p.ldx == 0) p.ldx = p.K;
  const size_t x_bytes = (((size_t)bmax * p.K * 2) + 15) & ~size_t(15);
  const size_t misc = 4096 + 128;
  int n_stages = (int)((113 * 1024 - (long long)x_bytes - (long long)misc) / RingCfg::STAGE_BYTES);   // two kernels co-resident per SM
  if (n_stages >= 3) n_stages = n_stages > 6 ? 6 : n_stages;
  else {
    n_stages = (int)((225 * 1024 - (long long)x_bytes - (long long)misc) / RingCfg::STAGE_BYTES);
    if (n_stages > RingCfg::MAX_STAGES) n_stages = RingCfg::MAX_STAGES;
    if (n_stages < 1) return fail(VLY_ERR_INVALID, "gemv: activation rows (B=%d, K=%d) do not fit in shared memory", p.B, p.K);
  }
  const size_t smem = (size_t)n_stages * RingCfg::STAGE_BYTES + x_bytes + misc;
  const int groups = (p.N + RingCfg::ROWS - 1) / RingCfg::ROWS;
  const LaunchCfg l = {dim3(groups < c->num_sms ? groups : c->num_sms), dim3(RingCfg::THREADS), smem, st, pdl, true};
  return with_bmax(p.B, [&](auto bm) { return launch(c, gemv_ring_kernel<decltype(bm)::value, MODE>, l, p, n_stages); });
}

// decode attention over the newest key *p.seq_len and the keys before it: one CTA per (row, head, 64-key split of Smax)
static int launch_decode_attention(vly_ctx* c, DecAttnParams p, bool pdl, cudaStream_t st) {
  p.nsplit = p.Smax / kDecSplitKeys;
  p.scale_log2e = 0.08838834764831845f * 1.4426950408889634f;
  return launch(c, decode_attention_v2_kernel, {dim3(p.B * p.nH, p.nsplit), dim3(128), 0, st, pdl, true}, p);
}

static int launch_logits_gemv(vly_ctx* c, vly_kv* kv, int b0, int nb, const bf16* x, long long ldx, long long* out_tokens, bool bump,
                              bool pdl, cudaStream_t st);

// Enqueue one decode step for batch rows [b0, b0+nb) of kv (nb <= 4).  Reads kv->cur_tokens, writes kv->cur_tokens.
static int enqueue_decode_step(vly_ctx* c, vly_kv* kv, int b0, int nb, bool bump, cudaStream_t st) {
  const vly_config& g = c->cfg;
  const int H = g.hidden_size, nH = g.num_attention_heads, I = g.intermediate_size, V = g.vocab_size;
  bf16 *x = kv->x + (size_t)b0 * H, *q = kv->q + (size_t)b0 * H, *attn = kv->attn + (size_t)b0 * H, *hb = kv->hb + (size_t)b0 * I;
  TRY(launch(c, decode_embed_kernel, {dim3(nb), dim3(256), 0, st}, kv->cur_tokens + b0, c->embed, x, H, V));
  for (int l = 0; l < g.num_hidden_layers; ++l) {
    const LlamaLayerW& w = c->layers[l];
    bf16* kc = kv->k_layer(l) + (size_t)b0 * nH * kv->Smax * 128;
    bf16* vc = kv->v_layer(l) + (size_t)b0 * nH * kv->Smax * 128;
    {
      GemvParams p = {};
      p.N = 3 * H; p.K = H; p.B = nb; p.W = w.wqkv; p.x = x; p.eps = g.rms_norm_eps;
      p.out = q; p.rope = c->rope; p.seq_len = kv->d_len; p.H = H; p.nH = nH; p.Smax = kv->Smax; p.kcache = kc; p.vcache = vc;
      TRY(launch_gemv_ring<GEMV_QKV_ROPE>(c, p, true, st));
    }
    {
      DecAttnParams p = {};
      p.B = nb; p.nH = nH; p.H = H; p.Smax = kv->Smax; p.seq_len = kv->d_len;
      p.q = q; p.kcache = kc; p.vcache = vc;
      p.part_o = kv->part_o + (size_t)b0 * nH * kv->nsplit * 128;
      p.part_ml = kv->part_ml + (size_t)b0 * nH * kv->nsplit;
      p.counters = kv->counters + (size_t)b0 * nH;
      p.out = attn;
      p.key_bits = kv->key_bits + (size_t)b0 * kv->mask_words(); p.mask_words = kv->mask_words();
      TRY(launch_decode_attention(c, p, true, st));
    }
    {
      GemvParams p = {};
      p.N = H; p.K = H; p.B = nb; p.W = w.wo; p.x = attn; p.out = x; p.res = x;
      TRY(launch_gemv_ring<GEMV_RESIDUAL>(c, p, true, st));
    }
    {
      GemvParams p = {};
      p.N = 2 * I; p.K = H; p.B = nb; p.W = w.wgu; p.x = x; p.eps = g.rms_norm_eps; p.out = hb;
      TRY(launch_gemv_ring<GEMV_SWIGLU>(c, p, true, st));
    }
    {
      GemvParams p = {};
      p.N = H; p.K = I; p.B = nb; p.W = w.wdown; p.x = hb; p.out = x; p.res = x;
      TRY(launch_gemv_ring<GEMV_RESIDUAL>(c, p, true, st));
    }
  }
  return launch_logits_gemv(c, kv, b0, nb, x, 0, kv->gen_tokens + (size_t)b0 * kv->Smax, bump, true, st);
}

// final RMSNorm (folded) + lm_head + arg-max for batch rows [b0, b0+nb) of kv (nb <= 4): x [nb, H] of row stride ldx (0 = H) ->
// kv->logits and kv->cur_tokens, and column *d_step of out_tokens [nb, Smax] (nullptr: none).  bump: the last batch group of a
// decode step, which advances the step / length counters.
static int launch_logits_gemv(vly_ctx* c, vly_kv* kv, int b0, int nb, const bf16* x, long long ldx, long long* out_tokens, bool bump,
                              bool pdl, cudaStream_t st) {
  const vly_config& g = c->cfg;
  GemvParams p = {};
  p.N = g.vocab_size; p.K = g.hidden_size; p.B = nb; p.W = c->lm_head; p.x = x; p.ldx = ldx; p.eps = g.rms_norm_eps;
  p.logits = kv->logits + (size_t)b0 * g.vocab_size;
  p.part_val = kv->part_val + (size_t)b0 * c->num_sms;
  p.part_idx = kv->part_idx + (size_t)b0 * c->num_sms;
  p.counter = kv->counters + (size_t)kv->B * g.num_attention_heads;
  p.next_tokens = kv->cur_tokens + b0;
  p.out_tokens = out_tokens; p.out_stride = kv->Smax;
  p.step = kv->d_step; p.seq_len_rw = kv->d_len; p.bump = bump ? 1 : 0;
  return launch_gemv_ring<GEMV_LOGITS>(c, p, pdl, st);
}

// ------------------------------------------------------------------------------------------------
// prefill
// ------------------------------------------------------------------------------------------------
// One layer's causal prefill attention: q [B*S, nH*128] against the K/V rows [0, past + S) of kcache / vcache [B, nH, Smax, 128];
// key_bits [B, Smax/32] (1 = attend) or NULL when no key is masked.
static int launch_prefill_attention(vly_ctx* c, const bf16* qbuf, const bf16* kcache, const bf16* vcache, int Smax, const uint32_t* key_bits,
                                    int B, int S, int past, int nH, bf16* out, cudaStream_t st) {
  const int H = nH * 128;
  using C = FlashCfg<128>;
  CUtensorMap tq, tk, tv;
  TRY(make_tmap_2d(c, &tq, qbuf, H, (uint64_t)B * S, (uint64_t)H * 2, 64, 64));
  TRY(make_tmap_3d(c, &tk, kcache, 128, Smax, (uint64_t)B * nH, 256, (uint64_t)Smax * 256, 64, 64));
  TRY(make_tmap_3d(c, &tv, vcache, 128, Smax, (uint64_t)B * nH, 256, (uint64_t)Smax * 256, 64, 64));
  PrefillAttnParams p;
  p.B = B; p.S = S; p.past = past; p.nH = nH; p.H = H; p.Smax = Smax; p.ctx = out;
  p.scale_log2e = 0.08838834764831845f * 1.4426950408889634f;
  p.key_bits = key_bits; p.mask_words = Smax / 32;
  const int n_qt = cdiv(S, 64);
  return launch(c, llama_prefill_attention_kernel, {dim3(B * nH * n_qt), dim3(C::THREADS), C::SMEM_BYTES, st, true}, tq, tk, tv, p);
}

extern "C" int vly_llama_prefill(vly_ctx* c, vly_kv* kv, const void* inputs_embeds, int B, int S, int logits_mode, void* logits_dev,
                                 int64_t* next_tokens_dev, void* stream) {
  if (!c || !kv || !inputs_embeds || B <= 0 || S <= 0) return fail(VLY_ERR_INVALID, "vly_llama_prefill: bad argument");
  if (kv->ctx != c || B != kv->B) return fail(VLY_ERR_INVALID, "vly_llama_prefill: batch %d does not match the kv cache (%d)", B, kv->B);
  if (logits_mode < 0 || logits_mode > 2 || (logits_mode && !logits_dev)) return fail(VLY_ERR_INVALID, "vly_llama_prefill: bad logits mode");
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->finalized || !c->has_llm) return fail(VLY_ERR_STATE, "vly_llama_prefill: LLM weights not finalised");
  TRY(sync_len(kv));
  const int past = kv->host_len;
  if (past + S > kv->Smax) return fail(VLY_ERR_INVALID, "vly_llama_prefill: %d cached + %d new tokens exceed the cache capacity %d", past, S, kv->Smax);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const vly_config& g = c->cfg;
  const int H = g.hidden_size, nH = g.num_attention_heads, I = g.intermediate_size, V = g.vocab_size;
  const int M = B * S;
  const int bn_h = pick_bn_m(c, H, M), nt = cdiv(H, bn_h);
  TRY(ensure(c->w_x, (size_t)M * H * 2));
  TRY(ensure(c->w_q, (size_t)M * H * 2));
  TRY(ensure(c->w_attn, (size_t)M * H * 2));
  TRY(ensure(c->w_hb, (size_t)M * I * 2));
  TRY(ensure(c->w_pstats, (size_t)M * nt * sizeof(float2)));
  bf16 *x = (bf16*)c->w_x.p, *qb = (bf16*)c->w_q.p, *attn = (bf16*)c->w_attn.p, *hb = (bf16*)c->w_hb.p;
  float2* stats = (float2*)c->w_pstats.p;
  TRY(launch(c, copy_rows_stats_kernel, {dim3(M), dim3(128), 0, st}, (const bf16*)inputs_embeds, x, stats, nt, H));
  for (int l = 0; l < g.num_hidden_layers; ++l) {
    const LlamaLayerW& w = c->layers[l];
    {
      GemmParams p = {};
      p.M = M; p.N = 3 * H; p.K = H; p.out = qb; p.ldo = H;
      p.stats_in = stats; p.stats_in_nt = nt; p.inv_dim = 1.f / H; p.eps = g.rms_norm_eps;
      p.rope = c->rope; p.S = S; p.past = past; p.H = H; p.nH = nH; p.Smax = kv->Smax;
      p.kcache = kv->k_layer(l); p.vcache = kv->v_layer(l);
      TRY(launch_gemm<EPI_RMS_QKV_ROPE>(c, pick_bn_m(c, 3 * H, M), x, H, w.wqkv, H, p, st));
    }
    TRY(launch_prefill_attention(c, qb, kv->k_layer(l), kv->v_layer(l), kv->Smax, kv->masked ? static_cast<uint32_t*>(kv->key_bits) : nullptr,
                                 B, S, past, nH, attn, st));
    {
      GemmParams p = {};
      p.M = M; p.N = H; p.K = H; p.out = x; p.ldo = H; p.residual = x; p.ldr = H; p.stats_out = stats;
      TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, bn_h, attn, H, w.wo, H, p, st));
    }
    {
      GemmParams p = {};
      p.M = M; p.N = 2 * I; p.K = H; p.out = hb; p.ldo = I;
      p.stats_in = stats; p.stats_in_nt = nt; p.inv_dim = 1.f / H; p.eps = g.rms_norm_eps;
      TRY(launch_gemm<EPI_RMS_SWIGLU>(c, pick_bn_m(c, 2 * I, M), x, H, w.wgu, H, p, st));
    }
    {
      GemmParams p = {};
      p.M = M; p.N = H; p.K = I; p.out = x; p.ldo = H; p.residual = x; p.ldr = H; p.stats_out = stats;
      TRY(launch_gemm<EPI_BIAS_RES_STATS>(c, bn_h, hb, I, w.wdown, I, p, st));
    }
  }
  if (logits_mode == 2) {  // lm_head over every position (valley_model.py:304-305)
    GemmParams p = {};
    p.M = M; p.N = V; p.K = H; p.out = logits_dev; p.ldo = V;
    p.stats_in = stats; p.stats_in_nt = nt; p.inv_dim = 1.f / H; p.eps = g.rms_norm_eps;
    TRY(launch_gemm<EPI_RMS_F32>(c, 256, x, H, c->lm_head, H, p, st));
  }
  // last position only: final RMSNorm (folded) + lm_head GEMV + greedy argmax (model_worker.py:389-391)
  for (int b0 = 0; b0 < B; b0 += 4)
    TRY(launch_logits_gemv(c, kv, b0, std::min(4, B - b0), x + ((size_t)b0 * S + (S - 1)) * H, (long long)S * H, nullptr, false, false, st));
  if (logits_mode == 1) CK(cudaMemcpyAsync(logits_dev, kv->logits, (size_t)B * V * 4, cudaMemcpyDeviceToDevice, st));
  if (next_tokens_dev) CK(cudaMemcpyAsync(next_tokens_dev, kv->cur_tokens, (size_t)B * 8, cudaMemcpyDeviceToDevice, st));
  kv->host_len = past + S;
  return launch(c, set_int_kernel, {dim3(1), dim3(1), 0, st}, kv->d_len, kv->host_len);
}

// ------------------------------------------------------------------------------------------------
// decode
// ------------------------------------------------------------------------------------------------
extern "C" int vly_kv_debug_counters(vly_kv* kv, long long* host_out, int n) {
  if (!kv || !host_out || n < 0) return fail(VLY_ERR_INVALID, "vly_kv_debug_counters: bad argument");
  if (!kv->dbg)
    return fail(VLY_ERR_STATE, "vly_kv_debug_counters: this cache has no counters (B %d; they need B <= 4 and VLY_MEGA_DBG set when it was created)", kv->B);
  if (n > kMegaDbgCounters) return fail(VLY_ERR_INVALID, "vly_kv_debug_counters: %d values requested, the cache holds %d", n, kMegaDbgCounters);
  CK(cudaSetDevice(kv->ctx->cfg.device));
  CK(cudaMemcpy(host_out, kv->dbg, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost));
  return VLY_OK;
}

// the launch was planned by vly_kv_create (plan_decode_mega); select = false: the step ends with the logits, another kernel selects
static int launch_decode_mega(vly_ctx* c, vly_kv* kv, bool select, cudaStream_t st) {
  StepParams p = kv->mega;
  p.select = select ? 1 : 0;
  LaunchCfg l = {dim3(c->num_sms), dim3(MegaCfg::THREADS), kv->mega_smem, st};
  l.cooperative = true;
  return with_bmax(kv->B, [&](auto bm) { return launch(c, decode_step_kernel<decltype(bm)::value>, l, p); });
}

// token selection over [B, V] logits (sampling.cuh), one CTA per row; a filter = 1 launch (a filter, stop strings, recording or
// logits processors) has room for a filtered row's staged scores and for the processors' two bitmaps in shared memory
static int launch_sample_filter(vly_ctx* c, const float* logits, int B, int V, SampleState* s, const int* seq_len, const int* step,
                                long long* next_tokens, long long* out_tokens, int out_stride, bool filter, bool per_op,
                                uint8_t* keep_out, cudaStream_t st) {
  const size_t smem = filter ? filter_stage_bytes(V) + proc_map_bytes(V) : 0;
  return launch(c, sample_filter_kernel, {dim3(B), dim3(kFilterThreads), smem, st}, logits, V, s, seq_len, step, next_tokens, out_tokens,
                out_stride, filter ? 1 : 0, per_op ? 1 : 0, keep_out);
}

// rows within groups of `group` take their parent's positions [*from_pos, *len) (kv_beam_reorder_kernel)
static int launch_kv_beam_reorder(vly_ctx* c, vly_kv* kv, int group, const int* parent, const int* from_pos, const int* skip,
                                  cudaStream_t st) {
  const int nH = c->cfg.num_attention_heads, L = c->cfg.num_hidden_layers;
  const size_t smem = (size_t)group * reorder_block_positions(group) * 256;
  return launch(c, kv_beam_reorder_kernel, {dim3(L * 2 * (kv->B / group) * nH), dim3(kReorderThreads), smem, st}, kv->cache, kv->B,
                nH, kv->Smax, group, parent, from_pos, (const int*)kv->d_len, skip);
}

static int launch_beam_step(vly_ctx* c, vly_kv* kv, int nb, const float* logits, cudaStream_t st) {
  const size_t half = (size_t)2 * kv->B * kv->Smax;       // [2 parities][B][Smax]: the running rows, then the finished ones
  return launch(c, beam_step_kernel, {dim3(kv->B / nb), dim3(kBeamThreads), 0, st}, logits, c->cfg.vocab_size, kv->d_beam,
                (long long*)kv->beam_tok, kv->beam_tok + half, (int*)kv->beam_bidx, kv->beam_bidx + half, kv->Smax,
                (const float*)kv->beam_div, (long long*)kv->cur_tokens, kv->d_sample);
}

// Enqueue one decode step of kv: the persistent kernel (B <= 4) or the per-op kernels per group of <= 4 rows, then what the
// step kind selects with.  nb: beams per item (STEP_BEAM only).
static int enqueue_step(vly_ctx* c, vly_kv* kv, StepKind kind, int nb, cudaStream_t st) {
  const bool per_op = kv->B > 4;
  if (!per_op) TRY(launch_decode_mega(c, kv, kind == STEP_TOKEN, st));
  else
    for (int b0 = 0; b0 < kv->B; b0 += 4) TRY(enqueue_decode_step(c, kv, b0, std::min(4, kv->B - b0), b0 + 4 >= kv->B, st));
  if (kind == STEP_BEAM) {      // beam_step_kernel selects, the cache follows the parents
    TRY(launch_beam_step(c, kv, nb, kv->logits, st));
    return launch_kv_beam_reorder(c, kv, nb, kv->d_beam->parent, &kv->d_beam->prompt_len, &kv->d_beam->done, st);
  }
  // a filtered token, or on the per-op path the sampling / eos bookkeeping (returns at once when greedy), is one more launch
  // over the step's logits (a filter needs set_sampling, which allows at most kMaxSampleRows rows)
  if (kind == STEP_FILTERED || (per_op && kv->B <= kMaxSampleRows))
    TRY(launch_sample_filter(c, kv->logits, kv->B, c->cfg.vocab_size, kv->d_sample, kv->d_len, kv->d_step, kv->cur_tokens,
                             kv->gen_tokens, kv->Smax, kind == STEP_FILTERED, per_op, nullptr, st));
  return VLY_OK;
}

// ---- token selection state ----
__global__ void set_sample_state_kernel(SampleState* s, const SampleState r, int reset_done) {
  if (threadIdx.x == 0) {
    s->temperature = r.temperature; s->inv_temp = r.inv_temp; s->enabled = r.enabled; s->filter = r.filter; s->top_k = r.top_k;
    s->top_p = r.top_p; s->seed_lo = r.seed_lo; s->seed_hi = r.seed_hi; s->eos = r.eos; s->pad = r.pad; s->stop2 = r.stop2;
    s->n_stop = r.n_stop; s->stop_walk = r.stop_walk; s->stop_masks = r.stop_masks; s->tok_len = r.tok_len; s->pause = r.pause;
    s->ring = r.ring; s->rec_scores = r.rec_scores; s->rec_logits = r.rec_logits; s->rec_temp = r.rec_temp;
    s->procs = r.procs; s->penalty = r.penalty; s->ngram = r.ngram; s->min_length = r.min_length; s->hist = r.hist;
    s->hist_stride = r.hist_stride;
    if (reset_done) { s->all_done = 0; s->steps_valid = 0; }
  }
  if (threadIdx.x < kMaxStopStrings) s->stop_len[threadIdx.x] = r.stop_len[threadIdx.x];
  if (reset_done && threadIdx.x < kMaxSampleRows) { s->done[threadIdx.x] = 0; s->ring_n[threadIdx.x] = r.ring_n[threadIdx.x]; }
}

// ---- stop strings ----
// kv->stop_buf: [kMaxStopStrings][V] ulonglong2 masks | [V] uint8 token lengths | [ceil(V/32)] uint32 pause bits |
// [kMaxSampleRows][kStopRing] int32 rings.  stop_stage (pinned) has the same layout.
struct StopLayout {
  size_t lens, pause, ring, bytes;
  explicit StopLayout(int V) {
    auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
    lens = (size_t)kMaxStopStrings * V * sizeof(ulonglong2);
    pause = up(lens + V);
    ring = up(pause + (size_t)cdiv(V, 32) * 4);
    bytes = ring + (size_t)kMaxSampleRows * kStopRing * 4;
  }
};

static int check_stop_tables(const vly_sampling* sp, int B, const char* who) {
  const int n = sp->n_stop_strings;
  if (n < 0 || n > kMaxStopStrings || !sp->stop_lens || !sp->stop_masks || !sp->stop_token_lens)
    return fail(VLY_ERR_INVALID, "%s: n_stop_strings %d must be in [1, %d] with stop_lens, stop_masks and stop_token_lens", who, n, kMaxStopStrings);
  for (int i = 0; i < n; ++i)
    if (sp->stop_lens[i] < 1 || sp->stop_lens[i] > kMaxStopChars)
      return fail(VLY_ERR_INVALID, "%s: stop string %d has %d characters (1..%d on the device)", who, i, sp->stop_lens[i], kMaxStopChars);
  if (sp->stop_tail_len < 0 || sp->stop_tail_len >= kStopRing || (sp->stop_tail_len > 0 && !sp->stop_tail))
    return fail(VLY_ERR_INVALID, "%s: stop_tail_len %d must be in [0, %d) with a stop_tail", who, sp->stop_tail_len, kStopRing);
  if (B > kMaxSampleRows) return fail(VLY_ERR_INVALID, "%s: stop strings support at most %d rows (%d)", who, kMaxSampleRows, B);
  return VLY_OK;
}

// The SampleState fields of sp's stop strings over the device buffer `dev` (StopLayout); ring_n from the tail length.
static void stop_state(const vly_sampling* sp, uint8_t* dev, int V, SampleState& r) {
  const StopLayout l(V);
  r.n_stop = sp->n_stop_strings;
  r.stop_walk = 0;
  for (int i = 0; i < r.n_stop; ++i) {
    r.stop_len[i] = sp->stop_lens[i];
    r.stop_walk = std::max(r.stop_walk, sp->stop_lens[i]);
  }
  r.stop_masks = (const ulonglong2*)dev;
  r.tok_len = dev + l.lens;
  r.pause = sp->pause_bits ? (const uint32_t*)(dev + l.pause) : nullptr;
  r.ring = (int*)(dev + l.ring);
  for (int b = 0; b < kMaxSampleRows; ++b) r.ring_n[b] = sp->stop_tail_len;
}

// Uploads sp's tables and each row's tail (seeding its ring) to `dev` through the pinned `stage`; every host array is read
// before this returns.  The wait on `ev` only blocks when the previous upload from `stage` has not run yet.
static int upload_stop_tables(const vly_sampling* sp, int B, int V, uint8_t* dev, uint8_t* stage, cudaEvent_t ev, cudaStream_t st) {
  const StopLayout l(V);
  const int n = sp->n_stop_strings, tail = sp->stop_tail_len;
  CK(cudaEventSynchronize(ev));
  const size_t mask_bytes = (size_t)n * V * sizeof(ulonglong2);
  memcpy(stage, sp->stop_masks, mask_bytes);
  for (int t = 0; t < V; ++t) stage[l.lens + t] = (uint8_t)std::min<int32_t>(sp->stop_token_lens[t], 255);
  const size_t pause_bytes = sp->pause_bits ? (size_t)cdiv(V, 32) * 4 : 0;
  if (pause_bytes) memcpy(stage + l.pause, sp->pause_bits, pause_bytes);
  int* ring = (int*)(stage + l.ring);
  for (int b = 0; b < B; ++b)
    for (int j = 0; j < tail; ++j) ring[b * kStopRing + j] = (int)sp->stop_tail[(size_t)b * tail + j];
  CK(cudaMemcpyAsync(dev, stage, mask_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(dev + l.lens, stage + l.lens, (size_t)V, cudaMemcpyHostToDevice, st));
  if (pause_bytes) CK(cudaMemcpyAsync(dev + l.pause, stage + l.pause, pause_bytes, cudaMemcpyHostToDevice, st));
  if (tail) CK(cudaMemcpyAsync(dev + l.ring, stage + l.ring, (size_t)B * kStopRing * 4, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(ev, st));
  return VLY_OK;
}

// sampling == nullptr: plain greedy, no stop token (skipped when the device state already says so, unless `force`: a beam
// search starts from that state and leaves all_done raised, so it always resets it and leaves it dirty)
// sp with stop strings: a call that resets the flags (or sets stop_restart) uploads the tables and seeds the rings; one that
// keeps them continues the running stop-string request.
static int set_sampling(vly_ctx* c, vly_kv* kv, const vly_sampling* sp, bool reset_done, cudaStream_t st, bool force = false) {
  SampleState r = {};
  kv->filtered = false;
  kv->recording = false;
  const bool had_stop = kv->stop_ready, had_procs = kv->procs_ready;
  kv->stop_ready = false;
  kv->procs_ready = false;
  if (!sp) {
    if (!kv->sample_dirty && !force) return VLY_OK;
    reset_done = true;
  } else {
    if (sp->n_stop_strings != 0) {
      const int V = c->cfg.vocab_size;
      TRY(check_stop_tables(sp, kv->B, "vly_sampling"));
      reset_done = reset_done || sp->stop_restart;
      if (!reset_done && !had_stop)
        return fail(VLY_ERR_STATE, "vly_generate: stop strings continue a request started by vly_sample_logits; set stop_restart to start one");
      if (!kv->stop_buf) {
        const StopLayout l(V);
        TRY(kv->stop_buf.alloc(l.bytes));
        TRY(kv->stop_stage.alloc(l.bytes, true));
        CK(cudaEventCreateWithFlags(&kv->stop_event, cudaEventDisableTiming));
      }
      if (reset_done) TRY(upload_stop_tables(sp, kv->B, V, kv->stop_buf, kv->stop_stage, kv->stop_event, st));
      stop_state(sp, kv->stop_buf, V, r);
      kv->stop_ready = true;
    }
    if (kv->B > kMaxSampleRows) return fail(VLY_ERR_INVALID, "sampling / eos bookkeeping supports at most %d sequences per cache", kMaxSampleRows);
    // logits processors (zero fields: off): a request that resets seeds every row's history from its prompt ids, one that
    // keeps the flags continues the processor request vly_sample_logits started
    if (!(sp->repetition_penalty >= 0.f) || sp->no_repeat_ngram_size < 0 || sp->min_length < 0)
      return fail(VLY_ERR_INVALID, "vly_sampling: repetition_penalty %g, no_repeat_ngram_size %d and min_length %d must be >= 0",
                  (double)sp->repetition_penalty, sp->no_repeat_ngram_size, sp->min_length);
    const float penalty = sp->repetition_penalty == 0.f ? 1.f : sp->repetition_penalty;
    if (penalty != 1.f || sp->no_repeat_ngram_size > 0 || (sp->min_length > 0 && sp->eos_token_id >= 0)) {
      if (!reset_done && !had_procs)
        return fail(VLY_ERR_STATE, "vly_generate: logits processors continue a request started by vly_sample_logits");
      const int S = kv->host_len;
      if (reset_done && (!sp->prompt_ids_dev || S <= 0))
        return fail(VLY_ERR_INVALID, "vly_sampling: logits processors need prompt_ids_dev [B, %d] when a request starts", S);
      if (!kv->hist) TRY(kv->hist.alloc((size_t)kv->B * kv->Smax * sizeof(int)));
      if (reset_done)
        TRY(launch(c, hist_seed_kernel, {dim3(kv->B), dim3(256), 0, st}, (int*)kv->hist, kv->Smax, (const long long*)sp->prompt_ids_dev, S));
      r.procs = 1; r.penalty = penalty; r.ngram = sp->no_repeat_ngram_size; r.min_length = sp->min_length;
      r.hist = kv->hist; r.hist_stride = kv->Smax;
      kv->procs_ready = true;
    }
    const bool on = sp->temperature >= 1e-4f;        // model_worker.py:390: below that the reference takes the arg-max
    if (on) {
      r.temperature = sp->temperature; r.inv_temp = 1.f / sp->temperature; r.enabled = 1; r.top_k = sp->top_k; r.top_p = sp->top_p;
    }
    r.seed_lo = (uint32_t)sp->seed; r.seed_hi = (uint32_t)(sp->seed >> 32);
    r.eos = sp->eos_token_id < 0 ? -1 : sp->eos_token_id;
    r.pad = sp->pad_token_id;
    r.stop2 = sp->stop_token_id < 0 ? -1 : sp->stop_token_id;
    // the filters apply only when sampling (HF ignores its warpers when it does not sample)
    kv->filtered = on && (sp->top_k > 0 || (sp->top_p > 0.f && sp->top_p < 1.f));
    r.filter = kv->filtered ? 1 : 0;
    // recording: HF records logits / temperature whenever it samples, also where the temperature is too low to draw with
    r.rec_scores = sp->scores_out;
    r.rec_logits = sp->logits_out;
    r.rec_temp = sp->temperature > 0.f ? sp->temperature : 1.f;
    kv->recording = sp->scores_out != nullptr || sp->logits_out != nullptr;
  }
  kv->sample_dirty = sp != nullptr || force;
  return launch(c, set_sample_state_kernel, {dim3(1), dim3(64), 0, st}, kv->d_sample, r, reset_done ? 1 : 0);
}

constexpr int kGraphSteps = 8;
// n steps of enqueue_step(stream) as one graph; *nodes receives the kernel launches per step
template <typename F>
static int capture_steps(vly_ctx* c, int n, F&& enqueue_step, cudaGraphExec_t* out, int* nodes) {
  const int64_t before = c->launches;
  CK(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeThreadLocal));
  int r = VLY_OK;
  for (int i = 0; i < n && r == VLY_OK; ++i) r = enqueue_step(c->cap_stream);
  cudaGraph_t graph = nullptr;
  const cudaError_t e = cudaStreamEndCapture(c->cap_stream, &graph);
  *nodes = (int)((c->launches - before) / n);
  c->launches = before;
  if (r != VLY_OK) {
    if (graph) cudaGraphDestroy(graph);
    return r;
  }
  if (e != cudaSuccess) return fail(VLY_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(e));
  const cudaError_t e2 = cudaGraphInstantiate(out, graph, 0);
  cudaGraphDestroy(graph);
  if (e2 != cudaSuccess) return fail(VLY_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e2));
  return VLY_OK;
}
// Run n decode steps of one kind on st as replays of its kGraphSteps-step graph, then of its 1-step graph; each replayed step
// counts its kernels.  VLY_NO_GRAPH=1 (profiling aid): eager launches instead.
static int run_steps(vly_ctx* c, vly_kv* kv, StepKind kind, int nb, int n, cudaStream_t st) {
  static const bool no_graph = getenv("VLY_NO_GRAPH") != nullptr;
  auto step = [&](cudaStream_t s) { return enqueue_step(c, kv, kind, nb, s); };
  if (no_graph) {
    for (int i = 0; i < n; ++i) TRY(step(st));
    return VLY_OK;
  }
  StepGraphs& g = kv->graphs[kind];
  if (!g.many || g.nb != nb) {
    g.reset();
    TRY(capture_steps(c, 1, step, &g.one, &g.nodes));
    TRY(capture_steps(c, kGraphSteps, step, &g.many, &g.nodes));
    g.nb = nb;
  }
  for (int i = 0; i < n;) {
    if (n - i >= kGraphSteps) { CK(cudaGraphLaunch(g.many, st)); i += kGraphSteps; }
    else { CK(cudaGraphLaunch(g.one, st)); ++i; }
  }
  c->launches += (int64_t)n * g.nodes;
  return VLY_OK;
}

// the request advanced the cache by n positions, or fewer when the device may have stopped early (a stop id, the end of a beam
// search): then the device's length is copied back behind the request, and sync_len reads it on the cache's next use
static int finish_request(vly_kv* kv, int n, bool may_stop_early, cudaStream_t st) {
  kv->host_len += n;
  if (!may_stop_early) return VLY_OK;
  CK(cudaMemcpyAsync(kv->h_len, kv->d_len, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(kv->len_event, st));
  kv->len_dirty = true;
  return VLY_OK;
}

extern "C" int vly_sample_logits(vly_ctx* c, vly_kv* kv, const float* logits, const vly_sampling* sp, int64_t* tokens_out, void* stream) {
  if (!c || !kv || !logits || !sp || !tokens_out || kv->ctx != c) return fail(VLY_ERR_INVALID, "vly_sample_logits: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  TRY(set_sampling(c, kv, sp, true, st));
  // (no step counter: the first token records into slot 0)
  return launch_sample_filter(c, logits, kv->B, c->cfg.vocab_size, kv->d_sample, kv->d_len, nullptr, (long long*)tokens_out, nullptr,
                              0, kv->filtered || kv->procs_ready, false, nullptr, st);
}

static int generate_impl(vly_ctx* c, vly_kv* kv, const int64_t* first_tokens, int n_steps, int64_t* out_tokens, const vly_sampling* sp,
                         int* steps_done_dev, void* stream);

extern "C" int vly_generate_greedy(vly_ctx* c, vly_kv* kv, const int64_t* first_tokens, int n_steps, int64_t* out_tokens, void* stream) {
  return generate_impl(c, kv, first_tokens, n_steps, out_tokens, nullptr, nullptr, stream);
}

extern "C" int vly_generate(vly_ctx* c, vly_kv* kv, const int64_t* first_tokens, int n_steps, int64_t* out_tokens, const vly_sampling* sp,
                            int* steps_done_dev, void* stream) {
  return generate_impl(c, kv, first_tokens, n_steps, out_tokens, sp, steps_done_dev, stream);
}

static int generate_impl(vly_ctx* c, vly_kv* kv, const int64_t* first_tokens, int n_steps, int64_t* out_tokens, const vly_sampling* sp,
                         int* steps_done_dev, void* stream) {
  if (!c || !kv || !first_tokens || n_steps <= 0 || kv->ctx != c) return fail(VLY_ERR_INVALID, "vly_generate: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  TRY(sync_len(kv));
  if (kv->host_len + n_steps > kv->Smax) return fail(VLY_ERR_INVALID, "vly_generate: %d cached + %d steps exceed the cache capacity %d", kv->host_len, n_steps, kv->Smax);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  // with a sampling struct the eos flags raised by vly_sample_logits (the first token) are kept, unless a stop-string request
  // restarts; greedy starts clean
  TRY(set_sampling(c, kv, sp, false, st));
  CK(cudaMemcpyAsync(kv->cur_tokens, first_tokens, (size_t)kv->B * 8, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync(kv->d_step, 0, 4, st));
  if (steps_done_dev) CK(cudaMemsetAsync(&kv->d_sample->steps_valid, 0, 4, st));
  // (a stop-string request selects in sample_filter_kernel, which runs the matcher; a recording one, which writes its slot;
  //  one with logits processors, which applies them)
  TRY(run_steps(c, kv, kv->filtered || kv->stop_ready || kv->recording || kv->procs_ready ? STEP_FILTERED : STEP_TOKEN, 0, n_steps,
                st));
  if (out_tokens)
    CK(cudaMemcpy2DAsync(out_tokens, (size_t)n_steps * 8, kv->gen_tokens, (size_t)kv->Smax * 8, (size_t)n_steps * 8, kv->B,
                         cudaMemcpyDeviceToDevice, st));
  if (steps_done_dev)      // (zeroed above, before the first step)
    CK(cudaMemcpyAsync(steps_done_dev, &kv->d_sample->steps_valid, 4, cudaMemcpyDeviceToDevice, st));
  return finish_request(kv, n_steps, sp && (sp->eos_token_id >= 0 || sp->stop_token_id >= 0 || sp->n_stop_strings > 0), st);
}

extern "C" int vly_llama_decode(vly_ctx* c, vly_kv* kv, const int64_t* tokens, int64_t* next_tokens, void* logits_dev, void* stream) {
  if (!c || !kv || !tokens || kv->ctx != c) return fail(VLY_ERR_INVALID, "vly_llama_decode: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  TRY(sync_len(kv));
  if (kv->host_len + 1 > kv->Smax) return fail(VLY_ERR_INVALID, "vly_llama_decode: cache full (%d)", kv->Smax);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  TRY(set_sampling(c, kv, nullptr, true, st));
  CK(cudaMemcpyAsync(kv->cur_tokens, tokens, (size_t)kv->B * 8, cudaMemcpyDeviceToDevice, st));
  CK(cudaMemsetAsync(kv->d_step, 0, 4, st));
  TRY(run_steps(c, kv, STEP_TOKEN, 0, 1, st));
  if (next_tokens) CK(cudaMemcpyAsync(next_tokens, kv->cur_tokens, (size_t)kv->B * 8, cudaMemcpyDeviceToDevice, st));
  if (logits_dev) CK(cudaMemcpyAsync(logits_dev, kv->logits, (size_t)kv->B * c->cfg.vocab_size * 4, cudaMemcpyDeviceToDevice, st));
  return finish_request(kv, 1, false, st);
}

// ------------------------------------------------------------------------------------------------
// beam search (beam.cuh)
// ------------------------------------------------------------------------------------------------
static int ensure_beam_buffers(vly_kv* kv) {
  if (kv->d_beam) return VLY_OK;
  TRY(kv->d_beam.alloc(sizeof(BeamState)));
  TRY(kv->beam_tok.alloc((size_t)4 * kv->B * kv->Smax * sizeof(long long)));
  TRY(kv->beam_bidx.alloc((size_t)4 * kv->B * kv->Smax * sizeof(int)));
  TRY(kv->beam_div.alloc((size_t)kv->Smax * sizeof(float)));
  TRY(kv->beam_from.alloc(sizeof(int)));
  return VLY_OK;
}

extern "C" int vly_beam_search(vly_ctx* c, vly_kv* kv, const vly_beam* bp, const float* first_logits, int prompt_len, int n_steps,
                               int64_t* seq_out, float* scores_out, int* gen_len_out, void* stream) {
  if (!c || !kv || !bp || !first_logits || !seq_out || !scores_out || !gen_len_out || n_steps <= 0 || kv->ctx != c)
    return fail(VLY_ERR_INVALID, "vly_beam_search: bad argument");
  const int nb = bp->num_beams, nrs = bp->num_return_sequences;
  if (nb < 1 || nb > kMaxBeams || kv->B % nb != 0)
    return fail(VLY_ERR_INVALID, "vly_beam_search: num_beams %d must be in [1, %d] and divide the cache's %d rows", nb, kMaxBeams, kv->B);
  if (kv->B > kMaxSampleRows) return fail(VLY_ERR_INVALID, "vly_beam_search: at most %d rows per cache (%d)", kMaxSampleRows, kv->B);
  if (nrs < 1 || nrs > nb) return fail(VLY_ERR_INVALID, "vly_beam_search: num_return_sequences %d must be in [1, num_beams %d]", nrs, nb);
  if (bp->early_stopping < 0 || bp->early_stopping > 2) return fail(VLY_ERR_INVALID, "vly_beam_search: early_stopping %d", bp->early_stopping);
  std::lock_guard<std::mutex> lk(c->mu);
  TRY(sync_len(kv));
  if (prompt_len != kv->host_len) return fail(VLY_ERR_STATE, "vly_beam_search: the cache holds %d tokens, not the %d-token prompt", kv->host_len, prompt_len);
  if (kv->host_len + n_steps - 1 > kv->Smax) return fail(VLY_ERR_INVALID, "vly_beam_search: %d cached + %d steps exceed the cache capacity %d", kv->host_len, n_steps - 1, kv->Smax);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  TRY(ensure_beam_buffers(kv));
  // plain selection state: the decode steps write logits only, and exit once beam_step_kernel raises all_done
  TRY(set_sampling(c, kv, nullptr, true, st, true));
  TRY(launch(c, beam_init_kernel, {dim3(1), dim3(256), 0, st}, kv->d_beam, kv->B, nb, n_steps, prompt_len, (int)bp->early_stopping,
             bp->length_penalty, (long long)(bp->eos_token_id < 0 ? -1 : bp->eos_token_id), (float*)kv->beam_div, bp->scores_out,
             bp->logits_out, (long long*)bp->beam_indices_out, (int*)bp->steps_out));
  TRY(launch_beam_step(c, kv, nb, first_logits, st));
  CK(cudaMemsetAsync(kv->d_step, 0, 4, st));
  TRY(run_steps(c, kv, STEP_BEAM, nb, n_steps - 1, st));
  const size_t half = (size_t)2 * kv->B * kv->Smax;
  TRY(launch(c, beam_output_kernel, {dim3(kv->B / nb * nrs), dim3(256), 0, st}, (const BeamState*)kv->d_beam,
             (const long long*)kv->beam_tok + half, (const int*)kv->beam_bidx + half, kv->Smax, kv->B, nrs, n_steps,
             (long long)bp->pad_token_id, (long long*)seq_out, scores_out, gen_len_out));
  // the steps after the end of the search did not advance the cache
  return finish_request(kv, n_steps - 1, true, st);
}

extern "C" int vly_kv_beam_reorder(vly_ctx* c, vly_kv* kv, const int32_t* parent_rows, int from_pos, void* stream) {
  if (!c || !kv || !parent_rows || kv->ctx != c || from_pos < 0) return fail(VLY_ERR_INVALID, "vly_kv_beam_reorder: bad argument");
  if (kv->B > kMaxSampleRows) return fail(VLY_ERR_INVALID, "vly_kv_beam_reorder: at most %d rows per cache (%d)", kMaxSampleRows, kv->B);
  TRY(sync_len(kv));
  std::lock_guard<std::mutex> lk(c->mu);
  if (from_pos >= kv->host_len) return VLY_OK;
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  TRY(ensure_beam_buffers(kv));
  TRY(launch(c, set_int_kernel, {dim3(1), dim3(1), 0, st}, (int*)kv->beam_from, from_pos));
  return launch_kv_beam_reorder(c, kv, kv->B, parent_rows, kv->beam_from, nullptr, st);
}

// ------------------------------------------------------------------------------------------------
// shifted cross-entropy over [B,S,V] logits (valley_model.py:308-318)
// ------------------------------------------------------------------------------------------------
extern "C" int vly_cross_entropy(vly_ctx* c, const float* logits, const int64_t* labels, int B, int S, int64_t ignore_index, float* loss_out,
                                 void* stream) {
  if (!c || !logits || !labels || !loss_out || B <= 0 || S < 2) return fail(VLY_ERR_INVALID, "vly_cross_entropy: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const int rows = B * (S - 1);
  TRY(ensure(c->w_score, (size_t)rows * 8));
  float* nll = (float*)c->w_score.p;
  int* cnt = (int*)(nll + rows);
  TRY(launch(c, ce_rows_kernel, {dim3(rows), dim3(256), 0, st}, logits, (const long long*)labels, S, c->cfg.vocab_size, ignore_index, nll,
             cnt));
  return launch(c, ce_mean_kernel, {dim3(1), dim3(1024), 0, st}, nll, cnt, rows, loss_out);
}

// ------------------------------------------------------------------------------------------------
// frame preprocessing (load_video's Resize(256) -> CenterCrop(224) -> /255 -> CLIP mean/std), SURVEY 8 f-2
// ------------------------------------------------------------------------------------------------
extern "C" int vly_preprocess_frames(vly_ctx* c, const uint8_t* frames, int T, int H, int W, int out_dtype, void* out, void* stream) {
  if (!c || !frames || !out || T <= 0 || H <= 0 || W <= 0 || out_dtype < VLY_F32 || out_dtype > VLY_F16)
    return fail(VLY_ERR_INVALID, "vly_preprocess_frames: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  PreprocParams& p = c->pre;
  if (c->pre_H != H || c->pre_W != W) {      // new geometry: rebuild the fixed-point tables on the host (exact, Pillow's arithmetic)
    int nh, nw, cy, cx, kh = 0, kv = 0;
    TRY(vly_preprocess_plan(H, W, &nh, &nw, &cy, &cx));
    TRY(vly_resample_coeffs(W, nw, &kh, nullptr, nullptr, nullptr));
    TRY(vly_resample_coeffs(H, nh, &kv, nullptr, nullptr, nullptr));
    std::vector<int32_t> tab((size_t)nw * (2 + kh) + (size_t)nh * (2 + kv));
    int32_t* xmin = tab.data(); int32_t* xcnt = xmin + nw; int32_t* xk = xcnt + nw;
    int32_t* ymin = xk + (size_t)nw * kh; int32_t* ycnt = ymin + nh; int32_t* yk = ycnt + nh;
    TRY(vly_resample_coeffs(W, nw, &kh, xmin, xcnt, xk));
    TRY(vly_resample_coeffs(H, nh, &kv, ymin, ycnt, yk));
    int row0 = H, row1 = 0;
    for (int y = cy; y < cy + 224; ++y) {
      row0 = std::min(row0, ymin[y]);
      row1 = std::max(row1, ymin[y] + ycnt[y]);
    }
    TRY(ensure(c->w_tables, tab.size() * 4));
    CK(cudaStreamSynchronize(st));           // the previous geometry's tables may still be in use on this stream
    CK(cudaMemcpy(c->w_tables.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
    const int32_t* d = (const int32_t*)c->w_tables.p;
    p.H = H; p.W = W; p.row0 = row0; p.rows = row1 - row0; p.crop_x = cx; p.crop_y = cy; p.ksize_h = kh; p.ksize_v = kv;
    p.xmin_h = d; p.cnt_h = d + nw; p.kk_h = d + 2 * (size_t)nw;
    p.ymin_v = p.kk_h + (size_t)nw * kh; p.cnt_v = p.ymin_v + nh; p.kk_v = p.cnt_v + nh;
    const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f}, sd[3] = {0.26862954f, 0.26130258f, 0.27577711f};   // data_util.py:272-273
    for (int i = 0; i < 3; ++i) { p.mean[i] = mean[i]; p.std[i] = sd[i]; }
    c->pre_H = H; c->pre_W = W;
  }
  TRY(ensure(c->w_strip, (size_t)T * p.rows * 224 * 3));
  p.frames = frames; p.T = T; p.strip = (uint8_t*)c->w_strip.p; p.out = out; p.out_dtype = out_dtype;
  TRY(launch(c, preprocess_horizontal_kernel, {dim3(p.rows, T), dim3(224), 0, st}, p));
  return with_dtype(out_dtype, [&](auto t) {
    return launch(c, preprocess_vertical_kernel<typename decltype(t)::type>, {dim3(224, T), dim3(224), 0, st}, p);
  });
}

// ------------------------------------------------------------------------------------------------
// per-kernel test hooks
// ------------------------------------------------------------------------------------------------
extern "C" int vly_test_gemm(vly_ctx* c, const void* a, const void* w, int M, int N, int K, int epi, const float* bias, const void* residual,
                             void* out, int block_n, const float* colsum, const void* stats_in, int stats_in_nt, float eps, void* stats_out,
                             void* kcache, void* vcache, int S, int past, int Smax, void* stream) {
  if (!c || !a || !w || !out || M <= 0 || N <= 0 || K <= 0 || (K % 8) || (block_n != 128 && block_n != 256))
    return fail(VLY_ERR_INVALID, "vly_test_gemm: bad argument (M %d, N %d, K %d, block_n %d)", M, N, K, block_n);
  const bool norm = epi == EPI_LN_BIAS || epi == EPI_LN_BIAS_GELU || epi == EPI_RMS_QKV_ROPE || epi == EPI_RMS_SWIGLU || epi == EPI_RMS_F32;
  if (norm && (!stats_in || stats_in_nt <= 0))
    return fail(VLY_ERR_INVALID, "vly_test_gemm: epilogue %d needs stats_in and stats_in_nt > 0", epi);
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const bf16 *A = (const bf16*)a, *W = (const bf16*)w;
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.out = out; p.ldo = N; p.bias = bias;
  p.stats_in = (const float2*)stats_in; p.stats_in_nt = stats_in_nt; p.inv_dim = 1.f / K; p.eps = eps;
  switch (epi) {
    case EPI_BIAS:
      return launch_gemm<EPI_BIAS>(c, block_n, A, K, W, K, p, st);
    case EPI_BIAS_RES_STATS:
      if (!residual || (N % 32)) return fail(VLY_ERR_INVALID, "vly_test_gemm: the residual epilogue needs a residual and N %% 32 == 0");
      p.residual = (const bf16*)residual; p.ldr = N; p.stats_out = (float2*)stats_out;
      return launch_gemm<EPI_BIAS_RES_STATS>(c, block_n, A, K, W, K, p, st);
    case EPI_LN_BIAS:
    case EPI_LN_BIAS_GELU:
      if (!colsum) return fail(VLY_ERR_INVALID, "vly_test_gemm: the LayerNorm epilogues need colsum");
      p.colsum = colsum;
      return epi == EPI_LN_BIAS ? launch_gemm<EPI_LN_BIAS>(c, block_n, A, K, W, K, p, st)
                                : launch_gemm<EPI_LN_BIAS_GELU>(c, block_n, A, K, W, K, p, st);
    case EPI_RMS_QKV_ROPE:
      if (!kcache || !vcache || (N % 384) || S <= 0 || (M % S) || past < 0 || past + S > Smax || Smax > c->cfg.max_position_embeddings ||
          !c->rope)
        return fail(VLY_ERR_INVALID, "vly_test_gemm: the QKV epilogue needs K/V caches, N %% 384 == 0, M %% S == 0, "
                    "past + S <= Smax <= max_position_embeddings and a RoPE table (S %d, past %d, Smax %d)", S, past, Smax);
      p.ldo = N / 3; p.rope = c->rope; p.S = S; p.past = past; p.H = N / 3; p.nH = N / 384; p.Smax = Smax;
      p.kcache = (bf16*)kcache; p.vcache = (bf16*)vcache;
      return launch_gemm<EPI_RMS_QKV_ROPE>(c, block_n, A, K, W, K, p, st);
    case EPI_RMS_SWIGLU:
      if (N % 32) return fail(VLY_ERR_INVALID, "vly_test_gemm: the SwiGLU epilogue needs N %% 32 == 0");
      p.ldo = N / 2;
      return launch_gemm<EPI_RMS_SWIGLU>(c, block_n, A, K, W, K, p, st);
    case EPI_RMS_F32:
      return launch_gemm<EPI_RMS_F32>(c, block_n, A, K, W, K, p, st);
  }
  return fail(VLY_ERR_INVALID, "vly_test_gemm: unsupported epilogue %d", epi);
}

extern "C" int vly_test_prefill_attention(vly_ctx* c, const void* q, const void* kcache, const void* vcache, int B, int S, int past, int nH,
                                          int Smax, const uint8_t* key_mask, void* out, void* stream) {
  if (!c || !q || !kcache || !vcache || !out || B <= 0 || S <= 0 || past < 0 || nH <= 0 || Smax <= 0 || (Smax % 128) || past + S > Smax)
    return fail(VLY_ERR_INVALID, "vly_test_prefill_attention: bad argument (B %d, S %d, past %d, heads %d, Smax %d)", B, S, past, nH, Smax);
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const int words = Smax / 32;
  uint32_t* key_bits = nullptr;
  if (key_mask) {
    TRY(ensure(c->w_tprefill, (size_t)B * words * 4));
    key_bits = (uint32_t*)c->w_tprefill.p;
    TRY(launch(c, pack_key_mask_kernel, {dim3(cdiv(words, 128), B), dim3(128), 0, st}, key_mask, past + S, words, key_bits));
  }
  return launch_prefill_attention(c, (const bf16*)q, (const bf16*)kcache, (const bf16*)vcache, Smax, key_bits, B, S, past, nH, (bf16*)out, st);
}

extern "C" int vly_test_vit_attention(vly_ctx* c, const void* qkv, int F, void* out, void* stream) {
  if (!c || !qkv || !out || F <= 0) return fail(VLY_ERR_INVALID, "vly_test_vit_attention: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  return launch_vit_attention(c, (const bf16*)qkv, F, (bf16*)out, (cudaStream_t)stream);
}

extern "C" int vly_test_sample_filter(vly_ctx* c, const float* logits, int B, int V, float temperature, int top_k, float top_p,
                                      uint8_t* keep_out, void* stream) {
  if (!c || !logits || !keep_out || B <= 0 || B > 65535 || V <= 0 || !(temperature > 0.f))
    return fail(VLY_ERR_INVALID, "vly_test_sample_filter: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  SampleState s = {};
  s.temperature = temperature; s.inv_temp = 1.f / temperature; s.enabled = 1; s.filter = 1; s.top_k = top_k; s.top_p = top_p;
  TRY(ensure(c->w_score, sizeof(SampleState)));
  CK(cudaMemcpyAsync(c->w_score.p, &s, sizeof(s), cudaMemcpyHostToDevice, st));
  return launch_sample_filter(c, logits, B, V, (SampleState*)c->w_score.p, nullptr, nullptr, nullptr, nullptr, 0, true, false, keep_out, st);
}

extern "C" int vly_test_logits_process(vly_ctx* c, const float* logits, int B, int V, const int64_t* ids, int L, float penalty,
                                       int ngram, int min_length, int64_t eos, float* out, void* stream) {
  if (!c || !logits || !ids || !out || B <= 0 || B > 65535 || V <= 0 || L <= 0 || !(penalty > 0.f) || ngram < 0 || min_length < 0)
    return fail(VLY_ERR_INVALID, "vly_test_logits_process: bad argument");
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  return launch(c, logits_process_test_kernel, {dim3(B), dim3(1024), proc_map_bytes(V), (cudaStream_t)stream}, logits, V,
                (const long long*)ids, L, penalty, ngram, min_length, (long long)eos, out);
}

extern "C" int vly_test_stop_strings(vly_ctx* c, const vly_sampling* sp, int V, const int64_t* tokens, int B, int n, uint8_t* out,
                                     void* stream) {
  if (!c || !sp || !tokens || !out || V <= 0 || B <= 0 || B > kMaxSampleRows || n <= 0 || sp->n_stop_strings < 1)
    return fail(VLY_ERR_INVALID, "vly_test_stop_strings: bad argument");
  TRY(check_stop_tables(sp, B, "vly_test_stop_strings"));
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const StopLayout l(V);
  Owned<uint8_t> dev, stage;
  TRY(dev.alloc(l.bytes));
  TRY(stage.alloc(l.bytes, true));
  cudaEvent_t ev;
  CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  SampleState s = {};
  int r = upload_stop_tables(sp, 0, V, dev, stage, ev, st);
  if (r == VLY_OK) {
    stop_state(sp, dev, V, s);
    r = launch(c, stop_match_test_kernel, {dim3(B), dim3(32), 0, st}, s, V, (const long long*)tokens, n, s.ring, out);
  }
  const cudaError_t e = cudaStreamSynchronize(st);      // (the scratch buffers are freed on return)
  cudaEventDestroy(ev);
  if (r != VLY_OK) return r;
  if (e != cudaSuccess) return fail(VLY_ERR_CUDA, "vly_test_stop_strings: %s", cudaGetErrorString(e));
  return VLY_OK;
}

// Grow-only scratch whose first `counter_bytes` are work counters: zeroed whenever the buffer is (re)allocated; the kernels
// reset them to zero themselves at the end of every launch.
static int ensure_counters(Mem& b, size_t bytes, size_t counter_bytes, cudaStream_t st) {
  if (b.bytes >= bytes) return VLY_OK;
  TRY(b.alloc(bytes));
  CK(cudaMemsetAsync(b.p, 0, counter_bytes, st));
  return VLY_OK;
}

extern "C" int vly_test_gemv(vly_ctx* c, int mode, const void* w, const void* x, int N, int K, int B, int64_t ldx, float eps,
                             const void* res, void* out, void* kcache, void* vcache, int Smax, int pos, float* logits,
                             int64_t* next_tokens, void* stream) {
  if (!c || !w || !x || (((uintptr_t)w | (uintptr_t)x) & 15) || N <= 0 || K <= 0 || (K % 8) || B <= 0 || B > 4 || ldx < 0 ||
      (ldx % 8) || (ldx > 0 && ldx < K))
    return fail(VLY_ERR_INVALID, "vly_test_gemv: bad argument (N %d, K %d, B %d, ldx %lld)", N, K, B, (long long)ldx);
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  GemvParams p = {};
  p.N = N; p.K = K; p.B = B; p.W = (const bf16*)w; p.x = (const bf16*)x; p.ldx = ldx; p.eps = eps;
  if (mode == GEMV_RESIDUAL) {
    if (!res || !out) return fail(VLY_ERR_INVALID, "vly_test_gemv: the residual mode needs res and out");
    p.res = (const bf16*)res; p.out = (bf16*)out;
    return launch_gemv_ring<GEMV_RESIDUAL>(c, p, false, st);
  }
  if (mode == GEMV_SWIGLU) {
    if (!out || (N % 2)) return fail(VLY_ERR_INVALID, "vly_test_gemv: the SwiGLU mode needs out and an even N");
    p.out = (bf16*)out;
    return launch_gemv_ring<GEMV_SWIGLU>(c, p, false, st);
  }
  // [0] position of the new token (QKV), [1] arg-max counter, [2] step, [3] length; then part_val, part_idx [B, grid]
  const size_t part = (size_t)4 * c->num_sms * 4;
  TRY(ensure_counters(c->w_tgemv, 16 + 2 * part, 16, st));
  int* scal = (int*)c->w_tgemv.p;
  if (mode == GEMV_QKV_ROPE) {
    if (!out || !kcache || !vcache || (N % 384) || Smax <= 0 || pos < 0 || pos >= Smax || !c->rope ||
        pos >= c->cfg.max_position_embeddings)
      return fail(VLY_ERR_INVALID, "vly_test_gemv: the QKV mode needs out, K/V caches, N %% 384 == 0, 0 <= pos < Smax and a RoPE table");
    CK(cudaMemcpyAsync(scal, &pos, sizeof(int), cudaMemcpyHostToDevice, st));
    p.out = (bf16*)out; p.rope = c->rope; p.seq_len = scal; p.H = N / 3; p.nH = N / 384; p.Smax = Smax;
    p.kcache = (bf16*)kcache; p.vcache = (bf16*)vcache;
    return launch_gemv_ring<GEMV_QKV_ROPE>(c, p, false, st);
  }
  if (mode == GEMV_LOGITS) {
    if (!next_tokens) return fail(VLY_ERR_INVALID, "vly_test_gemv: the logits mode needs next_tokens");
    p.logits = logits;
    p.counter = (unsigned int*)scal + 1;
    p.step = scal + 2; p.seq_len_rw = scal + 3; p.bump = 0;
    p.part_val = (float*)((uint8_t*)c->w_tgemv.p + 16);
    p.part_idx = (int*)((uint8_t*)c->w_tgemv.p + 16 + part);
    p.next_tokens = (long long*)next_tokens;
    return launch_gemv_ring<GEMV_LOGITS>(c, p, false, st);
  }
  return fail(VLY_ERR_INVALID, "vly_test_gemv: unknown mode %d", mode);
}

extern "C" int vly_test_decode_attention(vly_ctx* c, const void* q, const void* kcache, const void* vcache, int B, int nH, int Smax,
                                         int len, const uint8_t* key_mask, void* out, void* stream) {
  constexpr int kMaxHeads = 4 * 64;           // counters for up to 4 rows x 64 heads: one per-op step group of the widest LLaMA
  if (!c || !q || !kcache || !vcache || !out || B <= 0 || B > 4 || nH <= 0 || nH > 64 || Smax <= 0 || (Smax % 128) || len <= 0 ||
      len > Smax)
    return fail(VLY_ERR_INVALID, "vly_test_decode_attention: bad argument (B %d, heads %d, Smax %d, len %d)", B, nH, Smax, len);
  std::lock_guard<std::mutex> lk(c->mu);
  CK(cudaSetDevice(c->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const int nsplit = Smax / kDecSplitKeys, words = Smax / 32, bh = B * nH;
  // counters [kMaxHeads], seq_len, then key bits [B, words], part_ml [B*nH, nsplit], part_o [B*nH, nsplit, 128]
  const size_t cnt = kMaxHeads * 4, off_bits = cnt + 16, bits = (size_t)B * words * 4;
  const size_t off_ml = off_bits + ((bits + 15) & ~size_t(15)), off_o = off_ml + (size_t)bh * nsplit * sizeof(float2);
  TRY(ensure_counters(c->w_tattn, off_o + (size_t)bh * nsplit * 128 * 4, cnt, st));
  uint8_t* ws = (uint8_t*)c->w_tattn.p;
  const int old_len = len - 1;
  CK(cudaMemcpyAsync(ws + cnt, &old_len, sizeof(int), cudaMemcpyHostToDevice, st));
  uint32_t* key_bits = (uint32_t*)(ws + off_bits);
  if (key_mask) TRY(launch(c, pack_key_mask_kernel, {dim3(cdiv(words, 128), B), dim3(128), 0, st}, key_mask, len, words, key_bits));
  else CK(cudaMemsetAsync(key_bits, 0xff, bits, st));
  DecAttnParams p = {};
  p.B = B; p.nH = nH; p.H = nH * 128; p.Smax = Smax; p.seq_len = (const int*)(ws + cnt);
  p.q = (const bf16*)q; p.kcache = (const bf16*)kcache; p.vcache = (const bf16*)vcache;
  p.part_o = (float*)(ws + off_o); p.part_ml = (float2*)(ws + off_ml); p.counters = (unsigned int*)ws;
  p.out = (bf16*)out;
  p.key_bits = key_bits; p.mask_words = words;
  return launch_decode_attention(c, p, false, st);
}
