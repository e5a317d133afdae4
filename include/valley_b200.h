/* valley_b200.h -- C ABI of libvalley_b200.so: the H100-native (sm_90a) implementation of Valley's
 * multimodal forward hot path (CLIP ViT-L/14 encode -> temporal pool + mm_projector -> LLaMA decoder
 * with KV cache -> greedy, sampled or beam-searched tokens).
 *
 * The reference (RupertLuo/Valley) has NO FFI / plugin interface: the boundary it offers is the Python
 * nn.Module surface of valley/model/valley_model.py, whose arithmetic is delegated to HuggingFace
 * transformers + ATen.  Each entry point below therefore cites the Python code path it stands in for;
 * valley_b200/model.py re-exposes them under the reference's own class/method names.
 *
 * Conventions
 *   - plain C: opaque handles, raw device pointers + explicit sizes, no C++/torch types.
 *   - every call returns VLY_OK (0) or a negative vly_status; vly_last_error() gives a thread-local message.
 *   - "dev" pointers are CUDA device pointers owned by the caller (e.g. a torch tensor's data_ptr());
 *     the library owns only its packed weights, workspace and KV caches (tied to vly_ctx / vly_kv).
 *   - calls are stream-ordered on the cudaStream_t passed in (void* stream; NULL = legacy default stream).
 *   - there is NO CPU fallback: without a CUDA device of compute capability 9.x vly_create fails.
 *   - hot calls do not allocate once the workspace has grown to the largest shapes seen, so decode steps run
 *     as CUDA graph replays: a KV cache captures a 1-step and an 8-step graph per kind of step (token, filtered
 *     token, beam search step) on the kind's first use, the beam graphs again for another beam count, and
 *     vly_llama_decode, vly_generate(_greedy) and vly_beam_search replay them.  VLY_NO_GRAPH=1 (profiling)
 *     launches the steps eagerly instead.
 *   - thread safety: a vly_ctx serialises its workspace-using calls with an internal mutex
 *     (model_worker.py:467-474 may call the model from up to 5 threads); distinct vly_kv are independent.
 */
#ifndef VALLEY_B200_H_
#define VALLEY_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vly_ctx vly_ctx;
typedef struct vly_kv vly_kv;

typedef enum {
  VLY_OK = 0,
  VLY_ERR_INVALID = -1,          /* bad argument / shape                                          */
  VLY_ERR_CUDA = -2,             /* CUDA runtime / driver failure                                  */
  VLY_ERR_STATE = -3,            /* call order violated (e.g. weights not finalised)               */
  VLY_ERR_IM_COUNT = -10,        /* "The number of im_start_token and im_end_token should be the same" (valley_model.py:219-220) */
  VLY_ERR_IM_CUT = -11,          /* "Seems that the image is cut." (valley_model.py:226-227)       */
  VLY_ERR_INDEX = -12            /* IndexError the reference would raise reading past the ids row  */
} vly_status;

typedef enum { VLY_F32 = 0, VLY_BF16 = 1, VLY_F16 = 2 } vly_dtype;

/* ValleyConfig(LlamaConfig) keys + the CLIPVisionConfig of config.mm_vision_tower (valley_model.py:18-56). */
typedef struct {
  int32_t hidden_size, num_hidden_layers, num_attention_heads, intermediate_size, vocab_size;
  float rms_norm_eps, rope_theta;
  int32_t max_position_embeddings;   /* KV-cache capacity per sequence (model_max_length 2048, valley_stage2.yaml:54) */
  int32_t vit_hidden, vit_layers, vit_heads, vit_mlp, vit_patch, vit_image;
  float vit_eps;
  int32_t mm_vision_select_layer;    /* config.mm_vision_select_layer (default -1, yaml -2; valley_model.py:173) */
  int32_t device;                    /* CUDA device ordinal */
  int32_t patch_pooling_method;      /* vly_pooling: ValleyLlamaModel.patch_pooling_method (valley_model.py:27, :40-52, :205-213) */
} vly_config;

/* 'mean' (default), 'max', 'temporal_importance' (config.use_patch_importance_pooling: model.pooling_layer.{weight,bias}),
 * 'temporal_transformer' (config.use_delta_transformer: model.transformer_delta_encoder.layers.0.* + model.position_matrix) */
typedef enum { VLY_POOL_MEAN = 0, VLY_POOL_MAX = 1, VLY_POOL_TEMPORAL_IMPORTANCE = 2, VLY_POOL_TEMPORAL_TRANSFORMER = 3 } vly_pooling;

/* Sentinel token ids kept on vision_tower.config by every entry point (run_valley.py:13-18). -1 = unset. */
typedef struct {
  int64_t im_patch_token, im_start_token, im_end_token, vi_frame_token, vi_start_token, vi_end_token;
} vly_tokens;

const char* vly_last_error(void);
const char* vly_version(void);

/* ---- lifetime ---- replaces ValleyLlamaForCausalLM.from_pretrained / __init__ (valley_model.py:24-56, :260-267) */
int vly_create(const vly_config* cfg, vly_ctx** out);
void vly_destroy(vly_ctx* ctx);

/* ---- weights ---- accepts HF state_dict names (SURVEY 8b): model.embed_tokens.weight, model.layers.{i}.*,
 * model.norm.weight, lm_head.weight, model.mm_projector.{weight,bias}, model.vision_tower.vision_model.*
 * Data is copied (converted to bf16) immediately; vly_finalize_weights packs the kernel layouts
 * (fused QKV, LayerNorm/RMSNorm gamma folded into the following Linear, RoPE pair interleave,
 * gate/up interleave) and frees the staging copies. */
int vly_load_weight(vly_ctx* ctx, const char* hf_name, const void* dev_ptr, int dtype, const int64_t* shape, int ndim);
int vly_finalize_weights(vly_ctx* ctx);

/* ---- vision tower ---- vision_tower(images, output_hidden_states=True).hidden_states[select_layer]
 * (valley_model.py:172-184; HF modeling_clip.py:202-219, :363-385, :667-690).
 * pixels [F,3,224,224] of pixel_dtype -> out [F,257,1024] bf16.  Only the layers needed are run. */
int vly_vit_encode(vly_ctx* ctx, const void* pixels_dev, int pixel_dtype, int n_frames, int select_layer, void* out_dev,
                   void* stream);

/* ---- fused ViT encode + all-gather of frame features (multi-GPU; BASELINE north_star "all-gather of frame embeddings before
 * projection").  The reference has no inference collective (SURVEY 2.1); torch.distributed/NCCL is the plain path
 * (valley_b200/dist.py); this is the fused one: the LAST ViT layer's fc2+residual epilogue stores every finished tile
 * into the gather buffer of every rank over NVLink (peer-mapped pointers), followed by a flag exchange.
 *   vly_gather_create     : allocate this rank's gather buffer [rows_total, 1024] bf16 (+flags) and export its 64-byte CUDA IPC handle
 *   vly_gather_open_peers : map all ranks' buffers (handles gathered by the caller, e.g. torch.distributed.all_gather_object)
 *   vly_vit_encode_gather : encode n_frames local frames that start at global frame index frame_offset; on return (stream
 *                           order) the local gather buffer holds the features of ALL ranks' frames
 * vly_destroy unmaps the peers' buffers and frees this rank's, which the peers write into: every rank must have finished its
 * last vly_vit_encode_gather before any rank destroys its context. */
int vly_gather_create(vly_ctx* ctx, int64_t rows_total, void** local_buf_dev, void* ipc_handle_out_64B);
int vly_gather_open_peers(vly_ctx* ctx, const void* handles_64B_each, int world, int rank);
int vly_vit_encode_gather(vly_ctx* ctx, const void* pixels_dev, int pixel_dtype, int n_frames, int frame_offset, int select_layer,
                          void* stream);
/* the same with the local frames dealt round-robin: local frame i is global frame frame_offset + i * frame_stride (frame_stride =
 * world size, frame_offset = rank), so every video's frames are spread over all ranks and every rank needs remote frames */
int vly_vit_encode_gather_strided(vly_ctx* ctx, const void* pixels_dev, int pixel_dtype, int n_frames, int frame_offset,
                                  int frame_stride, int select_layer, void* stream);
/* enqueue after the kernels that read the gather buffer: lets the peers overwrite it in their next vly_vit_encode_gather */
int vly_gather_release(vly_ctx* ctx, void* stream);
/* A peer that never signals makes the device-side wait give up after ~10 s and raise a pinned flag in the context; from then on
 * vly_vit_encode_gather / vly_gather_release / vly_gather_status return VLY_ERR_STATE (the buffer holds stale rows).  Call
 * vly_gather_status after the synchronisation that follows a request (non-blocking read): *timed_out = 0 / 1. */
int vly_gather_status(vly_ctx* ctx, int* timed_out);

/* ---- frame preprocessing (SURVEY 8 f-2): what load_video does to the decoded uint8 frames before the vision tower
 * (valley/util/data_util.py:271-281): Resize(256) [PIL.Image.BILINEAR: video_transform.py:63-66 swaps the names] ->
 * CenterCrop(224) -> /255 -> CLIP mean/std.  Bit-exact with the reference (Pillow's 8-bit two-pass fixed-point convolution).
 *   vly_preprocess_plan   : host, exact: resized size (video_transform.py:56-60, :74-81) and crop origin (:542-543).  No GPU.
 *   vly_resample_coeffs   : host, exact: Pillow's precompute_coeffs + normalize_coeffs_8bpc for the triangle filter.
 *                           kk == NULL queries ksize only; else xmin[out], count[out], kk[out * ksize].  No GPU.
 *   vly_preprocess_frames : frames_dev [T,H,W,3] uint8 (decord's get_batch layout, data_util.py:262) -> out_dev [T,3,224,224]
 *                           of out_dtype (frames first, as every caller permutes it: model_worker.py:337, valley_model.py:430). */
int vly_preprocess_plan(int H, int W, int* new_h, int* new_w, int* crop_y, int* crop_x);
int vly_resample_coeffs(int in_size, int out_size, int* ksize_out, int32_t* xmin, int32_t* count, int32_t* kk);
int vly_preprocess_frames(vly_ctx* ctx, const uint8_t* frames_dev, int T, int H, int W, int out_dtype, void* out_dev, void* stream);

/* ---- mm_projector over every token, == encode_images' projection (valley_model.py:187-190):
 * feats [rows,1024] bf16 -> out [rows,hidden] bf16 */
int vly_project(vly_ctx* ctx, const void* feats_dev, int64_t rows, void* out_dev, void* stream);

/* ---- temporal pool + projector (valley_model.py:205-215 + :190), per cfg.patch_pooling_method:
 * feats [n_videos*T,257,1024] bf16 -> vis_rows [n_videos, 256+T, hidden] bf16
 * (rows 0..255 = pooled patch features in LLM space, rows 256.. = projected per-frame CLS features).
 * mean / temporal_importance pool first and project 256+T rows (the projector is linear and the weights sum to one);
 * max / temporal_transformer project all 257*T rows and pool in LLM space, as the reference does. */
int vly_pool_project(vly_ctx* ctx, const void* feats_dev, int n_videos, int T, void* vis_rows_dev, void* stream);

/* ---- splice plan (pure host integer logic, exact; valley_model.py:196-246).  ids_host [B,S] int64.
 * src_map_host [B,S] int32: -1 = keep the token embedding, j in [0,256) = pooled row j, 256+t = frame t's CLS row.
 * img_idx_host [B] int32: which entry of image_features the sample consumes (-1 = not multimodal).
 * Returns VLY_OK or VLY_ERR_IM_COUNT / VLY_ERR_IM_CUT / VLY_ERR_INDEX exactly where the reference raises.  Needs no GPU. */
int vly_build_splice_map(const int64_t* ids_host, int B, int S, int T, const vly_tokens* tok, int32_t* src_map_host,
                         int32_t* img_idx_host);

/* ---- embed_tokens gather + splice (valley_model.py:160, :223-247): -> inputs_embeds [B,S,hidden] bf16 */
int vly_embed_splice(vly_ctx* ctx, const int64_t* ids_dev, const int32_t* src_map_dev, const int32_t* img_idx_dev,
                     const void* vis_rows_dev, int rows_per_img, int B, int S, void* inputs_embeds_dev, void* stream);

/* ---- KV cache ---- replaces HF DynamicCache / the tuple cache (cache_utils.py:102-120): pre-allocated
 * [L][2][B][heads][max_seq][128] bf16, appended in place by the QKV epilogues. */
int vly_kv_create(vly_ctx* ctx, int batch, int max_seq, vly_kv** out);
void vly_kv_destroy(vly_kv* kv);
int vly_kv_seq_len(vly_kv* kv, int* out_len);   /* host-visible length (syncs the kv's stream state) */
/* which kernel a decode step of this cache launches ("decode_step_kernel<1>", "per-op TMA-ring decode kernels", ...): written,
 * NUL-terminated, into name (capacity cap).  For reports (bench.py names the kernel its roofline describes); no GPU work. */
int vly_kv_decode_kernel(vly_kv* kv, char* name, int cap);
int vly_kv_reset(vly_kv* kv, void* stream);
/* HF's 2-D attention_mask (HF masking_utils: the padding mask is AND-ed into the causal mask; build_inputs /
 * tokenizer(padding=True) pad on the LEFT, valley_model.py:249-254 passes the mask through): mask_dev [B, len] uint8 on the
 * device, 0 = cache position k of sequence b must never be attended.  Covers cache positions [0, len) -- set it before the
 * prefill that appends them; later positions (decode) are attendable.  Position ids are NOT shifted by padding (the
 * reference never passes position_ids, SURVEY Appendix A.8).  len = 0 clears the mask; vly_kv_reset clears it too. */
int vly_kv_set_key_mask(vly_kv* kv, const uint8_t* mask_dev, int len, void* stream);
/* copy layer l's K (which=0) or V (which=1) as HF-layout [B,heads,len,128] bf16 (de-interleaves K) -- for tests/drop-in */
int vly_kv_export(vly_ctx* ctx, vly_kv* kv, int layer, int which, void* out_dev, void* stream);

/* ---- LlamaModel.forward + lm_head on S new positions (valley_model.py:249-254, :304-305;
 * HF modeling_llama.py:375-426).  inputs_embeds [B,S,hidden] bf16.
 * logits_mode 0: none; 1: last position only -> logits_dev [B,V] fp32; 2: all positions -> [B,S,V] fp32.
 * hidden_out_dev (optional) receives the final-norm'ed hidden states is NOT provided: norm is folded into lm_head. */
int vly_llama_prefill(vly_ctx* ctx, vly_kv* kv, const void* inputs_embeds_dev, int B, int S, int logits_mode,
                      void* logits_dev, int64_t* next_tokens_dev, void* stream);

/* ---- one decode step for B sequences (model_worker.py:380-391): tokens_dev [B] int64 -> next_tokens_dev [B]
 * int64 = argmax (lowest index on ties); logits_dev optional [B,V] fp32. */
int vly_llama_decode(vly_ctx* ctx, vly_kv* kv, const int64_t* tokens_dev, int64_t* next_tokens_dev, void* logits_dev,
                     void* stream);

/* ---- n_steps greedy decode steps with no host round trip (CUDA graph replay): first_tokens_dev [B] is fed at step 0,
 * step i's argmax is fed to step i+1; out_tokens_dev [B, n_steps] int64 receives every argmax. */
int vly_generate_greedy(vly_ctx* ctx, vly_kv* kv, const int64_t* first_tokens_dev, int n_steps, int64_t* out_tokens_dev,
                        void* stream);

/* ---- loss of a forward with labels (SURVEY 8 f-4; valley_model.py:308-318): shift by one, CrossEntropyLoss() = mean of
 * logsumexp(logits[b,s,:]) - logits[b,s,labels[b,s+1]] over the labels != ignore_index (-100).  logits_dev [B,S,V] fp32
 * (vly_llama_prefill logits_mode 2), labels_dev [B,S] int64, loss_out_dev one fp32 (nan when no label counts, like torch). */
int vly_cross_entropy(vly_ctx* ctx, const float* logits_dev, const int64_t* labels_dev, int B, int S, int64_t ignore_index,
                      float* loss_out_dev, void* stream);

/* ---- token selection on the device (SURVEY 8 f-1; model_worker.py:388-397; HF generate as called at valley_model.py:432) ----
 * temperature < 1e-4: arg-max (model_worker.py:390-391); otherwise multinomial(softmax(logits / temperature)) (:392-395), drawn
 * with the Gumbel-max identity from counter-based Philox noise keyed by `seed` -- fused into the arg-max epilogue of the decode
 * step, so sampling costs no extra pass and no host round trip.  eos_token_id >= 0: a row that emits it is finished (:396-397);
 * finished rows emit pad_token_id (HF generate) and once every row has finished the remaining steps are skipped.
 * top_k / top_p (HF generate's TopKLogitsWarper / TopPLogitsWarper, applied after the temperature and only when sampling):
 * with s = logits / temperature, top_k keeps the tokens whose s is >= the k-th largest s (ties kept; k >= V keeps all);
 * top_p then keeps, among those, every token whose score has less than top_p of the softmax mass strictly above it (the
 * maximum is always kept; a tie group at the cut is kept whole).  The token is the same Gumbel-max draw restricted to the kept
 * set, so a filter that keeps everything draws what the unfiltered sampler draws.  With a filter on, one more kernel per step
 * (one CTA per row over the step's logits) makes the selection.  Zero-initialised fields mean no filter. */
typedef struct {
  float temperature;
  uint64_t seed;
  int64_t eos_token_id;      /* -1: none */
  int64_t pad_token_id;
  int64_t stop_token_id;     /* -1: none; a second id that ends a row: the worker's single-token stop string (model_worker.py:355-360, :396-397) */
  int32_t top_k;             /* <= 0: off */
  float top_p;               /* off unless 0 < top_p < 1 */
  /* Stop strings: transformers' StopStringCriteria (generate(stop_strings=...)), matched on the device after each token is
   * selected.  A row whose text -- the concatenation of its tokens' clean strings -- ends with a stop string, the last
   * characters inside the newest token, is finished; so is a row that emits a token of pause_bits.  A finished row emits
   * pad_token_id afterwards only when eos_token_id or stop_token_id is set (HF pads only with an eos criterion); the remaining
   * steps are skipped once every row has finished.  The tables are built by valley_b200/stop_strings.py (stop_tables); V is
   * the context's vocab_size.  Every host array is copied before the call returns.  At most 64 rows.  Zero: no stop strings. */
  int32_t n_stop_strings;          /* 0..8 */
  const int32_t* stop_lens;        /* host [n_stop_strings]: characters of each stop string, 1..64 */
  const uint64_t* stop_masks;      /* host [n_stop_strings][V][2]: per token, the end mask (bit L-1: the token can be the last one
                                    * with the last L characters of the string inside it, trailing characters allowed) and the
                                    * position mask (bit p: the token fits with its end p characters before the string's end) */
  const int32_t* stop_token_lens;  /* host [V]: each token's clean-string length */
  const uint32_t* pause_bits;      /* host [ceil(V / 32)] bit set of tokens that finish a row as a match does, or NULL */
  const int64_t* stop_tail;        /* host [B][stop_tail_len]: each row's last tokens before its first selected token */
  int32_t stop_tail_len;           /* 0..63 */
  int32_t stop_restart;            /* vly_generate: 1 = start the matcher here (upload the tables, seed the rows from stop_tail
                                    * and clear the finished flags); 0 = continue the request vly_sample_logits started.
                                    * vly_sample_logits always starts it. */
  /* Logits processors (transformers 5.5's RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor and
   * MinLengthLogitsProcessor, in that order, before the temperature and the top-k / top-p filter), over each row's input_ids as
   * HF holds them: the cache's tokens (prompt_ids_dev), then every emitted token (pad_token_id once the row finished).
   *   repetition_penalty > 0: the score s of every id in the row becomes s * penalty if s < 0, else s / penalty (IEEE fp32);
   *   no_repeat_ngram_size n > 0: every token that followed an earlier occurrence of the row's last n - 1 ids scores -inf;
   *   min_length > 0 (with eos_token_id >= 0): eos scores -inf while the row holds fewer than min_length ids.
   * scores_out records the processed scores (then tempered and filtered); logits_out stays raw.  The row histories live in a
   * buffer the cache allocates on its first processor request and keeps.  A request with processors selects in the
   * filtered-token step (one more kernel per step at B <= 4).  Zero fields (and a penalty of 1) mean off.
   * prompt_ids_dev: device [B, cache length] int64, read when a request starts (vly_sample_logits, or stop_restart).
   * vly_generate with processors must continue the processor request vly_sample_logits started (VLY_ERR_STATE otherwise). */
  float repetition_penalty;
  int32_t no_repeat_ngram_size;
  int32_t min_length;
  const int64_t* prompt_ids_dev;
  /* Recording (HF generate's output_scores / output_logits): device buffers [n_slots, B, V] fp32 owned by the caller, or NULL.
   * vly_sample_logits writes slot 0; vly_generate writes slot i for its step i (pass pointers offset by one slot to continue
   * the request vly_sample_logits started).  scores_out: the scores the token is selected from -- logits / temperature when
   * temperature > 0 (the raw logits when it is 0), with -inf at every token the top-k / top-p filter removed; logits_out:
   * the raw logits.  Every row is recorded, finished ones too; nothing is recorded after every row has finished.  A request
   * that records selects in the filtered-token step (one more kernel per step at B <= 4).  NULL: nothing is recorded. */
  float* scores_out;
  float* logits_out;
} vly_sampling;

/* the first generated token: select from the prefill's last-position logits [B,V] fp32 (vly_llama_prefill logits_mode 1);
 * starts a generation (clears the finished flags). */
int vly_sample_logits(vly_ctx* ctx, vly_kv* kv, const float* logits_dev, const vly_sampling* sampling, int64_t* tokens_out_dev,
                      void* stream);
/* vly_generate_greedy with token selection per `sampling` (NULL = greedy, no stop token).  steps_done_dev (optional, device
 * int32) receives the number of steps actually executed: n_steps, or fewer when every row reached eos -- columns
 * [0, steps_done) of out_tokens_dev are valid. */
int vly_generate(vly_ctx* ctx, vly_kv* kv, const int64_t* first_tokens_dev, int n_steps, int64_t* out_tokens_dev,
                 const vly_sampling* sampling, int* steps_done_dev, void* stream);

/* ---- beam search (HF generate with num_beams > 1, do_sample=False: transformers' GenerationMixin._beam_search) ----
 * The cache holds B = items * num_beams rows, each item's beams prefilled with the same prompt (HF's
 * _expand_inputs_for_generation).  Per step, on the device: log_softmax of every beam row + the running beam scores; the top
 * 2 * num_beams of the num_beams * V candidates (ties: lowest flat index); a candidate hits the stopping criteria when its
 * token is eos or at the last of n_steps steps; the next running beams are the best num_beams candidates that did not hit;
 * the finished hypotheses keep the best num_beams by score / generated_len ** length_penalty under HF's early_stopping rules;
 * the KV rows follow their parent beams (positions after the prompt only).  The search ends as HF's does, and the remaining
 * graph replays then exit at once.  log_softmax uses a float64 log-sum-exp (within an ulp of the fp32 one). */
typedef struct {
  int32_t num_beams;             /* 1..8, divides the cache's rows                                              */
  int32_t num_return_sequences;  /* 1..num_beams: the best finished hypotheses returned per item                 */
  float length_penalty;          /* HF default 1.0                                                              */
  int32_t early_stopping;        /* 0: False (HF default), 1: True, 2: "never"                                  */
  int64_t eos_token_id;          /* -1: none                                                                    */
  int64_t pad_token_id;          /* written beyond each sequence's end (HF's output_fill_value)                  */
  /* Recording (HF's output_scores / output_logits / beam_indices), device buffers owned by the caller, or NULL:
   *   scores_out / logits_out [n_steps, B, V] fp32: slot t = search step t (the first one selects from first_logits_dev):
   *     HF's log_probs (log_softmax of every beam row, float64 log-sum-exp, before the beam scores are added) / the raw logits;
   *   beam_indices_out [B / num_beams * num_return_sequences, n_steps] int64: per returned hypothesis and step, the cache row
   *     (item * num_beams + beam) the token was appended to, -1 from the hypothesis' generated length on;
   *   steps_out (one int32): the search steps run (HF's len(scores)).
   * The library allocates nothing per request for these; the beam-index rows it keeps on the device are allocated with the
   * cache's other beam buffers, on its first beam request. */
  float* scores_out;
  float* logits_out;
  int64_t* beam_indices_out;
  int32_t* steps_out;
} vly_beam;

/* Beam search after the prefill of the prompt_len-token prompt (the cache's length): the first step selects from
 * first_logits_dev [B, V] fp32 (vly_llama_prefill logits_mode 1), each of the following n_steps - 1 steps is one CUDA-graph
 * replay of decode step + beam_step_kernel + kv_beam_reorder_kernel.  Outputs, for item i and its r-th best hypothesis in
 * row i * num_return_sequences + r: seq_out_dev [., n_steps] int64 (generated tokens, pad_token_id after the end),
 * scores_out_dev [.] fp32 (HF's sequences_scores), gen_len_out_dev [.] int32 (generated length).  No host synchronisation. */
int vly_beam_search(vly_ctx* ctx, vly_kv* kv, const vly_beam* params, const float* first_logits_dev, int prompt_len, int n_steps,
                    int64_t* seq_out_dev, float* scores_out_dev, int* gen_len_out_dev, void* stream);
/* HF's Cache.reorder_cache(beam_idx) for positions [from_pos, length): every layer's K and V row r takes row
 * parent_rows_dev[r] (device int32 [B], any row of the cache), in place. */
int vly_kv_beam_reorder(vly_ctx* ctx, vly_kv* kv, const int32_t* parent_rows_dev, int from_pos, void* stream);

/* ---- introspection for bench / tests ---- */
int vly_kernel_launch_count(vly_ctx* ctx, int64_t* out);   /* kernels launched by this ctx so far */
/* bytes of device memory and of pinned host memory the library holds right now, summed over every context and KV cache of
 * the process (packed and staged weights, workspace, caches, gather buffers) */
int vly_held_bytes(int64_t* device_bytes, int64_t* pinned_bytes);
int vly_num_sms(vly_ctx* ctx, int* out);

/* in-kernel cycle counters of kv's last decode step (tools/bench_decode.py): copies n int64 values to host_out.  Only a
 * cache created with VLY_MEGA_DBG set, at B <= 4, has them (VLY_ERR_STATE otherwise); VLY_ERR_INVALID when n exceeds the
 * cache's 8192 values. */
int vly_kv_debug_counters(vly_kv* kv, long long* host_out, int n);
/* internal: lets the host-only translation units (host_splice.cpp, host_preprocess.cpp) set the thread-local error message */
void vly_set_error_(const char* message);

/* ---- low-level op hooks (per-kernel parity tests; SURVEY section 4) ----
 * One prefill / ViT GEMM through the launcher production uses: acc[M,N] = A[M,K] * W[N,K]^T (bf16, K a multiple of 8, fp32
 * accumulation) in 128 x block_n tiles (block_n 128 or 256), then the fused epilogue epi.  bias_dev / colsum_dev are fp32 [N].
 * The normalising epilogues (1, 2, 4, 5, 6) read stats_in_dev [M, stats_in_nt] float2 partial (sum, sumsq) of the rows of A
 * and form mean = sum / K, rstd = 1 / sqrt(sumsq / K - mean^2 + eps) (LayerNorm) or rstd = 1 / sqrt(sumsq / K + eps) (RMSNorm).
 *   0 bias:                 out [M,N] bf16 = acc (+ bias)
 *   1 LayerNorm + bias:     out [M,N] bf16 = rstd * (acc - mean * colsum) + bias
 *   2 ... + quick_gelu:     out [M,N] bf16 = quick_gelu(rstd * (acc - mean * colsum) + bias)
 *   3 bias + residual:      out [M,N] bf16 = acc (+ bias) + residual_dev [M,N] (in place allowed), N a multiple of 32;
 *                           stats_out_dev (or NULL) [M, ceil(N / block_n)] float2 = per-tile (sum, sumsq) of the bf16 outputs
 *   4 RMSNorm + QKV + RoPE: rows [q | k | v] of nH = N / 384 heads in pair-interleaved RoPE order; row m of A is token
 *                           (b = m / S, s = m % S) at position past + s (M a multiple of S, past + S <= Smax <=
 *                           max_position_embeddings); rstd * acc rotated by the context's RoPE table: q -> out [M, N/3],
 *                           k / v -> row past + s of kcache_dev / vcache_dev [M/S, nH, Smax, 128]
 *   5 RMSNorm + SwiGLU:     columns (2j, 2j+1) = (gate j, up j), N a multiple of 32: out [M, N/2] bf16 = silu(g) * u with
 *                           g = rstd * acc[2j], u = rstd * acc[2j+1] (neither rounded to bf16)
 *   6 RMSNorm, fp32:        out [M,N] fp32 = rstd * acc
 * Arguments an epilogue does not use may be NULL / 0. */
int vly_test_gemm(vly_ctx* ctx, const void* a_dev, const void* w_dev, int M, int N, int K, int epi, const float* bias_dev,
                  const void* residual_dev, void* out_dev, int block_n, const float* colsum_dev, const void* stats_in_dev,
                  int stats_in_nt, float eps, void* stats_out_dev, void* kcache_dev, void* vcache_dev, int S, int past, int Smax,
                  void* stream);
/* one layer's causal prefill attention, through the launcher the prefill uses: q_dev [B*S, nH*128] bf16 (RoPE pair-interleaved
 * like the cache's keys), kcache_dev / vcache_dev [B, nH, Smax, 128] bf16 (Smax a multiple of 128) holding keys [0, past + S),
 * key_mask_dev [B, past + S] uint8 (0 = key never attended) or NULL -> out_dev [B*S, nH*128] bf16: query s of row b, at position
 * past + s, = softmax(q k^T / sqrt(128)) v over the attended keys at positions <= past + s (0 when none is attended). */
int vly_test_prefill_attention(vly_ctx* ctx, const void* q_dev, const void* kcache_dev, const void* vcache_dev, int B, int S,
                               int past, int nH, int Smax, const uint8_t* key_mask_dev, void* out_dev, void* stream);
/* ViT attention on a packed qkv [F*257, 3072] bf16 -> ctx [F*257,1024] bf16 */
int vly_test_vit_attention(vly_ctx* ctx, const void* qkv_dev, int n_frames, void* out_dev, void* stream);
/* the top-k / top-p filter of vly_sampling over logits [B,V] fp32 (any V): keep_out [B,V] uint8 = 1 where the token is kept,
 * computed by the same device routine the decode loop selects with.  temperature > 0; top_k / top_p as in vly_sampling. */
int vly_test_sample_filter(vly_ctx* ctx, const float* logits_dev, int B, int V, float temperature, int top_k, float top_p,
                           uint8_t* keep_out_dev, void* stream);
/* the logits processors of vly_sampling alone, by the device routine the decode loop selects with: out_dev [B,V] fp32 = the
 * processed scores of logits_dev [B,V] fp32 (any V) for input_ids ids_dev [B,L] int64.  penalty > 0 (1: off), ngram >= 0
 * (0: off), min_length >= 0 with eos (< 0: off) as in vly_sampling. */
int vly_test_logits_process(vly_ctx* ctx, const float* logits_dev, int B, int V, const int64_t* ids_dev, int L, float penalty,
                            int ngram, int min_length, int64_t eos, float* out_dev, void* stream);
/* the stop-string matcher of vly_sampling alone: with the stop-string fields of `sampling` (tables over a vocabulary of V
 * tokens; the tail and pause fields are not used), out_dev[b] (uint8) = 1 when row b of tokens_dev [B, n] int64, read as a
 * row whose newest token is the last, matches.  B <= 64.  Synchronises the stream. */
int vly_test_stop_strings(vly_ctx* ctx, const vly_sampling* sampling, int V, const int64_t* tokens_dev, int B, int n,
                          uint8_t* out_dev, void* stream);
/* one weight-streaming GEMV of the per-op decode step, through the launcher the step uses: y[b,n] = sum_k x[b,k] W[n,k] with
 * W [N,K] bf16, x [B,K] bf16 of row stride ldx (0 = K), B <= 4, K and ldx multiples of 8, W and x 16-byte aligned.  rstd[b] = 1/sqrt(mean_k x[b,k]^2 + eps)
 * (the RMSNorm whose gamma is folded into W).  mode:
 *   0 QKV + RoPE: rows in pair-interleaved RoPE order, N = 3 * nH * 128; rstd * y rotated by the RoPE table of the context at
 *     position pos (0 <= pos < Smax): q -> out_dev [B, N/3]; k / v -> row pos of kcache_dev / vcache_dev [B, nH, Smax, 128]
 *   1 residual: out_dev [B,N] = bf16(y + res_dev) (in place allowed)
 *   2 SwiGLU: rows (2j, 2j+1) = (gate j, up j): out_dev [B,N/2] = silu(bf16(rstd*gate)) * bf16(rstd*up)
 *   3 logits: logits_dev [B,N] fp32 (or NULL) = rstd * y; next_tokens_dev [B] int64 = arg-max (lowest index on ties)
 * Arguments a mode does not use may be NULL / 0. */
int vly_test_gemv(vly_ctx* ctx, int mode, const void* w_dev, const void* x_dev, int N, int K, int B, int64_t ldx, float eps,
                  const void* res_dev, void* out_dev, void* kcache_dev, void* vcache_dev, int Smax, int pos, float* logits_dev,
                  int64_t* next_tokens_dev, void* stream);
/* the per-op decode step's attention, through the launcher the step uses: q_dev [B, nH*128] bf16 (RoPE pair-interleaved like the
 * cache's keys), kcache_dev / vcache_dev [B, nH, Smax, 128] bf16 (Smax a multiple of 128), keys [0, len) with the newest at
 * len - 1, key_mask_dev [B, len] uint8 (0 = key never attended) or NULL -> out_dev [B, nH*128] bf16 = softmax(q k^T / sqrt(128)) v
 * over the attended keys.  B <= 4, nH <= 64. */
int vly_test_decode_attention(vly_ctx* ctx, const void* q_dev, const void* kcache_dev, const void* vcache_dev, int B, int nH,
                              int Smax, int len, const uint8_t* key_mask_dev, void* out_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VALLEY_B200_H_ */
