"""Reference-facing Python surface: the same class / method names, argument meaning and error
behaviour as valley/model/valley_model.py, with every tensor op executed by libvalley_b200.so.

    ValleyConfig                      valley_model.py:18
    ValleyLlamaModel                  valley_model.py:21   (.vision_tower.config sentinel ids, .forward)
    ValleyLlamaForCausalLM            valley_model.py:257  (.forward, .get_model, .generate,
                                      .prepare_inputs_for_generation, .build_inputs, .process_response)
  + encode_images / prepare_inputs_labels_for_multimodal: the two inline blocks valley_model.py:163-190
    and :192-247 factored out under the names BASELINE.json's north_star uses (SURVEY.md 0.3).

PyTorch is used here only for device memory, streams and (optionally) sampling; there is no
eager / CPU fallback for any op on the path.
"""
from __future__ import annotations

import os
import ctypes as C
import types
from typing import Iterable, List, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib
from . import beam as _beam
from . import processors as _proc
from . import stop_strings as _ss
from ._lib import VlyBeam, VlySampling, VlyConfig, VlyTokens, check

# valley/util/config.py:1-13
IGNORE_INDEX = -100
DEFAULT_IMAGE_PATCH_TOKEN = "<im_patch>"
DEFAULT_IM_START_TOKEN = "<im_start>"
DEFAULT_IM_END_TOKEN = "<im_end>"
DEFAULT_VIDEO_FRAME_TOKEN = "<vi_frame>"
DEFAULT_VI_START_TOKEN = "<vi_start>"
DEFAULT_VI_END_TOKEN = "<vi_end>"

_DT = {torch.float32: _lib.VLY_F32, torch.bfloat16: _lib.VLY_BF16, torch.float16: _lib.VLY_F16}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class ValleyConfig:
    """ValleyConfig(LlamaConfig), model_type 'valley' (valley_model.py:18-19) plus the extra keys the reference
    reads: mm_vision_tower, use_mm_proj, mm_hidden_size, mm_vision_select_layer, mm_use_im_start_end,
    use_patch_importance_pooling / use_delta_transformer (:40-52; the pooling variant is fixed at construction, as in the
    reference -- ``patch_pooling_method="max"`` stands for setting that attribute on the reference model)."""
    model_type = "valley"

    def __init__(self, hidden_size=4096, num_hidden_layers=32, num_attention_heads=32, intermediate_size=11008,
                 vocab_size=32008, rms_norm_eps=1e-5, rope_theta=10000.0, max_position_embeddings=2048,
                 mm_vision_tower="openai/clip-vit-large-patch14", mm_hidden_size=1024, mm_vision_select_layer=-2,
                 use_mm_proj=True, mm_use_im_start_end=True, vit_layers=24, vit_heads=16, vit_mlp=4096, vit_patch=14,
                 vit_image=224, vit_eps=1e-5, use_patch_importance_pooling=False, use_delta_transformer=False,
                 patch_pooling_method=None, bos_token_id=1, eos_token_id=2, pad_token_id=None, **kw):
        self.hidden_size, self.num_hidden_layers = hidden_size, num_hidden_layers
        self.num_attention_heads, self.intermediate_size = num_attention_heads, intermediate_size
        self.vocab_size, self.rms_norm_eps, self.rope_theta = vocab_size, rms_norm_eps, rope_theta
        self.max_position_embeddings = max_position_embeddings
        self.mm_vision_tower, self.mm_hidden_size = mm_vision_tower, mm_hidden_size
        self.mm_vision_select_layer, self.use_mm_proj = mm_vision_select_layer, use_mm_proj
        self.mm_use_im_start_end = mm_use_im_start_end
        self.vit_layers, self.vit_heads, self.vit_mlp = vit_layers, vit_heads, vit_mlp
        self.vit_patch, self.vit_image, self.vit_eps = vit_patch, vit_image, vit_eps
        self.use_patch_importance_pooling, self.use_delta_transformer = use_patch_importance_pooling, use_delta_transformer
        if patch_pooling_method is None:          # valley_model.py:27, :40-52: the later flag wins
            patch_pooling_method = "temporal_transformer" if use_delta_transformer else (
                "temporal_importance" if use_patch_importance_pooling else "mean")
        if patch_pooling_method not in _lib.POOLING:
            raise ValueError(f"patch_pooling_method {patch_pooling_method!r} not in {sorted(_lib.POOLING)}")
        self.patch_pooling_method = patch_pooling_method
        # LlamaConfig defaults (HF:configuration_llama.py); HF generate() stops on config.eos_token_id unless told otherwise
        self.bos_token_id, self.eos_token_id, self.pad_token_id = bos_token_id, eos_token_id, pad_token_id
        self.use_return_dict, self.use_cache = True, True
        self.output_attentions = self.output_hidden_states = False
        for k, v in kw.items():
            setattr(self, k, v)

    @classmethod
    def from_spec(cls, spec, **kw):
        return cls(hidden_size=spec.hidden_size, num_hidden_layers=spec.num_hidden_layers,
                   num_attention_heads=spec.num_attention_heads, intermediate_size=spec.intermediate_size,
                   vocab_size=spec.vocab_size, rms_norm_eps=spec.rms_norm_eps, rope_theta=spec.rope_theta,
                   max_position_embeddings=spec.max_position_embeddings, mm_hidden_size=spec.vit_hidden,
                   mm_vision_select_layer=spec.mm_vision_select_layer, vit_layers=spec.vit_layers,
                   vit_heads=spec.vit_heads, vit_mlp=spec.vit_mlp, vit_patch=spec.vit_patch,
                   vit_image=spec.vit_image, vit_eps=spec.vit_eps,
                   patch_pooling_method=getattr(spec, "patch_pooling_method", "mean"),
                   **{"eos_token_id": None, **kw})          # synthetic specs have no eos: random-init ids must not stop a run


class CausalLMOutputWithPast(dict):
    """Attribute + index access like transformers.modeling_outputs.CausalLMOutputWithPast."""

    def __init__(self, loss=None, logits=None, past_key_values=None, hidden_states=None, attentions=None):
        super().__init__(loss=loss, logits=logits, past_key_values=past_key_values,
                         hidden_states=hidden_states, attentions=attentions)
        self.__dict__ = self

    def __getitem__(self, k):
        if isinstance(k, int):
            return [v for v in (self.loss, self.logits, self.past_key_values) if v is not None][k]
        return dict.__getitem__(self, k)


class _GenerateOutput(dict):
    """The surface of transformers' ``ModelOutput`` for generate()'s output classes: attribute, key and integer-index access.
    Fields that are None are attributes only: ``keys()``, integer indices and ``to_tuple()`` skip them, as in transformers."""
    _fields: Tuple[str, ...] = ()

    def __init__(self, **kw):
        unknown = set(kw) - set(self._fields)
        if unknown:
            raise TypeError(f"{type(self).__name__} has no field(s) {sorted(unknown)}")
        super().__init__((k, kw[k]) for k in self._fields if kw.get(k) is not None)
        self.__dict__.update({k: kw.get(k) for k in self._fields})

    def __getitem__(self, k):
        if isinstance(k, str):
            return dict.__getitem__(self, k)
        return self.to_tuple()[k]

    def to_tuple(self) -> tuple:
        return tuple(dict.__getitem__(self, k) for k in self._fields if k in self)


class GenerateDecoderOnlyOutput(_GenerateOutput):
    """transformers' ``GenerateDecoderOnlyOutput``: generate(return_dict_in_generate=True) with num_beams == 1."""
    _fields = ("sequences", "scores", "logits", "attentions", "hidden_states", "past_key_values")


class GenerateBeamDecoderOnlyOutput(_GenerateOutput):
    """transformers' ``GenerateBeamDecoderOnlyOutput``: generate(return_dict_in_generate=True) with num_beams > 1."""
    _fields = ("sequences", "sequences_scores", "scores", "logits", "beam_indices", "attentions", "hidden_states",
               "past_key_values")


def generation_output(sequences, steps: int, scores=None, logits=None, sequences_scores=None, beam_indices=None, beam=False):
    """generate()'s output object from what a request recorded: ``scores`` / ``logits`` are buffers [>= steps, rows, V] (or
    None when not asked for) of which the first ``steps`` slots were written; they become HF's per-step tuples (views)."""
    per_step = lambda buf: None if buf is None else tuple(buf[i] for i in range(steps))
    if beam:
        return GenerateBeamDecoderOnlyOutput(sequences=sequences, sequences_scores=sequences_scores, scores=per_step(scores),
                                             logits=per_step(logits), beam_indices=beam_indices)
    return GenerateDecoderOnlyOutput(sequences=sequences, scores=per_step(scores), logits=per_step(logits))


class _ShapeOnly:
    def __init__(self, shape):
        self.shape = torch.Size(shape)


class ValleyKVCache:
    """Opaque KV cache returned as ``past_key_values``.  Supports both access patterns callers use:
    ``past_key_values[0][0].shape[-2]`` (model_worker.py:253, :381, pinned-HF tuple cache) and
    ``.get_seq_length()`` (HF >= 4.36 DynamicCache).  Storage is the library's pre-allocated
    [L][2][B][heads][max_seq][128] bf16 buffer, appended in place by the QKV epilogues."""

    def __init__(self, model: "ValleyLlamaForCausalLM", batch: int, max_seq: int):
        self._model, self.batch, self.max_seq = model, batch, max_seq
        h = model._pop_handle(batch, max_seq)            # a handle (allocation + captured CUDA graph) freed by an earlier cache
        if h is None:
            h = C.c_void_p()
            check(model._lib.vly_kv_create(model._ctx, batch, max_seq, C.byref(h)))
        else:
            check(model._lib.vly_kv_reset(h, _stream()))
        self._h = h

    def get_seq_length(self, layer_idx: int = 0) -> int:
        n = C.c_int()
        check(self._model._lib.vly_kv_seq_len(self._h, C.byref(n)))
        return n.value

    def decode_kernel(self) -> str:
        """name of the kernel a decode step of this cache launches (for reports)"""
        buf = C.create_string_buffer(96)
        check(self._model._lib.vly_kv_decode_kernel(self._h, buf, 96))
        return buf.value.decode()

    def __len__(self):
        return self._model.config.num_hidden_layers

    def __bool__(self):
        return True

    def __getitem__(self, layer):
        c = self._model.config
        shp = (self.batch, c.num_attention_heads, self.get_seq_length(), c.hidden_size // c.num_attention_heads)
        return (_ShapeOnly(shp), _ShapeOnly(shp))

    def to_hf(self, layer: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """Materialise layer's (key, value) in HuggingFace layout [B, heads, len, 128] (keys de-interleaved)."""
        c, n = self._model.config, self.get_seq_length()
        out = []
        for which in (0, 1):
            t = torch.empty(self.batch, c.num_attention_heads, n, 128, dtype=torch.bfloat16, device=self._model.device)
            check(self._model._lib.vly_kv_export(self._model._ctx, self._h, layer, which, t.data_ptr(), _stream()))
            out.append(t)
        return tuple(out)

    def reset(self):
        check(self._model._lib.vly_kv_reset(self._h, _stream()))

    def reorder_cache(self, beam_idx: torch.Tensor, from_pos: int = 0):
        """HF's ``Cache.reorder_cache(beam_idx)``: row r of every layer's keys and values becomes row ``beam_idx[r]``, in place
        on the device.  Positions before ``from_pos`` are left alone (a beam search's prompt rows are identical)."""
        idx = beam_idx.to(self._model.device, torch.int32).contiguous()
        if idx.shape != (self.batch,):
            raise ValueError(f"beam_idx shape {tuple(idx.shape)} != ({self.batch},)")
        check(self._model._lib.vly_kv_beam_reorder(self._model._ctx, self._h, idx.data_ptr(), int(from_pos), _stream()))

    def set_attention_mask(self, attention_mask: Optional[torch.Tensor], total_len: int):
        """HF's 2-D ``attention_mask`` [B, total_len] over cache positions 0..total_len-1 (past + new): a 0 means
        the key is never attended (left padding from ``build_inputs``).  Later positions stay attendable."""
        if attention_mask is None:
            return
        if attention_mask.dim() != 2 or tuple(attention_mask.shape) != (self.batch, total_len):
            raise ValueError(f"attention_mask shape {tuple(attention_mask.shape)} != (batch {self.batch}, past+new {total_len})")
        m = (attention_mask != 0).to(self._model.device, torch.uint8).contiguous()
        check(self._model._lib.vly_kv_set_key_mask(self._h, m.data_ptr(), total_len, _stream()))

    def release(self):
        """Give the handle (allocation + captured CUDA graphs) back to the model for the next cache of the same shape, or
        destroy it when the model already keeps 2.  The cache is unusable afterwards."""
        h, self._h = getattr(self, "_h", None), None
        if h is not None and self._model._ctx and not self._model._push_handle(self.batch, self.max_seq, h):
            self._model._lib.vly_kv_destroy(h)

    def __del__(self):
        # forward() without past_key_values hands a fresh cache to the caller on every request (model_worker.py:371-379);
        # when the caller drops it, the allocation (1 GB / sequence at 7B) goes back to the model instead of to cudaFree
        try:
            self.release()
        except Exception:
            pass


def _same_device(have: torch.device, want) -> bool:
    want = torch.device(want) if not isinstance(want, torch.device) else want
    return want.type == "cuda" and (want.index is None or want.index == have.index)


class _ModuleSurface:
    """The slice of ``nn.Module`` the reference's callers touch on the model and on ``vision_tower``
    (model_worker.py:78,86; run_valley.py:42-43; run_valley_conv.py:113,126): ``.to()``, ``.cuda()``, ``.half()``,
    ``.eval()``, ``.device``, ``.dtype``.  Weights live packed (bf16) inside the library on the device chosen at
    construction, so these calls VALIDATE and return self: a 16-bit float dtype is accepted (fp16 checkpoints were
    converted to bf16 at load), the owning CUDA device is accepted, anything else raises -- there is no CPU path."""
    device: torch.device
    dtype = torch.bfloat16
    training = False

    def to(self, *args, **kwargs):
        device, dtype = kwargs.get("device"), kwargs.get("dtype")
        for a in args:
            if isinstance(a, torch.dtype):
                dtype = a
            elif isinstance(a, (str, torch.device, int)):
                device = a
            elif torch.is_tensor(a):
                device, dtype = a.device, a.dtype
        if device is not None:
            device = f"cuda:{device}" if isinstance(device, int) else device
            if not _same_device(self.device, device):
                raise _lib.VlyError(f"valley_b200 weights live on {self.device}; .to({device!r}) is not supported "
                                    "(there is no CPU path; build the model with device=... instead)")
        if dtype is not None and dtype not in (torch.float16, torch.bfloat16):
            raise _lib.VlyError(f".to({dtype}): the packed weights are bf16; only 16-bit float dtypes are accepted")
        return self

    def cuda(self, device=None):
        return self.to(device="cuda" if device is None else device)

    def half(self):
        return self.to(dtype=torch.float16)

    def bfloat16(self):
        return self.to(dtype=torch.bfloat16)

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise _lib.VlyError("valley_b200 is the inference hot path: forward only (SURVEY 8 f-4), no train() mode")
        return self.eval()

    def requires_grad_(self, requires_grad: bool = False):
        if requires_grad:
            raise _lib.VlyError("valley_b200 holds no autograd parameters")
        return self


class _VisionTower(_ModuleSurface):
    """Stands where CLIPVisionModel sits on the reference model: carries ``.config`` with the sentinel ids
    (run_valley.py:13-18, model_worker.py:80-84), takes the ``.to(device, dtype)`` the callers issue
    (model_worker.py:78, run_valley_conv.py:126) and is callable like the reference's use of it."""

    def __init__(self, model: "ValleyLlamaForCausalLM"):
        self._model = model
        self.device = model.device
        cfg = model.config
        self.config = types.SimpleNamespace(
            hidden_size=cfg.mm_hidden_size, image_size=cfg.vit_image, patch_size=cfg.vit_patch,
            num_hidden_layers=cfg.vit_layers, use_im_start_end=cfg.mm_use_im_start_end,
            im_patch_token=-1, im_start_token=-1, im_end_token=-1,
            _name_or_path=getattr(cfg, "mm_vision_tower", None))

    def __call__(self, pixel_values: torch.Tensor, output_hidden_states: bool = True, select_layer: Optional[int] = None):
        sel = self._model.config.mm_vision_select_layer if select_layer is None else select_layer
        hs = self._model._vit_encode(pixel_values, sel)
        return types.SimpleNamespace(selected_hidden_state=hs, select_layer=sel)


class _PackedLinear(_ModuleSurface):
    """Shape-carrying stand-in for an ``nn.Linear`` / ``nn.Embedding`` whose weight lives packed inside the library
    (fused / norm-folded / interleaved -- there is no per-module weight tensor to hand out)."""

    def __init__(self, owner, **dims):
        self.device = owner.device
        for k, v in dims.items():
            setattr(self, k, v)

    @property
    def weight(self):
        raise _lib.VlyError("weights are packed inside libvalley_b200.so (fused QKV, norm-folded, RoPE-interleaved); "
                            "load them with load_state_dict / from_pretrained -- they cannot be read back per module")


class ValleyLlamaModel(_ModuleSurface):
    """valley_model.py:21-254.  Holds the vision tower handle; ``forward`` returns final hidden states is NOT exposed
    separately (the final RMSNorm is folded into lm_head) -- callers in the reference only use the CausalLM wrapper.
    Plain attributes the callers set on it (``multi_image``, ``multi_image_mode``: model_worker.py:63-64 -- never read by
    the reference either, SURVEY App. C-3) are accepted like on any Python object."""

    def __init__(self, owner: "ValleyLlamaForCausalLM"):
        self._owner = owner
        self.device = owner.device
        self.config = owner.config
        self.vision_tower = _VisionTower(owner)
        self.patch_pooling_method = owner.config.patch_pooling_method      # valley_model.py:27, :40-52
        self.mm_projector = _PackedLinear(owner, in_features=owner.config.mm_hidden_size, out_features=owner.config.hidden_size)
        self.embed_tokens = _PackedLinear(owner, num_embeddings=owner.config.vocab_size, embedding_dim=owner.config.hidden_size)


class KeywordsStoppingCriteria:
    """valley/util/data_util.py:40-56 (a ``transformers.StoppingCriteria``): stop when the text decoded from the ids generated
    so far contains a keyword.  Same quirk as the reference: the FIRST call only records the prompt length (so the first
    generated token is never tested on its own), later calls decode row 0 of ``output_ids[:, start_len:]``."""

    def __init__(self, keywords, tokenizer, input_ids):
        self.keywords = keywords
        self.tokenizer = tokenizer
        self.start_len = None
        self.input_ids = input_ids

    def __call__(self, output_ids, scores=None, **kwargs) -> bool:
        if self.start_len is None:
            self.start_len = self.input_ids.shape[1]
        else:
            outputs = self.tokenizer.batch_decode(output_ids[:, self.start_len:], skip_special_tokens=True)[0]
            for keyword in self.keywords:
                if keyword in outputs:
                    return True
        return False


_UNSET = object()


def host_rows_step(seq, nxt, finished, eos_token_id, pad, tables=None, stopping_criteria=None):
    """One step of HF generate's row handling in the host-visible loop, after ``nxt`` [B] was selected for ``seq`` [B, n]:
    finished rows emit ``pad`` when an eos criterion exists (``eos_token_id`` set); a row finishes on eos or on a stop-string
    match (``tables``, ``stop_strings.match_rows``); the loop stops when every row has finished, or when a stopping criterion
    returns True (a plain bool stops every row, as the reference's criteria do).  Returns (seq, nxt, finished, stop)."""
    if eos_token_id is not None:
        nxt = torch.where(finished, torch.full_like(nxt, pad), nxt)
        finished = finished | (nxt == eos_token_id)
    seq = torch.cat([seq, nxt[:, None]], dim=1)
    if tables is not None:
        finished = finished | _ss.match_rows(seq, tables).to(finished.device)
    if (eos_token_id is not None or tables is not None) and bool(finished.all()):
        return seq, nxt, finished, True
    return seq, nxt, finished, bool(stopping_criteria) and any(sc(seq, None) for sc in stopping_criteria)


def _repeat_rows(t: torch.Tensor, n: int) -> torch.Tensor:
    """every row n times in a row (HF's _expand_inputs_for_generation), without a host synchronisation"""
    return t[:, None].expand(t.shape[0], n, *t.shape[1:]).reshape(t.shape[0] * n, *t.shape[1:]).contiguous()


def sampling_filters(top_k=None, top_p=None) -> Tuple[int, float]:
    """``generate``'s ``top_k`` / ``top_p`` as HF's generate reads them when it samples (generation/utils.py builds
    ``TopKLogitsWarper`` for ``top_k not in (None, 0)`` and ``TopPLogitsWarper`` for ``top_p`` below 1).  Returns
    ``(top_k, top_p)`` with 0 / 1.0 meaning off and raises HF's ``ValueError`` for values its warpers reject.
    ``top_p == 0`` is legal in HF and keeps one token: it becomes ``top_k = 1``."""
    k, p = 0, 1.0
    if top_k is not None and top_k != 0:
        if not isinstance(top_k, int) or top_k <= 0:
            raise ValueError(f"`top_k` has to be a strictly positive integer, but is {top_k}")
        k = top_k
    if top_p is not None:
        top_p = float(top_p)
        if top_p < 0 or top_p > 1.0:
            raise ValueError(f"`top_p` has to be a float > 0 and < 1, but is {top_p}")
        if top_p == 0.0:
            k = 1
        elif top_p < 1.0:
            p = top_p
    return k, p


def filter_scores(scores: torch.Tensor, top_k: int, top_p: float) -> torch.Tensor:
    """HF's ``TopKLogitsWarper`` then ``TopPLogitsWarper`` (generation/logits_process.py) on ``scores = logits / temperature``
    [B, V] fp32, with ``(top_k, top_p)`` from ``sampling_filters``: removed tokens become -inf.  The host-visible decode loop
    samples with it; the device loop applies the same filters in ``sample_filter_kernel``."""
    if top_k > 0:
        kth = torch.topk(scores, min(top_k, scores.size(-1)))[0][..., -1, None]
        scores = scores.masked_fill(scores < kth, -float("inf"))
    if top_p < 1.0:
        sorted_logits, sorted_indices = torch.sort(scores, descending=False)
        cumulative_probs = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
        sorted_indices_to_remove = cumulative_probs <= (1 - top_p)
        sorted_indices_to_remove[..., -1:] = 0
        indices_to_remove = sorted_indices_to_remove.scatter(1, sorted_indices, sorted_indices_to_remove)
        scores = scores.masked_fill(indices_to_remove, -float("inf"))
    return scores


def _open_video_reader(path: str):
    """Default file reader of ``completion(tokenizer, path, ...)``: decord, exactly as load_video opens it
    (data_util.py:258-260).  Container decoding is CPU work outside the hot path; inject another reader factory through
    ``model.video_reader_factory`` (anything with ``len()``, ``get_batch(idx)`` -> [n,H,W,3] uint8, ``get_avg_fps()``)."""
    try:
        import decord
    except ImportError as e:
        raise ImportError("completion() was given a video path but decord is not installed; set model.video_reader_factory "
                          "to a callable path -> reader, or pass the decoded clip tensor [3,T,224,224]") from e
    return decord.VideoReader(path, num_threads=1, ctx=decord.cpu(0))


class ValleyLlamaForCausalLM(_ModuleSurface):
    """valley_model.py:257-439 behind libvalley_b200.so."""
    config_class = ValleyConfig
    video_reader_factory = staticmethod(_open_video_reader)

    def __init__(self, config: ValleyConfig, device: Union[int, str, torch.device] = 0):
        self._lib = _lib.load()
        self._ctx = None
        self.config = config
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise _lib.VlyError("valley_b200 runs on a CUDA sm_90a device only; there is no CPU path")
        self.device = dev
        self.dtype = torch.bfloat16
        c = VlyConfig(config.hidden_size, config.num_hidden_layers, config.num_attention_heads, config.intermediate_size,
                      config.vocab_size, config.rms_norm_eps, config.rope_theta, config.max_position_embeddings,
                      config.mm_hidden_size, config.vit_layers, config.vit_heads, config.vit_mlp, config.vit_patch,
                      config.vit_image, config.vit_eps, config.mm_vision_select_layer, dev.index or 0,
                      _lib.POOLING[config.patch_pooling_method])
        h = C.c_void_p()
        check(self._lib.vly_create(C.byref(c), C.byref(h)))
        self._ctx = h
        self.model = ValleyLlamaModel(self)
        self.training = False
        self.logits_all_positions = True      # reference behaviour (valley_model.py:304-305); generate() uses last-only
        import threading
        self._pool_lock = threading.Lock()
        self._free_handles = {}               # (batch, max_seq) -> [vly_kv handles] released by ValleyKVCache.release()

    # ---------------- lifetime / weights ----------------
    def __del__(self):
        try:
            if getattr(self, "_ctx", None):
                for lst in getattr(self, "_free_handles", {}).values():
                    for h in lst:
                        self._lib.vly_kv_destroy(h)
                self._free_handles = {}
                self._lib.vly_destroy(self._ctx)
                self._ctx = None
        except Exception:
            pass

    def _pop_handle(self, batch: int, max_seq: int):
        with self._pool_lock:
            lst = self._free_handles.get((batch, max_seq))
            return lst.pop() if lst else None

    def _push_handle(self, batch: int, max_seq: int, h) -> bool:
        with self._pool_lock:
            lst = self._free_handles.setdefault((batch, max_seq), [])
            if len(lst) >= 2:
                return False
            lst.append(h)
            return True

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, torch_dtype=None, device=0, **kw) -> "ValleyLlamaForCausalLM":
        """``ValleyLlamaForCausalLM.from_pretrained(path, torch_dtype=torch.float16)`` (run_valley.py:39, model_worker.py:62): a
        local HF checkpoint directory (config.json + safetensors / .bin shards).  Weights are stored as bf16 whatever ``torch_dtype``
        says (fp16 checkpoints are converted on load)."""
        from . import checkpoint
        path = pretrained_model_name_or_path
        if checkpoint.is_lora_dir(path):       # run_valley.py:26-37: PeftModel.from_pretrained(base, path).merge_and_unload()
            base = checkpoint.resolve_lora_base(path)
            cfg = ValleyConfig(**{**checkpoint.read_config(base), **kw})
            m = cls(cfg, device)
            m.load_state_dict(checkpoint.iter_checkpoint_merged(base, path, device=m.device))
            return m
        cfg = ValleyConfig(**{**checkpoint.read_config(path), **kw})
        m = cls(cfg, device)
        m.load_state_dict(checkpoint.iter_checkpoint(path))
        return m

    @classmethod
    def from_state_dict(cls, config: ValleyConfig, state: Iterable, device=0) -> "ValleyLlamaForCausalLM":
        m = cls(config, device)
        m.load_state_dict(state)
        return m

    def load_state_dict(self, state, strict: bool = False):
        """Accepts a dict or an iterator of (hf_name, tensor).  Tensors may live on CPU or GPU, fp32/bf16/fp16.
        Unknown names (post_layernorm, rotary inv_freq, position_ids...) are ignored like HF non-strict loading."""
        items = state.items() if hasattr(state, "items") else state
        for name, t in items:
            if "post_layernorm" in name or name.endswith("position_ids") or name.endswith("inv_freq"):
                continue
            if "transforemr_adding_layer" in name:      # the template nn.TransformerEncoder deep-copies; never executed (valley_model.py:47-48)
                continue
            t = t.detach()
            if t.dtype not in _DT:
                t = t.float()
            t = t.to(self.device).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            check(self._lib.vly_load_weight(self._ctx, name.encode(), t.data_ptr(), _DT[t.dtype], shape, t.dim()))
        check(self._lib.vly_finalize_weights(self._ctx))
        return self

    def get_model(self) -> ValleyLlamaModel:      # valley_model.py:269
        return self.model

    def get_input_embeddings(self):
        return self.model.embed_tokens

    def get_output_embeddings(self):
        return _PackedLinear(self, in_features=self.config.hidden_size, out_features=self.config.vocab_size)

    def resize_token_embeddings(self, new_num_tokens: Optional[int] = None):
        """Growing the embedding table is a training-time step (train.py:147 -> initialize_vision_tokenizer); released
        checkpoints already contain the added tokens.  Accepted as a no-op when nothing has to grow."""
        if new_num_tokens is not None and new_num_tokens > self.config.vocab_size:
            raise _lib.VlyError(f"resize_token_embeddings({new_num_tokens}) > loaded vocab {self.config.vocab_size}: growing the "
                                "embeddings is a training-time operation; load a checkpoint that already holds the added tokens")
        return self.model.embed_tokens

    def initialize_vision_tokenizer(self, tokenizer):
        """valley_model.py:354-379 for an inference checkpoint: register the sentinel tokens with the tokenizer and record
        their ids on ``vision_tower.config``.  The reference also grows the embeddings and initialises the new rows with the
        mean embedding -- that is checkpoint construction (training); here the tokenizer must fit the loaded vocabulary."""
        vc = self.get_model().vision_tower.config
        vc.use_im_start_end = True
        tokenizer.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_VIDEO_FRAME_TOKEN], special_tokens=True)
        self.resize_token_embeddings(len(tokenizer))
        tokenizer.add_tokens([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN, DEFAULT_VI_START_TOKEN, DEFAULT_VI_END_TOKEN],
                             special_tokens=True)
        self.resize_token_embeddings(len(tokenizer))
        vc.im_start_token, vc.im_end_token = tokenizer.convert_tokens_to_ids([DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN])
        vc.vi_start_token, vc.vi_end_token = tokenizer.convert_tokens_to_ids([DEFAULT_VI_START_TOKEN, DEFAULT_VI_END_TOKEN])
        vc.vi_frame_token = tokenizer.convert_tokens_to_ids(DEFAULT_VIDEO_FRAME_TOKEN)
        vc.im_patch_token = tokenizer.convert_tokens_to_ids([DEFAULT_IMAGE_PATCH_TOKEN])[0]

    def launches(self) -> int:
        n = C.c_int64()
        check(self._lib.vly_kernel_launch_count(self._ctx, C.byref(n)))
        return n.value

    # ---------------- vision ----------------
    def _tokens(self) -> VlyTokens:
        vc = self.model.vision_tower.config
        g = lambda k: int(getattr(vc, k, -1) if getattr(vc, k, None) is not None else -1)
        return VlyTokens(g("im_patch_token"), g("im_start_token"), g("im_end_token"),
                         g("vi_frame_token"), g("vi_start_token"), g("vi_end_token"))

    def _vit_encode(self, pixels: torch.Tensor, select_layer: int) -> torch.Tensor:
        """[F,3,224,224] -> hidden_states[select_layer] [F,257,1024] bf16."""
        if pixels.dim() != 4 or pixels.shape[1] != 3 or pixels.shape[2] != self.config.vit_image or pixels.shape[3] != self.config.vit_image:
            # HF:modeling_clip.py:203-207
            raise ValueError(f"Input image size ({pixels.shape[-2]}*{pixels.shape[-1]}) doesn't match model "
                             f"({self.config.vit_image}*{self.config.vit_image}).")
        if pixels.dtype not in _DT:
            pixels = pixels.float()
        pixels = pixels.to(self.device, non_blocking=True).contiguous()
        tokens = (self.config.vit_image // self.config.vit_patch) ** 2 + 1
        out = torch.empty(pixels.shape[0], tokens, self.config.mm_hidden_size, dtype=torch.bfloat16, device=self.device)
        check(self._lib.vly_vit_encode(self._ctx, pixels.data_ptr(), _DT[pixels.dtype], pixels.shape[0], select_layer,
                                       out.data_ptr(), _stream()))
        return out

    def encode_frames(self, pixels: torch.Tensor) -> torch.Tensor:
        """Vision tower only: [F,3,224,224] -> [F,257,1024] (config.mm_vision_select_layer)."""
        return self._vit_encode(pixels, getattr(self.config, "mm_vision_select_layer", -1))

    def _project(self, feats: torch.Tensor) -> torch.Tensor:
        rows = feats.numel() // feats.shape[-1]
        out = torch.empty(*feats.shape[:-1], self.config.hidden_size, dtype=torch.bfloat16, device=self.device)
        check(self._lib.vly_project(self._ctx, feats.data_ptr(), rows, out.data_ptr(), _stream()))
        return out

    @torch.no_grad()
    def encode_images(self, images):
        """valley_model.py:163-190: tensor [B,T,3,H,W] -> [B,T,257,hidden]; list of [T_i,3,H,W] -> list."""
        if isinstance(images, (list, tuple)):
            return [self._project(self.encode_frames(img)) for img in images]
        B, T = images.shape[:2]
        feats = self.encode_frames(images.reshape(B * T, *images.shape[2:]))
        return self._project(feats).view(B, T, feats.shape[1], self.config.hidden_size)

    def _pool_project(self, feats: torch.Tensor, n_videos: int, T: int) -> torch.Tensor:
        """feats [n_videos*T,257,1024] -> [n_videos, 256+T, hidden] (pool-first)."""
        rows = feats.shape[1] - 1 + T
        out = torch.empty(n_videos, rows, self.config.hidden_size, dtype=torch.bfloat16, device=self.device)
        check(self._lib.vly_pool_project(self._ctx, feats.data_ptr(), n_videos, T, out.data_ptr(), _stream()))
        return out

    def _splice_plan(self, input_ids: torch.Tensor, T: int):
        ids = input_ids.detach().to("cpu", torch.int64).contiguous()
        B, S = ids.shape
        smap = torch.empty(B, S, dtype=torch.int32)
        iidx = torch.empty(B, dtype=torch.int32)
        tok = self._tokens()
        check(self._lib.vly_build_splice_map(C.cast(ids.data_ptr(), C.POINTER(C.c_int64)), B, S, T, C.byref(tok),
                                             C.cast(smap.data_ptr(), C.POINTER(C.c_int32)),
                                             C.cast(iidx.data_ptr(), C.POINTER(C.c_int32))))
        return smap, iidx

    @torch.no_grad()
    def prepare_inputs_labels_for_multimodal(self, input_ids, attention_mask=None, past_key_values=None, labels=None,
                                              images=None, frame_features: Optional[torch.Tensor] = None,
                                              n_frames: Optional[int] = None):
        """valley_model.py:155-247 -> (None, attention_mask, past_key_values, inputs_embeds, labels).

        Vision runs iff input_ids.shape[1] != 1 (or training) and images is not None (:163-164).
        ``frame_features`` ([n_videos*n_frames,257,1024], e.g. all-gathered from other ranks) skips the local ViT."""
        B, S = input_ids.shape
        ids_dev = input_ids.to(self.device, torch.int64).contiguous()
        embeds = torch.empty(B, S, self.config.hidden_size, dtype=torch.bfloat16, device=self.device)
        use_vision = (images is not None or frame_features is not None) and (S != 1 or self.training)
        if not use_vision:
            check(self._lib.vly_embed_splice(self._ctx, ids_dev.data_ptr(), None, None, None, 0, B, S, embeds.data_ptr(), _stream()))
            return None, attention_mask, past_key_values, embeds, labels
        if isinstance(images, (list, tuple)):
            # variable T per sample (valley_model.py:168-176): plan and pool per sample
            vis, smaps, cur = [], [], 0
            for b in range(B):
                T_b = images[min(cur, len(images) - 1)].shape[0]
                smap, iidx = self._splice_plan(input_ids[b:b + 1], T_b)
                if iidx[0] >= 0:
                    feats = self.encode_frames(images[cur])
                    vis.append(self._pool_project(feats, 1, T_b)[0])
                    cur += 1
                smaps.append((smap, int(iidx[0])))
            out = []
            for b, (smap, flag) in enumerate(smaps):
                e = torch.empty(1, S, self.config.hidden_size, dtype=torch.bfloat16, device=self.device)
                if flag < 0:
                    check(self._lib.vly_embed_splice(self._ctx, ids_dev[b:b + 1].data_ptr(), None, None, None, 0, 1, S, e.data_ptr(), _stream()))
                else:
                    v = vis.pop(0).contiguous()
                    sm = smap.to(self.device)
                    z = torch.zeros(1, dtype=torch.int32, device=self.device)
                    check(self._lib.vly_embed_splice(self._ctx, ids_dev[b:b + 1].data_ptr(), sm.data_ptr(), z.data_ptr(), v.data_ptr(),
                                                     v.shape[0], 1, S, e.data_ptr(), _stream()))
                out.append(e)
            return None, attention_mask, past_key_values, torch.cat(out, 0), labels
        if frame_features is None:
            Bi, T = images.shape[:2]
            frame_features = self.encode_frames(images.reshape(Bi * T, *images.shape[2:]))
        else:
            T = n_frames if n_frames is not None else images.shape[1]
            Bi = frame_features.shape[0] // T
        smap, iidx = self._splice_plan(input_ids, T)          # raises ValueError exactly where the reference does
        vis = self._pool_project(frame_features, Bi, T)        # [Bi, 256+T, H]
        n_mm = int((iidx >= 0).sum())
        if n_mm > Bi:
            raise IndexError("index out of range: more multimodal samples than images")   # image_features[cur_image_idx]
        sm, ii = smap.to(self.device, non_blocking=True), iidx.clamp(min=0).to(self.device, non_blocking=True)
        check(self._lib.vly_embed_splice(self._ctx, ids_dev.data_ptr(), sm.data_ptr(), ii.data_ptr(), vis.data_ptr(), vis.shape[1],
                                         B, S, embeds.data_ptr(), _stream()))
        return None, attention_mask, past_key_values, embeds, labels

    # ---------------- language model ----------------
    def new_cache(self, batch: int, max_seq: Optional[int] = None) -> ValleyKVCache:
        return ValleyKVCache(self, batch, max_seq or self.config.max_position_embeddings)

    def _prefill(self, cache: ValleyKVCache, embeds: torch.Tensor, logits_mode: int):
        B, S, _ = embeds.shape
        V = self.config.vocab_size
        logits = None
        if logits_mode == 2:
            logits = torch.empty(B, S, V, dtype=torch.float32, device=self.device)
        elif logits_mode == 1:
            logits = torch.empty(B, 1, V, dtype=torch.float32, device=self.device)
        nxt = torch.empty(B, dtype=torch.int64, device=self.device)
        check(self._lib.vly_llama_prefill(self._ctx, cache._h, embeds.data_ptr(), B, S, logits_mode, _ptr(logits), nxt.data_ptr(), _stream()))
        return logits, nxt

    def _decode(self, cache: ValleyKVCache, tokens: torch.Tensor, want_logits: bool):
        B = tokens.shape[0]
        nxt = torch.empty(B, dtype=torch.int64, device=self.device)
        logits = torch.empty(B, 1, self.config.vocab_size, dtype=torch.float32, device=self.device) if want_logits else None
        tk = tokens.reshape(B).to(self.device, torch.int64).contiguous()
        check(self._lib.vly_llama_decode(self._ctx, cache._h, tk.data_ptr(), nxt.data_ptr(), _ptr(logits), _stream()))
        return logits, nxt

    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, past_key_values=None, inputs_embeds=None, labels=None,
                use_cache=None, output_attentions=None, output_hidden_states=None, images=None, return_dict=None):
        """ValleyLlamaForCausalLM.forward (valley_model.py:272-330).  logits are fp32 [B,S,V]
        (the reference returns them in the model dtype; callers .float() them).  A 2-D attention_mask [B, past+S] masks
        keys exactly as HF does (padding mask AND causal mask; position ids are not shifted -- the reference never
        passes position_ids); rows that are themselves padding produce unspecified (finite) logits."""
        if output_hidden_states or output_attentions:
            # valley_model.py:285-300 forwards these to LlamaModel; the fused path never materialises per-layer hidden states
            # or attention probabilities (that is the point of it), so asking for them is an error rather than a silent None
            raise NotImplementedError("output_hidden_states / output_attentions are not produced by the fused kernels")
        if inputs_embeds is None:
            if input_ids is None:
                raise ValueError("You have to specify either input_ids or inputs_embeds")
            _, _, _, inputs_embeds, _ = self.prepare_inputs_labels_for_multimodal(
                input_ids, attention_mask, past_key_values, labels, images)
        else:
            if images is not None and input_ids is None:
                # the reference dereferences input_ids.shape here (valley_model.py:164)
                raise AttributeError("'NoneType' object has no attribute 'shape'")
            inputs_embeds = inputs_embeds.to(self.device, torch.bfloat16).contiguous()
        B, S, _ = inputs_embeds.shape
        cache = past_key_values if isinstance(past_key_values, ValleyKVCache) else None
        if cache is None:
            cache = self.new_cache(B)
        cache.set_attention_mask(attention_mask, cache.get_seq_length() + S)
        if S == 1 and cache.get_seq_length() > 0 and input_ids is not None:
            logits, nxt = self._decode(cache, input_ids, True)
        else:
            logits, nxt = self._prefill(cache, inputs_embeds, 2 if self.logits_all_positions else 1)
        loss = None
        if labels is not None:       # valley_model.py:308-318
            if logits.shape[1] != S:
                raise ValueError("labels need logits at every position (logits_all_positions=True, the reference behaviour)")
            lab = labels.to(self.device, torch.int64).contiguous()
            loss = torch.full((), float("nan"), dtype=torch.float32, device=self.device)     # S == 1: nothing to score (torch: nan)
            if S >= 2:
                check(self._lib.vly_cross_entropy(self._ctx, logits.data_ptr(), lab.data_ptr(), B, S, IGNORE_INDEX,
                                                  loss.data_ptr(), _stream()))
        out = CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=cache)
        out.next_tokens = nxt
        if return_dict is False:
            return tuple(v for v in (loss, logits, cache) if v is not None)
        return out

    __call__ = forward

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None, **kwargs):
        """valley_model.py:332-352 with the INTENDED semantics (SURVEY Appendix C-1): slice to the last token only
        once the cache actually holds tokens."""
        if past_key_values is not None and (not hasattr(past_key_values, "get_seq_length") or past_key_values.get_seq_length() > 0):
            input_ids = input_ids[:, -1:]
        if inputs_embeds is not None and past_key_values is None:
            model_inputs = {"inputs_embeds": inputs_embeds}
        else:
            model_inputs = {"input_ids": input_ids}
        model_inputs.update({"past_key_values": past_key_values, "use_cache": kwargs.get("use_cache"),
                             "attention_mask": attention_mask, "images": kwargs.get("images", None)})
        return model_inputs

    @torch.no_grad()
    def generate(self, input_ids=None, images=None, max_new_tokens: int = 1024, do_sample: bool = False,
                 temperature: float = 1.0, stopping_criteria=None, eos_token_id=_UNSET, top_k=None, top_p=None,
                 num_beams: int = 1, num_return_sequences: int = 1, length_penalty: float = 1.0, early_stopping=False,
                 stop_strings=None, tokenizer=None, return_dict_in_generate: bool = False, output_scores: bool = False,
                 output_logits: bool = False, output_attentions: bool = False, output_hidden_states: bool = False, **kw):
        """Greedy (or temperature) generation == the loop of model_worker.py:371-397 / HF generate as called at
        valley_model.py:432.  Returns [B, S + n_new] like HF.  With no stopping criteria, decoding runs
        entirely on the device (CUDA-graph replay, no per-token host sync).  ``attention_mask`` [B, S] (left padding)
        is honoured like HF generate does; generated positions are always attendable.

        ``top_k`` / ``top_p`` filter the sampled distribution after the temperature, as HF's warpers do (``sampling_filters``
        gives the argument handling).  They apply only when sampling: with ``do_sample=False`` or a temperature below 1e-4
        they are ignored.  Unlike HF, no ``top_k = 50`` is implied when none is given.

        HF defaults that the reference's callers rely on are kept: ``eos_token_id`` / ``pad_token_id`` default to the config's
        (generation stops when every row has emitted eos; finished rows are padded), and when no ``attention_mask`` is given
        but the prompt contains ``pad_token_id`` (!= eos) the mask is inferred as ``input_ids != pad_token_id``
        (HF:generation/utils.py _prepare_attention_mask_for_generation).  Pass ``eos_token_id=None`` to run the full length.

        ``num_beams > 1`` runs HF's beam search (``length_penalty``, ``early_stopping`` True / False / "never",
        ``num_return_sequences`` best hypotheses per row, returned as [B * num_return_sequences, S + L]).  Without stopping
        criteria (and up to 8 beams and 64 rows in all) the selection and the KV-cache reorder run inside the decode step's CUDA
        graph, with one device-to-host read per request; otherwise a host-visible loop runs the same search
        (valley_b200/beam.py).  The returned sequences' scores (HF's ``sequences_scores``) are left in
        ``model.last_beam_scores``.  Beam sampling (``do_sample=True``) is not implemented.

        ``stop_strings`` (a string or a list of strings) with ``tokenizer``: transformers' ``StopStringCriteria``.  A row
        finishes when its text ends with a stop string, the last characters inside the newest token; the text is the
        concatenation of the tokens' clean strings (``valley_b200/stop_strings.py``), prompt included.  Finished rows are padded
        only when ``eos_token_id`` is set, as in HF; generation ends when every row has finished.  With ``num_beams == 1``, no
        other stopping criteria, at most 64 rows, at most 8 stop strings and at most 64 characters each, the matcher runs on
        the device after every token (no per-token host sync); otherwise the host-visible loops check it.  ``stop_strings``
        without ``tokenizer`` raises HF's ``ValueError``.

        ``return_dict_in_generate=True`` returns HF's output object instead of the tensor: ``GenerateDecoderOnlyOutput``
        (``num_beams == 1``) or ``GenerateBeamDecoderOnlyOutput``, with transformers 5.5's fields.  ``output_scores`` adds
        ``scores``, one [rows, V] fp32 tensor per step run: the raw logits when not sampling; when sampling, logits /
        temperature with -inf at every token top_k / top_p removed; for beams, each beam row's log-softmax (and
        ``sequences_scores``).  ``output_logits`` adds the raw logits per step.  Beams always return ``beam_indices``
        [B * num_return_sequences, L]: the cache row (item * num_beams + beam) of each token, -1 after the hypothesis ended.
        The device routes record these inside the decode loop, with no extra host synchronisation; each requested output
        costs steps x rows x V x 4 bytes (128 KB per row and step at V = 32,000).  ``past_key_values`` is None: the KV cache
        goes back to the model's pool when the request ends.  ``output_attentions`` / ``output_hidden_states`` raise
        ``NotImplementedError``.  Without ``return_dict_in_generate`` the output flags are ignored, as in HF.

        ``repetition_penalty``, ``no_repeat_ngram_size``, ``min_new_tokens`` and ``min_length`` add transformers 5.5's logits
        processors, under HF's conditions and with HF's errors (``valley_b200/processors.py``), before the temperature and the
        filters; the min-length ones only with an eos id, ``min_new_tokens`` winning over ``min_length``.  They see each row as HF
        does: the prompt ids (padding and image placeholders included), then every emitted token, pad once the row finished.
        ``scores`` records the processed scores; ``logits`` stays raw.  With ``num_beams == 1`` they run on the device inside
        the selection kernel, with no extra host synchronisation; beams with processors run the host beam loop, on each beam
        row's log-softmax.  Other HF processors (``bad_words_ids``, ``suppress_tokens``, ...) are still ignored."""
        if output_hidden_states or output_attentions:
            raise NotImplementedError("output_hidden_states / output_attentions are not produced by the fused kernels")
        record = (bool(output_scores), bool(output_logits)) if return_dict_in_generate else None
        B, S = input_ids.shape
        procs = _proc.from_kwargs(kw, S, getattr(self.config, "eos_token_id", None) if eos_token_id is _UNSET else eos_token_id)
        tables = None
        if stop_strings is not None:
            if tokenizer is None:
                raise ValueError("There are one or more stop strings, either in the arguments to `generate` or in the model's "
                                 "generation config, but we could not locate a tokenizer. When generating with stop strings, "
                                 "you must pass the model's tokenizer to the `tokenizer` argument of `generate`.")
            tables = _ss.stop_tables(_ss.clean_token_strings(tokenizer), stop_strings, self.config.vocab_size)
        if num_beams != 1:
            return self._beam_generate(input_ids, images, max_new_tokens, do_sample, stopping_criteria, eos_token_id, num_beams,
                                       num_return_sequences, length_penalty, early_stopping, tables=tables, record=record,
                                       procs=procs, **kw)
        greedy = (not do_sample) or temperature < 1e-4
        filters = {} if greedy else dict(zip(("top_k", "top_p"), sampling_filters(top_k, top_p)))
        n_new, eos_token_id, pad_token_id, attention_mask = self._generation_defaults(input_ids, max_new_tokens, eos_token_id, kw)
        if n_new == 0:
            seq = input_ids.to(self.device)
            return seq if record is None else generation_output(seq, 0, *self._record_buffers(record, 0, B))
        _, _, _, embeds, _ = self.prepare_inputs_labels_for_multimodal(input_ids, None, None, None, images)
        cache = self.new_cache(B)
        try:
            cache.set_attention_mask(attention_mask, S)
            return self._generate_with_cache(cache, input_ids, embeds, n_new, do_sample, temperature, stopping_criteria, eos_token_id,
                                             pad_token_id, tables=tables, record=record, procs=procs, **filters)
        finally:
            cache.release()

    def _generation_defaults(self, input_ids, max_new_tokens, eos_token_id, kw):
        """(n_new, eos_token_id, pad_token_id, attention_mask) of a generate() request, with the HF defaults generate() describes:
        at most the tokens the context has room for, eos and pad from the config, pad falling back to eos, and the attention
        mask inferred from pad tokens in the prompt (pad != eos)."""
        n_new = max(0, min(max_new_tokens, self.config.max_position_embeddings - input_ids.shape[1]))
        if eos_token_id is _UNSET:
            eos_token_id = getattr(self.config, "eos_token_id", None)
        pad_token_id = kw.get("pad_token_id", getattr(self.config, "pad_token_id", None))
        if pad_token_id is None:
            pad_token_id = eos_token_id                       # HF generate: pad defaults to eos
        attention_mask = kw.get("attention_mask")
        if attention_mask is None and pad_token_id is not None and pad_token_id != eos_token_id:
            is_pad = input_ids == pad_token_id
            if bool(is_pad.any()):
                attention_mask = (~is_pad).to(torch.int64)
        return n_new, eos_token_id, pad_token_id, attention_mask

    def _record_buffers(self, record, n_steps: int, rows: int):
        """(scores, logits) buffers [n_steps, rows, V] fp32 for a request that records them (``record`` = (output_scores,
        output_logits), or None: nothing is recorded); None for an output not asked for"""
        V = self.config.vocab_size
        mk = lambda want: torch.empty(n_steps, rows, V, dtype=torch.float32, device=self.device) if want else None
        return (None, None) if record is None else (mk(record[0]), mk(record[1]))

    def _generate_with_cache(self, cache, input_ids, embeds, n_new, do_sample, temperature, stopping_criteria, eos_token_id,
                             pad_token_id=None, top_k=0, top_p=1.0, tables=None, record=None, procs=None):
        """the tokens after the prefill of ``embeds`` into ``cache``: [B, S + steps], or with ``record`` = (output_scores,
        output_logits) the output object of generate(return_dict_in_generate=True); ``procs``: the request's logits processors
        (``processors.Processors``) or None"""
        B = input_ids.shape[0]
        greedy = (not do_sample) or temperature < 1e-4
        plain = greedy and not stopping_criteria and eos_token_id is None and tables is None and procs is None
        device_select = (not stopping_criteria and not (plain and record is None) and B <= 64
                         and (tables is None or tables.on_device))
        rec_scores, rec_logits = self._record_buffers(record, n_new, B)
        tail = None
        if device_select and tables is not None:       # the prompt's last tokens seed the device matcher (the whole row counts)
            tail = input_ids[:, -min(input_ids.shape[1], 63):].to("cpu", torch.int64).numpy()
        logits, nxt = self._prefill(cache, embeds, 0 if (greedy and not device_select and record is None and procs is None) else 1)
        ids_dev = input_ids.to(self.device, torch.int64).contiguous()
        if plain and record is None:
            out = torch.empty(B, n_new, dtype=torch.int64, device=self.device)
            out[:, 0] = nxt
            if n_new > 1:
                rest = torch.empty(B, n_new - 1, dtype=torch.int64, device=self.device)
                check(self._lib.vly_generate_greedy(self._ctx, cache._h, nxt.data_ptr(), n_new - 1, rest.data_ptr(), _stream()))
                out[:, 1:] = rest
            return torch.cat([ids_dev, out], dim=1)
        if device_select:
            # temperature sampling and/or a stop token, still without a per-token host sync: the selection (Gumbel-max over
            # Philox noise) and the eos bookkeeping run inside the decode step; one 4-byte read at the end gives the length
            eos = -1 if eos_token_id is None else int(eos_token_id)
            pad = int(pad_token_id) if pad_token_id is not None else max(eos, 0)      # HF: pad defaults to eos
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())                         # torch.manual_seed() governs it
            # (a top-k / top-p filter: one more kernel per step selects over the step's logits, still on the device)
            # below a temperature of 1e-4 the library takes the arg-max; a sampling request still passes its temperature, which
            # its recorded scores divide by (HF's warper)
            sp = VlySampling(float(temperature) if do_sample else 0.0, seed, eos, pad, top_k=top_k, top_p=top_p)
            if tables is not None:
                sp.set_stop_strings(tables, tail)
            sp.scores_out, sp.logits_out = _ptr(rec_scores), _ptr(rec_logits)      # slot 0: the first token
            if procs is not None:       # (the rows' histories start from the prompt ids, on the device)
                sp.repetition_penalty, sp.no_repeat_ngram_size = procs.penalty, procs.ngram
                sp.min_length, sp.prompt_ids_dev = procs.min_length, ids_dev.data_ptr()
            out = torch.empty(B, n_new, dtype=torch.int64, device=self.device)
            first = torch.empty(B, dtype=torch.int64, device=self.device)
            check(self._lib.vly_sample_logits(self._ctx, cache._h, logits.data_ptr(), C.byref(sp), first.data_ptr(), _stream()))
            out[:, 0] = first
            n_valid = 1
            if n_new > 1:
                rest = torch.empty(B, n_new - 1, dtype=torch.int64, device=self.device)
                done = torch.zeros(1, dtype=torch.int32, device=self.device)
                sp.scores_out = None if rec_scores is None else rec_scores[1:].data_ptr()     # step i writes slot i + 1
                sp.logits_out = None if rec_logits is None else rec_logits[1:].data_ptr()
                check(self._lib.vly_generate(self._ctx, cache._h, first.data_ptr(), n_new - 1, rest.data_ptr(), C.byref(sp),
                                             done.data_ptr(), _stream()))
                out[:, 1:] = rest
                # (a greedy request without eos or stop strings -- here because it records or has processors -- runs every
                #  step: no read-back)
                runs_all = greedy and eos_token_id is None and tables is None
                n_valid += n_new - 1 if runs_all else int(done.item())
            seq = torch.cat([ids_dev, out[:, :n_valid]], dim=1)
            return seq if record is None else generation_output(seq, n_valid, rec_scores, rec_logits)
        # host-visible loop (stopping criteria present, B > 64, or stop strings past the device limits): one device->host
        # sync per token, as in the reference
        seq = ids_dev
        finished = torch.zeros(B, dtype=torch.bool, device=self.device)
        pad = int(pad_token_id) if pad_token_id is not None else (int(eos_token_id) if eos_token_id is not None else 0)
        steps = 0
        for i in range(n_new):
            # the processors (before the temperature and the filters, as in HF) see the row so far
            proc = None if logits is None else _proc.apply(logits[:, -1, :], seq, procs)
            if not greedy:
                scores = filter_scores(proc / temperature, top_k, top_p)     # model_worker.py:393-394
                probs = torch.softmax(scores, dim=-1)
                nxt = torch.multinomial(probs, num_samples=1).reshape(B)
            else:
                if procs is not None:
                    nxt = proc.argmax(-1)                   # (the first maximum, as on the device)
                if rec_scores is not None:
                    scores = proc / temperature if do_sample else proc
            if rec_scores is not None:
                rec_scores[i] = scores
            if rec_logits is not None:
                rec_logits[i] = logits[:, -1, :]
            steps = i + 1
            seq, nxt, finished, stop = host_rows_step(seq, nxt, finished, eos_token_id, pad, tables, stopping_criteria)
            if stop:
                break
            if i + 1 < n_new:
                logits, nxt = self._decode(cache, nxt, not greedy or record is not None or procs is not None)
        return seq if record is None else generation_output(seq, steps, rec_scores, rec_logits)

    def _beam_generate(self, input_ids, images, max_new_tokens, do_sample, stopping_criteria, eos_token_id, num_beams,
                       num_return_sequences, length_penalty, early_stopping, tables=None, record=None, procs=None, **kw):
        """generate(num_beams > 1): the vision part is encoded once per row, then every row's embeddings and attention mask
        are repeated num_beams times (HF's _expand_inputs_for_generation) and prefilled as B * num_beams cache rows."""
        if not isinstance(num_beams, int) or num_beams < 1:
            raise ValueError(f"`num_beams` has to be a strictly positive integer, but is {num_beams}")
        if do_sample:
            raise NotImplementedError("beam sampling (num_beams > 1 with do_sample=True) is not implemented")
        if not isinstance(num_return_sequences, int) or not 1 <= num_return_sequences <= num_beams:
            raise ValueError(f"`num_return_sequences` ({num_return_sequences}) has to be smaller or equal to `num_beams` ({num_beams}).")
        if early_stopping not in (True, False, "never"):
            raise ValueError(f"`early_stopping` must be a boolean or 'never', but is {early_stopping}.")
        B, S = input_ids.shape
        nb = num_beams
        n_new, eos_token_id, pad_token_id, attention_mask = self._generation_defaults(input_ids, max_new_tokens, eos_token_id, kw)
        ids_dev = input_ids.to(self.device, torch.int64)
        if n_new == 0:
            seq = _repeat_rows(ids_dev, num_return_sequences)
            if record is None:
                return seq
            empty = torch.empty(seq.shape[0], 0, dtype=torch.int64, device=self.device)
            return generation_output(seq, 0, *self._record_buffers(record, 0, B * nb), beam_indices=empty, beam=True)
        fill = _beam.output_fill_value(pad_token_id, eos_token_id)
        _, _, _, embeds, _ = self.prepare_inputs_labels_for_multimodal(input_ids, None, None, None, images)
        embeds = _repeat_rows(embeds, nb)
        ids_rep = _repeat_rows(ids_dev, nb)
        if attention_mask is not None:
            attention_mask = _repeat_rows(attention_mask, nb)
        cache = self.new_cache(B * nb)
        try:
            cache.set_attention_mask(attention_mask, S)
            logits, _ = self._prefill(cache, embeds, 1)
            logits = logits[:, -1].contiguous()
            if not stopping_criteria and tables is None and procs is None and nb <= 8 and B * nb <= 64:
                nrs = num_return_sequences
                es = {False: 0, True: 1, "never": 2}[early_stopping]
                bp = VlyBeam(nb, nrs, float(length_penalty), es, -1 if eos_token_id is None else int(eos_token_id), fill)
                seq = torch.empty(B * nrs, n_new, dtype=torch.int64, device=self.device)
                scores = torch.empty(B * nrs, dtype=torch.float32, device=self.device)
                lens = torch.empty(B * nrs, dtype=torch.int32, device=self.device)
                if record is not None:
                    rec_scores, rec_logits = self._record_buffers(record, n_new, B * nb)
                    bidx = torch.empty(B * nrs, n_new, dtype=torch.int64, device=self.device)
                    steps = torch.empty(1, dtype=torch.int32, device=self.device)
                    bp.scores_out, bp.logits_out = _ptr(rec_scores), _ptr(rec_logits)
                    bp.beam_indices_out, bp.steps_out = bidx.data_ptr(), steps.data_ptr()
                check(self._lib.vly_beam_search(self._ctx, cache._h, C.byref(bp), logits.data_ptr(), S, n_new, seq.data_ptr(),
                                                scores.data_ptr(), lens.data_ptr(), _stream()))
                self.last_beam_scores = scores
                if record is None:
                    L = int(lens.max())                      # the request's one device-to-host read
                    return torch.cat([_repeat_rows(ids_dev, nrs), seq[:, :L]], dim=1)
                L, n_steps = torch.stack([lens.max(), steps[0]]).tolist()      # (still one read)
                return generation_output(torch.cat([_repeat_rows(ids_dev, nrs), seq[:, :L]], dim=1), n_steps, rec_scores,
                                         rec_logits, sequences_scores=scores if record[0] else None,
                                         beam_indices=bidx[:, :L], beam=True)
            # host-visible loop: the same search in torch over the library's logits, with HF's stopping criteria on the
            # candidates (a criterion returning a plain bool applies to every row, as in HF's StoppingCriteriaList)
            bs = _beam.BeamSearch(ids_rep, nb, n_new, eos_token_id, fill, length_penalty, early_stopping,
                                  record_scores=record is not None and record[0], record_logits=record is not None and record[1],
                                  processors=procs)
            stop = None
            if stopping_criteria or tables is not None:
                def stop(seqs):
                    done = torch.zeros(seqs.shape[0], dtype=torch.bool, device=seqs.device)
                    for sc in stopping_criteria or ():
                        done = done | torch.as_tensor(sc(seqs, None), device=seqs.device)
                    if tables is not None:
                        done = done | _ss.match_rows(seqs, tables).to(seqs.device)
                    return done
            while True:
                parents, tokens = bs.step(logits, stop)
                if bs.done:
                    break
                cache.reorder_cache(parents, from_pos=S)
                step_logits, _ = self._decode(cache, tokens, True)
                logits = step_logits[:, -1]
            out, self.last_beam_scores = bs.result(num_return_sequences)
            if record is None:
                return out
            stacked = lambda steps: torch.stack(steps) if steps is not None else None
            return generation_output(out, bs.t, stacked(bs.scores), stacked(bs.logits),
                                     sequences_scores=self.last_beam_scores if record[0] else None,
                                     beam_indices=bs.beam_indices(num_return_sequences), beam=True)
        finally:
            cache.release()

    def compute_transition_scores(self, sequences: torch.Tensor, scores, beam_indices: Optional[torch.Tensor] = None,
                                  normalize_logits: bool = False) -> torch.Tensor:
        """transformers' ``GenerationMixin.compute_transition_scores``: the score of each generated token of ``sequences``
        [rows, S + L] at its step, from ``scores`` (generate's per-step tuple) and, after a beam search, ``beam_indices``;
        [rows, L], 0 after a hypothesis ended.  ``normalize_logits`` applies a log-softmax over the vocabulary first."""
        V = self.config.vocab_size
        if beam_indices is None:             # greedy / sampling: row r always continues row r
            beam_indices = torch.arange(scores[0].shape[0]).view(-1, 1).to(sequences.device)
            beam_indices = beam_indices.expand(-1, len(scores))
        stacked = torch.stack(scores).reshape(len(scores), -1).transpose(0, 1)       # [rows * V, steps]
        if normalize_logits:
            stacked = stacked.reshape(-1, V, stacked.shape[-1])
            stacked = torch.nn.functional.log_softmax(stacked, dim=1)
            stacked = stacked.reshape(-1, stacked.shape[-1])
        mask = beam_indices < 0
        max_len = (1 - mask.long()).sum(-1).max()
        beam_indices = beam_indices.clone()[:, :max_len]
        mask = mask[:, :max_len]
        beam_indices[mask] = 0
        indices = sequences[:, sequences.shape[-1] - max_len:] + beam_indices * V
        out = stacked.gather(0, indices)
        out[mask] = 0
        return out

    _KEYWORD_ROUTE_ARGS = frozenset({"max_new_tokens", "do_sample", "temperature", "eos_token_id", "pad_token_id",
                                     "attention_mask", "top_k", "top_p", "num_beams", "use_cache"})

    def _keyword_generate(self, input_ids, images, criterion: KeywordsStoppingCriteria, gen_kwargs):
        """``generate(stopping_criteria=[criterion], **gen_kwargs)`` for a greedy single-row request, with the keyword matched
        on the device instead of decoding the reply after every token; None when the request does not qualify (sampled,
        beams, more rows, other arguments, or a keyword past the device limits), and the host loop runs it instead.

        The criterion decides, as in the host loop: it is called after the first token (which only records the prompt
        length), and again whenever the device loop stops early -- on a stop-string match of a keyword over the generated
        tokens, or on a token the criterion's decode deletes (``stop_strings.pause_bits``: such a token can join two halves
        of a keyword) -- and True ends the request, False resumes the device loop.  A first token whose own text holds a
        keyword is followed by one host step, as the host loop's criterion only sees it then."""
        kw = dict(gen_kwargs)
        greedy = not kw.pop("do_sample", False) or kw.pop("temperature", 1.0) < 1e-4
        kw.pop("temperature", None)
        if (not greedy or kw.pop("num_beams", 1) != 1 or input_ids.shape[0] != 1 or set(kw) - self._KEYWORD_ROUTE_ARGS
                or not hasattr(criterion.tokenizer, "get_vocab")):
            return None
        tok = criterion.tokenizer
        V = self.config.vocab_size
        tables = _ss.stop_tables(_ss.clean_token_strings(tok), criterion.keywords, V)
        if not tables.on_device:
            return None
        S = input_ids.shape[1]
        n_new, eos, pad, attention_mask = self._generation_defaults(input_ids, kw.get("max_new_tokens", 1024),
                                                                    kw.get("eos_token_id", _UNSET), kw)
        if n_new == 0:
            return None
        pause = _ss.pause_bits(tok, V, exclude=() if eos is None else (int(eos),))
        paused = lambda t: bool((int(pause[t >> 5]) >> (t & 31)) & 1) if 0 <= t < V else False
        _, _, _, embeds, _ = self.prepare_inputs_labels_for_multimodal(input_ids, None, None, None, images)
        cache = self.new_cache(1)
        try:
            cache.set_attention_mask(attention_mask, S)
            _, nxt = self._prefill(cache, embeds, 0)
            seq = torch.cat([input_ids.to(self.device, torch.int64), nxt[:, None]], dim=1)
            gen = [int(nxt.item())]
            if eos is not None and gen[0] == eos:
                return seq
            if criterion(seq, None):                        # (records the prompt length)
                return seq
            if len(gen) < n_new and any(k in tok.decode(gen[:1], skip_special_tokens=True) for k in criterion.keywords):
                _, nxt = self._decode(cache, nxt, False)
                seq = torch.cat([seq, nxt[:, None]], dim=1)
                gen.append(int(nxt.item()))
                if (eos is not None and gen[-1] == eos) or criterion(seq, None):
                    return seq
            last = nxt
            while len(gen) < n_new:
                n = n_new - len(gen)
                tail = [t for t in gen if not paused(t)][-63:]
                sp = VlySampling(0.0, 0, -1 if eos is None else int(eos), int(pad) if pad is not None else 0)
                sp.set_stop_strings(tables, np.asarray([tail], dtype=np.int64).reshape(1, len(tail)), pause, restart=True)
                rest = torch.empty(1, n, dtype=torch.int64, device=self.device)
                done = torch.zeros(1, dtype=torch.int32, device=self.device)
                check(self._lib.vly_generate(self._ctx, cache._h, last.reshape(1).contiguous().data_ptr(), n, rest.data_ptr(),
                                             C.byref(sp), done.data_ptr(), _stream()))
                k = int(done.item())
                seq = torch.cat([seq, rest[:, :k]], dim=1)
                gen += rest[0, :k].tolist()
                if k == n or (eos is not None and gen[-1] == eos) or criterion(seq, None):
                    break
                last = rest[:, k - 1].clone()
            return seq
        finally:
            cache.release()

    # ---------------- prompt helpers (pure string logic; valley_model.py:381-422) ----------------
    def build_inputs(self, tokenizer, messages):
        prompt = ''
        for m in messages:
            if m['role'] == 'system':
                prompt += m['content'] + '\n\n' + '###'
            elif m['role'] == 'user':
                replace_token = DEFAULT_IM_START_TOKEN + DEFAULT_IMAGE_PATCH_TOKEN * 256 + DEFAULT_IM_END_TOKEN + \
                    DEFAULT_VI_START_TOKEN + DEFAULT_VIDEO_FRAME_TOKEN * 8 + DEFAULT_VI_END_TOKEN
                if '<video>' in m['content'] or '<image>' in m['content']:
                    message = m['content'].replace('<video>', replace_token).replace('<image>', replace_token)
                    prompt += ' ' + 'Human' + ": " + message + ' \n' + '###'
            elif m['role'] == 'assistent':
                prompt += ' ' + 'Assistent' + ": " + m['content'] + ' \n' + '###'
            else:
                raise ValueError("Role is only suport \"assistent\", \"human\" and \"system\".")
        if DEFAULT_IM_START_TOKEN not in prompt:
            raise ValueError("You need to specify the <video> token in the query")
        tokenizer.padding_side = 'left'
        return tokenizer([prompt], padding=True)

    def process_response(self, outputs):
        output = []
        for out in outputs:
            while True:
                cur_len = len(out)
                out = out.strip()
                for pattern in ['###', 'Assistant:', 'Response:', 'Valley:']:
                    if out.startswith(pattern):
                        out = out[len(pattern):].strip()
                if len(out) == cur_len:
                    break
            if '###' not in out:
                out += '###'
            output.append(out[:out.index('###')].strip())
        return output

    @torch.no_grad()
    def completion(self, tokenizer, video, message: list, gen_kwargs: dict, device=None):
        """valley_model.py:424-439, same call: ``model.completion(tokenizer, args.video_file, message, gen_kwargs, device)``
        (run_valley.py:56).  ``video`` is a file path -- opened by ``self.video_reader_factory`` (decord by default, as
        load_video does; container decoding is CPU work outside the hot path) and then sampled (8 frames, 'fixed'),
        resized, cropped and normalised ON THE DEVICE, bit-identical to load_video (valley_b200/video.py) -- or the decoded
        clip tensor [3,T,224,224] load_video would have returned.  Generation stops like the reference's: the
        ``KeywordsStoppingCriteria(['###'])`` it passes (:431-432) plus HF generate's default stop on ``config.eos_token_id``
        (overridable through ``gen_kwargs``)."""
        inputs = self.build_inputs(tokenizer, message)
        input_ids = torch.as_tensor(inputs.input_ids).to(self.device)
        if torch.is_tensor(video):
            images = video.permute(1, 0, 2, 3).unsqueeze(0).half().to(self.device)
        else:
            from . import video as _video
            if os.path.isdir(str(video)):              # load_video's directory-of-images branch (data_util.py:282-302)
                images = _video.load_image_dir(str(video), getattr(self, "image_processor", None)).unsqueeze(0).half().to(self.device)
            else:
                reader = self.video_reader_factory(str(video))
                images = _video.load_video(self, reader, "fixed", 8, dtype=torch.float16).unsqueeze(0)      # [1,T,3,224,224]
        gen_kwargs = dict(gen_kwargs)
        if "attention_mask" not in gen_kwargs and getattr(inputs, "attention_mask", None) is not None:
            am = torch.as_tensor(inputs.attention_mask)
            if bool((am == 0).any()):               # build_inputs pads on the left (valley_model.py:400-402); B == 1 -> no padding
                gen_kwargs["attention_mask"] = am
        if "eos_token_id" not in gen_kwargs and getattr(tokenizer, "eos_token_id", None) is not None \
                and getattr(self.config, "eos_token_id", None) is None:
            gen_kwargs["eos_token_id"] = tokenizer.eos_token_id
        stopping_criteria = KeywordsStoppingCriteria(['###'], tokenizer, input_ids)
        output_ids = self._keyword_generate(input_ids, images, stopping_criteria, gen_kwargs)
        if output_ids is None:
            output_ids = self.generate(input_ids=input_ids, images=images, stopping_criteria=[stopping_criteria], **gen_kwargs)
        input_token_len = input_ids.shape[1]
        n_diff_input_output = (input_ids != output_ids[:, :input_token_len]).sum().item()
        if n_diff_input_output > 0:
            print(f'[Warning] {n_diff_input_output} output_ids are not the same as the input_ids')
        outputs = tokenizer.batch_decode(output_ids[:, input_token_len:], skip_special_tokens=True)
        return self.process_response(outputs)
