"""ctypes binding of libvalley_b200.so (the C ABI in include/valley_b200.h).

There is no fallback: if the shared library is missing, import fails loudly with the build
command; if no sm_90 GPU is visible, ``vly_create`` fails with the library's own message.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# VLY_LIB_PATH: A/B measurements against another build of the same ABI (tools/); the product always loads the in-tree library
LIB_PATH = os.environ.get("VLY_LIB_PATH") or os.path.join(_HERE, "lib", "libvalley_b200.so")


class VlyConfig(C.Structure):
    _fields_ = [
        ("hidden_size", C.c_int32), ("num_hidden_layers", C.c_int32), ("num_attention_heads", C.c_int32),
        ("intermediate_size", C.c_int32), ("vocab_size", C.c_int32),
        ("rms_norm_eps", C.c_float), ("rope_theta", C.c_float),
        ("max_position_embeddings", C.c_int32),
        ("vit_hidden", C.c_int32), ("vit_layers", C.c_int32), ("vit_heads", C.c_int32), ("vit_mlp", C.c_int32),
        ("vit_patch", C.c_int32), ("vit_image", C.c_int32),
        ("vit_eps", C.c_float),
        ("mm_vision_select_layer", C.c_int32),
        ("device", C.c_int32),
        ("patch_pooling_method", C.c_int32),
    ]


class VlyTokens(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("im_patch_token", "im_start_token", "im_end_token",
                                          "vi_frame_token", "vi_start_token", "vi_end_token")]


class VlySampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("seed", C.c_uint64), ("eos_token_id", C.c_int64), ("pad_token_id", C.c_int64),
                ("stop_token_id", C.c_int64), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("n_stop_strings", C.c_int32), ("stop_lens", C.POINTER(C.c_int32)), ("stop_masks", C.POINTER(C.c_uint64)),
                ("stop_token_lens", C.POINTER(C.c_int32)), ("pause_bits", C.POINTER(C.c_uint32)),
                ("stop_tail", C.POINTER(C.c_int64)), ("stop_tail_len", C.c_int32), ("stop_restart", C.c_int32),
                ("repetition_penalty", C.c_float), ("no_repeat_ngram_size", C.c_int32), ("min_length", C.c_int32),
                ("prompt_ids_dev", C.c_void_p),
                ("scores_out", C.c_void_p), ("logits_out", C.c_void_p)]

    def __init__(self, temperature=0.0, seed=0, eos_token_id=-1, pad_token_id=0, stop_token_id=-1, top_k=0, top_p=1.0):
        super().__init__(temperature, seed, eos_token_id, pad_token_id, stop_token_id, top_k, top_p)
        self._keep = ()

    def set_stop_strings(self, tables, tail=None, pause=None, restart=False):
        """Point the stop-string fields at ``tables`` (``stop_strings.StopTables``), the rows' last tokens before the first
        selected one (``tail`` [B, <= 63] int64 CPU, or None) and the pause bit set (uint32 CPU, or None).  The arrays are
        kept alive with the struct; the library copies them during the call."""
        import numpy as np
        lens = np.ascontiguousarray(tables.lens, dtype=np.int32)
        masks = np.ascontiguousarray(tables.masks, dtype=np.uint64)
        tok = np.ascontiguousarray(tables.token_lens, dtype=np.int32)
        keep = [lens, masks, tok]
        self.n_stop_strings = len(lens)
        self.stop_lens = lens.ctypes.data_as(C.POINTER(C.c_int32))
        self.stop_masks = masks.ctypes.data_as(C.POINTER(C.c_uint64))
        self.stop_token_lens = tok.ctypes.data_as(C.POINTER(C.c_int32))
        if pause is not None:
            pause = np.ascontiguousarray(pause, dtype=np.uint32)
            keep.append(pause)
            self.pause_bits = pause.ctypes.data_as(C.POINTER(C.c_uint32))
        if tail is not None and tail.shape[1] > 0:
            t = np.ascontiguousarray(np.asarray(tail, dtype=np.int64))
            keep.append(t)
            self.stop_tail = t.ctypes.data_as(C.POINTER(C.c_int64))
            self.stop_tail_len = t.shape[1]
        self.stop_restart = 1 if restart else 0
        self._keep = tuple(keep)
        return self


class VlyBeam(C.Structure):
    _fields_ = [("num_beams", C.c_int32), ("num_return_sequences", C.c_int32), ("length_penalty", C.c_float),
                ("early_stopping", C.c_int32), ("eos_token_id", C.c_int64), ("pad_token_id", C.c_int64),
                ("scores_out", C.c_void_p), ("logits_out", C.c_void_p), ("beam_indices_out", C.c_void_p),
                ("steps_out", C.c_void_p)]


VLY_OK, VLY_ERR_INVALID, VLY_ERR_CUDA, VLY_ERR_STATE = 0, -1, -2, -3
VLY_ERR_IM_COUNT, VLY_ERR_IM_CUT, VLY_ERR_INDEX = -10, -11, -12
VLY_F32, VLY_BF16, VLY_F16 = 0, 1, 2
POOLING = {"mean": 0, "max": 1, "temporal_importance": 2, "temporal_transformer": 3}

# every symbol include/valley_b200.h declares: name -> (restype, argtypes)
_p, _i, _i64, _vp = C.POINTER, C.c_int, C.c_int64, C.c_void_p
SIGNATURES = {
    "vly_last_error": (C.c_char_p, []),
    "vly_version": (C.c_char_p, []),
    "vly_create": (_i, [_p(VlyConfig), _p(_vp)]),
    "vly_destroy": (None, [_vp]),
    "vly_load_weight": (_i, [_vp, C.c_char_p, _vp, _i, _p(_i64), _i]),
    "vly_finalize_weights": (_i, [_vp]),
    "vly_vit_encode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "vly_gather_create": (_i, [_vp, _i64, _p(_vp), _vp]),
    "vly_gather_open_peers": (_i, [_vp, _vp, _i, _i]),
    "vly_vit_encode_gather": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "vly_vit_encode_gather_strided": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "vly_gather_release": (_i, [_vp, _vp]),
    "vly_gather_status": (_i, [_vp, _p(_i)]),
    "vly_preprocess_plan": (_i, [_i, _i, _p(_i), _p(_i), _p(_i), _p(_i)]),
    "vly_resample_coeffs": (_i, [_i, _i, _p(_i), _p(C.c_int32), _p(C.c_int32), _p(C.c_int32)]),
    "vly_preprocess_frames": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "vly_project": (_i, [_vp, _vp, _i64, _vp, _vp]),
    "vly_pool_project": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "vly_build_splice_map": (_i, [_p(_i64), _i, _i, _i, _p(VlyTokens), _p(C.c_int32), _p(C.c_int32)]),
    "vly_embed_splice": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "vly_kv_create": (_i, [_vp, _i, _i, _p(_vp)]),
    "vly_kv_decode_kernel": (_i, [_vp, C.c_char_p, _i]),
    "vly_kv_destroy": (None, [_vp]),
    "vly_kv_seq_len": (_i, [_vp, _p(_i)]),
    "vly_kv_reset": (_i, [_vp, _vp]),
    "vly_kv_set_key_mask": (_i, [_vp, _vp, _i, _vp]),
    "vly_kv_export": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "vly_llama_prefill": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "vly_llama_decode": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "vly_generate_greedy": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "vly_cross_entropy": (_i, [_vp, _vp, _vp, _i, _i, _i64, _vp, _vp]),
    "vly_sample_logits": (_i, [_vp, _vp, _vp, _p(VlySampling), _vp, _vp]),
    "vly_generate": (_i, [_vp, _vp, _vp, _i, _vp, _p(VlySampling), _vp, _vp]),
    "vly_beam_search": (_i, [_vp, _vp, _p(VlyBeam), _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "vly_kv_beam_reorder": (_i, [_vp, _vp, _vp, _i, _vp]),
    "vly_kernel_launch_count": (_i, [_vp, _p(_i64)]),
    "vly_held_bytes": (_i, [_p(_i64), _p(_i64)]),
    "vly_num_sms": (_i, [_vp, _p(_i)]),
    "vly_kv_debug_counters": (_i, [_vp, _vp, _i]),
    "vly_set_error_": (None, [C.c_char_p]),
    "vly_test_gemm": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, C.c_float, _vp, _vp, _vp, _i, _i, _i,
                           _vp]),
    "vly_test_prefill_attention": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "vly_test_vit_attention": (_i, [_vp, _vp, _i, _vp, _vp]),
    "vly_test_sample_filter": (_i, [_vp, _vp, _i, _i, C.c_float, _i, C.c_float, _vp, _vp]),
    "vly_test_logits_process": (_i, [_vp, _vp, _i, _i, _vp, _i, C.c_float, _i, _i, _i64, _vp, _vp]),
    "vly_test_stop_strings": (_i, [_vp, _p(VlySampling), _i, _vp, _i, _i, _vp, _vp]),
    "vly_test_gemv":(_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i64, C.c_float, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "vly_test_decode_attention": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
}

_lib = None


def load():
    """Load the shared library (once) and attach the signatures."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). valley_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        if not hasattr(lib, name) and os.environ.get("VLY_LIB_PATH"):
            continue                     # an OLDER build loaded on purpose for a same-box A/B (tools/): it may predate an entry point
        fn = getattr(lib, name)          # AttributeError here == the .so does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


class VlyError(RuntimeError):
    pass


def check(code: int):
    """Map a vly_status to the exception the reference raises on the same path
    (valley_model.py:220/227 ValueError; torch IndexError; model_worker.py:436-449 catches
    ValueError / CUDA errors)."""
    if code == VLY_OK:
        return
    msg = load().vly_last_error().decode()
    if code in (VLY_ERR_IM_COUNT, VLY_ERR_IM_CUT, VLY_ERR_INVALID):
        raise ValueError(msg)
    if code == VLY_ERR_INDEX:
        raise IndexError(msg)
    raise VlyError(f"[vly {code}] {msg}")
