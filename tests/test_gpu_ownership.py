"""GPU: every allocation the library makes is owned by a context or a KV cache and freed with it, on success and on every
error path.  Each test compares the exact byte counts vly_held_bytes reports (device-wide free memory means nothing on a
shared GPU)."""
import ctypes as C
import gc

import pytest
import torch

import helpers as Hh
from valley_b200 import _lib, synthetic as syn
from valley_b200._lib import check

pytestmark = pytest.mark.gpu


def held():
    d, p = C.c_int64(), C.c_int64()
    check(_lib.load().vly_held_bytes(C.byref(d), C.byref(p)))
    return d.value, p.value


def settled():
    gc.collect()
    return held()


def packed_weight_bytes(spec):
    """What vly_finalize_weights keeps: matrices bf16; vectors and the ViT position table fp32; the patch weights padded to
    kpad columns; the RoPE table as max_pos x 64 float2."""
    H, I, V, L = spec.hidden_size, spec.intermediate_size, spec.vocab_size, spec.num_hidden_layers
    D, M, P = spec.vit_hidden, spec.vit_mlp, spec.vit_patch
    kpad = (3 * P * P + 63) // 64 * 64
    NP = (spec.vit_image // P) ** 2
    vit = D * kpad * 2 + (3 * D + (NP + 1) * D) * 4
    vit += spec.vit_layers * ((3 * D * D + D * D + M * D + D * M) * 2 + (3 * D + 3 * D + D + M + M + D) * 4)
    vit += H * D * 2 + H * 4
    if spec.patch_pooling_method == "temporal_importance":
        vit += NP * D * 4
    if spec.patch_pooling_method == "temporal_transformer":
        ffn = max_pos = 2048                        # synthetic linear1 / position_matrix rows
        vit += (3 * H * H + H * H + 2 * ffn * H + max_pos * H) * 2 + (3 * H + H + ffn + H + 4 * H) * 4
    llm = V * H * 2 + L * (3 * H * H + H * H + 2 * I * H + H * I) * 2 + V * H * 2 + spec.max_position_embeddings * 64 * 8
    return vit + llm


@pytest.mark.parametrize("name", ["tiny", "tiny-v2", "tiny-v3"])
def test_finalize_keeps_only_the_packed_weights(name):
    spec = syn.SPECS[name]
    dev0, pin0 = settled()
    m = Hh.build_model(spec, syn.make_state_dict(spec, 0))
    dev, pin = held()
    assert (dev - dev0, pin - pin0) == (packed_weight_bytes(spec), 0)
    del m
    assert settled() == (dev0, pin0)


def _generate(m, spec, B, seed):
    ids, px = syn.make_prompt_ids(spec, B, 2, seed), syn.make_pixels(B, 2, seed)
    out = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=6)
    torch.cuda.synchronize()
    return out.cpu()


def test_dropping_the_model_frees_caches_and_gather_buffer():
    """The persistent decode path (B = 2) and the per-op path (B = 6) leave pooled KV-cache handles; the fused gather adds a
    buffer, its pinned timeout flag and (world 1) no peer mapping.  Dropping the model frees all of it."""
    spec = syn.TINY
    before = settled()
    m = Hh.build_model(spec, syn.make_state_dict(spec, 0))
    _generate(m, spec, 2, 0)
    _generate(m, spec, 6, 1)
    rows = 2 * ((spec.vit_image // spec.vit_patch) ** 2 + 1)
    buf, handle = C.c_void_p(), C.create_string_buffer(64)
    check(m._lib.vly_gather_create(m._ctx, rows, C.byref(buf), handle))
    check(m._lib.vly_gather_open_peers(m._ctx, handle, 1, 0))
    assert held() != before
    del m
    assert settled() == before


def test_rejected_weight_dtype_allocates_nothing():
    from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM
    m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(syn.TINY), 0)
    t = torch.zeros(64, 64, device="cuda")
    before = held()
    with pytest.raises(ValueError, match="unknown dtype 7"):
        check(m._lib.vly_load_weight(m._ctx, b"model.layers.0.self_attn.q_proj.weight", t.data_ptr(), 7,
                                     (C.c_int64 * 2)(64, 64), 2))
    assert held() == before


def test_failed_cache_creation_allocates_nothing(monkeypatch):
    spec = syn.SPECS["tiny-umma-ragged"]
    m = Hh.build_model(spec, syn.make_state_dict(spec, 0, vision=False))
    before = held()
    monkeypatch.setenv("VLY_MEGA_STAGES", "1")
    with pytest.raises(ValueError, match="weight ring"):
        m.new_cache(2)
    assert held() == before


def test_second_generate_reuses_the_cache():
    spec = syn.TINY
    m = Hh.build_model(spec, syn.make_state_dict(spec, 0))
    first = _generate(m, spec, 2, 0)
    after_first = held()
    assert torch.equal(_generate(m, spec, 2, 0), first)
    assert held() == after_first
