"""How many kernels each entry point launches, as vly_kernel_launch_count reports it.  The counter is what bench.py reports
as gpu_launches and what the decode graphs' node counts are derived from, so every number here is written out as a formula
in the model's layer counts and the batch, read off the host code: a launch that is added, dropped or miscounted shows up."""
import ctypes as C

import pytest
import torch

import helpers as Hh
from valley_b200 import synthetic as syn
from valley_b200._lib import VlySampling, check

_models = {}


def get(spec_name):
    if spec_name not in _models:
        spec = syn.SPECS[spec_name]
        _models[spec_name] = (spec, Hh.build_model(spec, Hh.bf16_weights(spec, 0)))
    return _models[spec_name]


def launched(m, fn):
    before = m.launches()
    fn()
    torch.cuda.synchronize()
    return m.launches() - before


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _embeds(m, spec, B, S, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, spec.vocab_size - 8, (B, S), generator=g)
    return m.prepare_inputs_labels_for_multimodal(ids)[3]


def _per_op_step(spec, B):
    """one decode step at B > 4: per group of <= 4 rows the embedding, 5 kernels per layer and the lm_head GEMV; then one
    selection kernel over all rows"""
    return -(-B // 4) * (1 + 5 * spec.num_hidden_layers + 1) + 1


def _step(spec, B):
    return 1 if B <= 4 else _per_op_step(spec, B)      # B <= 4: the persistent kernel alone


@pytest.mark.gpu
def test_weight_preparation_is_counted():
    """every tensor of the fp32 state dict is converted once by vly_load_weight; vly_finalize_weights then packs the patch
    embedding, q / k / v and fc1 of every ViT layer, q / k / v and gate / up of every LLaMA layer and the lm_head, and writes
    the RoPE table"""
    spec = syn.TINY
    sd = Hh.bf16_weights(spec, 0)
    m = Hh.build_model(spec, sd)
    L, VL = spec.num_hidden_layers, spec.vit_layers
    assert m.launches() == len(sd) + 1 + 4 * VL + 5 * L + 1 + 1


@pytest.mark.gpu
@pytest.mark.parametrize("select_layer", [-2, -1])
def test_vit_encode(select_layer):
    """im2col, patch GEMM and embedding LayerNorm, then 5 kernels per encoder layer up to the selected one"""
    spec, m = get("tiny")
    px = syn.make_pixels(1, 2, 0).reshape(2, 3, 224, 224).cuda()
    layers = spec.vit_layers + 1 + select_layer
    assert launched(m, lambda: m._vit_encode(px, select_layer)) == 3 + 5 * layers


@pytest.mark.gpu
def test_project():
    spec, m = get("tiny")
    feats = torch.randn(2, 257, 1024, device="cuda").bfloat16()
    assert launched(m, lambda: m._project(feats)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("spec_name,per_call,per_video", [
    ("tiny", 2, 0),          # mean: temporal pool + projector GEMM
    ("tiny-v2", 3, 0),       # temporal_importance: scores + weighted pool + projector GEMM
    ("tiny-max", 0, 2),      # max: per video a projector GEMM + temporal max
    ("tiny-v3", 0, 12),      # temporal_transformer: per video the projector GEMM, 5 encoder-layer GEMMs and 6 other kernels
])
def test_pool_project(spec_name, per_call, per_video):
    spec, m = get(spec_name)
    NV, T = 2, 3
    feats = torch.randn(NV * T, 257, 1024, device="cuda").bfloat16()
    assert launched(m, lambda: m._pool_project(feats, NV, T)) == per_call + NV * per_video


@pytest.mark.gpu
def test_embed_splice():
    spec, m = get("tiny")
    assert launched(m, lambda: _embeds(m, spec, 2, 16)) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 6])
@pytest.mark.parametrize("logits_mode", [0, 1, 2])
def test_prefill(B, logits_mode):
    """row copy + statistics, 5 kernels per layer, the lm_head over every position (mode 2), the last-token lm_head GEMV per
    group of <= 4 rows, and the length update"""
    spec, m = get("tiny")
    e = _embeds(m, spec, B, 16)
    cache = m.new_cache(B, 256)
    try:
        n = launched(m, lambda: m._prefill(cache, e, logits_mode))
    finally:
        cache.release()
    assert n == 1 + 5 * spec.num_hidden_layers + (logits_mode == 2) + -(-B // 4) + 1


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 6])
def test_decode_and_generate(B):
    """a decode step and generate replay the step's graph: its nodes are counted, its capture is not.  A sampled request
    leaves the selection state dirty, and the next greedy call resets it with one more kernel"""
    spec, m = get("tiny")
    cache = m.new_cache(B, 256)
    try:
        _, nxt = m._prefill(cache, _embeds(m, spec, B, 16), 0)
        assert launched(m, lambda: m._decode(cache, nxt, False)) == _step(spec, B)
        assert launched(m, lambda: m._decode(cache, nxt, True)) == _step(spec, B)
        out = torch.empty(B, 9, dtype=torch.int64, device="cuda")

        def greedy():
            check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), 9, out.data_ptr(), _stream()))

        assert launched(m, greedy) == 9 * _step(spec, B)             # one 8-step graph and one 1-step graph
        logits = torch.randn(B, spec.vocab_size, device="cuda")
        first = torch.empty(B, dtype=torch.int64, device="cuda")
        sp = VlySampling(temperature=0.8, seed=3)

        def sample():
            check(m._lib.vly_sample_logits(m._ctx, cache._h, logits.data_ptr(), C.byref(sp), first.data_ptr(), _stream()))

        assert launched(m, sample) == 2                                # state update + selection
        assert launched(m, greedy) == 1 + 9 * _step(spec, B)
        assert launched(m, greedy) == 9 * _step(spec, B)
    finally:
        cache.release()


@pytest.mark.gpu
def test_key_mask_and_export():
    spec, m = get("tiny")
    B, S = 2, 16
    cache = m.new_cache(B, 256)
    try:
        assert launched(m, lambda: cache.set_attention_mask(torch.ones(B, S, dtype=torch.int64), S)) == 1
        m._prefill(cache, _embeds(m, spec, B, S), 0)
        assert launched(m, lambda: cache.to_hf(0)) == 2                # keys and values
    finally:
        cache.release()


@pytest.mark.gpu
def test_cross_entropy_and_preprocess():
    spec, m = get("tiny")
    B, S = 2, 8
    logits = torch.randn(B, S, spec.vocab_size, device="cuda")
    labels = torch.randint(0, spec.vocab_size, (B, S), device="cuda")
    loss = torch.empty(1, device="cuda")
    assert launched(m, lambda: check(m._lib.vly_cross_entropy(m._ctx, logits.data_ptr(), labels.data_ptr(), B, S, -100,
                                                               loss.data_ptr(), _stream()))) == 2
    T = 2
    frames = torch.randint(0, 256, (T, 240, 320, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty(T, 3, 224, 224, device="cuda")
    assert launched(m, lambda: check(m._lib.vly_preprocess_frames(m._ctx, frames.data_ptr(), T, 240, 320, 0, out.data_ptr(),
                                                                   _stream()))) == 2


@pytest.mark.gpu
def test_export_rejects_a_cache_of_another_model():
    """two models of the same shapes: indexing one model's cache with the other's context must be refused, not tolerated"""
    spec, m = get("tiny")
    other = Hh.build_model(spec, Hh.bf16_weights(spec, 1))
    cache = other.new_cache(2, 256)
    try:
        other._prefill(cache, _embeds(other, spec, 2, 16), 0)
        t = torch.empty(2, spec.num_attention_heads, 16, 128, dtype=torch.bfloat16, device="cuda")
        with pytest.raises(ValueError):
            check(m._lib.vly_kv_export(m._ctx, cache._h, 0, 0, t.data_ptr(), _stream()))
    finally:
        cache.release()
