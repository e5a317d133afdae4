"""Synthetic random-init weights, prompts and pixels for the BASELINE.json configurations.

There is no network for checkpoints or datasets, so every configuration is run on
random-init weights of the named architecture and synthetic inputs of the named shape
(SURVEY.md 8d "Synthetic inputs").  Tensors are produced per HF state_dict name
(SURVEY.md 8b "Weight names to accept") so the same dict can be handed to the CUDA path
(``ValleyLlamaForCausalLM.load_state_dict``), to the CPU oracle, and -- in the build
container -- to the reference class itself.
"""
from __future__ import annotations

import dataclasses
from typing import Dict, Iterator, Optional, Tuple

import torch

VIT_PFX = "model.vision_tower.vision_model."


@dataclasses.dataclass
class ShapeSpec:
    """Architecture of one Valley checkpoint family (SURVEY.md section 8, model constants)."""
    name: str
    hidden_size: int
    num_hidden_layers: int
    num_attention_heads: int
    intermediate_size: int
    vocab_size: int = 32008          # 32000 + 7 added tokens (SURVEY 8), padded to 8-element alignment
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    max_position_embeddings: int = 2048
    vit_hidden: int = 1024
    vit_layers: int = 24
    vit_heads: int = 16
    vit_mlp: int = 4096
    vit_patch: int = 14
    vit_image: int = 224
    vit_eps: float = 1e-5
    mm_vision_select_layer: int = -2
    patch_pooling_method: str = "mean"   # "mean" | "max" | "temporal_importance" (v2) | "temporal_transformer" (v3)


VALLEY2_7B = ShapeSpec("valley2-7b", 4096, 32, 32, 11008, rms_norm_eps=1e-5)          # Llama-2-7B shape
VALLEY_13B = ShapeSpec("valley-13b", 5120, 40, 40, 13824, rms_norm_eps=1e-6)          # LLaMA-13B shape
TINY = ShapeSpec("tiny", 512, 2, 4, 1024, vocab_size=1032, vit_layers=3)               # parity-test size
TINY_WIDE = ShapeSpec("tiny-wide", 768, 3, 6, 1536, vocab_size=2056, vit_layers=2, rms_norm_eps=1e-6)

# one decoder layer / one ViT layer at the real widths: parity at the production shapes (K tails, 40 heads, V = 32008)
SHAPE_7B_1L = ShapeSpec("shape-7b-1l", 4096, 1, 32, 11008, vit_layers=2)
SHAPE_13B_1L = ShapeSpec("shape-13b-1l", 5120, 1, 40, 13824, rms_norm_eps=1e-6, vit_layers=2)

# pooling variants (valley_model.py:40-52): v2 = learned temporal importance, v3 = temporal transformer delta
TINY_V2 = ShapeSpec("tiny-v2", 512, 2, 4, 1024, vocab_size=1032, vit_layers=2, patch_pooling_method="temporal_importance")
TINY_V3 = ShapeSpec("tiny-v3", 512, 2, 4, 1024, vocab_size=1032, vit_layers=2, patch_pooling_method="temporal_transformer")
TINY_MAX = ShapeSpec("tiny-max", 512, 2, 4, 1024, vocab_size=1032, vit_layers=2, patch_pooling_method="max")
SHAPE_7B_1L_V3 = ShapeSpec("shape-7b-1l-v3", 4096, 1, 32, 11008, vit_layers=2, patch_pooling_method="temporal_transformer")

# intermediate_size = 7 x 512: a wide down_proj K for the tensor-core decode consumer (B = 2..4)
TINY_UMMA = ShapeSpec("tiny-umma", 512, 2, 4, 3584, vocab_size=1032, vit_layers=2)
# intermediate_size = 59 x 64 (not a multiple of 512, like Llama-2-7B's 11008): down_proj's K does not divide into whole ring stages
TINY_UMMA_RAGGED = ShapeSpec("tiny-umma-ragged", 512, 2, 4, 3776, vocab_size=1032, vit_layers=2)

SPECS = {s.name: s for s in (VALLEY2_7B, VALLEY_13B, TINY, TINY_WIDE, SHAPE_7B_1L, SHAPE_13B_1L, TINY_V2, TINY_V3, TINY_MAX,
                             SHAPE_7B_1L_V3, TINY_UMMA, TINY_UMMA_RAGGED)}


def weight_shapes(spec: ShapeSpec, *, vision: bool = True, llm: bool = True) -> Iterator[Tuple[str, Tuple[int, ...], str]]:
    """Yield (hf_name, shape, kind) for every tensor on the path; kind picks the init."""
    H, I, V, D, M = spec.hidden_size, spec.intermediate_size, spec.vocab_size, spec.vit_hidden, spec.vit_mlp
    if vision:
        p = VIT_PFX
        yield p + "embeddings.class_embedding", (D,), "emb"
        yield p + "embeddings.patch_embedding.weight", (D, 3, spec.vit_patch, spec.vit_patch), "conv"
        n_pos = (spec.vit_image // spec.vit_patch) ** 2 + 1
        yield p + "embeddings.position_embedding.weight", (n_pos, D), "emb"
        yield p + "pre_layrnorm.weight", (D,), "ln_w"
        yield p + "pre_layrnorm.bias", (D,), "ln_b"
        for i in range(spec.vit_layers):
            q = f"{p}encoder.layers.{i}."
            for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
                yield q + f"self_attn.{nm}.weight", (D, D), "lin"
                yield q + f"self_attn.{nm}.bias", (D,), "bias"
            yield q + "layer_norm1.weight", (D,), "ln_w"
            yield q + "layer_norm1.bias", (D,), "ln_b"
            yield q + "mlp.fc1.weight", (M, D), "lin"
            yield q + "mlp.fc1.bias", (M,), "bias"
            yield q + "mlp.fc2.weight", (D, M), "lin_out"
            yield q + "mlp.fc2.bias", (D,), "bias"
            yield q + "layer_norm2.weight", (D,), "ln_w"
            yield q + "layer_norm2.bias", (D,), "ln_b"
        yield "model.mm_projector.weight", (H, D), "lin"
        yield "model.mm_projector.bias", (H,), "bias"
        if spec.patch_pooling_method == "temporal_importance":          # valley_model.py:40-43
            yield "model.pooling_layer.weight", (1, H * 256), "pool"
            yield "model.pooling_layer.bias", (1,), "bias"
        if spec.patch_pooling_method == "temporal_transformer":         # valley_model.py:45-52
            q = "model.transformer_delta_encoder.layers.0."
            yield "model.position_matrix", (2048, H), "emb"
            yield q + "self_attn.in_proj_weight", (3 * H, H), "lin"
            yield q + "self_attn.in_proj_bias", (3 * H,), "bias"
            yield q + "self_attn.out_proj.weight", (H, H), "lin"
            yield q + "self_attn.out_proj.bias", (H,), "bias"
            yield q + "linear1.weight", (2048, H), "lin"
            yield q + "linear1.bias", (2048,), "bias"
            yield q + "linear2.weight", (H, 2048), "lin_out"
            yield q + "linear2.bias", (H,), "bias"
            yield q + "norm1.weight", (H,), "ln_w"
            yield q + "norm1.bias", (H,), "ln_b"
            yield q + "norm2.weight", (H,), "ln_w"
            yield q + "norm2.bias", (H,), "ln_b"
    if llm:
        yield "model.embed_tokens.weight", (V, H), "tok"
        for i in range(spec.num_hidden_layers):
            q = f"model.layers.{i}."
            for nm in ("q_proj", "k_proj", "v_proj", "o_proj"):
                yield q + f"self_attn.{nm}.weight", (H, H), "lin"
            yield q + "mlp.gate_proj.weight", (I, H), "lin"
            yield q + "mlp.up_proj.weight", (I, H), "lin"
            yield q + "mlp.down_proj.weight", (H, I), "lin_out"
            yield q + "input_layernorm.weight", (H,), "ln_w"
            yield q + "post_attention_layernorm.weight", (H,), "ln_w"
        yield "model.norm.weight", (H,), "ln_w"
        yield "lm_head.weight", (V, H), "head"


def _init(kind: str, shape, gen: torch.Generator, device, fan_in: int) -> torch.Tensor:
    r = torch.randn(shape, generator=gen, device=device, dtype=torch.float32)
    if kind in ("lin", "conv"):
        return r * 0.02
    if kind == "lin_out":
        return r * (0.02 * 0.5)
    if kind == "head":
        return r * 0.05
    if kind == "tok":
        return r * 0.5
    if kind == "pool":
        return r * 0.002          # scores = w . flatten(256*H features): keeps the softmax over frames informative
    if kind == "emb":
        return r * 0.02
    if kind == "bias":
        return r * 0.02
    if kind == "ln_w":
        return 1.0 + 0.1 * r
    if kind == "ln_b":
        return 0.05 * r
    raise ValueError(kind)


def iter_state_dict(spec: ShapeSpec, seed: int = 0, device="cpu", dtype=torch.float32, *,
                    vision: bool = True, llm: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
    """Stream (name, tensor) pairs -- one tensor resident at a time, so a 13B model can be
    loaded into the CUDA library without a second full copy."""
    gen = torch.Generator(device=device)
    for idx, (name, shape, kind) in enumerate(weight_shapes(spec, vision=vision, llm=llm)):
        gen.manual_seed(seed * 1000003 + idx)
        yield name, _init(kind, shape, gen, device, shape[-1]).to(dtype)


def make_state_dict(spec: ShapeSpec, seed: int = 0, device="cpu", dtype=torch.float32, **kw) -> Dict[str, torch.Tensor]:
    return dict(iter_state_dict(spec, seed, device, dtype, **kw))


def sentinel_ids(spec: ShapeSpec) -> Dict[str, int]:
    """The six highest vocabulary ids (SURVEY.md 8d)."""
    V = spec.vocab_size
    return dict(im_patch_token=V - 6, im_start_token=V - 5, im_end_token=V - 4,
                vi_frame_token=V - 3, vi_start_token=V - 2, vi_end_token=V - 1)


def make_prompt_ids(spec: ShapeSpec, batch: int, frames: int, seed: int = 0, len_a: int = 40, len_b: int = 24,
                    n_patches: int = 256) -> torch.Tensor:
    """[1] + text_a + <im_start> <im_patch>*256 <im_end> <vi_start> <vi_frame>*T <vi_end> + text_b
    (model_worker.py:338-341 layout; SURVEY.md 8d).  S = 1+len_a+1+256+2+T+1+len_b."""
    t = sentinel_ids(spec)
    gen = torch.Generator().manual_seed(seed + 7919)
    rows = []
    for _ in range(batch):
        a = torch.randint(3, spec.vocab_size - 8, (len_a,), generator=gen)
        b = torch.randint(3, spec.vocab_size - 8, (len_b,), generator=gen)
        mid = [t["im_start_token"]] + [t["im_patch_token"]] * n_patches + [t["im_end_token"], t["vi_start_token"]] \
            + [t["vi_frame_token"]] * frames + [t["vi_end_token"]]
        rows.append(torch.cat([torch.tensor([1]), a, torch.tensor(mid), b]))
    return torch.stack(rows).to(torch.int64)


def make_pixels(batch: int, frames: int, seed: int = 0, image: int = 224, dtype=torch.float32) -> torch.Tensor:
    """CLIP-normalised pixels are ~N(0,1) per channel (data_util.py:272-273)."""
    gen = torch.Generator().manual_seed(seed + 104729)
    return torch.randn(batch, frames, 3, image, image, generator=gen).to(dtype)
