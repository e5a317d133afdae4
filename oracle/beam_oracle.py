"""Beam search on the fp32 CPU oracle model: HF generate's beam search (valley_b200/beam.py, the torch restatement of
transformers' GenerationMixin._beam_search that generate's host-visible loop runs) driven by valley_oracle's LLaMA forward.
HF's ``_expand_inputs_for_generation`` repeats every row num_beams times, and ``Cache.reorder_cache(beam_idx)`` becomes an
``index_select`` of the oracle's growing K/V tensors.  tests/golden/ref_beam_search.pt (transformers' own generate on the same
weights) pins it."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from oracle import valley_oracle as O
from valley_b200.beam import BeamSearch


@torch.no_grad()
def beam_generate(w, cfg: O.OracleConfig, tok: O.SentinelIds, input_ids: torch.Tensor, images, max_new_tokens: int,
                  num_beams: int, eos_token_id: Optional[int], fill: int, length_penalty: float = 1.0, early_stopping=False,
                  attention_mask: Optional[torch.Tensor] = None) -> BeamSearch:
    """-> the finished BeamSearch (``.result(nrs)``, ``.margins``)"""
    nb = num_beams
    if images is not None:
        feats = O.encode_images(w, images, cfg.mm_vision_select_layer, num_layers=cfg.vit_layers, heads=cfg.vit_heads,
                                patch=cfg.vit_patch, eps=cfg.vit_eps)
        embeds = O.prepare_inputs_embeds(w, input_ids, feats, tok, cfg.patch_pooling_method)
    else:
        embeds = F.embedding(input_ids, w["model.embed_tokens.weight"])
    embeds = embeds.repeat_interleave(nb, 0)
    mask = attention_mask.repeat_interleave(nb, 0) if attention_mask is not None else None
    cache = O.KVCache(cfg.num_hidden_layers)

    def forward(x):
        h = O.llama_model(w, x, cache, n_layers=cfg.num_hidden_layers, heads=cfg.num_attention_heads, eps=cfg.rms_norm_eps,
                          theta=cfg.rope_theta, attention_mask=mask)
        return F.linear(h[:, -1], w["lm_head.weight"]).float()

    logits = forward(embeds)
    bs = BeamSearch(input_ids.repeat_interleave(nb, 0), nb, max_new_tokens, eos_token_id, fill, length_penalty, early_stopping)
    while True:
        parents, tokens = bs.step(logits)
        if bs.done:
            return bs
        for layer in range(cfg.num_hidden_layers):
            cache.k[layer] = cache.k[layer].index_select(0, parents)
            cache.v[layer] = cache.v[layer].index_select(0, parents)
        if mask is not None:
            mask = torch.cat([mask, torch.ones_like(mask[:, :1])], dim=1)
        logits = forward(F.embedding(tokens[:, None], w["model.embed_tokens.weight"]))
