"""Writes tests/golden/ref_beam_search.pt: transformers' own ``LlamaForCausalLM.generate`` beam search (CPU, fp32) on the
``tiny`` synthetic weights (bf16-rounded, as the library holds them), with the oracle's beam search (oracle/beam_oracle.py)
run next to it for each step's smallest decision margin.

    python -m oracle.make_golden_beam_search

Cases (``CASES``): a text prompt over num_beams {2, 4} x num_return_sequences {1, num_beams} x length_penalty {1.0, 0.0, 2.0}
x early_stopping {False, True, "never"}; a left-padded batch of 2 with an attention mask; a multimodal prompt (given to
transformers as ``inputs_embeds`` + ``input_ids``); and batch 2 x 4 beams = 8 cache rows.  eos is a token of the greedy
continuation, so that finished hypotheses occur before the last step.  Position ids are passed explicitly as 0..S-1 on every
row: Valley never shifts them for padding (HF would otherwise derive them from the attention mask).  Each entry keeps the
sequences, HF's sequences_scores and the oracle's per-step margins (the smallest gap between consecutive top-(K+1)
accumulated scores)."""
from __future__ import annotations

import os

import torch

SPEC = "tiny"
N_NEW = 10
PAD = 0
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_beam_search.pt")


def _cases():
    out = []
    for nb in (2, 4):
        for nrs in sorted({1, nb}):
            for lp in (1.0, 0.0, 2.0):
                for es in (False, True, "never"):
                    out.append(dict(prompt="text", num_beams=nb, num_return_sequences=nrs, length_penalty=lp, early_stopping=es))
    out.append(dict(prompt="padded", num_beams=2, num_return_sequences=2, length_penalty=1.0, early_stopping=False))
    out.append(dict(prompt="multimodal", num_beams=4, num_return_sequences=1, length_penalty=1.0, early_stopping=False))
    out.append(dict(prompt="multimodal", num_beams=2, num_return_sequences=2, length_penalty=2.0, early_stopping=True))
    out.append(dict(prompt="padded", num_beams=4, num_return_sequences=4, length_penalty=1.0, early_stopping=False))
    out.append(dict(prompt="padded", num_beams=4, num_return_sequences=1, length_penalty=0.0, early_stopping="never"))
    return out


CASES = _cases()


def prompts(spec):
    """name -> (input_ids [B, S], attention_mask or None, images [B, T, 3, 224, 224] or None)"""
    from valley_b200 import synthetic as syn
    g = torch.Generator().manual_seed(20261017)
    text = torch.randint(3, spec.vocab_size - 8, (1, 12), generator=g)
    padded = torch.randint(3, spec.vocab_size - 8, (2, 11), generator=g)
    padded[1, :3] = PAD
    mask = torch.ones_like(padded)
    mask[1, :3] = 0
    mm = syn.make_prompt_ids(spec, 1, 2, 5, len_a=8, len_b=6)
    return {"text": (text, None, None), "padded": (padded, mask, None), "multimodal": (mm, None, syn.make_pixels(1, 2, 5))}


def weights(spec):
    from valley_b200 import synthetic as syn
    return {k: v.bfloat16().float() for k, v in syn.make_state_dict(spec, 0).items()}


def hf_model(spec, w):
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=spec.hidden_size, num_hidden_layers=spec.num_hidden_layers,
                      num_attention_heads=spec.num_attention_heads, num_key_value_heads=spec.num_attention_heads,
                      intermediate_size=spec.intermediate_size, vocab_size=spec.vocab_size, rms_norm_eps=spec.rms_norm_eps,
                      rope_theta=spec.rope_theta, max_position_embeddings=spec.max_position_embeddings,
                      tie_word_embeddings=False, attn_implementation="eager")
    m = LlamaForCausalLM(cfg).to(torch.float32).eval()
    llm = {k: v for k, v in w.items() if k.startswith("model.layers.") or k in ("model.embed_tokens.weight", "model.norm.weight", "lm_head.weight")}
    missing, unexpected = m.load_state_dict(llm, strict=False)
    assert not unexpected and all("rotary" in k for k in missing), (missing, unexpected)
    return m


def main():
    import transformers
    from oracle import beam_oracle as BO
    from oracle import valley_oracle as O
    from valley_b200 import synthetic as syn
    from valley_b200.beam import output_fill_value
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import helpers as Hh

    spec = syn.SPECS[SPEC]
    w = weights(spec)
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    m = hf_model(spec, w)
    inputs = {}
    for name, (ids, mask, images) in prompts(spec).items():
        embeds = None
        if images is not None:
            feats = O.encode_images(w, images, cfg.mm_vision_select_layer, num_layers=cfg.vit_layers, heads=cfg.vit_heads,
                                    patch=cfg.vit_patch, eps=cfg.vit_eps)
            embeds = O.prepare_inputs_embeds(w, ids, feats, tok, cfg.patch_pooling_method)
        B, S = ids.shape
        kw = dict(input_ids=ids, attention_mask=mask if mask is not None else torch.ones_like(ids),
                  position_ids=torch.arange(S)[None].expand(B, S).contiguous(), pad_token_id=PAD)
        if embeds is not None:
            kw["inputs_embeds"] = embeds
        with torch.no_grad():
            greedy = m.generate(**kw, max_new_tokens=4, do_sample=False, eos_token_id=None)
        inputs[name] = (kw, int(greedy[0, S + 3]))
    entries = []
    for case in CASES:
        kw, eos = inputs[case["prompt"]]
        ids, mask, images = prompts(spec)[case["prompt"]]
        with torch.no_grad():
            out = m.generate(**kw, max_new_tokens=N_NEW, do_sample=False, eos_token_id=eos, num_beams=case["num_beams"],
                             num_return_sequences=case["num_return_sequences"], length_penalty=case["length_penalty"],
                             early_stopping=case["early_stopping"], return_dict_in_generate=True, output_scores=True)
        fill = output_fill_value(PAD, eos)
        bs = BO.beam_generate(w, cfg, tok, ids, images, N_NEW, case["num_beams"], eos, fill, case["length_penalty"],
                              case["early_stopping"], attention_mask=mask)
        seq, scores = bs.result(case["num_return_sequences"])
        ok = torch.equal(seq, out.sequences)
        print(case, "eos", eos, "steps", bs.t, "min margin %.2e" % min(bs.margins), "oracle == transformers" if ok else "DIFFERENT",
              "max score diff %.1e" % float((scores - out.sequences_scores).abs().max()) if ok else "")
        assert ok, (seq, out.sequences)
        entries.append(dict(case=case, eos=eos, fill=fill, sequences=out.sequences.clone(),
                            scores=out.sequences_scores.float().clone(), margins=torch.tensor(bs.margins)))
    torch.save({"transformers": transformers.__version__, "spec": SPEC, "n_new": N_NEW, "pad": PAD, "entries": entries}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(entries)} cases")


if __name__ == "__main__":
    main()
