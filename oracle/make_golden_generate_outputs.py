"""Writes tests/golden/ref_generate_outputs.pt: transformers' own ``LlamaForCausalLM.generate(return_dict_in_generate=True,
output_scores=True, output_logits=True)`` (CPU, fp32) on the ``tiny`` synthetic weights, with the prompts, eos choice and
model of oracle/make_golden_beam_search.py.

    python -m oracle.make_golden_generate_outputs

Runs (``CASES``, each with its own ``max_new_tokens``):
  * greedy on the text prompt and on the left-padded batch, with and without eos;
  * sampling at temperature 0.7 with top_k = 0, top_k = 20 and top_p = 0.8 (top_k = 0 there, so that HF's implied top_k = 50
    is off): the draws cannot be compared across samplers, so only ``scores`` and ``logits`` are of use;
  * beam search: 2 beams; 4 beams returning 2 with eos ending hypotheses early; the padded batch with 2 beams returning 2.
Each entry keeps ``sequences`` and, stacked [steps, rows, V] fp32, what the tests need of ``scores`` / ``logits``: greedy keeps
``logits`` only (its scores are the same tensors, checked here), sampling keeps both, beams keep ``scores`` (and ``logits`` for
the 2-beam run).  Beams add ``sequences_scores`` and ``beam_indices``; greedy and beams add HF's ``compute_transition_scores``
with normalize_logits False and True.  (V = 1032: every stored step-row costs 4 KB, so the runs are short.)"""
from __future__ import annotations

import os

import torch

from oracle import make_golden_beam_search as GB

SPEC = GB.SPEC
PAD = GB.PAD
TEMPERATURE = 0.7
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_generate_outputs.pt")

CASES = [
    dict(kind="greedy", prompt="text", eos=False, n_new=5),
    dict(kind="greedy", prompt="text", eos=True, n_new=5),
    dict(kind="greedy", prompt="padded", eos=False, n_new=5),
    dict(kind="greedy", prompt="padded", eos=True, n_new=5),
    dict(kind="sample", prompt="text", eos=False, n_new=2, top_k=0, top_p=1.0),
    dict(kind="sample", prompt="text", eos=False, n_new=2, top_k=20, top_p=1.0),
    dict(kind="sample", prompt="text", eos=False, n_new=2, top_k=0, top_p=0.8),
    dict(kind="beam", prompt="text", eos=False, n_new=5, num_beams=2, num_return_sequences=1, length_penalty=1.0,
         early_stopping=False, keep_logits=True),
    dict(kind="beam", prompt="text", eos=True, n_new=5, num_beams=4, num_return_sequences=2, length_penalty=2.0,
         early_stopping=True),
    dict(kind="beam", prompt="padded", eos=True, n_new=5, num_beams=2, num_return_sequences=2, length_penalty=1.0,
         early_stopping=False),
]


def scores(e):
    """an entry's per-step scores [steps, rows, V]: greedy records its logits as its scores"""
    return e["scores"] if "scores" in e else e["logits"]


def main():
    import transformers
    from valley_b200 import synthetic as syn

    spec = syn.SPECS[SPEC]
    w = GB.weights(spec)
    m = GB.hf_model(spec, w)
    prompts = GB.prompts(spec)
    inputs = {}
    for name in ("text", "padded"):
        ids, mask, _ = prompts[name]
        B, S = ids.shape
        kw = dict(input_ids=ids, attention_mask=mask if mask is not None else torch.ones_like(ids),
                  position_ids=torch.arange(S)[None].expand(B, S).contiguous(), pad_token_id=PAD)
        with torch.no_grad():
            greedy = m.generate(**kw, max_new_tokens=4, do_sample=False, eos_token_id=None)
        inputs[name] = (kw, int(greedy[0, S + 3]))       # eos: a token of row 0's greedy continuation (make_golden_beam_search)
    entries = []
    for i, case in enumerate(CASES):
        kw, eos_id = inputs[case["prompt"]]
        eos = eos_id if case["eos"] else None
        gen = dict(max_new_tokens=case["n_new"], eos_token_id=eos, return_dict_in_generate=True, output_scores=True, output_logits=True)
        if case["kind"] == "greedy":
            gen.update(do_sample=False)
        elif case["kind"] == "sample":
            torch.manual_seed(1000 + i)
            gen.update(do_sample=True, temperature=TEMPERATURE, top_k=case["top_k"], top_p=case["top_p"])
        else:
            gen.update(do_sample=False, num_beams=case["num_beams"], num_return_sequences=case["num_return_sequences"],
                       length_penalty=case["length_penalty"], early_stopping=case["early_stopping"])
        with torch.no_grad():
            out = m.generate(**kw, **gen)
        sc, lg = torch.stack(out.scores).clone(), torch.stack(out.logits).clone()
        e = dict(case=case, eos=eos, sequences=out.sequences.clone())
        if case["kind"] == "greedy":
            assert torch.equal(sc, lg)
            e["logits"] = lg
        else:
            e["scores"] = sc
            if case["kind"] == "sample" or case.get("keep_logits"):
                e["logits"] = lg
        if case["kind"] != "sample":
            bi = out.beam_indices if case["kind"] == "beam" else None
            e["transition"] = m.compute_transition_scores(out.sequences, out.scores, bi, normalize_logits=False).clone()
            e["transition_normalized"] = m.compute_transition_scores(out.sequences, out.scores, bi, normalize_logits=True).clone()
        if case["kind"] == "beam":
            e["sequences_scores"] = out.sequences_scores.clone()
            e["beam_indices"] = out.beam_indices.clone()
        print(case, "steps", len(out.scores), "sequences", tuple(out.sequences.shape))
        entries.append(e)
    torch.save({"transformers": transformers.__version__, "spec": SPEC, "pad": PAD, "temperature": TEMPERATURE,
                "entries": entries}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(entries)} runs")


if __name__ == "__main__":
    main()
