"""Writes tests/golden/ref_logits_processors.pt: transformers' own logits processors (``RepetitionPenaltyLogitsProcessor``,
``NoRepeatNGramLogitsProcessor``, ``MinLengthLogitsProcessor`` / ``MinNewTokensLengthLogitsProcessor``) and
``LlamaForCausalLM.generate`` with them (CPU, fp32), on the ``tiny`` synthetic weights with the prompts, eos choice and model
of oracle/make_golden_beam_search.py.

    python -m oracle.make_golden_logits_processors

(a) ``process``: recorded fp32 logits [R, V] (mixed signs, exact ties, +-0 and -inf) and id rows [R, L] (repeats, pads,
    lengths 1 ... 300) at V = 1032, and one small batch at V = 32008 (its logits regenerated from a seed: ``wide_inputs``).  Each
    entry keeps, per setting -- penalty {0.5, 1.2, 2.0}, n {1, 2, 3, 5} and min_length {L - 1, L, L + 1} alone, and the list
    ``_get_logits_processor`` builds from all three -- only the scores the processors changed (flat index, value).
(b) ``generate``: greedy on the text and padded prompts with each processor alone and all three together, with and without
    eos; one tempered top-k sampling run (scores only); 2- and 4-beam runs with penalty + n-gram.  Greedy keeps ``logits``
    (its scores are checked here to equal ``processors.apply`` of them, bit for bit), sampling keeps ``scores``, beams their
    ``sequences_scores`` and the scores of their first steps.
(c) ``conditions``: for a set of generate() arguments, the processors transformers adds (class name and parameters), or the
    ValueError it raises.

``greedy_generate`` / ``beam_generate`` run the same requests on the fp32 CPU oracle model (oracle/valley_oracle.py) with
``valley_b200.processors``; tests/test_logits_processors.py compares them with (b)."""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F

from oracle import make_golden_beam_search as GB

SPEC = GB.SPEC
PAD = GB.PAD
TEMPERATURE = 0.7
N_NEW = 5
BEAM_SCORE_STEPS = 2            # the beam runs keep the scores of their first steps
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_logits_processors.pt")

LENGTHS = (1, 2, 3, 4, 6, 12, 40, 300)
PENALTIES = (0.5, 1.2, 2.0)
NGRAMS = (1, 2, 3, 5)

# (b): generate() arguments; "eos" True takes the prompt's eos of make_golden_beam_search (a token greedy emits early)
GEN_CASES = [
    dict(kind="greedy", prompt=p, eos=e, args=a)
    for p in ("text", "padded")
    for e, a in ((False, dict(repetition_penalty=1.3)), (False, dict(no_repeat_ngram_size=2)),
                 (True, dict(min_new_tokens=5)), (True, dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=5)),
                 (False, dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=5)))
    if p == "text" or e or len(a) == 1
] + [
    dict(kind="sample", prompt="text", eos=True, args=dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3),
         top_k=20),
    dict(kind="beam", prompt="text", eos=True, args=dict(repetition_penalty=1.3, no_repeat_ngram_size=2), num_beams=2),
    dict(kind="beam", prompt="text", eos=True, args=dict(repetition_penalty=1.3, no_repeat_ngram_size=2), num_beams=4),
]

# (c): generate() arguments -> HF's processors or error (prompt of 12 ids; eos: whether an eos id is set)
COND_CASES = [
    (dict(), True), (dict(repetition_penalty=1.0), True), (dict(repetition_penalty=None), True),
    (dict(repetition_penalty=1.2), False), (dict(repetition_penalty=0.5), True), (dict(repetition_penalty=2), True),
    (dict(repetition_penalty=0.0), True), (dict(repetition_penalty=-1.5), True),
    (dict(no_repeat_ngram_size=0), True), (dict(no_repeat_ngram_size=None), True), (dict(no_repeat_ngram_size=3), False),
    (dict(no_repeat_ngram_size=-2), True), (dict(no_repeat_ngram_size=2.0), True),
    (dict(min_length=0), True), (dict(min_length=20), True), (dict(min_length=20), False), (dict(min_length=5), True),
    (dict(min_new_tokens=0), True), (dict(min_new_tokens=None), True), (dict(min_new_tokens=4), True),
    (dict(min_new_tokens=4), False), (dict(min_new_tokens=4, min_length=40), True), (dict(min_new_tokens=0, min_length=40), True),
    (dict(min_new_tokens=2.5), True),
    (dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=16), True),
]


def _logits(R, V, g):
    z = torch.randn(R, V, generator=g) * 3
    z[:, 5:9] = z[:, 4:5]                                      # exact ties
    z[:, 10], z[:, 11] = 0.0, -0.0
    z[:, 12:14] = -float("inf")
    z[0, 20:26] = z[0, 30]                                     # ties among the ids' scores
    return z


def _ids(R, L, V, g):
    ids = torch.randint(0, 40, (R, L), generator=g)           # a small alphabet: repeats and n-gram matches
    ids[0, :min(L, 3)] = PAD                                   # left padding
    if L > 4:
        ids[-1, -2] = V - 1
        ids[-1, -4:-2] = ids[-1, -2:]                          # the tail's 2-gram occurs earlier
    return ids


def _hf_settings(L):
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    out = [(dict(penalty=p), [RepetitionPenaltyLogitsProcessor(p)]) for p in PENALTIES]
    out += [(dict(ngram=n), [NoRepeatNGramLogitsProcessor(n)]) for n in NGRAMS]
    out += [(dict(min_length=ml), [MinLengthLogitsProcessor(ml, 7)]) for ml in (max(L - 1, 0), L, L + 1)]
    return out


def _processor_list(model, penalty, ngram, min_length, S, eos):
    """the list GenerationMixin._get_logits_processor builds for these arguments"""
    from transformers import GenerationConfig
    gc = GenerationConfig(repetition_penalty=penalty, no_repeat_ngram_size=ngram, min_length=min_length, eos_token_id=eos)
    model._prepare_special_tokens(gc, True, device="cpu")
    return model._get_logits_processor(generation_config=gc, input_ids_seq_length=S, encoder_input_ids=None,
                                       prefix_allowed_tokens_fn=None, logits_processor=None, device="cpu", model_kwargs={})


def _changed(before, after):
    diff = ~((before == after) | (torch.isnan(before) & torch.isnan(after)))
    diff |= torch.signbit(before) != torch.signbit(after)
    idx = diff.reshape(-1).nonzero()[:, 0]
    return idx, after.reshape(-1)[idx].clone()


def make_process(model):
    g = torch.Generator().manual_seed(20261018)
    entries = []
    for L in LENGTHS:
        V = 1032
        z, ids = _logits(3, V, g), _ids(3, L, V, g)
        e = dict(V=V, logits=z, ids=ids, settings=[])
        for kw, procs in _hf_settings(L):
            out = z.clone()
            for p in procs:
                out = p(ids, out)
            e["settings"].append((dict(kw, eos=7), *_changed(z, out)))
        lst = _processor_list(model, 1.2, 2, L + 1, L, 7)
        assert len(lst) == 3, lst
        out = lst(ids, z.clone())
        e["settings"].append((dict(penalty=1.2, ngram=2, min_length=L + 1, eos=7), *_changed(z, out)))
        entries.append(e)
    z, ids = wide_inputs()
    lst = _processor_list(model, 2.0, 3, ids.shape[1] + 1, ids.shape[1], 2)
    out = lst(ids, z.clone())
    entries.append(dict(V=z.shape[1], logits=None, logits_sum=float(z.double().sum()), ids=ids,
                        settings=[(dict(penalty=2.0, ngram=3, min_length=ids.shape[1] + 1, eos=2), *_changed(z, out))]))
    return entries


def wide_inputs():
    """the V = 32008 batch of (a): its logits are regenerated from the seed (the fixture keeps their sum to check them)"""
    g = torch.Generator().manual_seed(32008)
    V, L = 32008, 50
    z = _logits(2, V, g)
    ids = torch.randint(0, V, (2, L), generator=g)
    ids[:, 30:40] = ids[:, 10:20]
    ids[1, :5] = PAD
    return z, ids


def _describe(lst):
    out = []
    for p in lst:
        name = type(p).__name__
        if name == "RepetitionPenaltyLogitsProcessor":
            out.append((name, p.penalty))
        elif name == "NoRepeatNGramLogitsProcessor":
            out.append((name, p.ngram_size))
        elif name == "MinLengthLogitsProcessor":
            out.append((name, p.min_length))
        elif name == "MinNewTokensLengthLogitsProcessor":
            out.append((name, p.prompt_length_to_skip + p.min_new_tokens))
        else:
            out.append((name, None))
    return out


def make_conditions(model, eos_id):
    """what transformers' generate adds for COND_CASES on a 12-id prompt: the processors of its _get_logits_processor call"""
    ids = torch.randint(3, 1000, (1, 12), generator=torch.Generator().manual_seed(5))
    got = []
    orig = model._get_logits_processor

    def spy(*a, **k):
        lst = orig(*a, **k)
        got.append(lst)
        return lst

    model._get_logits_processor = spy
    out = []
    try:
        for kw, with_eos in COND_CASES:
            got.clear()
            try:
                with torch.no_grad():
                    model.generate(input_ids=ids, attention_mask=torch.ones_like(ids), max_new_tokens=2, do_sample=False,
                                   eos_token_id=eos_id if with_eos else None, pad_token_id=PAD, **kw)
                out.append(dict(kwargs=kw, eos=with_eos, processors=_describe(got[0])))
            except ValueError as err:
                out.append(dict(kwargs=kw, eos=with_eos, error=str(err)))
    finally:
        del model._get_logits_processor
    return out


def make_generate(model, spec):
    from valley_b200 import processors as P
    prompts = GB.prompts(spec)
    inputs = {}
    for name in ("text", "padded"):
        ids, mask, _ = prompts[name]
        B, S = ids.shape
        kw = dict(input_ids=ids, attention_mask=mask if mask is not None else torch.ones_like(ids),
                  position_ids=torch.arange(S)[None].expand(B, S).contiguous(), pad_token_id=PAD)
        with torch.no_grad():
            greedy = model.generate(**kw, max_new_tokens=4, do_sample=False, eos_token_id=None)
        inputs[name] = (kw, int(greedy[0, S + 3]))
    entries = []
    for i, case in enumerate(GEN_CASES):
        kw, eos_id = inputs[case["prompt"]]
        eos = eos_id if case["eos"] else None
        gen = dict(max_new_tokens=N_NEW, eos_token_id=eos, return_dict_in_generate=True, output_scores=True, output_logits=True,
                   **case["args"])
        if case["kind"] == "greedy":
            gen.update(do_sample=False)
        elif case["kind"] == "sample":
            torch.manual_seed(2000 + i)
            gen.update(do_sample=True, temperature=TEMPERATURE, top_k=case["top_k"])
        else:
            gen.update(do_sample=False, num_beams=case["num_beams"])
        with torch.no_grad():
            out = model.generate(**kw, **gen)
        sc, lg = torch.stack(out.scores).clone(), torch.stack(out.logits).clone()
        e = dict(case=case, eos=eos, sequences=out.sequences.clone())
        S = kw["input_ids"].shape[1]
        if case["kind"] == "greedy":
            spec_p = P.from_kwargs(dict(case["args"]), S, eos)
            for t in range(sc.shape[0]):          # HF's scores are processors.apply of its logits, bit for bit
                assert torch.equal(sc[t], P.apply(lg[t], out.sequences[:, :S + t], spec_p)), (case, t)
            e["logits"] = lg
        else:
            e["scores"] = sc[:BEAM_SCORE_STEPS].clone() if case["kind"] == "beam" else sc
        if case["kind"] == "beam":
            e["sequences_scores"] = out.sequences_scores.clone()
        print(case, "steps", sc.shape[0], "sequences", tuple(out.sequences.shape))
        entries.append(e)
    return entries


@torch.no_grad()
def greedy_generate(w, cfg, ids: torch.Tensor, mask: Optional[torch.Tensor], max_new_tokens: int, eos: Optional[int], pad: int,
                    procs):
    """HF greedy generate with ``procs`` on the fp32 CPU oracle model: (sequences, per-step raw logits [steps, B, V])"""
    from oracle import valley_oracle as O
    from valley_b200 import processors as P
    cache = O.KVCache(cfg.num_hidden_layers)

    def forward(x):
        h = O.llama_model(w, x, cache, n_layers=cfg.num_hidden_layers, heads=cfg.num_attention_heads, eps=cfg.rms_norm_eps,
                          theta=cfg.rope_theta, attention_mask=mask)
        return F.linear(h[:, -1], w["lm_head.weight"]).float()

    logits = forward(F.embedding(ids, w["model.embed_tokens.weight"]))
    seq, finished, out = ids, torch.zeros(ids.shape[0], dtype=torch.bool), []
    for i in range(max_new_tokens):
        out.append(logits)
        nxt = P.apply(logits, seq, procs).argmax(-1)
        if eos is not None:
            nxt = torch.where(finished, torch.full_like(nxt, pad), nxt)
            finished = finished | (nxt == eos)
        seq = torch.cat([seq, nxt[:, None]], 1)
        if (eos is not None and bool(finished.all())) or i + 1 == max_new_tokens:
            break
        if mask is not None:
            mask = torch.cat([mask, torch.ones_like(mask[:, :1])], dim=1)
        logits = forward(F.embedding(nxt[:, None], w["model.embed_tokens.weight"]))
    return seq, torch.stack(out)


@torch.no_grad()
def beam_generate(w, cfg, ids: torch.Tensor, max_new_tokens: int, num_beams: int, eos: Optional[int], fill: int, procs):
    """HF beam search with ``procs`` on the fp32 CPU oracle model (valley_b200.beam.BeamSearch): the finished search"""
    from oracle import valley_oracle as O
    from valley_b200.beam import BeamSearch
    nb = num_beams
    cache = O.KVCache(cfg.num_hidden_layers)

    def forward(x):
        h = O.llama_model(w, x, cache, n_layers=cfg.num_hidden_layers, heads=cfg.num_attention_heads, eps=cfg.rms_norm_eps,
                          theta=cfg.rope_theta)
        return F.linear(h[:, -1], w["lm_head.weight"]).float()

    logits = forward(F.embedding(ids, w["model.embed_tokens.weight"]).repeat_interleave(nb, 0))
    bs = BeamSearch(ids.repeat_interleave(nb, 0), nb, max_new_tokens, eos, fill, record_scores=True, processors=procs)
    while True:
        parents, tokens = bs.step(logits)
        if bs.done:
            return bs
        for layer in range(cfg.num_hidden_layers):
            cache.k[layer] = cache.k[layer].index_select(0, parents)
            cache.v[layer] = cache.v[layer].index_select(0, parents)
        logits = forward(F.embedding(tokens[:, None], w["model.embed_tokens.weight"]))


def main():
    import transformers
    from valley_b200 import synthetic as syn

    spec = syn.SPECS[SPEC]
    model = GB.hf_model(spec, GB.weights(spec))
    process = make_process(model)
    gen = make_generate(model, spec)
    eos_id = next(e["eos"] for e in gen if e["eos"] is not None)
    cond = make_conditions(model, eos_id)
    for c in cond:
        print(c)
    torch.save({"transformers": transformers.__version__, "spec": SPEC, "pad": PAD, "temperature": TEMPERATURE, "n_new": N_NEW,
                "process": process, "generate": gen, "conditions": cond}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
