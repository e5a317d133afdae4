"""generate()'s logits processors on the CPU: ``valley_b200.processors`` against transformers' own (tests/golden/
ref_logits_processors.pt, written by oracle/make_golden_logits_processors.py).  ``apply`` equals transformers' processors bit
for bit; ``from_kwargs`` adds what transformers adds and raises what it raises; the oracle model's greedy loop and beam search
with the processors reproduce transformers' generate."""
import os
import re

import pytest
import torch

import helpers as Hh
from oracle import make_golden_beam_search as GB
from oracle import make_golden_logits_processors as G
from valley_b200 import processors as P
from valley_b200 import synthetic as syn
from valley_b200.beam import output_fill_value

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_logits_processors.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _expected(z, idx, val):
    out = z.clone()
    out.view(-1)[idx] = val
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


def process_cases(gold):
    """(logits, ids, Processors, expected scores) of fixture (a)"""
    for e in gold["process"]:
        z = e["logits"]
        if z is None:
            z = G.wide_inputs()[0]
            assert float(z.double().sum()) == e["logits_sum"]
        for kw, idx, val in e["settings"]:
            p = P.Processors(penalty=kw.get("penalty", 1.0), ngram=kw.get("ngram", 0), min_length=kw.get("min_length", 0),
                             eos=kw["eos"])
            yield z, e["ids"], p, _expected(z, idx, val)


def test_fixture_covers_the_settings(gold):
    lengths = {e["ids"].shape[1] for e in gold["process"]}
    assert {1, 300} <= lengths and {e["V"] for e in gold["process"]} == {1032, 32008}
    n_inf = sum(int(torch.isinf(want).sum() - torch.isinf(z).sum()) for z, _, _, want in process_cases(gold))
    assert n_inf > 0                                        # the bans occur
    assert any(p.min_length > ids.shape[1] for _, ids, p, _ in process_cases(gold))


def test_apply_equals_transformers_bit_for_bit(gold):
    n = 0
    for z, ids, p, want in process_cases(gold):
        got = P.apply(z, ids, p)
        assert torch.equal(_bits(got), _bits(want)), (p, ids.shape)
        assert torch.equal(_bits(z), _bits(z.clone()))    # (the input is not modified)
        n += 1
    assert n == 8 * 11 + 1


def test_banned_ngrams_follow_hf_by_hand():
    ids = torch.tensor([[1, 2, 3, 1, 2, 4, 1, 2]])
    assert P.banned_ngram_tokens(ids, 3) == [[3, 4]]
    assert P.banned_ngram_tokens(ids, 1) == [[1, 2, 3, 1, 2, 4, 1, 2]]
    assert P.banned_ngram_tokens(ids[:, :2], 4) == [[]]            # cur_len + 1 < n: nothing
    assert P.banned_ngram_tokens(ids[:, :3], 4) == [[]]            # cur_len + 1 == n: no complete n-gram yet


def test_conditions_and_errors_match_transformers(gold):
    eos, S = 2, 12
    for c in gold["conditions"]:
        kw = dict(c["kwargs"])
        if "error" in c:
            with pytest.raises(ValueError, match=re.escape(c["error"])):
                P.from_kwargs(kw, S, eos if c["eos"] else None)
            continue
        spec = P.from_kwargs(kw, S, eos if c["eos"] else None)
        assert not set(kw) & set(P.KWARGS)                          # the arguments were consumed
        procs = dict(c["processors"])
        want_len = max((v for k, v in c["processors"] if k.startswith("MinLength") or k.startswith("MinNewTokens")), default=0)
        want = P.Processors(penalty=procs.get("RepetitionPenaltyLogitsProcessor", 1.0),
                            ngram=procs.get("NoRepeatNGramLogitsProcessor", 0),
                            min_length=want_len if want_len > S else 0, eos=eos if c["eos"] else -1)
        if want.penalty == 1.0 and want.ngram == 0 and want.min_length == 0:
            assert spec is None, c                                  # (a min length the prompt reaches bans nothing)
        else:
            assert spec == want, c


def test_hf_defaults_give_no_processors():
    for kw in (dict(), dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=None, min_length=0),
               dict(min_new_tokens=0), dict(repetition_penalty=None, no_repeat_ngram_size=None)):
        assert P.from_kwargs(dict(kw), 10, 2) is None and P.from_kwargs(dict(kw), 10, None) is None


@pytest.fixture(scope="module")
def model():
    spec = syn.SPECS[G.SPEC]
    return spec, GB.weights(spec), Hh.oracle_cfg(spec), GB.prompts(spec)


def _entries(gold, kind):
    return [i for i, e in enumerate(gold["generate"]) if e["case"]["kind"] == kind]


@pytest.mark.parametrize("i", range(9))
def test_oracle_greedy_with_processors_matches_transformers(gold, model, i):
    spec, w, cfg, prompts = model
    e = gold["generate"][_entries(gold, "greedy")[i]]
    c = e["case"]
    ids, mask, _ = prompts[c["prompt"]]
    procs = P.from_kwargs(dict(c["args"]), ids.shape[1], e["eos"])
    assert procs is not None
    seq, logits = G.greedy_generate(w, cfg, ids, mask, gold["n_new"], e["eos"], gold["pad"], procs)
    assert torch.equal(seq, e["sequences"]), (c, seq, e["sequences"])
    torch.testing.assert_close(logits, e["logits"], rtol=1e-4, atol=1e-4)


def test_the_processors_change_greedy(gold, model):
    """at least one processor run differs from the plain greedy continuation of its prompt"""
    spec, w, cfg, prompts = model
    differ = 0
    for i in _entries(gold, "greedy"):
        e = gold["generate"][i]
        ids, mask, _ = prompts[e["case"]["prompt"]]
        plain, _ = G.greedy_generate(w, cfg, ids, mask, gold["n_new"], None, gold["pad"], None)
        differ += not torch.equal(plain, e["sequences"][:, :plain.shape[1]]) or plain.shape != e["sequences"].shape
    assert differ >= 3


@pytest.mark.parametrize("i", range(2))
def test_oracle_beam_search_with_processors_matches_transformers(gold, model, i):
    spec, w, cfg, prompts = model
    e = gold["generate"][_entries(gold, "beam")[i]]
    c = e["case"]
    ids, _, _ = prompts[c["prompt"]]
    procs = P.from_kwargs(dict(c["args"]), ids.shape[1], e["eos"])
    bs = G.beam_generate(w, cfg, ids, gold["n_new"], c["num_beams"], e["eos"], output_fill_value(gold["pad"], e["eos"]), procs)
    seq, scores = bs.result(1)
    assert torch.equal(seq, e["sequences"])
    torch.testing.assert_close(scores, e["sequences_scores"], rtol=1e-5, atol=1e-5)
    n = e["scores"].shape[0]
    torch.testing.assert_close(torch.stack(bs.scores[:n]), e["scores"], rtol=1e-5, atol=1e-4)
