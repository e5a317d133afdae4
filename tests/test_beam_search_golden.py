"""The oracle's beam search (valley_b200/beam.py over the fp32 CPU model, oracle/beam_oracle.py) reproduces transformers' own
beam search (tests/golden/ref_beam_search.pt, written by oracle/make_golden_beam_search.py): ids exact, scores within fp32
rounding."""
import os

import pytest
import torch

import helpers as Hh
from oracle import beam_oracle as BO
from oracle import make_golden_beam_search as G
from valley_b200 import synthetic as syn
from valley_b200.beam import BeamSearch, output_fill_value

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_beam_search.pt")


@pytest.fixture(scope="module")
def setup():
    spec = syn.SPECS[G.SPEC]
    return spec, G.weights(spec), Hh.oracle_cfg(spec), Hh.oracle_tok(spec), G.prompts(spec), torch.load(GOLD)


def test_golden_covers_the_cases():
    gold = torch.load(GOLD)
    assert [e["case"] for e in gold["entries"]] == G.CASES
    assert any(int((e["sequences"] == e["eos"]).sum()) > 0 for e in gold["entries"])   # finished hypotheses occur


@pytest.mark.parametrize("i", range(len(G.CASES)))
def test_oracle_beam_search_matches_transformers(setup, i):
    spec, w, cfg, tok, prompts, gold = setup
    e = gold["entries"][i]
    c = e["case"]
    ids, mask, images = prompts[c["prompt"]]
    bs = BO.beam_generate(w, cfg, tok, ids, images, gold["n_new"], c["num_beams"], e["eos"], e["fill"], c["length_penalty"],
                          c["early_stopping"], attention_mask=mask)
    seq, scores = bs.result(c["num_return_sequences"])
    assert torch.equal(seq, e["sequences"])
    torch.testing.assert_close(scores, e["scores"], rtol=1e-5, atol=1e-5)


def test_output_fill_value_follows_hf():
    assert output_fill_value(None, None) == -1 and output_fill_value(5, None) == -1
    assert output_fill_value(5, 2) == 5 and output_fill_value(0, 2) == 2 and output_fill_value(None, 2) == 2


def test_restatement_rules_on_hand_made_logits():
    """eos on the best candidate finishes a hypothesis at once; early_stopping=True then ends the search when every slot
    of the item is finished; the cache parents and fed tokens follow the surviving candidates"""
    V, nb = 6, 2
    bs = BeamSearch(torch.zeros(nb, 3, dtype=torch.int64), nb, 5, eos_token_id=1, fill=9, early_stopping=True)
    lg = torch.full((nb, V), -10.0)
    lg[:, 1], lg[:, 2], lg[:, 3] = 3.0, 2.0, 1.0          # eos best, then 2, then 3
    parents, tokens = bs.step(lg)
    assert parents.tolist() == [0, 0] and tokens.tolist() == [2, 3]
    assert bool(bs.fin[0, 0]) and not bool(bs.fin[0, 1]) and not bs.done
    parents, tokens = bs.step(lg)
    assert bool(bs.fin.all()) and bs.done
    seq, scores = bs.result(2)
    assert seq.shape == (2, 3 + 2) and seq[0, 3].item() == 1 and seq[0, 4].item() == 9
