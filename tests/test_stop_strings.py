"""Stop strings on the host (valley_b200/stop_strings.py): the clean strings, the tables and ``match_rows`` reproduce
transformers' own StopStringCriteria, and the host loop's row handling reproduces HF generate(stop_strings=...)
(tests/golden/ref_stop_strings.pt, written by oracle/make_golden_stop_strings.py)."""
import os
import types

import pytest
import torch

from valley_b200 import stop_strings as ss
from valley_b200.model import ValleyLlamaForCausalLM, host_rows_step

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_stop_strings.pt")


@pytest.fixture(scope="module")
def gold():
    g = torch.load(GOLD)
    g["rows"] = list(torch.split(g["row_tokens"].long(), g["row_lens"].tolist()))
    return g


def test_clean_token_strings_match_hf(gold):
    pytest.importorskip("tokenizers")
    pytest.importorskip("transformers")
    from oracle import make_golden_stop_strings as G
    assert list(ss.clean_token_strings(G.toy_tokenizer())) == gold["clean"]


def test_golden_covers_the_cases(gold):
    clean = gold["clean"]
    for w in ("#", "##", "#a", " ###", "", "x###y"):
        assert w in clean
    assert len(gold["rows"]) == 2000 and max(len(r) for r in gold["rows"]) == 80
    assert any(len(s) == 64 for st in gold["sets"] for s in st) and any(len(st) == 9 for st in gold["sets"])
    for res in gold["results"]:
        assert 0 < int(res.sum()) < len(res)


@pytest.mark.parametrize("k", range(7))
def test_match_rows_reproduces_hf(gold, k):
    t = ss.stop_tables(gold["clean"], gold["sets"][k])
    assert t.on_device == (len(gold["sets"][k]) <= 8 and max(map(len, gold["sets"][k])) <= 64)
    got = torch.tensor([bool(ss.match_rows(r[None], t)[0]) for r in gold["rows"]])
    assert torch.equal(got, gold["results"][k])


def test_tables_are_cached_and_pad_to_the_model_vocabulary(gold):
    a = ss.stop_tables(gold["clean"], "###", 32008)
    assert ss.stop_tables(gold["clean"], ["###"], 32008) is a
    assert a.masks.shape == (1, 32008, 2) and int(a.masks[0, len(gold["clean"]):].max()) == 0
    assert int(a.token_lens[len(gold["clean"]):].max()) == 0


@pytest.mark.parametrize("run", [0, 1])
def test_host_loop_row_handling_reproduces_hf_generate(gold, run):
    g = gold["generate"]
    r = g["runs"][run]
    clean = [f" w{i}" for i in range(g["V"])]
    tables = ss.stop_tables(clean, g["stop_strings"])
    seq = g["prompt"].clone()
    B = seq.shape[0]
    finished = torch.zeros(B, dtype=torch.bool)
    for i in range(r["scores"].shape[1]):
        nxt = r["scores"][:, i].argmax(-1)
        seq, nxt, finished, stop = host_rows_step(seq, nxt, finished, r["eos"], g["pad"], tables)
        if stop:
            break
    assert torch.equal(seq, r["sequences"])


def test_stop_strings_without_tokenizer_raise():
    fake = types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=100))
    with pytest.raises(ValueError, match="tokenizer"):
        ValleyLlamaForCausalLM.generate(fake, input_ids=torch.zeros(1, 3, dtype=torch.int64), stop_strings="###")


def test_match_rows_walks_no_further_than_the_longest_string():
    # ["#", "", "", "", "##"]: the empty tokens fit anywhere, but HF looks back only 3 tokens for "###"
    clean = ["#", "", "##", "b"]
    t = ss.stop_tables(clean, "###")
    assert bool(ss.match_rows(torch.tensor([[0, 1, 2]]), t)[0])
    assert not bool(ss.match_rows(torch.tensor([[0, 1, 1, 2]]), t)[0])
    assert not bool(ss.match_rows(torch.tensor([[0, 3, 2]]), t)[0])
