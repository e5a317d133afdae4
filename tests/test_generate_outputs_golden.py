"""generate(return_dict_in_generate=True)'s outputs against transformers' own (tests/golden/ref_generate_outputs.pt, written by
oracle/make_golden_generate_outputs.py), without a GPU: compute_transition_scores, the sampling scores' filter, the torch beam
restatement's recorded scores / logits / beam_indices, the output classes, and the ctypes layout of the recording fields."""
import functools
import os
import types

import pytest
import torch

import helpers as Hh
from oracle import beam_oracle as BO
from oracle import make_golden_beam_search as GB
from oracle import make_golden_generate_outputs as G
from valley_b200 import synthetic as syn
from valley_b200.beam import BeamSearch, output_fill_value
from valley_b200.model import (GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput, ValleyLlamaForCausalLM,
                               filter_scores, generation_output, sampling_filters)

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_generate_outputs.pt")
# fp32 CPU oracle vs transformers' fp32 CPU model on the same bf16-rounded weights: the logits agree exactly, the
# log-probabilities within an ulp (a float64 log-sum-exp against HF's fp32 log_softmax; measured 9.5e-7)
TOL = 1e-5


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _model_surface(spec):
    return types.SimpleNamespace(config=types.SimpleNamespace(vocab_size=spec.vocab_size))


def test_golden_covers_the_cases(gold):
    assert [e["case"] for e in gold["entries"]] == G.CASES
    beams = [e for e in gold["entries"] if e["case"]["kind"] == "beam"]
    assert any(bool((e["beam_indices"] < 0).any()) for e in beams)          # a hypothesis ended before the longest one
    assert any(len(G.scores(e)) < e["case"]["n_new"] for e in gold["entries"] if e["case"]["kind"] == "greedy")   # eos ended a run


@pytest.mark.parametrize("i", [i for i, c in enumerate(G.CASES) if c["kind"] != "sample"])
def test_compute_transition_scores_equals_transformers(gold, i):
    e = gold["entries"][i]
    spec = syn.SPECS[gold["spec"]]
    scores = tuple(G.scores(e))
    bi = e.get("beam_indices")
    for norm, key in ((False, "transition"), (True, "transition_normalized")):
        got = ValleyLlamaForCausalLM.compute_transition_scores(_model_surface(spec), e["sequences"], scores, bi, normalize_logits=norm)
        assert torch.equal(got, e[key]), (e["case"], norm)


@pytest.mark.parametrize("i", [i for i, c in enumerate(G.CASES) if c["kind"] == "sample"])
def test_sampling_scores_are_the_filtered_tempered_logits(gold, i):
    """HF's recorded scores == filter_scores(logits / T, k, p) on HF's recorded logits, bit for bit: the recorded -inf are the
    tokens the draw excludes"""
    e = gold["entries"][i]
    k, p = sampling_filters(e["case"]["top_k"], e["case"]["top_p"])
    for z, want in zip(e["logits"], e["scores"]):
        assert torch.equal(filter_scores(z / gold["temperature"], k, p), want), e["case"]
    if k or p < 1.0:
        assert bool(torch.isinf(e["scores"]).any())


@pytest.mark.parametrize("i", [i for i, c in enumerate(G.CASES) if c["kind"] == "beam"])
def test_beam_restatement_records_what_transformers_records(gold, i, monkeypatch):
    """the torch restatement (driven by the fp32 oracle, as tests/test_beam_search_golden.py drives it) records transformers'
    beam_indices and sequences exactly, and its log-probabilities (and, where the fixture keeps them, logits) per step within
    TOL"""
    e = gold["entries"][i]
    c = e["case"]
    spec = syn.SPECS[gold["spec"]]
    ids, mask, images = GB.prompts(spec)[c["prompt"]]
    monkeypatch.setattr(BO, "BeamSearch", functools.partial(BeamSearch, record_scores=True, record_logits=True))
    bs = BO.beam_generate(GB.weights(spec), Hh.oracle_cfg(spec), Hh.oracle_tok(spec), ids, images, c["n_new"],
                          c["num_beams"], e["eos"], output_fill_value(gold["pad"], e["eos"]), c["length_penalty"],
                          c["early_stopping"], attention_mask=mask)
    seq, seq_scores = bs.result(c["num_return_sequences"])
    assert torch.equal(seq, e["sequences"])
    assert torch.equal(bs.beam_indices(c["num_return_sequences"]), e["beam_indices"].long())
    assert bs.t == len(e["scores"]) == len(bs.scores) == len(bs.logits)
    err_s = float((torch.stack(bs.scores) - e["scores"]).abs().max())
    print(f"{c}: max |scores - HF| {err_s:.2e}")
    assert err_s <= TOL
    if "logits" in e:
        err_l = float((torch.stack(bs.logits) - e["logits"]).abs().max())
        print(f"  max |logits - HF| {err_l:.2e}")
        assert err_l <= TOL
    torch.testing.assert_close(seq_scores, e["sequences_scores"], rtol=1e-5, atol=1e-5)


def test_output_classes_follow_model_output():
    seq = torch.zeros(2, 5, dtype=torch.int64)
    buf = torch.randn(4, 2, 7)
    out = generation_output(seq, 3, buf, None)
    assert isinstance(out, GenerateDecoderOnlyOutput)
    assert out.sequences is seq and out["sequences"] is seq and out[0] is seq
    assert len(out.scores) == 3 and torch.equal(out.scores[2], buf[2]) and out[1] is out.scores
    assert out.logits is None and "logits" not in out and list(out.keys()) == ["sequences", "scores"]
    assert out.past_key_values is None and out.attentions is None and len(out.to_tuple()) == 2
    with pytest.raises(KeyError):
        out["logits"]
    b = generation_output(seq, 2, None, buf, sequences_scores=torch.zeros(2), beam_indices=torch.zeros(2, 2), beam=True)
    assert isinstance(b, GenerateBeamDecoderOnlyOutput)
    assert list(b.keys()) == ["sequences", "sequences_scores", "logits", "beam_indices"] and b.scores is None
    assert b[3] is b.beam_indices and len(b.logits) == 2
    sequences, = generation_output(seq, 0).to_tuple()
    assert sequences is seq


def test_beam_restatement_indices_on_hand_made_logits():
    """the finished hypothesis keeps the indices it had when it ended (-1 after), the running ones continue their parents'"""
    V, nb = 6, 2
    bs = BeamSearch(torch.zeros(nb, 3, dtype=torch.int64), nb, 5, eos_token_id=1, fill=9, early_stopping=True,
                    record_scores=True)
    lg = torch.full((nb, V), -10.0)
    lg[:, 1], lg[:, 2], lg[:, 3] = 3.0, 2.0, 1.0
    bs.step(lg)
    bs.step(lg)
    assert bs.done and bs.t == 2 and len(bs.scores) == 2 and bs.logits is None
    assert bs.beam_indices(2).tolist() == [[0, -1], [0, 0]]


def test_ctypes_structs_with_recording_match_the_c_header(tmp_path):
    """vly_beam (not covered by the older probe) and the extended vly_sampling have the layout gcc gives the header's structs"""
    import ctypes as C
    import shutil
    import subprocess
    from valley_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    structs = {"vly_sampling": _lib.VlySampling, "vly_beam": _lib.VlyBeam}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "valley_b200.h"', "int main(void) {"]
    for cname, ct in structs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi_probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi_probe"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {tuple(l.split()[:2]): int(l.split()[2]) for l in out if l}
    for cname, ct in structs.items():
        assert got[(cname, "size")] == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert got[(cname, fname)] == getattr(ct, fname).offset, (cname, fname)
    assert [f for f, _ in _lib.VlySampling._fields_][-2:] == ["scores_out", "logits_out"]
    assert [f for f, _ in _lib.VlyBeam._fields_][-4:] == ["scores_out", "logits_out", "beam_indices_out", "steps_out"]
