"""GPU (-m gpu): generate(return_dict_in_generate=True, output_scores=True, output_logits=True).  Recording changes no token
on any route; the device routes record bit for bit what the host-visible loop records; sampled scores are the filtered
tempered logits the draw used; the logits follow transformers' (tests/golden/ref_generate_outputs.pt) within the bf16
tolerance of test_gpu_parity.py; a recording request costs no host round trip, no allocation by the library and, after the
persistent decode kernel, one kernel per step; and the output objects behave like transformers'."""
import ctypes as C
import os
import warnings

import pytest
import torch

import helpers as Hh
from oracle import make_golden_beam_search as GB
from oracle import make_golden_generate_outputs as G
from valley_b200 import _lib
from valley_b200 import synthetic as syn
from valley_b200.model import KeywordsStoppingCriteria, filter_scores, sampling_filters

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_generate_outputs.pt")
N_NEW = 12
T = 0.7
_m = {}


def get():
    if "m" not in _m:
        spec = syn.SPECS[G.SPEC]
        _m["m"] = (spec, Hh.build_model(spec, GB.weights(spec)))
    return _m["m"]


def never(ids, scores):
    return False


def _prompt(spec, B, seed, S=10):
    return torch.randint(3, spec.vocab_size - 8, (B, S), generator=torch.Generator().manual_seed(seed)).cuda()


def _eos(m, ids):
    """a token of the last row's greedy continuation: rows finish at different steps"""
    free = m.generate(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=None)[:, ids.shape[1]:]
    return int(free[-1, 5])


ROUTES = {
    "greedy": dict(),
    "greedy_eos": dict(eos="gen"),
    "sample": dict(do_sample=True, temperature=T),
    "top_k": dict(do_sample=True, temperature=T, top_k=20),
    "top_p": dict(do_sample=True, temperature=T, top_p=0.8),
}


def _kw(m, ids, route):
    kw = dict(ROUTES[route])
    eos = kw.pop("eos", None)
    # (no pad_token_id: pad falls back to eos, so no attention mask is inferred from the prompt -- a read-back of its own)
    return dict(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=_eos(m, ids) if eos else None, **kw)


def _record(m, seed=7, **kw):
    torch.manual_seed(seed)
    return m.generate(return_dict_in_generate=True, output_scores=True, output_logits=True, **kw)


def _plain(m, seed=7, **kw):
    torch.manual_seed(seed)
    return m.generate(**kw)


class _Count:
    """counts the host's decode calls (vly_llama_decode)"""
    def __init__(self, lib):
        self._lib, self.decodes = lib, 0

    def __getattr__(self, name):
        if name == "vly_llama_decode":
            self.decodes += 1
        return getattr(self._lib, name)


def _no_host_decode(m, fn):
    lib = m._lib
    m._lib = cnt = _Count(lib)
    try:
        out = fn()
    finally:
        m._lib = lib
    assert cnt.decodes == 0
    return out


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return len([c for c in caught if "called a synchronizing CUDA operation" in str(c.message)])


def _launched(m, fn):
    before = m.launches()
    fn()
    torch.cuda.synchronize()
    return m.launches() - before


def _held():
    d, p = C.c_int64(), C.c_int64()
    _lib.check(_lib.load().vly_held_bytes(C.byref(d), C.byref(p)))
    return d.value, p.value


def _tokenizer(spec, ids, free):
    from test_gpu_stop_strings import PieceTokenizer, _pieces
    return PieceTokenizer(spec.vocab_size, _pieces(ids, free))


# ---- 1. recording changes no token ----
@pytest.mark.parametrize("B", [1, 3, 4, 6, 8])
@pytest.mark.parametrize("route", list(ROUTES))
def test_recording_does_not_change_tokens(B, route):
    """same tokens with recording on and off (same torch seed), on the persistent kernel (B <= 4) and the per-op kernels;
    one recorded step per generated token, without a decode call from the host"""
    spec, m = get()
    ids = _prompt(spec, B, 100 + B)
    kw = _kw(m, ids, route)
    plain = _plain(m, **kw)
    out = _no_host_decode(m, lambda: _record(m, **kw))
    assert torch.equal(out.sequences, plain)
    steps = plain.shape[1] - ids.shape[1]
    assert len(out.scores) == len(out.logits) == steps and out.scores[0].shape == (B, spec.vocab_size)
    if route == "greedy_eos":
        assert steps <= N_NEW


@pytest.mark.parametrize("B", [3, 6])
def test_recording_with_stop_strings_does_not_change_tokens_and_equals_the_host_loop(B):
    spec, m = get()
    ids = _prompt(spec, B, B)
    free = m.generate(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=None)[:, ids.shape[1]:]
    kw = dict(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=None, pad_token_id=0, stop_strings=["###", "a#"],
              tokenizer=_tokenizer(spec, ids, free))
    plain = m.generate(**kw)
    dev = _no_host_decode(m, lambda: _record(m, **kw))
    host = _record(m, **kw, stopping_criteria=[never])
    assert torch.equal(dev.sequences, plain) and torch.equal(host.sequences, plain)
    assert len(dev.scores) == len(host.scores) == plain.shape[1] - ids.shape[1]
    assert torch.equal(torch.stack(dev.scores), torch.stack(host.scores))
    assert torch.equal(torch.stack(dev.logits), torch.stack(host.logits))


# ---- 2. device == host loop ----
@pytest.mark.parametrize("B", [1, 3, 6])
@pytest.mark.parametrize("route", ["greedy", "greedy_eos"])
def test_device_records_what_the_host_loop_records(B, route):
    spec, m = get()
    ids = _prompt(spec, B, 200 + B)
    kw = _kw(m, ids, route)
    dev = _record(m, **kw)
    host = _record(m, **kw, stopping_criteria=[never])
    assert torch.equal(dev.sequences, host.sequences)
    assert len(dev.scores) == len(host.scores) == len(dev.logits) == len(host.logits)
    assert torch.equal(torch.stack(dev.scores), torch.stack(host.scores))
    assert torch.equal(torch.stack(dev.logits), torch.stack(host.logits))
    assert torch.equal(torch.stack(dev.scores), torch.stack(dev.logits))          # greedy: the scores are the raw logits


def _beam_settings():
    return [dict(num_beams=4, num_return_sequences=2, length_penalty=lp, early_stopping=es)
            for lp in (1.0, 0.0, 2.0) for es in (False, True, "never")]


@pytest.mark.parametrize("prompt,rows", [("text", 4), ("padded", 8)])
@pytest.mark.parametrize("setting", range(9))
def test_beam_device_records_what_the_host_loop_records(prompt, rows, setting):
    spec, m = get()
    ids, mask, _ = GB.prompts(spec)[prompt]
    gold = torch.load(GOLD)
    eos = next(e["eos"] for e in gold["entries"] if e["case"]["prompt"] == prompt and e["eos"] is not None)
    c = _beam_settings()[setting]
    assert ids.shape[0] * c["num_beams"] == rows
    kw = dict(input_ids=ids.cuda(), attention_mask=None if mask is None else mask.cuda(), max_new_tokens=10,
              eos_token_id=eos, pad_token_id=0, **c)
    plain = m.generate(**kw)
    dev = _no_host_decode(m, lambda: _record(m, **kw))
    host = _record(m, **kw, stopping_criteria=[never])
    assert torch.equal(dev.sequences, plain) and torch.equal(host.sequences, plain)
    for k in ("sequences_scores", "beam_indices"):
        assert torch.equal(dev[k], host[k]), k
    assert dev.beam_indices.dtype == torch.int64 and dev.beam_indices.shape == (plain.shape[0], plain.shape[1] - ids.shape[1])
    assert len(dev.scores) == len(host.scores) == len(dev.logits)
    assert torch.equal(torch.stack(dev.scores), torch.stack(host.scores))
    assert torch.equal(torch.stack(dev.logits), torch.stack(host.logits))


# ---- 3. sampling ----
def _teacher_forced_logits(m, ids, gen, steps):
    """the logits of every step when the returned tokens are fed back through _decode (the same kernels)"""
    cache = m.new_cache(ids.shape[0])
    try:
        embeds = m.prepare_inputs_labels_for_multimodal(ids, None, None, None, None)[3]
        logits, _ = m._prefill(cache, embeds, 1)
        out = [logits[:, -1].clone()]
        for i in range(steps - 1):
            logits, _ = m._decode(cache, gen[:, i], True)
            out.append(logits[:, -1].clone())
        return torch.stack(out)
    finally:
        cache.release()


@pytest.mark.parametrize("B", [3, 6])
@pytest.mark.parametrize("route", ["sample", "top_k", "top_p"])
def test_sampled_scores_are_the_filtered_tempered_logits(B, route):
    spec, m = get()
    ids = _prompt(spec, B, 300 + B)
    kw = _kw(m, ids, route)
    out = _record(m, **kw)
    gen = out.sequences[:, ids.shape[1]:]
    scores, logits = torch.stack(out.scores).cpu(), torch.stack(out.logits).cpu()
    k, p = sampling_filters(kw.get("top_k"), kw.get("top_p"))
    for i in range(len(out.scores)):
        assert torch.equal(scores[i], filter_scores(logits[i] / T, k, p)), i      # (CPU: an IEEE division, as on the device)
    chosen = scores.gather(2, gen.cpu().T[:, :, None])
    assert bool(torch.isfinite(chosen).all())
    if route != "sample":
        assert bool(torch.isinf(scores).any())
    assert torch.equal(torch.stack(out.logits), _teacher_forced_logits(m, ids, gen, len(out.logits)))


# ---- 4. against transformers ----
def test_logits_follow_transformers():
    """per step, the logits within test_gpu_parity.py's bf16 tolerance (relative Frobenius error 2e-2) wherever the device's
    prefix equals transformers' (always at the prefill step); beam runs are reported with their token agreement, as
    test_gpu_beam_search.py reports them"""
    spec, m = get()
    gold = torch.load(GOLD)
    report = []
    for e in gold["entries"]:
        c = e["case"]
        ids, mask, _ = GB.prompts(spec)[c["prompt"]]
        kw = dict(input_ids=ids.cuda(), attention_mask=None if mask is None else mask.cuda(), max_new_tokens=c["n_new"],
                  eos_token_id=e["eos"], pad_token_id=gold["pad"])
        if c["kind"] == "sample":
            kw.update(do_sample=True, temperature=gold["temperature"], top_k=c["top_k"], top_p=c["top_p"])
        elif c["kind"] == "beam":
            kw.update(num_beams=c["num_beams"], num_return_sequences=c["num_return_sequences"],
                      length_penalty=c["length_penalty"], early_stopping=c["early_stopping"])
        out = _record(m, **kw)
        S = ids.shape[1]
        if c["kind"] == "beam":
            # (the fixture keeps every beam run's log-probabilities, and the logits of one)
            err = Hh.rel_fro(out.logits[0], e["logits"][0]) if "logits" in e else 0.0
            err = max(err, Hh.rel_fro(out.scores[0], e["scores"][0]))
            assert err < 2e-2, (c, err)
            same = torch.equal(out.sequences.cpu(), e["sequences"])
            report.append((c["num_beams"], c["prompt"], "prefill err %.1e" % err, "ids equal" if same else "ids differ"))
            continue
        compared = 0
        for i in range(min(len(out.logits), len(e["logits"]))):
            if not torch.equal(out.sequences[:, :S + i].cpu(), e["sequences"][:, :S + i]):
                break
            err = Hh.rel_fro(out.logits[i], e["logits"][i])
            assert err < 2e-2, (c, i, err)
            compared += 1
        assert compared >= 1
        report.append((c["kind"], c["prompt"], c.get("top_k"), c.get("top_p"), f"{compared} steps compared"))
    print(report)


# ---- 5. cost ----
@pytest.mark.parametrize("B", [1, 4, 6])
@pytest.mark.parametrize("route", ["greedy", "greedy_eos", "top_k"])
def test_recording_costs_no_extra_host_reads(B, route):
    """as many device-to-host reads as without recording: none for plain greedy, one with eos or sampling"""
    spec, m = get()
    ids = _prompt(spec, B, 400 + B)
    kw = _kw(m, ids, route)
    _record(m, **kw)
    plain, rec = _syncs(lambda: _plain(m, **kw)), _syncs(lambda: _record(m, **kw))
    assert rec == plain == (0 if route == "greedy" else 1), (plain, rec)


@pytest.mark.parametrize("prompt,nb", [("text", 4), ("padded", 4)])
def test_beam_recording_costs_one_read_and_the_same_kernels(prompt, nb):
    spec, m = get()
    ids, mask, _ = GB.prompts(spec)[prompt]
    kw = dict(input_ids=ids.cuda(), num_beams=nb, eos_token_id=None, attention_mask=None if mask is None else mask.cuda())
    m.generate(max_new_tokens=4, **kw)
    held = _held()
    _record(m, max_new_tokens=4, **kw)
    assert _held() == held                            # the beam-index rows came with the cache's other beam buffers
    plain = _launched(m, lambda: m.generate(max_new_tokens=10, **kw)) - _launched(m, lambda: m.generate(max_new_tokens=6, **kw))
    rec = _launched(m, lambda: _record(m, max_new_tokens=10, **kw)) - _launched(m, lambda: _record(m, max_new_tokens=6, **kw))
    assert rec == plain
    assert _syncs(lambda: _record(m, max_new_tokens=10, **kw)) == 1


@pytest.mark.parametrize("B", [1, 4, 6])
def test_recording_greedy_kernels_per_step_and_no_library_allocation(B):
    """a recording greedy step at B <= 4 is the persistent kernel (writing logits) + sample_filter_kernel; at B > 4 the per-op
    step launches what it launches without recording (its selection kernel already runs every step).  vly_held_bytes does
    not move."""
    spec, m = get()
    ids = _prompt(spec, B, 500 + B)
    kw = dict(input_ids=ids, eos_token_id=None)
    _record(m, max_new_tokens=4, **kw)
    held = _held()
    rec = _launched(m, lambda: _record(m, max_new_tokens=10, **kw)) - _launched(m, lambda: _record(m, max_new_tokens=6, **kw))
    assert _held() == held
    per_op = ((B + 3) // 4) * (1 + 5 * spec.num_hidden_layers + 1)
    assert rec == 4 * ((1 + 1) if B <= 4 else per_op + 1)


def test_recording_leaves_the_next_plain_request_as_it_was():
    """the graphs a recording request ran keep no recording pointer: the next plain request's tokens and launches are unchanged"""
    spec, m = get()
    for B in (3, 6):
        ids = _prompt(spec, B, 600 + B)
        for route in ("greedy", "greedy_eos", "top_k"):
            kw = _kw(m, ids, route)
            _plain(m, **kw)
            n0 = _launched(m, lambda: _plain(m, **kw))
            want = _plain(m, **kw)
            _record(m, **kw)
            assert torch.equal(_plain(m, **kw), want), (B, route)
            assert _launched(m, lambda: _plain(m, **kw)) == n0, (B, route)


# ---- 6. interface ----
def test_output_objects_and_flags():
    spec, m = get()
    ids = _prompt(spec, 2, 700)
    out = m.generate(input_ids=ids, max_new_tokens=5, eos_token_id=None, return_dict_in_generate=True)
    assert type(out).__name__ == "GenerateDecoderOnlyOutput"
    assert out.scores is None and out.logits is None and out.past_key_values is None and list(out.keys()) == ["sequences"]
    assert out["sequences"] is out.sequences and out[0] is out.sequences and out.to_tuple() == (out.sequences,)
    only = m.generate(input_ids=ids, max_new_tokens=5, eos_token_id=None, return_dict_in_generate=True, output_scores=True)
    assert len(only.scores) == 5 and only.logits is None
    assert torch.equal(m.generate(input_ids=ids, max_new_tokens=5, eos_token_id=None, output_scores=True), out.sequences)
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=ids, max_new_tokens=5, return_dict_in_generate=True, output_attentions=True)
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=ids, max_new_tokens=5, return_dict_in_generate=True, output_hidden_states=True)
    b = m.generate(input_ids=ids, max_new_tokens=5, eos_token_id=None, num_beams=2, return_dict_in_generate=True)
    assert type(b).__name__ == "GenerateBeamDecoderOnlyOutput"
    assert b.sequences_scores is None and b.scores is None and list(b.keys()) == ["sequences", "beam_indices"]


def test_transition_scores():
    """greedy: normalize_logits=True gives the log-softmax at the chosen tokens; beams: summed transition scores over
    length ** length_penalty give sequences_scores (transformers' documented identity)"""
    spec, m = get()
    ids = _prompt(spec, 3, 800)
    out = _record(m, input_ids=ids, max_new_tokens=8, eos_token_id=None)
    got = m.compute_transition_scores(out.sequences, out.scores, normalize_logits=True)
    lp = torch.log_softmax(torch.stack(out.logits), -1)
    want = lp.gather(2, out.sequences[:, ids.shape[1]:].T[:, :, None])[:, :, 0].T
    torch.testing.assert_close(got, want)
    gold = torch.load(GOLD)
    eos = next(e["eos"] for e in gold["entries"] if e["case"]["prompt"] == "text" and e["eos"] is not None)
    for lpen in (1.0, 2.0):
        b = _record(m, input_ids=ids[:1], max_new_tokens=10, eos_token_id=eos, num_beams=4, num_return_sequences=4,
                    length_penalty=lpen)
        ts = m.compute_transition_scores(b.sequences, b.scores, b.beam_indices)
        length = (b.beam_indices >= 0).sum(1)
        torch.testing.assert_close(ts.sum(1) / length.float() ** lpen, b.sequences_scores, rtol=1e-5, atol=1e-5)


def test_trainer_call_shape():
    """the reference trainer's call: a keyword stopping criterion, num_beams=1, return_dict_in_generate=True, .sequences"""
    spec, m = get()
    ids = _prompt(spec, 1, 900)

    class Tok:
        def batch_decode(self, rows, skip_special_tokens=True):
            return [" ".join(f"w{int(t)}" for t in r) for r in rows]

    free = m.generate(input_ids=ids, max_new_tokens=8, eos_token_id=None)
    kw = dict(input_ids=ids, max_new_tokens=8, eos_token_id=None, num_beams=1)
    crit = KeywordsStoppingCriteria([f"w{int(free[0, -4])}"], Tok(), ids)
    out = m.generate(**kw, stopping_criteria=[crit], return_dict_in_generate=True)
    crit2 = KeywordsStoppingCriteria([f"w{int(free[0, -4])}"], Tok(), ids)
    assert torch.equal(out.sequences, m.generate(**kw, stopping_criteria=[crit2]))
    assert out.sequences.shape[1] < free.shape[1]
