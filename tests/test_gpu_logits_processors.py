"""GPU (-m gpu): generate(repetition_penalty=, no_repeat_ngram_size=, min_new_tokens=, min_length=).  The device routine
(vly_test_logits_process) equals transformers' processors (tests/golden/ref_logits_processors.pt) and processors.apply bit for
bit; the device route selects and records what the host-visible loop does, on the persistent (B <= 4) and per-op kernels; the
processors change what plain greedy emits on the tiny weights; logits follow transformers'; a processor request costs no host
decode, no extra device-to-host read, the launches of a recording request (B <= 4) or of a plain one (B > 4) and no allocation
after the first; beams with processors run the host beam loop and record the processed log-probabilities."""
import ctypes as C
import os

import pytest
import torch

import helpers as Hh
import test_gpu_generate_outputs as GO
from oracle import make_golden_beam_search as GB
from oracle import make_golden_logits_processors as G
from test_logits_processors import process_cases
from valley_b200 import _lib
from valley_b200 import beam as _beam
from valley_b200 import processors as P
from valley_b200.model import filter_scores, sampling_filters

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_logits_processors.pt")
N_NEW = 12
T = 0.7

SETTINGS = {
    "penalty": dict(repetition_penalty=1.3),
    "ngram": dict(no_repeat_ngram_size=2),
    "min_new": dict(min_new_tokens=6),
    "all": dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=6),
}


def _kw(m, ids, route, setting):
    kw = GO._kw(m, ids, route)
    kw.update(SETTINGS[setting])
    return kw


def _process(m, z, ids, p):
    out = torch.empty_like(z)
    _lib.check(m._lib.vly_test_logits_process(m._ctx, z.data_ptr(), z.shape[0], z.shape[1], ids.data_ptr(), ids.shape[1],
                                              p.penalty, p.ngram, p.min_length, p.eos, out.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- 1. the device routine ----
def test_kernel_equals_transformers_fixture():
    spec, m = GO.get()
    gold = torch.load(GOLD)
    n = 0
    for z, ids, p, want in process_cases(gold):
        got = _process(m, z.cuda().contiguous(), ids.cuda().contiguous(), p).cpu()
        assert torch.equal(_bits(got), _bits(want)), (p, ids.shape, z.shape)
        n += 1
    assert n == 8 * 11 + 1


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6])
def test_kernel_equals_apply_on_random_rows(n):
    """V = 32008, histories up to the cache capacity (2048), a small alphabet so that n-grams repeat"""
    spec, m = GO.get()
    g = torch.Generator().manual_seed(n)
    for L in (1, n - 1 if n > 1 else 2, 257, 2048):
        z = torch.randn(3, 32008, generator=g) * 4
        ids = torch.randint(0, 6, (3, L), generator=g)
        ids[1] = torch.randint(0, 32008, (L,), generator=g)
        for p in (P.Processors(1.2, n, L + 1, 3), P.Processors(0.5, n, 0, -1), P.Processors(1.0, n, L, 5)):
            got = _process(m, z.cuda(), ids.cuda(), p).cpu()
            assert torch.equal(_bits(got), _bits(P.apply(z, ids, p))), (L, p)


# ---- 2. device route == host loop ----
@pytest.mark.parametrize("B", [1, 3, 4, 6, 8])
@pytest.mark.parametrize("setting", list(SETTINGS))
@pytest.mark.parametrize("route", ["greedy", "greedy_eos"])
def test_device_equals_host_loop(B, setting, route):
    spec, m = GO.get()
    ids = GO._prompt(spec, B, 1000 + B)
    kw = _kw(m, ids, route, setting)
    dev = GO._no_host_decode(m, lambda: GO._record(m, **kw))
    host = GO._record(m, **kw, stopping_criteria=[GO.never])
    assert torch.equal(dev.sequences, host.sequences)
    assert torch.equal(GO._no_host_decode(m, lambda: GO._plain(m, **kw)), dev.sequences)     # recording changes nothing
    assert len(dev.scores) == len(host.scores) == len(dev.logits) == len(host.logits)
    assert torch.equal(torch.stack(dev.scores), torch.stack(host.scores))
    assert torch.equal(torch.stack(dev.logits), torch.stack(host.logits))


@pytest.mark.parametrize("B", [3, 6])
def test_device_equals_host_loop_with_stop_strings(B):
    spec, m = GO.get()
    ids = GO._prompt(spec, B, 1100 + B)
    free = m.generate(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=None)[:, ids.shape[1]:]
    kw = dict(input_ids=ids, max_new_tokens=N_NEW, eos_token_id=None, pad_token_id=0, stop_strings=["###", "a#"],
              tokenizer=GO._tokenizer(spec, ids, free), **SETTINGS["all"])
    dev = GO._no_host_decode(m, lambda: GO._record(m, **kw))
    host = GO._record(m, **kw, stopping_criteria=[GO.never])
    assert torch.equal(dev.sequences, host.sequences)
    assert torch.equal(torch.stack(dev.scores), torch.stack(host.scores))


@pytest.mark.parametrize("B", [3, 6])
@pytest.mark.parametrize("route", ["sample", "top_k", "top_p"])
def test_sampled_scores_are_the_processed_filtered_tempered_logits(B, route):
    spec, m = GO.get()
    ids = GO._prompt(spec, B, 1200 + B)
    kw = GO._kw(m, ids, route)
    kw.update(SETTINGS["all"], eos_token_id=GO._eos(m, ids))
    out = GO._no_host_decode(m, lambda: GO._record(m, **kw))
    S = ids.shape[1]
    procs = P.from_kwargs(dict(SETTINGS["all"]), S, kw["eos_token_id"])
    k, p = sampling_filters(kw.get("top_k"), kw.get("top_p"))
    seq = out.sequences.cpu()
    for i in range(len(out.scores)):
        want = filter_scores(P.apply(out.logits[i].cpu(), seq[:, :S + i], procs) / T, k, p)
        assert torch.equal(out.scores[i].cpu(), want), i
        chosen = want.gather(1, seq[:, S + i:S + i + 1])
        done = (seq[:, S:S + i] == kw["eos_token_id"]).any(1)
        assert bool(torch.isfinite(chosen[~done]).all()), i                 # (finished rows emit pad)


# ---- 3. the processors bite ----
def _ngrams(row, n):
    return [tuple(row[j:j + n]) for j in range(len(row) - n + 1)]


def test_processors_change_what_plain_greedy_emits():
    spec, m = GO.get()
    ids = GO._prompt(spec, 4, 1300, S=8)
    n_new = 48
    plain = m.generate(input_ids=ids, max_new_tokens=n_new, eos_token_id=None).tolist()
    rep = [r for r in range(4) if len(set(_ngrams(plain[r], 3))) < len(_ngrams(plain[r], 3))]
    assert rep, "precondition: plain greedy repeats a 3-gram on the tiny weights"
    out = m.generate(input_ids=ids, max_new_tokens=n_new, eos_token_id=None, no_repeat_ngram_size=3).tolist()
    for row in out:
        assert len(set(_ngrams(row, 3))) == len(_ngrams(row, 3))
    pen = m.generate(input_ids=ids, max_new_tokens=n_new, eos_token_id=None, repetition_penalty=1.5).tolist()
    assert all(pen[r] != plain[r] for r in rep)
    eos = plain[0][8 + 1]                                      # emitted by plain greedy as row 0's second new token
    k = 10
    first = m.generate(input_ids=ids, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=0, min_new_tokens=k)[:, 8:].tolist()
    assert first[0][1] != eos
    for row in first:
        assert eos not in row[:k]


# ---- 4. against transformers ----
def test_logits_follow_transformers():
    spec, m = GO.get()
    gold = torch.load(GOLD)
    report = []
    for e in gold["generate"]:
        c = e["case"]
        ids, mask, _ = GB.prompts(spec)[c["prompt"]]
        kw = dict(input_ids=ids.cuda(), attention_mask=None if mask is None else mask.cuda(), max_new_tokens=gold["n_new"],
                  eos_token_id=e["eos"], pad_token_id=gold["pad"], **c["args"])
        if c["kind"] == "sample":
            kw.update(do_sample=True, temperature=gold["temperature"], top_k=c["top_k"])
        elif c["kind"] == "beam":
            kw.update(num_beams=c["num_beams"])
        out = GO._record(m, **kw)
        S = ids.shape[1]
        same = torch.equal(out.sequences.cpu(), e["sequences"])
        if c["kind"] != "greedy":
            err = Hh.rel_fro(torch.nan_to_num(out.scores[0], neginf=0.0), torch.nan_to_num(e["scores"][0], neginf=0.0))
            assert err < 2e-2, (c, err)
            report.append((c["kind"], c.get("num_beams"), "first-step err %.1e" % err, "ids equal" if same else "ids differ"))
            continue
        compared = 0
        for i in range(min(len(out.logits), len(e["logits"]))):
            if not torch.equal(out.sequences[:, :S + i].cpu(), e["sequences"][:, :S + i]):
                break
            err = Hh.rel_fro(out.logits[i], e["logits"][i])
            assert err < 2e-2, (c, i, err)
            compared += 1
        assert compared >= 1
        report.append((c["prompt"], tuple(c["args"]), e["eos"] is not None, f"{compared} steps compared",
                       "ids equal" if same else "ids differ"))
    print(report)


# ---- 5. cost ----
@pytest.mark.parametrize("B", [1, 4, 6])
@pytest.mark.parametrize("route", ["greedy", "greedy_eos", "top_k"])
def test_no_extra_host_reads(B, route):
    """greedy with processors and no eos reads nothing back; otherwise as many reads as without processors"""
    spec, m = GO.get()
    ids = GO._prompt(spec, B, 1400 + B)
    kw = GO._kw(m, ids, route)
    procs = dict(kw, **SETTINGS["all"])
    GO._plain(m, **procs)
    plain, with_procs = GO._syncs(lambda: GO._plain(m, **kw)), GO._syncs(lambda: GO._plain(m, **procs))
    assert with_procs == (0 if route == "greedy" else plain), (plain, with_procs)


@pytest.mark.parametrize("B", [1, 4, 6])
def test_launches_per_step_and_no_allocation(B):
    """per step: a recording request's launches at B <= 4 (persistent kernel + sample_filter_kernel), a plain request's at
    B > 4; a second processor request leaves vly_held_bytes unchanged"""
    spec, m = GO.get()
    ids = GO._prompt(spec, B, 1500 + B)
    kw = dict(input_ids=ids, eos_token_id=None)
    per_step = lambda **k: (GO._launched(m, lambda: GO._plain(m, max_new_tokens=10, **kw, **k))
                            - GO._launched(m, lambda: GO._plain(m, max_new_tokens=6, **kw, **k)))
    # (each arm after a request of its own kind: the first plain request after another kind resets the selection state)
    GO._plain(m, max_new_tokens=4, **kw)
    plain = per_step()
    GO._plain(m, max_new_tokens=4, **kw, **SETTINGS["all"])
    held = GO._held()
    procs = per_step(**SETTINGS["all"])
    assert GO._held() == held
    rec = (GO._launched(m, lambda: GO._record(m, max_new_tokens=10, **kw))
           - GO._launched(m, lambda: GO._record(m, max_new_tokens=6, **kw)))
    assert procs == (rec if B <= 4 else plain)


def test_hf_defaults_change_nothing():
    spec, m = GO.get()
    defaults = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=None, min_length=0)
    for B in (3, 6):
        ids = GO._prompt(spec, B, 1600 + B)
        for route in ("greedy", "greedy_eos", "top_k"):
            kw = GO._kw(m, ids, route)
            want = GO._plain(m, **kw)
            assert torch.equal(GO._plain(m, **kw, **defaults), want)
            assert GO._launched(m, lambda: GO._plain(m, **kw, **defaults)) == GO._launched(m, lambda: GO._plain(m, **kw))
            assert GO._syncs(lambda: GO._plain(m, **kw, **defaults)) == GO._syncs(lambda: GO._plain(m, **kw))


def test_generate_must_continue_a_processor_request():
    spec, m = GO.get()
    ids = GO._prompt(spec, 2, 1700)
    cache = m.new_cache(2)
    try:
        embeds = m.prepare_inputs_labels_for_multimodal(ids, None, None, None, None)[3]
        _, nxt = m._prefill(cache, embeds, 0)
        sp = _lib.VlySampling(0.0, 0, -1, 0)
        sp.repetition_penalty, sp.prompt_ids_dev = 1.2, ids.data_ptr()
        out = torch.empty(2, 3, dtype=torch.int64, device="cuda")
        code = m._lib.vly_generate(m._ctx, cache._h, nxt.data_ptr(), 3, out.data_ptr(), C.byref(sp), None,
                                   torch.cuda.current_stream().cuda_stream)
        assert code == _lib.VLY_ERR_STATE
    finally:
        cache.release()


# ---- 6. beams ----
def test_beams_with_processors_run_the_host_loop_and_record_processed_log_probs():
    spec, m = GO.get()
    ids, _, _ = GB.prompts(spec)["text"]
    ids = ids.cuda()

    class NoDeviceBeam:
        def __init__(self, lib):
            self._lib = lib

        def __getattr__(self, name):
            assert name != "vly_beam_search"
            return getattr(self._lib, name)

    lib = m._lib
    m._lib = NoDeviceBeam(lib)
    try:
        out = GO._record(m, input_ids=ids, max_new_tokens=8, eos_token_id=None, num_beams=4, repetition_penalty=1.3,
                         no_repeat_ngram_size=2)
    finally:
        m._lib = lib
    procs = P.Processors(1.3, 2, 0, -1)
    first = P.apply(_beam.log_softmax(out.logits[0]), ids.repeat_interleave(4, 0), procs)
    assert torch.equal(out.scores[0], first)
    assert any(not torch.equal(out.scores[i], _beam.log_softmax(out.logits[i])) for i in range(len(out.scores)))
