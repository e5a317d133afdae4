"""Beam search in generate (num_beams > 1): the KV-cache reorder against HF's index_select, the device path
(beam_step_kernel + kv_beam_reorder_kernel in the decode step's graph) against the host-visible torch loop on the same logits,
both against transformers' own beam search (tests/golden/ref_beam_search.pt), completion() with a beam request, and the
cost of a request (one device-to-host read, a fixed number of kernels per step)."""
import hashlib
import os
import re
import types
import warnings

import pytest
import torch

import helpers as Hh
from oracle import make_golden_beam_search as G
from oracle import valley_oracle as O
from valley_b200 import synthetic as syn
from valley_b200.model import KeywordsStoppingCriteria

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_beam_search.pt")
_models = {}


def get():
    if "m" not in _models:
        spec = syn.SPECS[G.SPEC]
        w = G.weights(spec)
        _models["m"] = (spec, w, Hh.build_model(spec, w))
    return _models["m"]


def launched(m, fn):
    before = m.launches()
    out = fn()
    torch.cuda.synchronize()
    return m.launches() - before, out


def never(ids, scores):
    return False


def _run(m, prompt, case, eos, host, n_new=None):
    ids, mask, images = prompt
    kw = dict(input_ids=ids.cuda(), images=None if images is None else images.cuda(), max_new_tokens=n_new or G.N_NEW,
              num_beams=case["num_beams"], num_return_sequences=case["num_return_sequences"],
              length_penalty=case["length_penalty"], early_stopping=case["early_stopping"], eos_token_id=eos, pad_token_id=G.PAD,
              stopping_criteria=[never] if host else None)
    if mask is not None:
        kw["attention_mask"] = mask.cuda()
    out = m.generate(**kw)
    return out, m.last_beam_scores.clone()


# ---- 1. the reorder ----
@pytest.mark.gpu
@pytest.mark.parametrize("B,perm", [(4, [0, 1, 2, 3]), (4, [2, 2, 2, 2]), (4, [1, 2, 3, 0]), (4, [0, 0, 3, 3]),
                                    (8, [3, 3, 0, 7, 1, 1, 6, 2]), (8, [1, 2, 3, 0, 5, 6, 7, 4])])
@pytest.mark.parametrize("S,from_pos", [(77, 0), (77, 30), (40, 39)])
def test_reorder_cache_matches_index_select(B, perm, S, from_pos):
    """bit-exact against to_hf() + index_select over positions [from_pos, S) (77 and 47 positions are not whole blocks of the
    kernel: 32 positions at 4 rows, 16 at 8); positions before from_pos keep their rows"""
    spec, w, m = get()
    cache = m.new_cache(B, 128)
    try:
        g = torch.Generator().manual_seed(B * 1000 + S)
        ids = torch.randint(3, spec.vocab_size - 8, (B, S), generator=g)
        m._prefill(cache, m.prepare_inputs_labels_for_multimodal(ids)[3], 0)
        before = [cache.to_hf(layer) for layer in range(spec.num_hidden_layers)]
        idx = torch.tensor(perm)
        cache.reorder_cache(idx, from_pos)
        for layer in range(spec.num_hidden_layers):
            after = cache.to_hf(layer)
            for b, a in zip(before[layer], after):
                want = b.clone()
                want[:, :, from_pos:] = b.index_select(0, idx.cuda())[:, :, from_pos:]
                assert torch.equal(a, want), (layer, perm)
    finally:
        cache.release()


# ---- 2. device path == host loop ----
def _settings():
    out = []
    for lp in (1.0, 0.0, 2.0):
        for es in (False, True, "never"):
            out.append(dict(num_beams=4, num_return_sequences=2, length_penalty=lp, early_stopping=es))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("prompt,nb_rows", [("text", 4), ("multimodal", 4), ("padded", 8)])
@pytest.mark.parametrize("setting", range(9))
def test_device_path_equals_host_loop(prompt, nb_rows, setting):
    """token for token and bit for bit: both select over the library's logits with the same arithmetic"""
    spec, w, m = get()
    gold = torch.load(GOLD)
    eos = next(e["eos"] for e in gold["entries"] if e["case"]["prompt"] == prompt)
    case = _settings()[setting]
    p = G.prompts(spec)[prompt]
    assert p[0].shape[0] * case["num_beams"] == nb_rows
    dev, dev_s = _run(m, p, case, eos, host=False)
    host, host_s = _run(m, p, case, eos, host=True)
    assert torch.equal(dev, host), (dev, host)
    assert torch.equal(dev_s, host_s), (dev_s, host_s)


@pytest.mark.gpu
def test_default_settings_and_early_end():
    """generate(num_beams=2) with HF's defaults; a request that ends before max_new_tokens (eos everywhere) leaves the cache
    usable for the next request"""
    spec, w, m = get()
    ids = G.prompts(spec)["text"][0].cuda()
    a = m.generate(input_ids=ids, max_new_tokens=8, num_beams=2, eos_token_id=None)
    b = m.generate(input_ids=ids, max_new_tokens=8, num_beams=2, eos_token_id=None, stopping_criteria=[never])
    assert torch.equal(a, b) and a.shape == (1, ids.shape[1] + 8)
    g1 = m.generate(input_ids=ids, max_new_tokens=6, eos_token_id=None)
    c = m.generate(input_ids=ids, max_new_tokens=8, num_beams=2, eos_token_id=int(g1[0, -6]))
    assert c.shape[1] <= ids.shape[1] + 8
    g2 = m.generate(input_ids=ids, max_new_tokens=6, eos_token_id=None)       # the selection state was reset
    assert torch.equal(g1, g2)


# ---- 3. against transformers ----
@pytest.mark.gpu
def test_device_path_matches_transformers():
    """ids exact and scores close wherever every recorded decision margin exceeds twice the device's max logit error
    (measured on the prefill against the fp32 oracle), the policy DESIGN section 2 sets for greedy.  A case with a lower margin
    is reported with the step of its first low-margin decision and not compared: which of two candidates that close wins is
    not fixed by bf16 arithmetic.  (The device path is pinned bit for bit to the host loop above, and the host loop's
    restatement to transformers on CPU by tests/test_beam_search_golden.py.)"""
    spec, w, m = get()
    gold = torch.load(GOLD)
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    err = {}
    for name, (ids, mask, images) in G.prompts(spec).items():
        ref = O.causal_lm_forward(w, cfg, tok, ids, images, attention_mask=mask)[:, -1].float()
        m.logits_all_positions = False
        got = m(input_ids=ids.cuda(), images=None if images is None else images.cuda(),
                attention_mask=None if mask is None else mask.cuda()).logits[:, -1].float().cpu()
        m.logits_all_positions = True
        err[name] = float((got - ref).abs().max())
    compared, skipped = 0, []
    for e in gold["entries"]:
        c = e["case"]
        margins = e["margins"]
        low = margins <= 2 * err[c["prompt"]]
        if bool(low.any()):
            skipped.append((c, int(low.nonzero()[0])))
            continue
        out, scores = _run(m, G.prompts(spec)[c["prompt"]], c, e["eos"], host=False)
        assert torch.equal(out.cpu(), e["sequences"]), c
        torch.testing.assert_close(scores.cpu(), e["scores"], rtol=0, atol=4 * err[c["prompt"]] * G.N_NEW)
        compared += 1
    print(f"max logit error {err}; compared {compared} cases exactly; {len(skipped)} cases have a low-margin decision "
          f"(case, first such step): {skipped}")


# ---- 4. completion() ----
class WordTokenizer:
    """word-level tokenizer over the model's id space with the HF surface completion() uses; sentinel strings map to the six
    highest ids, ``stop_id`` decodes to '###'"""
    eos_token_id = 2
    pad_token_id = 0
    padding_side = "right"

    def __init__(self, spec, stop_id=None):
        t = syn.sentinel_ids(spec)
        self.V = spec.vocab_size
        self.special = {"<im_patch>": t["im_patch_token"], "<im_start>": t["im_start_token"], "<im_end>": t["im_end_token"],
                        "<vi_frame>": t["vi_frame_token"], "<vi_start>": t["vi_start_token"], "<vi_end>": t["vi_end_token"]}
        self.stop_id = stop_id
        self.rx = re.compile(r"<[a-z_]+>|###|w\d+|[A-Za-z']+|[^\sA-Za-z]")

    def _word(self, w):
        if w in self.special:
            return self.special[w]
        if re.fullmatch(r"w\d+", w):
            return int(w[1:])
        return 3 + int(hashlib.md5(w.encode()).hexdigest(), 16) % (self.V - 12)

    def __call__(self, text, padding=False):
        rows = [[1] + [self._word(w) for w in self.rx.findall(t)] for t in ([text] if isinstance(text, str) else text)]
        return types.SimpleNamespace(input_ids=rows, attention_mask=[[1] * len(r) for r in rows])

    def decode(self, ids, skip_special_tokens=True):
        return "".join(" ###" if int(i) == self.stop_id else f" w{int(i)}" for i in ids if int(i) not in (0, 1, 2))

    def batch_decode(self, rows, skip_special_tokens=True):
        return [self.decode(r.tolist() if torch.is_tensor(r) else r, skip_special_tokens) for r in rows]


class _NoDevicePath:
    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name == "vly_beam_search":
            raise AssertionError("completion() must take the host loop: it passes a stopping criterion")
        return getattr(self._lib, name)


@pytest.mark.gpu
def test_completion_with_beams_runs_the_host_loop():
    spec, w, m = get()
    clip = torch.randn(3, 8, 224, 224, generator=torch.Generator().manual_seed(1))
    message = [{"role": "system", "content": "You are a helpful assistant."},
               {"role": "user", "content": "<video> What happens in the video?"}]
    ids = m.build_inputs(WordTokenizer(spec), message).input_ids
    # the stop id: a token of the beam search's own output, so that '###' ends the reply early
    plain = m.generate(input_ids=torch.as_tensor(ids).cuda(), images=clip.permute(1, 0, 2, 3)[None].half().cuda(),
                       max_new_tokens=8, num_beams=2, eos_token_id=None)
    stop_id = int(plain[0, len(ids[0]) + 4])
    tk = WordTokenizer(spec, stop_id=stop_id)
    lib = m._lib
    m._lib = _NoDevicePath(lib)
    try:
        reply = m.completion(tk, clip, message, {"num_beams": 2, "max_new_tokens": 8}, "cuda")
    finally:
        m._lib = lib
    crit = KeywordsStoppingCriteria(["###"], tk, torch.as_tensor(ids).cuda())
    want = m.generate(input_ids=torch.as_tensor(ids).cuda(), images=clip.permute(1, 0, 2, 3)[None].half().cuda(),
                      max_new_tokens=8, num_beams=2, eos_token_id=2, stopping_criteria=[crit])
    assert reply == m.process_response(tk.batch_decode(want[:, len(ids[0]):]))
    assert isinstance(reply, list) and len(reply) == 1


# ---- 5. num_beams = 1 and beam sampling ----
@pytest.mark.gpu
def test_one_beam_is_todays_generate_and_beam_sampling_is_refused():
    spec, w, m = get()
    ids = G.prompts(spec)["text"][0].cuda()
    assert torch.equal(m.generate(input_ids=ids, max_new_tokens=6, num_beams=1), m.generate(input_ids=ids, max_new_tokens=6))
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=ids, max_new_tokens=6, num_beams=2, do_sample=True)
    with pytest.raises(ValueError):
        m.generate(input_ids=ids, max_new_tokens=6, num_beams=2, num_return_sequences=3)


# ---- 6. cost of a request ----
@pytest.mark.gpu
@pytest.mark.parametrize("prompt,nb", [("text", 4), ("padded", 4)])
def test_one_host_read_and_fixed_kernels_per_step(prompt, nb):
    """the device path synchronises with the host once per request; every step after the first replays the same kernels:
    the persistent decode kernel + beam_step_kernel + kv_beam_reorder_kernel at <= 4 rows, the per-op step + the same two
    above"""
    spec, w, m = get()
    ids, mask, _ = G.prompts(spec)[prompt]
    kw = dict(input_ids=ids.cuda(), num_beams=nb, eos_token_id=None, attention_mask=None if mask is None else mask.cuda())
    m.generate(max_new_tokens=4, **kw)                         # captures the graphs
    n6, _ = launched(m, lambda: m.generate(max_new_tokens=6, **kw))
    n10, _ = launched(m, lambda: m.generate(max_new_tokens=10, **kw))
    rows = ids.shape[0] * nb
    per_op = ((rows + 3) // 4) * (1 + 5 * spec.num_hidden_layers + 1)
    assert n10 - n6 == 4 * ((1 if rows <= 4 else per_op) + 2)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            m.generate(max_new_tokens=10, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [c for c in caught if "called a synchronizing CUDA operation" in str(c.message)]
    assert len(syncs) == 1, [str(c.message) for c in syncs]
