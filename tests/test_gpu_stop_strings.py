"""GPU (-m gpu): stop strings on the device.  The matcher (vly_test_stop_strings) reproduces transformers' StopStringCriteria
(tests/golden/ref_stop_strings.pt) bit for bit; generate(stop_strings=...) on the device loop equals the host loop token for
token with no per-token host sync; completion()'s '###' keyword on the device returns the host loop's reply."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import helpers as Hh
from valley_b200 import stop_strings as ss
from valley_b200 import synthetic as syn
from valley_b200._lib import VlySampling, check
from valley_b200.model import KeywordsStoppingCriteria, host_rows_step

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_stop_strings.pt")
_m = {}


def get():
    if "m" not in _m:
        spec = syn.SPECS["tiny"]
        _m["m"] = (spec, Hh.build_model(spec, Hh.bf16_weights(spec, 0)))
    return _m["m"]


class PieceTokenizer:
    """A word tokenizer over the model's ids with the HF surface stop strings use: token i is ``t<i>`` with text
    ``pieces.get(i, ' w<i>')``; ids 0, 1, 2 are special (``<unk>``, ``<s>``, ``</s>``: literal text, deleted by decode with
    skip_special_tokens), and so is ``sentinel`` (text ``<vi_frame>``).  The static-prefix token sits past the model's ids."""
    eos_token_id = 2

    def __init__(self, V, pieces=None, sentinel=None):
        self.V, self.pieces, self.sentinel = V, dict(pieces or {}), sentinel
        self.special = {0: "<unk>", 1: "<s>", 2: "</s>"}
        if sentinel is not None:
            self.special[sentinel] = "<vi_frame>"

    def text(self, i):
        return self.special.get(i) or self.pieces.get(i, f" w{i}")

    def get_vocab(self):
        return {f"t{i}": i for i in range(self.V + 1)}

    def __len__(self):
        return self.V + 1

    def __call__(self, text, add_special_tokens=True):
        assert text == ss.STATIC_PREFIX
        return {"input_ids": [self.V]}

    def convert_ids_to_tokens(self, ids):
        return [f"t{i}" for i in ids]

    def convert_tokens_to_string(self, toks):
        return "".join("abcdef" if t == f"t{self.V}" else self.text(int(t[1:])) for t in toks)

    def decode(self, ids, skip_special_tokens=True):
        ids = ids.tolist() if torch.is_tensor(ids) else ids
        return "".join("" if (skip_special_tokens and int(i) in self.special) else self.text(int(i)) for i in ids)

    def batch_decode(self, rows, skip_special_tokens=True):
        return [self.decode(r, skip_special_tokens) for r in rows]


# ---- 1. the device matcher against transformers ----
@pytest.mark.parametrize("V", [32008, 1032])
def test_device_matcher_reproduces_hf(V):
    spec, m = get()
    g = torch.load(GOLD)
    rows = list(torch.split(g["row_tokens"].long(), g["row_lens"].tolist()))
    clean = list(g["clean"]) + ["~"] * (V - len(g["clean"]))      # filler tokens fit nowhere
    filler = len(g["clean"])
    for k, strings in enumerate(g["sets"]):
        t = ss.stop_tables(clean, strings, V)
        if not t.on_device:
            continue
        sp = VlySampling().set_stop_strings(t)
        got = []
        for i in range(0, len(rows), 64):
            chunk = rows[i:i + 64]
            n = max(len(r) for r in chunk)
            tok = torch.full((len(chunk), n), filler, dtype=torch.int64)
            for b, r in enumerate(chunk):
                tok[b, n - len(r):] = r
            tok = tok.cuda()
            out = torch.empty(len(chunk), dtype=torch.uint8, device="cuda")
            check(m._lib.vly_test_stop_strings(m._ctx, C.byref(sp), V, tok.data_ptr(), len(chunk), n, out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
            got.append(out.cpu().bool())
        assert torch.equal(torch.cat(got), g["results"][k]), strings


# ---- 2. generate(stop_strings=...): device loop == host loop ----
def _prompt(spec, B, seed):
    return torch.randint(3, spec.vocab_size - 8, (B, 7), generator=torch.Generator().manual_seed(seed)).cuda()


def _pieces(ids, free):
    """'#' / '##' pieces on tokens of the free-running continuation so that '###' appears at several steps, one of them
    spanning the prompt/generation boundary of row 0"""
    p = {int(ids[0, -1]): "#", int(free[0, 0]): "##"}
    for b in range(1, free.shape[0], 2):
        k = 2 + b % 5
        p.setdefault(int(free[b, k]), "##")
        p.setdefault(int(free[b, k + 1]), "#a")
    return p


def _replay(ids, out, eos, pad, tables):
    """the host loop's row handling over out's own tokens: the sequence it returns"""
    seq, fin = ids, torch.zeros(ids.shape[0], dtype=torch.bool, device=ids.device)
    for i in range(ids.shape[1], out.shape[1]):
        seq, _, fin, stop = host_rows_step(seq, out[:, i].clone(), fin, eos, pad, tables)
        if stop:
            break
    return seq


class _Count:
    def __init__(self, lib):
        self._lib, self.decodes = lib, 0

    def __getattr__(self, name):
        if name == "vly_llama_decode":
            self.decodes += 1
        return getattr(self._lib, name)


@pytest.mark.parametrize("B", [1, 3, 6, 64])
@pytest.mark.parametrize("eos", [None, "gen"])
def test_generate_stop_strings_device_equals_host(B, eos):
    spec, m = get()
    ids = _prompt(spec, B, B)
    free = m.generate(input_ids=ids, max_new_tokens=16, eos_token_id=None)[:, ids.shape[1]:]
    tok = PieceTokenizer(spec.vocab_size, _pieces(ids, free))
    e = None if eos is None else int(free[-1, 10])
    kw = dict(input_ids=ids, max_new_tokens=16, eos_token_id=e, pad_token_id=0, stop_strings=["###", "a#"], tokenizer=tok)
    lib = m._lib
    m._lib = cnt = _Count(lib)
    try:
        dev = m.generate(**kw)
    finally:
        m._lib = lib
    assert cnt.decodes == 0                                    # no per-token host round trip
    host = m.generate(**kw, stopping_criteria=[lambda s, sc: False])
    assert torch.equal(dev, host)
    tables = ss.stop_tables(ss.clean_token_strings(tok), ["###", "a#"], spec.vocab_size)
    assert bool(ss.match_rows(dev[:1, :ids.shape[1] + 1], tables)[0])          # row 0 stops on the boundary-spanning string


@pytest.mark.parametrize("B", [1, 6])
def test_generate_stop_strings_sampled_rows_follow_hf_row_handling(B):
    spec, m = get()
    ids = _prompt(spec, B, 40 + B)
    free = m.generate(input_ids=ids, max_new_tokens=16, eos_token_id=None)[:, ids.shape[1]:]
    tok = PieceTokenizer(spec.vocab_size, _pieces(ids, free))
    tables = ss.stop_tables(ss.clean_token_strings(tok), "###", spec.vocab_size)
    for e in (None, int(free[0, 12])):
        torch.manual_seed(5)
        out = m.generate(input_ids=ids, max_new_tokens=16, do_sample=True, temperature=0.5, top_k=4, eos_token_id=e,
                         pad_token_id=0, stop_strings="###", tokenizer=tok)
        assert torch.equal(_replay(ids, out, e, 0, tables), out)


def test_beam_search_with_stop_strings_equals_the_host_beam_loop():
    spec, m = get()
    ids = _prompt(spec, 2, 9)
    free = m.generate(input_ids=ids, max_new_tokens=10, num_beams=2, eos_token_id=None)[:, ids.shape[1]:]
    tok = PieceTokenizer(spec.vocab_size, {int(free[0, 3]): "##", int(free[0, 4]): "#"})
    tables = ss.stop_tables(ss.clean_token_strings(tok), "###", spec.vocab_size)
    got = m.generate(input_ids=ids, max_new_tokens=10, num_beams=2, eos_token_id=2, stop_strings="###", tokenizer=tok)
    want = m.generate(input_ids=ids, max_new_tokens=10, num_beams=2, eos_token_id=2,
                      stopping_criteria=[lambda s, sc: ss.match_rows(s, tables).to(s.device)])
    assert torch.equal(got, want)


# ---- 3. completion()'s '###' on the device ----
MESSAGE = [{"role": "system", "content": "You are a helpful assistant."},
           {"role": "user", "content": "<video> What happens in the video?"}]


def _completion_case(case):
    """(tokenizer pieces, sentinel, eos) for a keyword at step 1, at step k, split over two tokens, split by a special token,
    or never (ending by eos or by length)"""
    spec, m = get()
    from test_gpu_dropin import WordTokenizer
    wt = WordTokenizer(spec)
    ids = torch.as_tensor(m.build_inputs(wt, MESSAGE).input_ids).cuda()
    clip = torch.randn(3, 8, 224, 224, generator=torch.Generator().manual_seed(1))
    images = clip.permute(1, 0, 2, 3)[None].half().cuda()
    free = m.generate(input_ids=ids, images=images, max_new_tokens=24, eos_token_id=None)[0, ids.shape[1]:].tolist()
    pieces, sentinel, eos = {}, None, None
    if case == "step1":
        pieces = {free[0]: " ###"}
    elif case == "stepk":
        pieces = {free[5]: " ###"}
    elif case == "split":
        pieces = {free[6]: "##", free[7]: "#b"}
    elif case == "special":
        pieces, sentinel = {free[4]: " #", free[6]: "##"}, free[5]
    elif case == "eos":
        eos = free[9]
    return wt, ids, clip, free, pieces, sentinel, eos


class _Tok(PieceTokenizer):
    """PieceTokenizer plus the prompt encoding of test_gpu_dropin.WordTokenizer, for build_inputs"""

    def __init__(self, wt, V, pieces, sentinel, eos):
        super().__init__(V, pieces, sentinel)
        self.wt, self.eos_token_id, self.padding_side = wt, 2 if eos is None else eos, "left"
        if eos is not None:
            self.special[eos] = "</s>"

    def __call__(self, text, add_special_tokens=True, padding=False):
        if text == ss.STATIC_PREFIX:
            return {"input_ids": [self.V]}
        self.wt.padding_side = self.padding_side
        return self.wt(text, padding=padding)


@pytest.mark.parametrize("case", ["step1", "stepk", "split", "special", "eos", "length"])
def test_completion_keyword_on_the_device_equals_the_host_loop(case):
    spec, m = get()
    wt, ids, clip, free, pieces, sentinel, eos = _completion_case(case)
    tok = _Tok(wt, spec.vocab_size, pieces, sentinel, eos)
    gen_kwargs = {"max_new_tokens": 24, "do_sample": False}
    lib = m._lib
    m._lib = cnt = _Count(lib)
    try:
        reply = m.completion(tok, clip, MESSAGE, gen_kwargs, "cuda")
    finally:
        m._lib = lib
    crit = KeywordsStoppingCriteria(["###"], tok, ids)
    want_ids = m.generate(input_ids=ids, images=clip.permute(1, 0, 2, 3)[None].half().cuda(), stopping_criteria=[crit],
                          eos_token_id=tok.eos_token_id, **gen_kwargs)
    assert reply == m.process_response(tok.batch_decode(want_ids[:, ids.shape[1]:]))
    assert cnt.decodes <= 1                                   # (one host step when the first token holds the keyword)
