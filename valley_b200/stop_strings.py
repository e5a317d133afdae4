"""Stop strings: transformers' ``StopStringCriteria`` (``generate(stop_strings=..., tokenizer=...)``) as bit-mask tables.

A row's text is the concatenation of its tokens' *clean strings*: what ``convert_tokens_to_string`` makes of the token after a
fixed prefix, minus that prefix (so ``▁`` / ``Ġ`` become spaces, byte tokens their byte; special tokens keep their literal
text).  After each step, a row matches when its text ends with a stop string, the last characters inside the newest token
(trailing characters after the stop string allowed there).  As in HF, the whole sequence counts, prompt included, and a match
spans at most as many tokens as the longest stop string has characters.

For stop string s and token t, ``stop_tables`` records
  end bit L-1: t can be the newest token with the last L characters of s inside it (L = len(s): t holds all of s);
  pos bit p:   t fits with its end p characters before the end of s (0 < p < len(s)); it may reach past the start of s;
and the token's length.  A row matches s when, for some end bit L of its newest token, walking back over the earlier tokens
from pos = L -- each must have pos bit ``pos`` set, and adds its length -- reaches pos >= len(s).  The device matcher
(``sampling.cuh``, ``stop_match_warp``) and ``match_rows`` below both walk these tables.
"""
from __future__ import annotations

import threading
from collections import OrderedDict
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

MAX_DEVICE_STOP_STRINGS = 8      # kMaxStopStrings
MAX_DEVICE_STOP_CHARS = 64       # kMaxStopChars: the masks are uint64
STATIC_PREFIX = "abcdef"

_lock = threading.Lock()
_clean_cache: OrderedDict = OrderedDict()          # tokenizer key -> (tokenizer, clean strings or pause bits)
_table_cache: "OrderedDict[tuple, StopTables]" = OrderedDict()
_CACHE_SIZE = 8


def _remember(cache: OrderedDict, key, value):
    cache[key] = value
    cache.move_to_end(key)
    while len(cache) > _CACHE_SIZE:
        cache.popitem(last=False)
    return value


def _tokenizer_key(tokenizer) -> tuple:
    """a tokenizer's cache key: the object (checked by identity on a hit) and its size, which adding tokens changes"""
    return (id(tokenizer), len(tokenizer) if hasattr(tokenizer, "__len__") else len(tokenizer.get_vocab()))


def normalize(stop_strings) -> Tuple[str, ...]:
    """``stop_strings`` as HF accepts it: one string or a list of strings"""
    if isinstance(stop_strings, str):
        stop_strings = [stop_strings]
    out = tuple(stop_strings)
    if not out or not all(isinstance(s, str) and s for s in out):
        raise ValueError(f"`stop_strings` must be a non-empty string or a list of non-empty strings, got {stop_strings!r}")
    return out


def clean_token_strings(tokenizer) -> Tuple[Optional[str], ...]:
    """The clean string of every token id (None for an id the vocabulary does not have), through the tokenizer surface HF
    uses: ``get_vocab``, ``__call__(..., add_special_tokens=False)``, ``convert_ids_to_tokens`` and
    ``convert_tokens_to_string``.  Cached per tokenizer and vocabulary size."""
    key = _tokenizer_key(tokenizer)
    with _lock:
        hit = _clean_cache.get(key)
        if hit is not None and hit[0] is tokenizer:
            _clean_cache.move_to_end(key)
            return hit[1]
    vocab = tokenizer.get_vocab()
    base = tokenizer.convert_ids_to_tokens(tokenizer(STATIC_PREFIX, add_special_tokens=False)["input_ids"])
    clean: List[Optional[str]] = [None] * (max(vocab.values()) + 1)
    for token, idx in vocab.items():
        text = tokenizer.convert_tokens_to_string(list(base) + [token])
        clean[idx] = text[text.index(STATIC_PREFIX) + len(STATIC_PREFIX):]
    clean = tuple(clean)
    with _lock:
        return _remember(_clean_cache, key, (tokenizer, clean))[1]


def _masks(c: str, s: str) -> Tuple[int, int]:
    """(end mask, pos mask) of clean string c for stop string s, as Python ints"""
    n = len(s)
    if c == "":
        return 0, ((1 << n) - 1) & ~1           # an empty token fits at every inner position and ends nothing
    if not set(c) & set(s):
        return 0, 0
    end = 0
    for k in range(len(c)):                     # k trailing characters of c after the end of s
        u = c[:len(c) - k]
        L = min(len(u), n)
        if u[len(u) - L:] == s[n - L:]:
            end |= 1 << (L - 1)
    pos = 0
    for p in range(1, n):
        m = min(len(c), n - p)
        if c[len(c) - m:] == s[n - p - m:n - p]:
            pos |= 1 << p
    return end, pos


class StopTables:
    """The tables of one (vocabulary, stop strings) pair over token ids [0, V).

    strings: the stop strings; lens: int32 [n] their lengths; walk: tokens a match may span (the longest length);
    token_lens: int32 [V] clean-string lengths (0 for ids the vocabulary lacks); end / pos: per string, Python-int masks
    [V] (any width); masks: uint64 [n, V, 2] (end, pos) when ``on_device``, else None.
    on_device: at most MAX_DEVICE_STOP_STRINGS strings of at most MAX_DEVICE_STOP_CHARS characters."""

    def __init__(self, clean: Sequence[Optional[str]], strings: Sequence[str], V: int):
        self.strings = tuple(strings)
        self.lens = np.array([len(s) for s in self.strings], dtype=np.int32)
        self.walk = int(self.lens.max())
        self.V = V
        self.token_lens = np.zeros(V, dtype=np.int32)
        self.end: List[List[int]] = [[0] * V for _ in self.strings]
        self.pos: List[List[int]] = [[0] * V for _ in self.strings]
        for t in range(min(V, len(clean))):
            c = clean[t]
            if c is None:
                continue
            self.token_lens[t] = len(c)
            for i, s in enumerate(self.strings):
                self.end[i][t], self.pos[i][t] = _masks(c, s)
        self.on_device = len(self.strings) <= MAX_DEVICE_STOP_STRINGS and self.walk <= MAX_DEVICE_STOP_CHARS
        self.masks = None
        if self.on_device:
            self.masks = np.zeros((len(self.strings), V, 2), dtype=np.uint64)
            for i in range(len(self.strings)):
                self.masks[i, :, 0] = np.array(self.end[i], dtype=np.uint64)
                self.masks[i, :, 1] = np.array(self.pos[i], dtype=np.uint64)


def stop_tables(clean: Sequence[Optional[str]], stop_strings, V: Optional[int] = None) -> StopTables:
    """``StopTables`` of the clean strings (``clean_token_strings``) for ``stop_strings`` over V token ids (default: the
    vocabulary's size; a model's larger vocabulary pads with ids that fit nowhere).  Cached per (vocabulary, strings, V)."""
    strings = normalize(stop_strings)
    V = len(clean) if V is None else int(V)
    key = (id(clean), len(clean), strings, V)
    with _lock:
        hit = _table_cache.get(key)
        if hit is not None and hit._clean is clean:
            _table_cache.move_to_end(key)
            return hit
    t = StopTables(clean, strings, V)
    t._clean = clean                       # (keeps the cached clean tuple, and so its id, alive)
    with _lock:
        return _remember(_table_cache, key, t)


def match_rows(tokens: torch.Tensor, tables: StopTables) -> torch.Tensor:
    """HF's StopStringCriteria on tokens [B, n]: bool [B], True where the row's text ends with a stop string, the last
    characters inside its last token.  The host loops use it; it is the reference the device matcher is tested against."""
    rows = tokens.detach().to("cpu", torch.int64).tolist()
    out = torch.zeros(len(rows), dtype=torch.bool)
    V = tables.V
    for b, row in enumerate(rows):
        if not row:
            continue
        recent = row[::-1][:tables.walk]
        if not 0 <= recent[0] < V:
            continue
        for i, n in enumerate(tables.lens.tolist()):
            end = tables.end[i][recent[0]]
            if not end:
                continue
            if end >> (n - 1):
                out[b] = True
                break
            reach = (end << 1) & ((1 << n) - 1)         # bit p: a walk stands p characters before the end of the string
            for t in recent[1:]:
                if not 0 <= t < V:
                    break
                reach &= tables.pos[i][t]
                if not reach:
                    break
                reach <<= int(tables.token_lens[t])
                if reach >> n:
                    break
                reach &= (1 << n) - 1
            if reach >> n:
                out[b] = True
                break
    return out


def pause_bits(tokenizer, V: int, exclude: Sequence[int] = ()) -> np.ndarray:
    """uint32 [ceil(V / 32)]: the ids whose ``tokenizer.decode([id], skip_special_tokens=True)`` is empty, less ``exclude``.
    ``KeywordsStoppingCriteria`` decodes with special tokens skipped, so such a token can join two halves of a keyword."""
    key = ("pause",) + _tokenizer_key(tokenizer) + (V, tuple(exclude))
    with _lock:
        hit = _clean_cache.get(key)
    if hit is None or hit[0] is not tokenizer:
        bits = np.zeros((V + 31) // 32, dtype=np.uint32)
        for idx in tokenizer.get_vocab().values():
            if 0 <= idx < V and idx not in exclude and tokenizer.decode([idx], skip_special_tokens=True) == "":
                bits[idx >> 5] |= np.uint32(1 << (idx & 31))
        with _lock:
            hit = _remember(_clean_cache, key, (tokenizer, bits))
    return hit[1]
