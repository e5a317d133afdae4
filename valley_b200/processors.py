"""generate()'s logits processors: transformers 5.5's ``RepetitionPenaltyLogitsProcessor``, ``NoRepeatNGramLogitsProcessor``
and ``MinLengthLogitsProcessor`` / ``MinNewTokensLengthLogitsProcessor``, as ``GenerationMixin._get_logits_processor`` adds
them, in its order and before the temperature and the top-k / top-p warpers.

``from_kwargs`` turns generate()'s keyword arguments into a ``Processors`` spec (or None when HF would add none of them, or
only ones that cannot change a score), with HF's add conditions and HF's errors.  ``apply`` restates the three processors in
torch with HF's arithmetic; the host-visible loops (greedy / sampling and beam search) run it, and the device path
(``sample_filter_kernel``, csrc/sampling.cuh) is pinned to it bit for bit.

Each row's ``input_ids`` is the row as HF holds it: the prompt (left padding and the image / frame placeholder ids
included), then every emitted token -- pad once the row has finished, as HF keeps processing finished rows."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

KWARGS = ("repetition_penalty", "no_repeat_ngram_size", "min_new_tokens", "min_length")


@dataclass(frozen=True)
class Processors:
    """the processors of one request: ``penalty`` 1.0 = off, ``ngram`` 0 = off, ``min_length`` 0 = off (the length, prompt
    included, below which ``eos`` scores -inf)"""
    penalty: float = 1.0
    ngram: int = 0
    min_length: int = 0
    eos: int = -1


def from_kwargs(kw: dict, prompt_len: int, eos_token_id: Optional[int]) -> Optional[Processors]:
    """Pops generate()'s processor arguments from ``kw`` and returns their spec, or None.  HF's conditions:

    * ``RepetitionPenaltyLogitsProcessor`` when ``repetition_penalty is not None and != 1.0``; it requires a float > 0;
    * ``NoRepeatNGramLogitsProcessor`` when ``no_repeat_ngram_size is not None and > 0``; it requires an int;
    * min length only with an eos id: ``min_new_tokens`` (when not None) becomes ``min_length = min_new_tokens + prompt_len``
      and wins over ``min_length``; ``MinLengthLogitsProcessor`` is added when ``min_length > 0`` and requires an int,
      ``MinNewTokensLengthLogitsProcessor`` when ``min_new_tokens > 0`` and requires an int >= 0.  A min length the prompt
      already reaches bans nothing, so it is left out."""
    vals = {k: kw.pop(k, None) for k in KWARGS}
    penalty, ngram = 1.0, 0
    rp = vals["repetition_penalty"]
    if rp is not None and rp != 1.0:
        if not isinstance(rp, float) or not (rp > 0):
            raise ValueError(f"`penalty` has to be a strictly positive float, but is {rp}")
        penalty = rp
    nr = vals["no_repeat_ngram_size"]
    if nr is not None and nr > 0:
        if not isinstance(nr, int) or nr <= 0:
            raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {nr}")
        ngram = nr
    min_length = 0
    mnt, ml = vals["min_new_tokens"], vals["min_length"]
    if mnt is not None:
        ml = mnt + prompt_len
    if eos_token_id is not None:
        if ml is not None and ml > 0:
            if not isinstance(ml, int) or ml < 0:
                raise ValueError(f"`min_length` has to be a non-negative integer, but is {ml}")
            min_length = ml
        if mnt is not None and mnt > 0:
            for name, v in (("prompt_length_to_skip", prompt_len), ("min_new_tokens", mnt)):
                if not isinstance(v, int) or v < 0:
                    raise ValueError(f"`{name}` has to be a positive integer, but is {v}")
    if min_length <= prompt_len:
        min_length = 0
    if penalty == 1.0 and ngram == 0 and min_length == 0:
        return None
    return Processors(float(penalty), int(ngram), int(min_length), -1 if eos_token_id is None else int(eos_token_id))


def banned_ngram_tokens(ids: torch.Tensor, n: int):
    """HF's ``_calc_banned_ngram_tokens`` for every row of ``ids`` [R, L]: per row, the tokens that followed an earlier
    occurrence of its last n - 1 ids (list of lists)"""
    R, L = ids.shape
    if L + 1 < n:
        return [[] for _ in range(R)]
    rows = ids.tolist()
    out = []
    for row in rows:
        tail = tuple(row[L - n + 1:])
        out.append([row[j + n - 1] for j in range(L - n + 1) if tuple(row[j:j + n - 1]) == tail])
    return out


def apply(scores: torch.Tensor, ids: torch.Tensor, p: Optional[Processors]) -> torch.Tensor:
    """HF's processors on ``scores`` [R, V] fp32 for ``input_ids`` ``ids`` [R, L] int64, in HF's order and arithmetic:
    the penalty gathers each id's score and scatters ``s * penalty`` if ``s < 0`` else ``s / penalty`` (a true fp32 division,
    also on CUDA, where torch divides by a Python scalar through its reciprocal), then the n-gram and min-length bans write
    -inf.  Ids outside [0, V) are not scored (HF would raise on them)."""
    if p is None:
        return scores
    V = scores.shape[-1]
    ids = ids.to(scores.device, torch.int64)
    out = scores
    if p.penalty != 1.0:
        # (HF's gather / scatter of the same per-element values, as a mask: no host synchronisation)
        seen = torch.zeros(ids.shape[0], V + 1, dtype=torch.bool, device=scores.device)
        seen.scatter_(1, torch.where((ids >= 0) & (ids < V), ids, V), True)
        pen = torch.tensor(p.penalty, dtype=scores.dtype, device=scores.device)
        out = torch.where(seen[:, :V], torch.where(out < 0, out * pen, out / pen), out)
    if p.ngram > 0:
        banned = banned_ngram_tokens(ids, p.ngram)
        if any(banned):
            out = out.clone() if out is scores else out
            for i, toks in enumerate(banned):
                toks = [t for t in toks if 0 <= t < V]
                if toks:
                    out[i, toks] = -float("inf")
    if p.min_length > 0 and p.eos >= 0 and ids.shape[-1] < p.min_length and p.eos < V:
        out = out.clone() if out is scores else out
        out[:, p.eos] = -float("inf")
    return out
