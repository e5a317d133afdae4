"""Writes tests/golden/ref_sampling_filters.pt: the kept masks of HF transformers' own sampling warpers
(TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper, the order HF generate applies them in) on seeded fp32 rows.

    python -m oracle.make_golden_sampling_filters

Rows (V = 1032 and V = 32008): one seeded normal row per V, scaled by powers of two (exact in fp32) to several scales and to a
nearly flat row, plus a row with ties at the 20th and 50th largest value and a row whose top-p cut falls inside a tie group.
Only the base rows are stored; ``build_rows`` derives the others exactly.  A mask is stored as the number of tokens kept when
it is the top of the row in descending order (ties in index order, ``mask_from_count``), which holds for every mask without a
tie group cut by the top-p threshold; the others are stored as packed bits.
"""
from __future__ import annotations

import os

import numpy as np
import torch

VOCABS = (1032, 32008)
TEMPERATURES = (0.2, 0.7, 1.0)
TOP_KS = (None, 1, 20, 50, "V")
TOP_PS = (None, 0.05, 0.5, 0.9, 0.999)
SETTINGS = [(t, k, p) for t in TEMPERATURES for k in TOP_KS for p in TOP_PS]
TIE_ROWS = ("tie_k", "tie_p")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_sampling_filters.pt")


def base_row(V: int, seed: int) -> torch.Tensor:
    """seeded N(0, 1) fp32 row on a 2^-16 grid with no two values on the same grid point (colliding values are moved up by
    one point), so that dividing by any of the temperatures cannot round two values to the same score"""
    z = torch.randn(V, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    q = torch.round(z * 65536).to(torch.int64)
    srt, idx = torch.sort(q)
    for i in range(1, V):
        if srt[i] <= srt[i - 1]:
            srt[i] = srt[i - 1] + 1
    q[idx] = srt
    return (q.double() / 65536).float()


def build_rows(base: torch.Tensor):
    """[(name, logits fp32 [V])] derived exactly from one base row"""
    order = torch.argsort(base, descending=True, stable=True)
    rows = [("normal_x0.5", base * 0.5), ("normal_x2", base * 2.0), ("normal_x8", base * 8.0), ("flat", base * 2.0 ** -10)]
    tk = base * 2.0
    tk[order[15:24]] = float(tk[order[19]])         # ranks 16..24 equal the 20th largest
    tk[order[44:55]] = float(tk[order[49]])         # ranks 45..55 equal the 50th largest
    rows.append(("tie_k", tk))
    tp = base * 2.0
    tp[order[1:41]] = float(tp[order[1]])          # ranks 2..41 tie: their mass straddles small and middle top_p cuts
    rows.append(("tie_p", tp))
    return rows


def mask_from_count(z: torch.Tensor, m: int) -> torch.Tensor:
    mask = torch.zeros(z.shape[-1], dtype=torch.bool)
    mask[torch.argsort(z, descending=True, stable=True)[:m]] = True
    return mask


def resolve_top_k(top_k, V):
    return V if top_k == "V" else top_k


def hf_mask(z: torch.Tensor, t: float, top_k, top_p) -> torch.Tensor:
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    scores = TemperatureLogitsWarper(t)(None, z[None].clone())
    if top_k is not None:
        scores = TopKLogitsWarper(top_k=top_k)(None, scores)
    if top_p is not None:
        scores = TopPLogitsWarper(top_p=top_p)(None, scores)
    return torch.isfinite(scores[0])


def main():
    import transformers
    bases, entries = {}, []
    for V in VOCABS:
        bases[V] = base_row(V, 20261016 + V)
        for name, z in build_rows(bases[V]):
            for t in TEMPERATURES:             # the division creates no ties: only the deliberate ones exist
                assert len(torch.unique(z / t)) == len(torch.unique(z)), (V, name, t)
            if name not in TIE_ROWS:
                assert len(torch.unique(z)) == V, (V, name)
            counts, packed = [], {}
            for i, (t, k, p) in enumerate(SETTINGS):
                mask = hf_mask(z, t, resolve_top_k(k, V), p)
                m = int(mask.sum())
                if torch.equal(mask, mask_from_count(z, m)):
                    counts.append(m)
                else:
                    assert name in TIE_ROWS, (V, name, t, k, p)
                    counts.append(-1)
                    packed[i] = torch.from_numpy(np.packbits(mask.numpy()))
            entries.append({"V": V, "name": name, "counts": torch.tensor(counts, dtype=torch.int32), "packed": packed})
    torch.save({"transformers": transformers.__version__, "settings": SETTINGS, "bases": bases, "rows": entries}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(entries)} rows x {len(SETTINGS)} settings")


def load_masks(gold):
    """[(V, name, z, setting_index, (T, top_k, top_p), kept mask)] from the golden dict (top_k resolved, None kept)"""
    out = []
    for e in gold["rows"]:
        z = dict(build_rows(gold["bases"][e["V"]]))[e["name"]]
        for i, (t, k, p) in enumerate(gold["settings"]):
            m = int(e["counts"][i])
            if m >= 0:
                mask = mask_from_count(z, m)
            else:
                mask = torch.from_numpy(np.unpackbits(e["packed"][i].numpy())[:e["V"]].astype(bool))
            out.append((e["V"], e["name"], z, i, (t, resolve_top_k(k, e["V"]), p), mask))
    return out


if __name__ == "__main__":
    main()
