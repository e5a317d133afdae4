"""Beam search as transformers 5.5 ``GenerationMixin._beam_search`` runs it (non-sampling branch), restated in torch over
logits that come from anywhere: ``generate``'s host-visible loop feeds it the library's logits (and reorders the library's KV
cache by the parents it returns), the oracle feeds it the fp32 CPU model's.  The device path (csrc/beam.cuh) computes the same
thing; the two agree bit for bit on the same logits because both

  * compute log_softmax as ``z - lse`` with ``lse = max + log(sum(exp(z - max)))`` summed in float64 (within an ulp of HF's
    fp32 log_softmax, and independent of the summation order), and
  * break every tie of a top-k by the lowest index (a stable descending sort; HF's ``torch.topk`` leaves ties unspecified).

Everything else is HF's arithmetic in HF's order, fp32: the ``-1e9`` masks, ``score / generated_len ** length_penalty``
(a true division by the fp32 divisor), the early-stop heuristic and the stopping rule."""
from __future__ import annotations

from typing import Callable, Optional

import torch

from . import processors as _proc

NEG = -1.0e9


def log_softmax(logits: torch.Tensor) -> torch.Tensor:
    """[R, V] fp32 -> fp32 log-probabilities with a float64 log-sum-exp"""
    m = logits.max(-1, keepdim=True).values
    s = torch.exp(logits - m).double().sum(-1, keepdim=True)
    return (logits.double() - (m.double() + torch.log(s))).float()


def topk(x: torch.Tensor, k: int):
    """top k along the last dim, descending, ties by the lowest index"""
    v, i = torch.sort(x, dim=-1, descending=True, stable=True)
    return v[..., :k], i[..., :k]


def output_fill_value(pad_token_id, eos_token_id) -> int:
    """HF's ``pad_token_id or eos_token_id[0] if eos_token_id is not None else -1``: the value written after a sequence's end"""
    if eos_token_id is None:
        return -1
    return int(pad_token_id) if pad_token_id else int(eos_token_id)


class BeamSearch:
    """The state of one beam request over ``prompt_ids`` [B * num_beams, S] (each item's prompt repeated num_beams times).

    ``step(logits)`` takes the step's logits [B * num_beams, V] and returns ``(parent_rows, tokens)``: the row of the previous
    step every new beam continues (what the KV cache must be reordered by) and the tokens to feed next; ``done`` is set when
    HF's loop would stop.  ``result(num_return_sequences)`` gives ``(sequences [B * nrs, S + L], sequences_scores [B * nrs])``,
    ``beam_indices(num_return_sequences)`` HF's ``beam_indices`` [B * nrs, L] next to them.  ``record_scores`` / ``record_logits``
    keep every step's log-probabilities / logits [B * num_beams, V] in ``scores`` / ``logits`` (HF's output_scores /
    output_logits); ``t`` is the number of steps run.  ``processors`` (``processors.Processors``) are applied to every beam row's
    log-probabilities with the running hypotheses as input_ids, before the beam scores are added, as HF does; the recorded
    scores are the processed log-probabilities."""

    def __init__(self, prompt_ids: torch.Tensor, num_beams: int, max_new_tokens: int, eos_token_id: Optional[int], fill: int,
                 length_penalty: float = 1.0, early_stopping=False, record_scores: bool = False, record_logits: bool = False,
                 processors: Optional[_proc.Processors] = None):
        rows, S = prompt_ids.shape
        self.nb, self.B, self.S, self.n_new = num_beams, rows // num_beams, S, max_new_tokens
        self.K = 2 * num_beams                     # max(2, 1 + n_eos) * num_beams with at most one eos id
        self.eos, self.lp, self.es = eos_token_id, float(length_penalty), early_stopping
        dev = prompt_ids.device
        self.seq = torch.full((self.B, num_beams, S + max_new_tokens), fill, dtype=torch.int64, device=dev)
        self.seq[:, :, :S] = prompt_ids.reshape(self.B, num_beams, S)
        self.fin_seq = self.seq.clone()
        self.run_scores = torch.zeros(self.B, num_beams, dtype=torch.float32, device=dev)
        self.run_scores[:, 1:] = NEG
        self.fin_scores = torch.full((self.B, num_beams), NEG, dtype=torch.float32, device=dev)
        self.fin = torch.zeros(self.B, num_beams, dtype=torch.bool, device=dev)
        self.fin_len = torch.zeros(self.B, num_beams, dtype=torch.int64, device=dev)
        self.heur = torch.ones(self.B, 1, dtype=torch.bool, device=dev)
        self.top_mask = (torch.arange(self.K, device=dev) < num_beams)[None]
        # beam indices of the running / finished hypotheses: per generated position, the cache row the token was appended to
        self.bidx = torch.full((self.B, num_beams, max_new_tokens), -1, dtype=torch.int64, device=dev)
        self.fin_bidx = self.bidx.clone()
        self.scores = [] if record_scores else None
        self.logits = [] if record_logits else None
        self.t, self.done = 0, False
        self.processors = processors
        self.margins = []                          # per step: the smallest gap between consecutive top-(K+1) candidates

    def _div(self, length: int) -> torch.Tensor:
        return torch.tensor(float(length ** self.lp), dtype=torch.float32, device=self.seq.device)

    def step(self, logits: torch.Tensor, stopping: Optional[Callable[[torch.Tensor], object]] = None):
        B, nb, K, t = self.B, self.nb, self.K, self.t
        V = logits.shape[-1]
        cur = self.S + t
        log_probs = log_softmax(logits.float())
        if self.processors is not None:
            log_probs = _proc.apply(log_probs, self.seq[:, :, :cur].reshape(B * nb, cur), self.processors)
        if self.scores is not None:
            self.scores.append(log_probs)
        if self.logits is not None:
            self.logits.append(logits.float())
        acc = (log_probs.reshape(B, nb, V) + self.run_scores[:, :, None]).reshape(B, nb * V)
        top_v, top_i = topk(acc, K + 1)
        self.margins.append(float((top_v[:, :-1] - top_v[:, 1:]).min()))
        vals, idx = top_v[:, :K], top_i[:, :K]
        parent, tok = idx // V, idx % V
        cand = torch.take_along_dim(self.seq, parent[:, :, None], dim=1)
        cand[:, :, cur] = tok
        cand_bidx = torch.take_along_dim(self.bidx, parent[:, :, None], dim=1)
        cand_bidx[:, :, t] = parent + torch.arange(B, device=parent.device)[:, None] * nb
        hits = tok == self.eos if self.eos is not None else torch.zeros_like(tok, dtype=torch.bool)
        if t + 1 >= self.n_new:                    # MaxLengthCriteria
            hits = torch.ones_like(hits)
        if stopping is not None:
            r = stopping(cand[:, :, :cur + 1].reshape(B * K, cur + 1))
            hits = hits | torch.as_tensor(r, device=hits.device).reshape(-1).expand(B * K).reshape(B, K)
        # the next running beams (_get_running_beams_for_next_iteration)
        adj = vals + hits.to(torch.float32) * NEG
        run_v, run_i = topk(adj, nb)
        self.seq = torch.take_along_dim(cand, run_i[:, :, None], dim=1)
        self.bidx = torch.take_along_dim(cand_bidx, run_i[:, :, None], dim=1)
        self.run_scores = run_v
        run_parent = torch.take_along_dim(parent, run_i, dim=1)
        # the finished hypotheses (_update_finished_beams)
        just = hits & self.top_mask
        fs = vals / self._div(t + 1)
        fs = fs + (self.fin.all(-1, keepdim=True) & (self.es is True)).to(torch.float32) * NEG
        fs = fs + (~self.heur).to(torch.float32) * NEG
        fs = fs + (~just).to(torch.float32) * NEG
        m_seq = torch.cat((self.fin_seq, cand), 1)
        m_s = torch.cat((self.fin_scores, fs), 1)
        m_f = torch.cat((self.fin, just), 1)
        m_len = torch.cat((self.fin_len, torch.full_like(vals, t + 1, dtype=torch.int64)), 1)
        _, mi = topk(m_s, nb)
        self.fin_seq = torch.take_along_dim(m_seq, mi[:, :, None], dim=1)
        self.fin_bidx = torch.take_along_dim(torch.cat((self.fin_bidx, cand_bidx), 1), mi[:, :, None], dim=1)
        self.fin_scores = torch.take_along_dim(m_s, mi, dim=1)
        self.fin = torch.take_along_dim(m_f, mi, dim=1)
        self.fin_len = torch.take_along_dim(m_len, mi, dim=1)
        # the early-stop heuristic at the new length, and the loop condition (_beam_search_has_unfinished_sequences)
        best_len = self.n_new if (self.es == "never" and self.lp > 0.0) else t + 1
        best = self.run_scores[:, :1] / self._div(best_len)
        worst = torch.where(self.fin, torch.min(self.fin_scores, dim=1, keepdim=True)[0], NEG)
        self.heur = self.heur & torch.any(best > worst, dim=-1, keepdim=True)
        go_on = bool(self.heur.any()) and not (bool(self.fin.all()) and self.es is True) and not bool(hits.all())
        self.t, self.done = t + 1, not go_on
        rows = (torch.arange(B, device=run_parent.device)[:, None] * nb + run_parent).reshape(-1)
        return rows, self.seq[:, :, cur].reshape(-1)

    def result(self, num_return_sequences: int = 1):
        n = num_return_sequences
        seq = self.fin_seq[:, :n].reshape(self.B * n, -1)
        L = int(self.fin_len[:, :n].max())
        return seq[:, :self.S + L], self.fin_scores[:, :n].reshape(-1)

    def beam_indices(self, num_return_sequences: int = 1) -> torch.Tensor:
        """HF's ``beam_indices`` of the hypotheses ``result`` returns: [B * nrs, L] int64, -1 after each one's end"""
        n = num_return_sequences
        L = int(self.fin_len[:, :n].max())
        return self.fin_bidx[:, :n].reshape(self.B * n, -1)[:, :L]
