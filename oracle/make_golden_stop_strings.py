"""Writes tests/golden/ref_stop_strings.pt: transformers' own ``StopStringCriteria`` on a toy tokenizer, and one run of HF
``generate(stop_strings=...)`` with a tiny seeded ``LlamaForCausalLM``, with and without eos.

    python -m oracle.make_golden_stop_strings

The toy tokenizer is a ``PreTrainedTokenizerFast`` over a ``tokenizers`` WordLevel model with Metaspace pre-tokenizer and
ByteFallback + Metaspace decoders.  Its vocabulary has the static-prefix token ``▁abcdef`` HF's ``clean_tokenizer_vocab``
needs, the tokens ``#``, ``##``, ``#a``, ``▁###``, ``<0x23>``, tokens that hold a whole stop string, tokens that overlap
several stop strings, special tokens and an empty-string token.  Stop-string sets (``SETS``) include one of 64 characters
and one of 9 strings.  Rows: ``N_ROWS`` seeded rows of lengths 1..80 drawn with extra weight on the ``#``-bearing tokens.
Stored: the vocabulary, HF's clean strings, the rows (``HANDMADE`` first; concatenated, with their lengths), HF's per-row
booleans per set.

Generate: the ``tiny`` synthetic LLM weights (bf16-rounded) as an HF ``LlamaForCausalLM``, 3 prompts of 6 tokens, greedy,
12 new tokens, with a word tokenizer over the model's vocabulary (token i is ``▁w<i>``) and stop strings chosen from its
greedy continuation so that row 0 stops at step 4 (a string spanning two tokens) and row 1 at step 7; row 2 never stops.
Stored for eos unset and for eos = a token of row 2's continuation: the sequences and HF's per-step scores."""
from __future__ import annotations

import os

import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_stop_strings.pt")
SPECIALS = ["<unk>", "<s>", "</s>", "<vi_frame>"]
WORDS = ["▁abcdef", "▁a", "a", "b", "▁b", "#", "##", "#a", "a#", "b#", "▁###", "<0x23>", "<0x61>", "▁", "", "x###y", "###",
         "#a#a", "a#a#", "ab", "ba", "▁ab", "#b", "##b", "a##", "▁#", "▁▁"]
SETS = [
    ["###"],
    ["###", "#a", "a#b"],
    ["ab", "ba", "a"],
    [" ###", "### "],
    ["#a" * 32],                                           # 64 characters: the device limit
    ["a" * 3 + "#" * 62],                                  # 65 characters: past it
    ["#", "##", "a", "b", "ab", "#b", " #", "a a", "b#"],  # 9 strings: past the device's 8
]
N_ROWS = 2000
GEN_NEW = 12


def toy_tokenizer():
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    vocab = {w: i for i, w in enumerate(SPECIALS + WORDS)}
    tk = Tokenizer(models.WordLevel(vocab=vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.Metaspace()
    tk.decoder = decoders.Sequence([decoders.ByteFallback(), decoders.Metaspace()])
    tok = PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>", bos_token="<s>", eos_token="</s>")
    tok.add_special_tokens({"additional_special_tokens": ["<vi_frame>"]})
    return tok


def word_tokenizer(V: int):
    """token i is ``▁w<i>`` (clean string `` w<i>``), plus the static-prefix token at id V"""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    vocab = {f"▁w{i}": i for i in range(V)}
    vocab["▁abcdef"] = V
    vocab["<unk>"] = V + 1
    tk = Tokenizer(models.WordLevel(vocab=vocab, unk_token="<unk>"))
    tk.pre_tokenizer = pre_tokenizers.Metaspace()
    tk.decoder = decoders.Metaspace()
    return PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="<unk>")


HANDMADE = [
    ["▁a", "##", "#a"], ["▁a", "▁###"], ["▁a", "<0x23>", "<0x23>", "<0x23>"], ["▁a", "#", "#", "b"], ["▁a", "##", "</s>", "#"],
    ["▁a", "b", "▁###", "b"], ["▁a", "##", "", "#"], ["#", "", "", "##"], ["x###y"], ["b", "x###y"], ["<vi_frame>", "###"],
    ["#a"] * 32, ["b"] + ["#a"] * 32, ["#a"] * 31, ["#a#a"] * 16, ["a#"] + ["#a"] * 31 + ["#"], ["a#a#"] * 16 + ["b"],
    ["a", "a", "a"] + ["##"] * 31, ["a", "a", "a"] + ["##"] * 30 + ["#"], ["a", "a"] + ["##"] * 31,
    ["▁ab", "a"], ["▁", "###"], ["###", "▁"], ["▁▁", "#", "##"],
]


def rows(n_vocab: int):
    vocab = {w: i for i, w in enumerate(SPECIALS + WORDS)}
    out = [torch.tensor([vocab[w] for w in r]) for r in HANDMADE]
    g = torch.Generator().manual_seed(20261017)
    hashy = [len(SPECIALS) + i for i, w in enumerate(WORDS) if "#" in w or w in ("<0x23>", "")]
    w = torch.ones(n_vocab)
    w[hashy] = 4.0
    for _ in range(N_ROWS - len(out)):
        n = int(torch.randint(1, 81, (1,), generator=g))
        out.append(torch.multinomial(w, n, replacement=True, generator=g))
    return out


def generate_run():
    from transformers.generation.stopping_criteria import StopStringCriteria  # noqa: F401  (the criterion generate builds)
    from oracle.make_golden_beam_search import hf_model, weights
    from valley_b200 import synthetic as syn
    spec = syn.SPECS["tiny"]
    m = hf_model(spec, weights(spec))
    V = spec.vocab_size
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(3, V - 8, (3, 6), generator=g)
    kw = dict(input_ids=ids, attention_mask=torch.ones_like(ids), position_ids=torch.arange(6)[None].expand(3, 6).contiguous(),
              max_new_tokens=GEN_NEW, do_sample=False, pad_token_id=0)
    with torch.no_grad():
        free = m.generate(**kw, eos_token_id=None)[:, 6:]
    # row 0: the last digit of its step-3 token, a space and the first characters of its step-4 token
    t3, t4 = f"w{int(free[0, 3])}", f"w{int(free[0, 4])}"
    stops = [t3[-1] + " " + t4[:2], f" w{int(free[1, 6])}"]
    tok = word_tokenizer(V)
    eos = int(free[2, 9])
    runs = []
    for e in (None, eos):
        with torch.no_grad():
            out = m.generate(**kw, eos_token_id=e, stop_strings=stops, tokenizer=tok, return_dict_in_generate=True,
                             output_scores=True)
        runs.append(dict(eos=e, sequences=out.sequences.clone(), scores=torch.stack(out.scores, 1).float().clone()))
        print("eos", e, "->", out.sequences[:, 6:].tolist())
    return dict(prompt=ids, free=free, stop_strings=stops, V=V, pad=0, runs=runs)


def main():
    import transformers
    from transformers.generation.stopping_criteria import StopStringCriteria
    tok = toy_tokenizer()
    vocab = tok.get_vocab()
    clean, idx = StopStringCriteria.clean_tokenizer_vocab(tok)
    clean_by_id = [None] * (max(idx) + 1)
    for c, i in zip(clean, idx):
        clean_by_id[i] = c
    data = rows(len(clean_by_id))
    results = []
    for stops in SETS:
        crit = StopStringCriteria(tok, stops)
        res = torch.tensor([bool(crit(r[None], None)[0]) for r in data])
        print(stops[:3], "...", int(res.sum()), "of", len(data), "rows match")
        results.append(res)
    torch.save({"transformers": transformers.__version__, "vocab": vocab, "clean": clean_by_id, "sets": SETS,
                "row_lens": torch.tensor([len(r) for r in data], dtype=torch.int16),
                "row_tokens": torch.cat(data).to(torch.int16), "results": results, "generate": generate_run()}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
