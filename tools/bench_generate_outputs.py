"""The cost of recording scores and logits in generate (return_dict_in_generate=True, output_scores=True, output_logits=True),
on an H100.

    python tools/bench_generate_outputs.py [--specs valley-13b,valley2-7b] [--batches 1,4] [--new 256] [--reps 3]

Per spec (synthetic random-init weights, one 8-frame video per row, --new tokens, no eos) and batch, CUDA events around whole
requests, the two arms of each pair alternated and the median of --reps taken:
  greedy   plain (the persistent kernel's fused arg-max) vs recording (the decode step writes its logits, then
           sample_filter_kernel selects and writes the row's score and logit)
  beam     4 beams plain vs recording (beam_step_kernel also writes every beam row's log-probabilities and logits, and keeps
           the beam-index rows)
Reports ms per step for each arm, the difference, and whether the two arms returned the same ids.  Prints the card's name and
power limit."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from valley_b200 import synthetic as syn  # noqa: E402
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM  # noqa: E402


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def alternate(plain, record, reps):
    """(plain output, record output, median ms plain, median ms record), the arms alternated after one warm-up each"""
    plain()
    record()
    tp, tr = [], []
    for _ in range(reps):
        p, t = timed(plain)
        tp.append(t)
        r, t = timed(record)
        tr.append(t)
    return p, r, sorted(tp)[reps // 2], sorted(tr)[reps // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--specs", default="valley-13b,valley2-7b")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("gpu:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                 capture_output=True, text=True).stdout.strip())
    for name in a.specs.split(","):
        spec = syn.SPECS[name]
        m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
        m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0"))
        for k, v in syn.sentinel_ids(spec).items():
            setattr(m.get_model().vision_tower.config, k, v)
        for B in (int(x) for x in a.batches.split(",")):
            ids = syn.make_prompt_ids(spec, B, 8, 0).cuda()
            images = syn.make_pixels(B, 8, 0).half().cuda()
            S = ids.shape[1]
            rec = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
            for arm, kw in (("greedy", dict()), ("4-beam", dict(num_beams=4))):
                kw = dict(input_ids=ids, images=images, max_new_tokens=a.new, eos_token_id=None, **kw)
                p, r, tp, tr = alternate(lambda: m.generate(**kw), lambda: m.generate(**kw, **rec), a.reps)
                steps = len(r.scores)
                same = torch.equal(p, r.sequences)
                del r
                print(f"{name} B={B} {arm}: {steps} steps  plain {tp / steps:.3f} ms/step  recording {tr / steps:.3f} ms/step  "
                      f"difference {1000 * (tr - tp) / steps:+.1f} us/step ({100 * (tr / tp - 1):+.1f} %)  same ids: {same}  "
                      f"(prompt {S} tokens)")
                torch.cuda.empty_cache()
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
