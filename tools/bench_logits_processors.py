"""The cost of generate()'s logits processors (repetition_penalty, no_repeat_ngram_size, min_new_tokens) on an H100.

    python tools/bench_logits_processors.py [--spec valley-13b] [--batches 4,8] [--new 256] [--reps 3]

The bench configuration: synthetic random-init weights, one 8-frame video per row, --new greedy tokens.  Per batch, CUDA
events around whole requests, alternated in one process and the median of --reps taken:
  plain       generate() with no processors (eos set, so that both arms select with the same eos bookkeeping)
  processors  repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=16
Reports ms per decode step for each arm and the difference, then, from a torch.profiler run of one processor request of its
own, sample_filter_kernel's launches per step and mean time.  Prints the card's name and power limit."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from valley_b200 import synthetic as syn  # noqa: E402
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM  # noqa: E402

PROCS = dict(repetition_penalty=1.1, no_repeat_ngram_size=3, min_new_tokens=16)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def alternate(plain, procs, reps):
    plain()
    procs()
    tp, tq = [], []
    for _ in range(reps):
        p, t = timed(plain)
        tp.append(t)
        q, t = timed(procs)
        tq.append(t)
    return p, q, sorted(tp)[reps // 2], sorted(tq)[reps // 2]


def filter_kernel_time(fn):
    """(launches, mean us) of sample_filter_kernel in one run of fn, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    n, total = 0, 0.0
    for ev in prof.events():
        if "sample_filter_kernel" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
            n += 1
            total += ev.device_time
    return n, (total / n if n else float("nan"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spec", default="valley-13b")
    ap.add_argument("--batches", default="4,8")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("gpu:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                 capture_output=True, text=True).stdout.strip())
    spec = syn.SPECS[a.spec]
    m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
    m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0"))
    for k, v in syn.sentinel_ids(spec).items():
        setattr(m.get_model().vision_tower.config, k, v)
    for B in (int(x) for x in a.batches.split(",")):
        ids = syn.make_prompt_ids(spec, B, 8, 0).cuda()
        images = syn.make_pixels(B, 8, 0).half().cuda()
        # eos: a token no row emits (the last id), so that every request runs all its steps
        kw = dict(input_ids=ids, images=images, max_new_tokens=a.new, eos_token_id=spec.vocab_size - 1, pad_token_id=0)
        p, q, tp, tq = alternate(lambda: m.generate(**kw), lambda: m.generate(**kw, **PROCS), a.reps)
        steps = q.shape[1] - ids.shape[1]
        n, us = filter_kernel_time(lambda: m.generate(**kw, **PROCS))
        print(f"{a.spec} B={B}: {steps} steps  plain {tp / steps:.3f} ms/step  processors {tq / steps:.3f} ms/step  "
              f"difference {1000 * (tq - tp) / steps:+.1f} us/step ({100 * (tq / tp - 1):+.1f} %)  "
              f"same length: {p.shape == q.shape}  ids differ: {not torch.equal(p, q) if p.shape == q.shape else True}  "
              f"sample_filter_kernel: {n} launches ({n / steps:.2f} per step), {us:.1f} us each  (prompt {ids.shape[1]} tokens)")
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
