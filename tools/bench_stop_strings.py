"""completion()-shaped requests with the '###' keyword: the host-visible loop against the device route, on an H100.

    python tools/bench_stop_strings.py [--specs valley-13b,valley2-7b] [--new 256] [--hit 200] [--reps 3]

Per spec (synthetic random-init weights, B = 1, 8 frames, greedy, --new tokens), CUDA events around whole requests:
  host     generate(stopping_criteria=[KeywordsStoppingCriteria(['###'])]): one decode, one sync and one batch_decode per token
  device   the route completion() takes (_keyword_generate): the keyword as a stop string matched in sample_filter_kernel
each with the keyword never hit and with the keyword on the token of step --hit (the reply ends where that token first occurs); and the plain greedy request (no keyword, STEP_TOKEN graphs), whose
difference to the device route's never-hit time, per token, is the cost of sample_filter_kernel + the matcher per step.
The tokenizer is a word tokenizer over the model's ids; the keyword is placed by mapping one token of the greedy continuation
to ' ###'.  Prints the card's name and power limit."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from valley_b200 import synthetic as syn  # noqa: E402
from valley_b200.model import KeywordsStoppingCriteria, ValleyConfig, ValleyLlamaForCausalLM  # noqa: E402


class Tok:
    """token i reads ' w<i>' (``keyword_id``: ' ###'); ids 0-2 are special; the static-prefix token is id V"""
    eos_token_id = 2

    def __init__(self, V, keyword_id=None):
        self.V, self.kw = V, keyword_id

    def text(self, i):
        return {0: "<unk>", 1: "<s>", 2: "</s>"}.get(i) or (" ###" if i == self.kw else f" w{i}")

    def get_vocab(self):
        return {f"t{i}": i for i in range(self.V + 1)}

    def __len__(self):
        return self.V + 1

    def __call__(self, text, add_special_tokens=True):
        return {"input_ids": [self.V]}

    def convert_ids_to_tokens(self, ids):
        return [f"t{i}" for i in ids]

    def convert_tokens_to_string(self, toks):
        return "".join("abcdef" if t == f"t{self.V}" else self.text(int(t[1:])) for t in toks)

    def decode(self, ids, skip_special_tokens=True):
        return "".join("" if int(i) in (0, 1, 2) else self.text(int(i)) for i in ids)

    def batch_decode(self, rows, skip_special_tokens=True):
        return [self.decode(r.tolist() if torch.is_tensor(r) else r) for r in rows]


def timed(fn, reps):
    out, ms = None, []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, sorted(ms)[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--specs", default="valley-13b,valley2-7b")
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--hit", type=int, default=200)
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
        ids = syn.make_prompt_ids(spec, 1, 8, 0).cuda()
        images = syn.make_pixels(1, 8, 0).half().cuda()
        V, S = spec.vocab_size, ids.shape[1]
        kw = dict(max_new_tokens=a.new, do_sample=False, eos_token_id=None)
        plain, t_plain = timed(lambda: m.generate(input_ids=ids, images=images, **kw), a.reps)
        print(f"{name}: plain greedy {t_plain:.1f} ms / {a.new} tokens")
        for case, kid in (("never", None), (f"on the token of step {a.hit}", int(plain[0, S + a.hit - 1]))):
            tok = Tok(V, kid)
            host, t_host = timed(lambda: m.generate(input_ids=ids, images=images, stopping_criteria=[
                KeywordsStoppingCriteria(["###"], tok, ids)], **kw), a.reps)
            dev, t_dev = timed(lambda: m._keyword_generate(ids, images, KeywordsStoppingCriteria(["###"], tok, ids), kw),
                               a.reps)
            n = host.shape[1] - S
            print(f"  keyword {case}: ends after {n} tokens  host loop {t_host:.1f} ms  device route {t_dev:.1f} ms  "
                  f"gain {100 * (t_host / t_dev - 1):.1f} %  same ids: {torch.equal(host, dev)}")
            if kid is None:
                print(f"  per step: device route - plain greedy = {1000 * (t_dev - t_plain) / a.new:.1f} us")
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
