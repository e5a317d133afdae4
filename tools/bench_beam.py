"""Cost of beam search on the device (LLM only): python tools/bench_beam.py [--model valley-13b] [--beams 4] [--new 256]

One video x 8 frames (the prompt's shape; the vision part is not timed), num_beams beams, --new generated tokens with no stop
token, so every step runs.  Prints, with the card's name and power limit read in the same process:
  * ms per step of vly_beam_search next to vly_generate_greedy at B = num_beams rows (the same decode step without the beam
    kernels), CUDA events around whole requests, alternated for --rounds rounds (medians);
  * torch.profiler device times of beam_step_kernel and kv_beam_reorder_kernel in one request (separate run);
  * the stand-alone reorder (every row takes another parent) over 64 / 256 / 1024 generated positions, CUDA events over
    --iters launches, with the bytes it moves computed from the shapes."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from valley_b200 import synthetic as syn  # noqa: E402
from valley_b200._lib import VlyBeam, check  # noqa: E402
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="valley-13b")
ap.add_argument("--beams", type=int, default=4)
ap.add_argument("--new", type=int, default=256)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=20)
a = ap.parse_args()
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True, timeout=30).stdout.strip()
print("gpu:", gpu)
spec = syn.SPECS[a.model]
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0", vision=False))
nb, n_new = a.beams, a.new
ids = syn.make_prompt_ids(spec, 1, 8, 0).cuda()
S = ids.shape[1]
emb = m.prepare_inputs_labels_for_multimodal(ids)[3].expand(nb, -1, -1).contiguous()
st = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
cache = m.new_cache(nb, S + 1024 + 8)
seq = torch.empty(1, n_new, dtype=torch.int64, device="cuda")
scores = torch.empty(1, dtype=torch.float32, device="cuda")
lens = torch.empty(1, dtype=torch.int32, device="cuda")
greedy_out = torch.empty(nb, n_new, dtype=torch.int64, device="cuda")


def prefill():
    cache.reset()
    logits, nxt = m._prefill(cache, emb, 1)
    return logits[:, -1].contiguous(), nxt


def beam():
    logits, _ = prefill()
    bp = VlyBeam(nb, 1, 1.0, 0, -1, 0)
    check(m._lib.vly_beam_search(m._ctx, cache._h, C.byref(bp), logits.data_ptr(), S, n_new, seq.data_ptr(), scores.data_ptr(),
                                 lens.data_ptr(), st()))


def greedy():
    _, nxt = prefill()
    check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), n_new - 1, greedy_out.data_ptr(), st()))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    _, nxt = prefill()          # (the prefill is outside the window: time it alone and subtract)
    torch.cuda.synchronize()
    e0.record()
    prefill()
    e1.record()
    torch.cuda.synchronize()
    t_prefill = e0.elapsed_time(e1)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return (e0.elapsed_time(e1) - t_prefill) / (n_new - 1)


beam(); greedy()                # warm-up: graph captures
torch.cuda.synchronize()
t_beam, t_greedy = [], []
for _ in range(a.rounds):
    t_beam.append(timed(beam))
    t_greedy.append(timed(greedy))
res = {"gpu": gpu, "model": a.model, "beams": nb, "new_tokens": n_new, "prompt_len": S,
       "beam_ms_per_step": statistics.median(t_beam), "greedy_ms_per_step_B%d" % nb: statistics.median(t_greedy)}

from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    beam()
    torch.cuda.synchronize()
for ev in prof.key_averages():
    for k in ("beam_step_kernel", "kv_beam_reorder_kernel"):
        if k in ev.key:
            res[k + "_us_mean"] = ev.device_time_total / max(ev.count, 1)   # (device_time_total is in us)
            res[k + "_count"] = ev.count

# the reorder alone after g generated positions: every row takes another parent
parent = torch.tensor([1, 2, 3, 0][:nb] if nb == 4 else [(i + 1) % nb for i in range(nb)], dtype=torch.int32, device="cuda")
g_ids = torch.randint(3, spec.vocab_size - 8, (nb, 1024), generator=torch.Generator().manual_seed(1)).cuda()
tail = m.prepare_inputs_labels_for_multimodal(g_ids)[3]
L, nH = spec.num_hidden_layers, spec.num_attention_heads
for g in (64, 256, 1024):
    cache.reset()
    m._prefill(cache, torch.cat([emb, tail[:, :g]], 1).contiguous(), 0)
    check(m._lib.vly_kv_beam_reorder(m._ctx, cache._h, parent.data_ptr(), S, st()))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(a.iters):
        check(m._lib.vly_kv_beam_reorder(m._ctx, cache._h, parent.data_ptr(), S, st()))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    moved = 2 * nb * g * 2 * L * nH * 128 * 2        # read once + written once, every row changes
    res[f"reorder_ms_{g}"] = ms
    res[f"reorder_GBps_{g}"] = moved / ms / 1e6
print(json.dumps(res))
