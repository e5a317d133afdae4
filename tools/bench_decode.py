"""Steady-state decode timing (LLM only): python tools/bench_decode.py [--model valley2-7b] [--batch 1] [--steps 120] [--ctx 340]"""
import argparse, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from valley_b200 import synthetic as syn
from valley_b200._lib import check
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="valley2-7b")
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--steps", type=int, default=120)
a = ap.parse_args()
spec = syn.SPECS[a.model]
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0", vision=False))
ids = syn.make_prompt_ids(spec, a.batch, 8, 0).cuda()
cache = m.new_cache(a.batch)
_, _, _, emb, _ = m.prepare_inputs_labels_for_multimodal(ids, None, None, None, None)
_, nxt = m._prefill(cache, emb, 0)
out = torch.empty(a.batch, a.steps, dtype=torch.int64, device="cuda")
run = lambda n: check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), n, out.data_ptr(), 0))
run(8)
torch.cuda.synchronize()
best = 1e9
for rep in range(3):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(a.steps); e1.record(); torch.cuda.synchronize()
    best = min(best, e0.elapsed_time(e1) / a.steps)
S = cache.get_seq_length()
H, I, V, L = spec.hidden_size, spec.intermediate_size, spec.vocab_size, spec.num_hidden_layers
bytes_step = 2 * (L * (4 * H * H + 3 * H * I) + V * H) + a.batch * (S - a.steps // 2) * 2 * L * H * 2
print(f"{a.model} B={a.batch}: {best:.3f} ms/token  {a.batch / best * 1e3:.1f} tok/s  {bytes_step / best / 1e6:.0f} GB/s  "
      f"env V1={os.environ.get('VLY_DECODE_V1')} NO_PDL={os.environ.get('VLY_NO_PDL')}  tokens[0,:6]={out[0,:6].tolist()}")
if os.environ.get("VLY_MEGA_DBG"):
    import ctypes as C
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    buf = (C.c_longlong * (n_sm * 32))()
    rc = m._lib.vly_debug_mega_counters(buf, n_sm * 32)
    import numpy as np
    arr = np.array(buf[:]).reshape(n_sm, 32)
    names = ["grid sync", "stage x", "weight loop", "attention"]
    print("last step, cycle breakdown (mean over CTAs | min | max), SM clock cycles (~1.9 GHz):")
    for i, nme in enumerate(names):
        print(f"  {nme:24s} {arr[:, i].mean():12.0f} {arr[:, i].min():12d} {arr[:, i].max():12d}")
    print("  per phase type: stage-x | loop | trailing grid sync   (mean over CTAs, us at 1.9 GHz; [min..max] of loop)")
    for t, nme in enumerate(["QKV", "ATTN", "OPROJ", "GATEUP", "DOWN", "LOGITS"]):
        a = arr[:, 8 + 3 * t: 11 + 3 * t] / 1.9e3
        print(f"  {nme:8s} {a[:, 0].mean():9.1f} {a[:, 1].mean():9.1f} {a[:, 2].mean():9.1f}   [{a[:, 1].min():.1f} .. {a[:, 1].max():.1f}]")
