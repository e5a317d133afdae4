"""Device time of the top-k / top-p selection kernel alone: python tools/bench_sample_filter.py [--vocab 32008] [--batch 1,4,64]

Runs sample_filter_kernel through vly_test_sample_filter (the same routine the decode loop selects with) on [B, V] fp32 logits
and reads its time per launch from torch.profiler's CUDA activity (so the host-side copy of the settings is not counted).
--settings 'T,top_k,top_p;...' (top_k 0 / top_p 1 = off)."""
import argparse, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import ProfilerActivity, profile
from valley_b200 import synthetic as syn
from valley_b200._lib import check
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM

ap = argparse.ArgumentParser()
ap.add_argument("--vocab", type=int, default=32008)
ap.add_argument("--batch", default="1,4,64")
ap.add_argument("--settings", default="0.7,50,1;0.7,0,0.9;0.7,50,0.9;0.7,32008,1")
ap.add_argument("--launches", type=int, default=200)
a = ap.parse_args()
print("gpu:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True).stdout.strip())
spec = syn.SPECS["tiny"]                     # any context will do: the hook takes V from its arguments
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0", vision=False))
V = a.vocab
for B in map(int, a.batch.split(",")):
    logits = torch.randn(B, V, generator=torch.Generator().manual_seed(B)).mul(2.0).cuda()
    keep = torch.empty(B, V, dtype=torch.uint8, device="cuda")
    for st in a.settings.split(";"):
        t, k, p = st.split(",")
        call = lambda: check(m._lib.vly_test_sample_filter(m._ctx, logits.data_ptr(), B, V, float(t), int(k), float(p),
                                                           keep.data_ptr(), 0))
        for _ in range(20):
            call()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.launches):
                call()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "sample_filter_kernel" in e.key]
        n = sum(e.count for e in ev)
        us = sum(e.device_time_total for e in ev) / max(n, 1)
        print(f"B={B:3d} V={V} T={t} top_k={k} top_p={p}: {us:8.1f} us per launch ({n} launches), "
              f"kept/row {keep.sum(1).float().mean().item():.1f}")
