"""ViT encode timing: python tools/bench_vit.py [--frames 8 64 256]"""
import argparse, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from valley_b200 import synthetic as syn
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM
ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, nargs="+", default=[8, 64, 256])
a = ap.parse_args()
spec = syn.VALLEY2_7B
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0", llm=False))
for F in a.frames:
    px = syn.make_pixels(1, F, 1, dtype=torch.float16)[0].cuda()
    for _ in range(3): m.encode_frames(px)
    torch.cuda.synchronize()
    best = 1e9
    for rep in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); out = m.encode_frames(px); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    print(f"ViT-L/14 F={F}: {best:.3f} ms  {F / best * 1e3:.0f} frames/s  {F / best * 1e3 * 155.29 / 1e3:.0f} TFLOP/s  nan={int(torch.isnan(out.float()).sum())}")
