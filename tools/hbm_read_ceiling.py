"""Plain streaming-read rate of this GPU's HBM: python tools/hbm_read_ceiling.py [--gb 4] [--reps 20]

Reads a multi-GB bf16 buffer (far larger than L2) with whole-tensor reductions and reports the best and median rate of each.
The decode step streams its weights once per step, so this read rate -- not the data-sheet figure -- is the ceiling its
achieved rate is judged against.  The buffer is read, never written; one small result per pass goes back to HBM."""
import argparse, json, statistics, subprocess
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--gb", type=float, default=4.0)
ap.add_argument("--reps", type=int, default=20)
a = ap.parse_args()
assert torch.cuda.is_available(), "needs a GPU"
n = int(a.gb * 1e9) // 2
x = torch.empty(n, dtype=torch.bfloat16, device="cuda").uniform_(-1, 1)
gpu = torch.cuda.get_device_name(0)
try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.max.mem", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=20).stdout.strip() or gpu
except Exception:
    pass
ops = {
    "sum(fp32 accumulate)": lambda: x.sum(dtype=torch.float32),
    "amax": lambda: x.amax(),
    "max of the int32 view": lambda: x.view(torch.int32).max(),
}
res = {}
for name, fn in ops.items():
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    best, med = n * 2 / min(ts) / 1e12, n * 2 / statistics.median(ts) / 1e12
    res[name] = {"best_TBps": round(best, 3), "median_TBps": round(med, 3)}
    print(f"{name:36s} best {best:.3f} TB/s  median {med:.3f} TB/s  ({n * 2 / 1e9:.1f} GB read per pass)")
print(json.dumps({"gpu": gpu, "bytes": n * 2, "read_TBps": res, "ceiling_TBps": max(r["best_TBps"] for r in res.values())}))
