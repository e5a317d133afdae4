"""Steady-state decode timing (LLM only): python tools/bench_decode.py [--model valley2-7b] [--batch 1] [--steps 120]

--configs 'A=1,B=2;A=0' times several settings of the persistent decode kernel's overrides (VLY_MEGA_*, VLY_ATTN_IKEYS) in
one process (the weights are loaded once).  The library reads them when a KV cache is created and the cache keeps them, so
every configuration gets a KV cache of its own, created with its variables set, and the configurations are timed
round-robin for --rounds rounds.  '' (an empty configuration) is the library's defaults.  With VLY_MEGA_DBG=1 each
configuration's cycle counters are read from its own cache.

--sampling 'greedy;0.7;0.7,50;0.7,50,0.9' times token selection settings the same way: 'greedy', or 'T[,top_k[,top_p]]'
(temperature sampling, with HF generate's top-k / top-p filters).  Every configuration is timed with every setting."""
import argparse, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from valley_b200 import synthetic as syn
from valley_b200._lib import VlySampling, check
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM

ap = argparse.ArgumentParser()
ap.add_argument("--model", default="valley2-7b")
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--steps", type=int, default=120)
ap.add_argument("--configs", default=None, help="';'-separated list of 'VAR=value,VAR=value' environment settings")
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--sampling", default=None, help="';'-separated list of 'greedy' or 'T[,top_k[,top_p]]'")
a = ap.parse_args()
spec = syn.SPECS[a.model]
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 0, device="cuda:0", vision=False))
ids = syn.make_prompt_ids(spec, a.batch, 8, 0).cuda()
_, _, _, emb, _ = m.prepare_inputs_labels_for_multimodal(ids, None, None, None, None)
H, I, V, L = spec.hidden_size, spec.intermediate_size, spec.vocab_size, spec.num_hidden_layers
n_sm = torch.cuda.get_device_properties(0).multi_processor_count
try:   # the card and its power limit belong beside every number this prints
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=20).stdout.strip()
    print("gpu:", q)
except Exception:
    pass


def parse(cfg):
    env = {}
    for kv in filter(None, cfg.split(",")):
        k, v = kv.split("=", 1)
        env[k.strip()] = v.strip()
    return env


def parse_sampling(text):
    """'greedy' -> None; 'T[,top_k[,top_p]]' -> VlySampling (fixed seed, no stop token)"""
    if text.strip() == "greedy":
        return None
    f = text.split(",")
    return VlySampling(float(f[0]), 1234, -1, 0, -1, int(f[1]) if len(f) > 1 else 0, float(f[2]) if len(f) > 2 else 1.0)


configs = [(c, s) for c in ([""] if a.configs is None else a.configs.split(";"))
           for s in (["greedy"] if a.sampling is None else a.sampling.split(";"))]
base_env = dict(os.environ)


def run_config(ci, cfg_samp):
    """one timed run of configuration ci: fresh prefill, 8 warm-up steps, a.steps timed steps (ms per step)"""
    import ctypes as C
    cfg, samp = cfg_samp
    sp = parse_sampling(samp)
    os.environ.clear()
    os.environ.update(base_env)
    os.environ.update(parse(cfg))
    # a distinct capacity per configuration: cache handles are pooled by (batch, capacity), so each configuration keeps
    # the handle (and the settings) it was created with
    cache = m.new_cache(a.batch, ids.shape[1] + a.steps + 160 + 128 * ci)
    _, nxt = m._prefill(cache, emb, 0)
    out = torch.empty(a.batch, a.steps, dtype=torch.int64, device="cuda")
    if sp is None:
        run = lambda n: check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), n, out.data_ptr(), 0))
    else:
        run = lambda n: check(m._lib.vly_generate(m._ctx, cache._h, nxt.data_ptr(), n, out.data_ptr(), C.byref(sp), None, 0))
    run(8)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); run(a.steps); e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    S = cache.get_seq_length()
    return ms, S, out[0, :6].tolist(), counters(cache)


def counters(cache):
    """the cycle counters of cache's last decode step, or None (the cache was not created with VLY_MEGA_DBG set, or B > 4)"""
    import ctypes as C
    import numpy as np
    buf = (C.c_longlong * (n_sm * 32))()
    if m._lib.vly_kv_debug_counters(cache._h, buf, n_sm * 32) != 0:
        return None
    return np.array(buf[:]).reshape(n_sm, 32)


def print_counters(arr, ms_step):
    names = ["grid sync", "stage x", "weight loop", "attention"]
    # a power-capped card runs below its maximum SM clock: convert cycles at the clock the counters imply for one step
    clk_mhz = arr[:, :4].sum(1).mean() / (ms_step * 1e3)
    print(f"  last step, cycle breakdown (mean over CTAs | min | max), SM clock cycles; us below at the implied {clk_mhz / 1e3:.2f} GHz:")
    for i, nme in enumerate(names):
        print(f"    {nme:24s} {arr[:, i].mean():12.0f} {arr[:, i].min():12d} {arr[:, i].max():12d}")
    print("    per phase type: stage-x | loop | trailing grid sync | producer blocked on a full ring (mean over CTAs, us; [min..max] of loop)")
    tot = [0.0] * 4
    for t, nme in enumerate(["QKV", "ATTN", "OPROJ", "GATEUP", "DOWN", "LOGITS"]):
        c = arr[:, 8 + 3 * t: 11 + 3 * t] / clk_mhz
        blk = arr[:, 26 + t] / clk_mhz
        vals = [c[:, 0].mean(), c[:, 1].mean(), c[:, 2].mean(), blk.mean()]
        tot = [x + y for x, y in zip(tot, vals)]
        print(f"    {nme:8s} {vals[0]:9.1f} {vals[1]:9.1f} {vals[2]:9.1f} {vals[3]:9.1f}   [{c[:, 1].min():.1f} .. {c[:, 1].max():.1f}]")
    print(f"    {'total':8s} {tot[0]:9.1f} {tot[1]:9.1f} {tot[2]:9.1f} {tot[3]:9.1f}")


res = {i: [] for i in range(len(configs))}
for rnd in range(a.rounds):
    for ci, cfg in enumerate(configs):
        ms, S, toks, arr = run_config(ci, cfg)
        res[ci].append(ms)
        if rnd == a.rounds - 1:
            res[ci] = (res[ci], S, toks, arr)
os.environ.clear()
os.environ.update(base_env)
for ci, (cfg, samp) in enumerate(configs):
    times, S, toks, arr = res[ci]
    med = statistics.median(times)
    bytes_step = 2 * (L * (4 * H * H + 3 * H * I) + V * H) + a.batch * (S - a.steps // 2) * 2 * L * H * 2
    print(f"{a.model} B={a.batch} [{cfg or 'defaults'}] [{samp}]: median {med:.3f} ms/token  (min {min(times):.3f}, max {max(times):.3f}, "
          f"{len(times)} runs)  {a.batch / med * 1e3:.1f} tok/s  {bytes_step / med / 1e6:.0f} GB/s  tokens[0,:6]={toks}  "
          f"lib={os.environ.get('VLY_LIB_PATH', 'default')}")
    if arr is not None:
        print_counters(arr, med)
