"""GPU (-m gpu): parity at the BASELINE.json configurations THEMSELVES -- full depth, real widths.

The tiny / one-layer tests prove the kernels; bf16 error grows with depth (every layer adds its own rounding to the residual
stream), so the stated bar is checked here at depth:  rel-Frobenius against the fp32 oracle <= 2e-2, or -- where 32-40 layers of
bf16 rounding exceed that for ANY bf16 implementation -- no worse than 1.5x the error of the same oracle run as eager torch-bf16
ops (which is what a user of the reference runs on a GPU); greedy ids exact wherever the oracle's top-1/top-2 margin exceeds 2x
the max logit error.  Measured numbers are printed (pytest -s) and recorded in BASELINE.md.  Checked on

    (a) ViT-L/14, all 24 layers loaded, ``select_layer=-2`` (23 executed) and ``-1`` (24), F = 8 frames       [configs 2-5]
    (b) valley2-7b  (Llama-2-7B shape, 32 layers), B = 1, 8 frames: prefill + 8 teacher-forced decode steps    [config 2]
    (c) valley-13b  (LLaMA-13B shape, 40 layers), B = 4, 8 frames each: prefill + 8 teacher-forced steps       [config 3]

against the SAME oracle (oracle/valley_oracle.py, pinned bit-exact to the live reference) evaluated in fp32 on the GPU with
TF32 disabled -- it is device-agnostic plain torch, and a 13B fp32 forward on the CPU would take minutes.  The weights are the
synthetic random-init tensors bench.py times (bf16-representable values, handed to both sides).
"""
import gc

import pytest
import torch

import helpers as Hh
from oracle import valley_oracle as O
from valley_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _true_fp32():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    gc.collect()
    torch.cuda.empty_cache()


class _Fp32View(dict):
    """bf16 tensors on the GPU, handed out as fp32 one access at a time: the fp32 oracle sees exactly the values of a bf16
    checkpoint without 4 bytes per parameter staying resident (the 13B model's 52 GB of fp32 weights do not fit an 80 GB GPU
    next to the packed model)."""

    def __getitem__(self, k):
        return dict.__getitem__(self, k).float()

    def get(self, k, default=None):
        return self[k] if k in self else default

    def items(self):
        return ((k, self[k]) for k in self.keys())

    def values(self):
        return (self[k] for k in self.keys())

    def bf16(self):
        return {k: dict.__getitem__(self, k) for k in self.keys()}


def _gpu_weights(spec, seed=0, **kw):
    """the weights as bf16 tensors on the GPU (what a bf16 checkpoint contains), read as fp32; one pass, no host copy"""
    return _Fp32View((k, v.bfloat16()) for k, v in syn.iter_state_dict(spec, seed, device="cuda", **kw))


def _build(spec, sd):
    m = Hh.build_model(spec, sd)
    torch.cuda.synchronize()
    return m


@pytest.mark.parametrize("sel", [-2, -1])
def test_vit_l14_full_depth_vs_fp32_oracle(sel):
    """CLIP ViT-L/14 at full depth on 8 frames: hidden_states[-2] (what Valley reads, 23 layers) and [-1] (24 layers)."""
    spec = syn.VALLEY2_7B
    assert spec.vit_layers == 24 and spec.vit_hidden == 1024
    sd = _gpu_weights(spec, 0, llm=False)
    m = _build(spec, sd)
    px = syn.make_pixels(1, 8, 3)[0].cuda()
    got = m._vit_encode(px.half(), sel)                                   # callers send fp16 pixels (valley_model.py:430)
    with torch.no_grad():
        ref = O.vit_hidden_state(sd, px.half().float(), sel, num_layers=24)
        ref_bf = O.vit_hidden_state(sd.bf16(), px.half().bfloat16(), sel, num_layers=24)
    e, eb = Hh.rel_fro(got, ref), Hh.rel_fro(ref_bf, ref)
    print(f"ViT-L/14 select {sel}: rel-Fro ours {e:.3e}, torch-bf16 {eb:.3e}, absmax ref {ref.abs().max().item():.2f}")
    assert torch.isfinite(got.float()).all()
    assert e <= 2e-2 and e <= max(1.5 * eb, 5e-3), (e, eb)
    # per-frame error is uniform (no frame / tile is special)
    per = ((got.float() - ref).flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1))
    assert float(per.max()) <= 2.5e-2, per.tolist()


def _llm_parity(spec, B, T, n_steps, seed=0):
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    sd = _gpu_weights(spec, seed)
    m = _build(spec, sd)
    ids, px = syn.make_prompt_ids(spec, B, T, seed), syn.make_pixels(B, T, seed, dtype=torch.float16)
    S = ids.shape[1]
    with torch.no_grad():
        r_tok, r_log = O.greedy_generate(sd, cfg, tok, ids.cuda(), px.float().cuda(), n_steps, return_logits=True)
        # the SAME oracle as eager torch-bf16 ops, teacher-forced with the fp32 oracle's tokens: the error any bf16 run has at this depth
        sd_bf = sd.bf16()
        cache_bf, bf_logs = O.KVCache(spec.num_hidden_layers), []
        for i in range(n_steps):
            cur = ids.cuda() if i == 0 else r_tok[:, i - 1:i]
            lg = O.causal_lm_forward(sd_bf, cfg, tok, cur, px.bfloat16().cuda() if i == 0 else None, cache_bf)
            bf_logs.append(lg[:, -1].float().cpu())
        probe_layers = (0, spec.num_hidden_layers // 2, spec.num_hidden_layers - 1)
        kv_bf = {l: (cache_bf.k[l][:, :, :S].float().cpu(), cache_bf.v[l][:, :, :S].float().cpu()) for l in probe_layers}
        del sd_bf, cache_bf
    bf_logs = torch.stack(bf_logs, 1)
    r_tok, r_log = r_tok.cpu(), r_log.cpu()
    errs_bf = [Hh.rel_fro(bf_logs[:, i], r_log[:, i]) for i in range(n_steps)]
    m.logits_all_positions = False                                         # last-position logits only ([B,S,V] fp32 is 170 MB at B = 4)
    out = m(input_ids=ids.cuda(), images=px.cuda())
    cache, logs = out.past_key_values, [out.logits[:, -1].cpu()]
    for i in range(1, n_steps):                                            # teacher-forced with the ORACLE's tokens, like model_worker.py:380-391
        o = m(input_ids=r_tok[:, i - 1:i].cuda(), past_key_values=cache,
              attention_mask=torch.ones(B, cache[0][0].shape[-2] + 1, device="cuda"))
        logs.append(o.logits[:, -1].cpu())
        assert cache.get_seq_length() == S + i
    logs = torch.stack(logs, 1)
    assert torch.isfinite(logs).all()
    errs = [Hh.rel_fro(logs[:, i], r_log[:, i]) for i in range(n_steps)]
    max_err = (logs - r_log).abs().max().item()
    top2 = r_log.topk(2, -1).values
    margin = top2[..., 0] - top2[..., 1]
    safe = margin > 2 * max_err
    print(f"{spec.name} B={B} S={S}: rel-Fro per step ours {['%.2e' % e for e in errs]}  torch-bf16 {['%.2e' % e for e in errs_bf]}, "
          f"max|d logit| {max_err:.3e}, logit std {r_log.std().item():.3f}, safe positions {int(safe.sum())}/{safe.numel()}")
    for e, eb in zip(errs, errs_bf):
        assert e <= max(2e-2, 1.5 * eb), (errs, errs_bf)
    assert torch.equal(logs.argmax(-1)[safe], r_tok[safe])
    # free-running device loop (CUDA-graph replay): identical to the oracle's ids up to the first near-tie of each row
    del cache, out
    gen = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=n_steps)[:, S:].cpu()
    agree = 0
    for b in range(B):
        for i in range(n_steps):
            if not safe[b, i]:
                break
            assert gen[b, i] == r_tok[b, i], (b, i, margin[b, i].item())
            agree += 1
    assert agree > 0 or not safe[:, 0].any()
    # KV cache after the prefill, first / middle / last layer, vs the oracle's cache
    c2 = O.KVCache(spec.num_hidden_layers)
    with torch.no_grad():
        O.causal_lm_forward(sd, cfg, tok, ids.cuda(), px.float().cuda(), c2)
    mine = m(input_ids=ids.cuda(), images=px.cuda()).past_key_values
    for layer in probe_layers:          # same bar as the logits: 2e-2, or 1.5x what torch-bf16 has at that depth
        k, v = mine.to_hf(layer)
        ek, ev = Hh.rel_fro(k, c2.k[layer]), Hh.rel_fro(v, c2.v[layer])
        bk, bv = Hh.rel_fro(kv_bf[layer][0], c2.k[layer]), Hh.rel_fro(kv_bf[layer][1], c2.v[layer])
        print(f"  KV cache layer {layer}: rel-Fro K ours {ek:.2e} / torch-bf16 {bk:.2e}, V ours {ev:.2e} / torch-bf16 {bv:.2e}")
        assert ek <= max(2e-2, 1.5 * bk) and ev <= max(2e-2, 1.5 * bv), (layer, ek, bk, ev, bv)
    return errs


def test_valley2_7b_full_depth_prefill_and_decode_vs_fp32_oracle():
    """BASELINE config 2: valley2-7b (32 layers), one 8-frame video, S = 333."""
    _llm_parity(syn.VALLEY2_7B, B=1, T=8, n_steps=9)


def test_valley_13b_b4_full_depth_prefill_and_decode_vs_fp32_oracle():
    """BASELINE config 3 (the metric's model): valley-13b (40 layers), 4 videos x 8 frames; the decode steps run
    decode_step_kernel<4> (tensor-core consumer), the prefill the 256-wide GEMM tiles at M = 1332."""
    free = torch.cuda.mem_get_info()[0]
    if free < 64e9:
        pytest.skip(f"needs ~60 GB of device memory for the bf16 oracle weights + the packed model (free: {free / 1e9:.0f} GB)")
    _llm_parity(syn.VALLEY_13B, B=4, T=8, n_steps=9)
