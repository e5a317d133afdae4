"""Stage-by-stage GPU diagnostics against the oracle (test infrastructure; prints metrics, never hides a failure).  Run each stage under `timeout`:
    timeout 180 python tests/diag_gpu.py gemm | vitattn | vit | splice | prefill | decode | e2e
"""
import ctypes as C
import os
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from valley_b200 import _lib, synthetic as syn  # noqa: E402
import helpers as Hh  # noqa: E402
from oracle import valley_oracle as O  # noqa: E402

torch.manual_seed(0)
dev = "cuda:0"


def bare_ctx(spec=syn.TINY):
    from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM
    return ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)


def stage_gemm():
    m = bare_ctx()
    lib = m._lib
    for (M, N, K, bn) in [(128, 128, 64, 128), (128, 256, 64, 256), (300, 512, 256, 128), (300, 512, 256, 256),
                          (1000, 1024, 640, 256), (257 * 6, 3072, 1024, 256), (77, 1032, 512, 128), (2056, 1024, 4096, 256)]:
        a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
        w = (torch.randn(N, K, device=dev) * 0.05).bfloat16()
        bias = torch.randn(N, device=dev)
        out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        _lib.check(lib.vly_test_gemm(m._ctx, a.data_ptr(), w.data_ptr(), M, N, K, 0, bias.data_ptr(), None, out.data_ptr(), bn,
                                     None, None, 0, 0.0, None, None, None, 0, 0, 0, None))
        torch.cuda.synchronize()
        ref = a.float() @ w.float().T + bias
        err = Hh.rel_fro(out, ref)
        bad = (out.float() - ref).abs().max().item()
        print(f"gemm M={M} N={N} K={K} bn={bn} epi=bias: rel_fro={err:.3e} max_abs={bad:.3e} {'OK' if err < 5e-3 else 'FAIL'}")
        if err >= 5e-3:
            d = (out.float() - ref).abs()
            rows = (d.max(dim=1).values > 0.1).nonzero().flatten()[:10].tolist()
            cols = (d.max(dim=0).values > 0.1).nonzero().flatten()[:10].tolist()
            print("   bad rows", rows, "bad cols", cols, " out[0,:8]", out[0, :8].float().tolist(), "ref", ref[0, :8].tolist())
        if N % 32 == 0:
            res = (torch.randn(M, N, device=dev)).bfloat16()
            out2 = res.clone()
            _lib.check(lib.vly_test_gemm(m._ctx, a.data_ptr(), w.data_ptr(), M, N, K, 3, bias.data_ptr(), out2.data_ptr(), out2.data_ptr(), bn,
                                         None, None, 0, 0.0, None, None, None, 0, 0, 0, None))
            torch.cuda.synchronize()
            ref2 = ref + res.float()
            err2 = Hh.rel_fro(out2, ref2)
            print(f"     epi=bias+residual(in place): rel_fro={err2:.3e} {'OK' if err2 < 5e-3 else 'FAIL'}")


def stage_vitattn():
    m = bare_ctx()
    for F in (1, 3, 20):
        qkv = (torch.randn(F * 257, 3072, device=dev)).bfloat16()
        out = torch.zeros(F * 257, 1024, device=dev, dtype=torch.bfloat16)
        _lib.check(m._lib.vly_test_vit_attention(m._ctx, qkv.data_ptr(), F, out.data_ptr(), 0))
        torch.cuda.synchronize()
        x = qkv.float().view(F, 257, 3, 16, 64)
        q, k, v = x[:, :, 0].transpose(1, 2), x[:, :, 1].transpose(1, 2), x[:, :, 2].transpose(1, 2)
        p = torch.softmax(q @ k.transpose(-1, -2) * 0.125, dim=-1)
        ref = (p @ v).transpose(1, 2).reshape(F * 257, 1024)
        err = Hh.rel_fro(out, ref)
        print(f"vit attention F={F}: rel_fro={err:.3e} {'OK' if err < 1e-2 else 'FAIL'}  nan={torch.isnan(out.float()).sum().item()}")
        if err >= 1e-2:
            d = (out.float() - ref).abs().view(F, 257, 16, 64)
            print("   per-row-tile err:", [d[:, a:b].max().item() for a, b in ((0, 128), (128, 256), (256, 257))],
                  " per-head err:", [round(d[:, :, h].max().item(), 3) for h in range(16)])


def stage_vit(spec=syn.TINY, F=6):
    sd = Hh.bf16_weights(spec, 0)
    m = Hh.build_model(spec, sd)
    px = syn.make_pixels(1, F, 0)[0]
    for sel in (0, 1, -2, -1):
        t0 = time.time()
        got = m._vit_encode(px.cuda(), sel)
        torch.cuda.synchronize()
        with torch.no_grad():
            ref = O.vit_hidden_state(sd, px, sel, num_layers=spec.vit_layers)
            ref_bf = O.vit_hidden_state({k: v.bfloat16() for k, v in sd.items()}, px.bfloat16(), sel, num_layers=spec.vit_layers)
        e, eb = Hh.rel_fro(got, ref), Hh.rel_fro(ref_bf, ref)
        print(f"vit hidden_states[{sel}] F={F}: ours-vs-fp32 {e:.3e}  torch-bf16-vs-fp32 {eb:.3e}  nan={torch.isnan(got.float()).sum().item()} "
              f"{'OK' if e < 2e-2 and e < max(1.5 * eb, 5e-3) else 'FAIL'}  ({time.time() - t0:.2f}s)")


def stage_splice(spec=syn.TINY):
    sd = Hh.bf16_weights(spec, 0)
    m = Hh.build_model(spec, sd)
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    B, T = 2, 3
    ids, px = syn.make_prompt_ids(spec, B, T, 0), syn.make_pixels(B, T, 0)
    enc = m.encode_images(px.cuda())
    with torch.no_grad():
        ref_enc = O.encode_images(sd, px, cfg.mm_vision_select_layer, num_layers=cfg.vit_layers)
        ref_emb = O.prepare_inputs_embeds(sd, ids, ref_enc, tok)
    print(f"encode_images: rel_fro={Hh.rel_fro(enc, ref_enc):.3e}")
    _, _, _, emb, _ = m.prepare_inputs_labels_for_multimodal(ids.cuda(), None, None, None, px.cuda())
    torch.cuda.synchronize()
    print(f"inputs_embeds after splice: rel_fro={Hh.rel_fro(emb, ref_emb):.3e}")
    text_rows = (ids[0] < spec.vocab_size - 6)
    print("   text rows exact:", torch.equal(emb[0][text_rows.cuda()].float().cpu(), ref_emb[0][text_rows].bfloat16().float()))


def stage_prefill(spec=syn.TINY):
    sd = Hh.bf16_weights(spec, 0)
    m = Hh.build_model(spec, sd)
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    B, T = 2, 3
    ids, px = syn.make_prompt_ids(spec, B, T, 0), syn.make_pixels(B, T, 0)
    with torch.no_grad():
        ref = O.causal_lm_forward(sd, cfg, tok, ids, px, None)
        ref_bf = O.causal_lm_forward({k: v.bfloat16() for k, v in sd.items()}, cfg, tok, ids, px.bfloat16(), None)
    # text-only first (isolates the decoder), then multimodal
    with torch.no_grad():
        ref_txt = O.causal_lm_forward(sd, cfg, tok, ids, None, None)
    out_txt = m(input_ids=ids.cuda())
    torch.cuda.synchronize()
    print(f"prefill logits (text only): rel_fro={Hh.rel_fro(out_txt.logits, ref_txt):.3e}  nan={torch.isnan(out_txt.logits).sum().item()}")
    out = m(input_ids=ids.cuda(), images=px.cuda())
    torch.cuda.synchronize()
    e, eb = Hh.rel_fro(out.logits, ref), Hh.rel_fro(ref_bf, ref)
    print(f"prefill logits (multimodal): ours-vs-fp32 {e:.3e}  torch-bf16-vs-fp32 {eb:.3e}  argmax agree "
          f"{(out.logits.argmax(-1).cpu() == ref.argmax(-1)).float().mean().item():.3f}  next_tokens {out.next_tokens.tolist()} ref {ref[:, -1].argmax(-1).tolist()}")
    k, v = out.past_key_values.to_hf(0)
    print("   kv len", out.past_key_values.get_seq_length(), "k finite", torch.isfinite(k.float()).all().item())


def stage_decode(spec=syn.TINY, n=12):
    sd = Hh.bf16_weights(spec, 0)
    m = Hh.build_model(spec, sd)
    cfg, tok = Hh.oracle_cfg(spec), Hh.oracle_tok(spec)
    B, T = 2, 3
    ids, px = syn.make_prompt_ids(spec, B, T, 0), syn.make_pixels(B, T, 0)
    with torch.no_grad():
        r_tok, r_log = O.greedy_generate(sd, cfg, tok, ids, px, n, return_logits=True)
    # teacher-forced: feed the oracle's tokens, compare each step's logits
    out = m(input_ids=ids.cuda(), images=px.cuda())
    cache = out.past_key_values
    errs, agree = [Hh.rel_fro(out.logits[:, -1], r_log[:, 0])], [(out.logits[:, -1].argmax(-1).cpu() == r_tok[:, 0]).all().item()]
    for i in range(1, n):
        o = m(input_ids=r_tok[:, i - 1:i].cuda(), past_key_values=cache)
        errs.append(Hh.rel_fro(o.logits[:, -1], r_log[:, i]))
        agree.append((o.next_tokens.cpu() == r_tok[:, i]).all().item())
    torch.cuda.synchronize()
    print("teacher-forced decode: rel_fro per step", [f"{e:.2e}" for e in errs])
    print("   argmax == oracle token per step", agree)
    top2 = r_log.topk(2, dim=-1).values
    print("   oracle top1-top2 margins", [f"{x:.3f}" for x in (top2[..., 0] - top2[..., 1]).min(0).values.tolist()])
    gen = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=n)
    torch.cuda.synchronize()
    print("free-running generate:", gen[:, -n:].tolist(), "\n               oracle:", r_tok.tolist())


def stage_e2e():
    import __graft_entry__ as g
    g.smoke()


if __name__ == "__main__":
    for st in sys.argv[1:]:
        print(f"===== stage {st} =====", flush=True)
        try:
            globals()["stage_" + st]()
        except Exception:
            traceback.print_exc()
        sys.stdout.flush()
