"""GPU: the persistent decode kernel's settings (DecodeSettings in api.cu: VLY_MEGA_*, VLY_ATTN_IKEYS) are read when a KV
cache is created and stay with that cache.  Those tested here change only scheduling -- the L2 eviction hint on the weight
stream, the ring depth, the bytes of copies in flight, and (VLY_NO_GRAPH) eager launches instead of graph replays -- never
what is computed: logits, greedy, sampled and beam token ids and beam scores must be equal bit for bit to those of the
reference configuration.  Each configuration runs in a subprocess of its own on the same seeded weights and prompt; one
in-process test checks that a cache keeps its settings when the environment changes."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from valley_b200 import synthetic as syn
from valley_b200._lib import check
from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM
spec_name, B, S, out_path = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), sys.argv[5]
spec = syn.SPECS[spec_name]
m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
m.load_state_dict(syn.iter_state_dict(spec, 1, device="cuda:0", vision=False))
m.logits_all_positions = False
g = torch.Generator().manual_seed(7)
ids = torch.randint(8, min(spec.vocab_size, 32000) - 16, (B, S), generator=g)
with torch.no_grad():
    out = m(input_ids=ids.cuda())
    cache, logs, tok = out.past_key_values, [out.logits[:, -1].float().cpu()], []
    for i in range(6):                     # single decode steps: logits of every step
        t = logs[-1].argmax(-1, keepdim=True)
        tok.append(t)
        o = m(input_ids=t.cuda(), past_key_values=cache)
        logs.append(o.logits[:, -1].float().cpu())
    nxt = logs[-1].argmax(-1).cuda().contiguous()
    n = 40                                 # then free-running greedy steps (graph replays)
    gen = torch.empty(B, n, dtype=torch.int64, device="cuda")
    check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), n, gen.data_ptr(), 0))
    torch.cuda.synchronize()
    seq_len = cache.get_seq_length()
    # seeded sampling through a top-k filter, then a 2-beam search on the device: 11 steps each after the first token,
    # one 8-step graph and three 1-step graphs
    torch.manual_seed(11)
    sampled = m.generate(input_ids=ids.cuda(), max_new_tokens=12, do_sample=True, temperature=0.8, top_k=20, eos_token_id=None)
    beam = m.generate(input_ids=ids[:max(B // 2, 1)].cuda(), max_new_tokens=12, num_beams=2, eos_token_id=None)
    beam_scores = m.last_beam_scores
np.savez(out_path, logits=torch.stack(logs, 1).numpy(), tokens=torch.cat(tok, 1).numpy(), gen=gen.cpu().numpy(),
         seq_len=np.array([seq_len]), sampled=sampled.cpu().numpy(), beam=beam.cpu().numpy(),
         beam_scores=beam_scores.float().cpu().numpy())
"""

# the plain ring (no hint) first: the reference of the others
CONFIGS = {
    "all off": {"VLY_MEGA_L2_HINT": "0"},
    "defaults": {},
    "2 stages": {"VLY_MEGA_STAGES": "2"},
    "64 KB in flight": {"VLY_MEGA_INFLIGHT_KB": "64"},
    "eager": {"VLY_NO_GRAPH": "1"},
}
SETTINGS = ("VLY_MEGA_STAGE_KB", "VLY_MEGA_ROWS", "VLY_MEGA_INFLIGHT_KB", "VLY_MEGA_STAGES", "VLY_MEGA_INFLIGHT", "VLY_ATTN_IKEYS",
            "VLY_MEGA_L2_HINT", "VLY_MEGA_DBG")


def _run(tmp_path, spec_name, B, S, name, env_over):
    env = dict(os.environ)
    for k in SETTINGS + ("VLY_LIB_PATH", "VLY_NO_GRAPH"):
        env.pop(k, None)
    env.update(env_over)
    out = str(tmp_path / f"{spec_name}_{B}_{name.replace(' ', '_').replace('/', '')}.npz")
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, spec_name, str(B), str(S), out], env=env, capture_output=True,
                       text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, f"{name}: " + r.stdout[-2000:] + r.stderr[-3000:]
    return np.load(out)


@pytest.mark.parametrize("spec_name,B,S", [("shape-13b-1l", 4, 560), ("tiny-umma-ragged", 2, 300), ("tiny-umma-ragged", 4, 300)])
def test_decode_ring_options_are_bit_identical(tmp_path, spec_name, B, S):
    """shape-13b-1l at B = 4 ends at ~610 keys: 40 heads x 4 sequences of multi-pass attention items; tiny-umma-ragged has a
    down-projection K that is not a multiple of the ring stage width."""
    ref = _run(tmp_path, spec_name, B, S, "all off", CONFIGS["all off"])
    assert np.isfinite(ref["logits"]).all()
    assert int(ref["seq_len"][0]) == S + 6 + 40
    for name, env in CONFIGS.items():
        if name == "all off":
            continue
        got = _run(tmp_path, spec_name, B, S, name, env)
        assert np.array_equal(got["logits"].view(np.uint32), ref["logits"].view(np.uint32)), f"{spec_name} B={B}: logits differ with {name}"
        assert np.array_equal(got["tokens"], ref["tokens"]), f"{spec_name} B={B}: token ids differ with {name}"
        assert np.array_equal(got["gen"], ref["gen"]), f"{spec_name} B={B}: generated ids differ with {name}"
        assert np.array_equal(got["sampled"], ref["sampled"]), f"{spec_name} B={B}: sampled ids differ with {name}"
        assert np.array_equal(got["beam"], ref["beam"]), f"{spec_name} B={B}: beam ids differ with {name}"
        assert np.array_equal(got["beam_scores"].view(np.uint32), ref["beam_scores"].view(np.uint32)), \
            f"{spec_name} B={B}: beam scores differ with {name}"


def test_decode_settings_are_fixed_per_cache(monkeypatch):
    """One model, one process: a ring depth below 2 makes creating a cache fail; a cache created without the setting keeps
    decoding the same tokens after the variable is set."""
    import torch
    from valley_b200 import synthetic as syn
    from valley_b200._lib import check
    from valley_b200.model import ValleyConfig, ValleyLlamaForCausalLM
    for k in SETTINGS:
        monkeypatch.delenv(k, raising=False)
    spec, B, n = syn.SPECS["tiny-umma-ragged"], 2, 24
    m = ValleyLlamaForCausalLM(ValleyConfig.from_spec(spec), 0)
    m.load_state_dict(syn.iter_state_dict(spec, 1, device="cuda:0", vision=False))
    m.logits_all_positions = False
    ids = torch.randint(8, min(spec.vocab_size, 32000) - 16, (B, 40), generator=torch.Generator().manual_seed(7)).cuda()

    monkeypatch.setenv("VLY_MEGA_STAGES", "1")
    with pytest.raises(ValueError, match="weight ring"):
        m.new_cache(B, 256)
    monkeypatch.delenv("VLY_MEGA_STAGES")
    cache = m.new_cache(B, 384)

    def prefill_and_generate():
        cache.reset()
        with torch.no_grad():
            nxt = m(input_ids=ids, past_key_values=cache).logits[:, -1].argmax(-1).contiguous()
        gen = torch.empty(B, n, dtype=torch.int64, device="cuda")
        check(m._lib.vly_generate_greedy(m._ctx, cache._h, nxt.data_ptr(), n, gen.data_ptr(), 0))
        torch.cuda.synchronize()
        return gen.cpu()

    first = prefill_and_generate()
    monkeypatch.setenv("VLY_MEGA_STAGES", "1")
    assert torch.equal(prefill_and_generate(), first)
