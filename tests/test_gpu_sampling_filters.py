"""top-k / top-p (nucleus) filtering of the sampled distribution, as HF generate's TopKLogitsWarper / TopPLogitsWarper apply it
after the temperature.  Pinned against transformers' own warpers (tests/golden/ref_sampling_filters.pt, written by
oracle/make_golden_sampling_filters.py); the device selection (sample_filter_kernel) is checked against those masks, for the
distribution it draws, and for drawing the same token on every decode path (first token, persistent kernel, per-op kernels)."""
import ctypes as C
import os

import pytest
import torch

import helpers as Hh
from oracle import make_golden_sampling_filters as G
from valley_b200 import synthetic as syn
from valley_b200._lib import VlySampling, check
from valley_b200.model import filter_scores, sampling_filters

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_sampling_filters.pt")
_models = {}


def get(spec_name):
    if spec_name not in _models:
        spec = syn.SPECS[spec_name]
        _models[spec_name] = (spec, Hh.build_model(spec, Hh.bf16_weights(spec, 0)))
    return _models[spec_name]


def _golden():
    return G.load_masks(torch.load(GOLD))


def test_torch_filter_reproduces_the_hf_warper_masks():
    """The host-loop helper (model.filter_scores after sampling_filters) keeps exactly what transformers' warpers keep."""
    for V, name, z, i, (t, k, p), want in _golden():
        kk, pp = sampling_filters(k, p)
        got = torch.isfinite(filter_scores(z[None] / t, kk, pp))[0]
        assert torch.equal(got, want), (V, name, t, k, p)


def test_sampling_filter_arguments_follow_hf():
    assert sampling_filters(None, None) == (0, 1.0) and sampling_filters(0, 1.0) == (0, 1.0)
    assert sampling_filters(50, 0.9) == (50, 0.9) and sampling_filters(None, 0.0) == (1, 1.0) and sampling_filters(7, 0) == (1, 1.0)
    with pytest.raises(ValueError, match="`top_k` has to be a strictly positive integer, but is -1"):
        sampling_filters(-1, None)
    with pytest.raises(ValueError, match="`top_k` has to be a strictly positive integer"):
        sampling_filters(2.5, None)
    for bad in (1.5, -0.1):
        with pytest.raises(ValueError, match=f"`top_p` has to be a float > 0 and < 1, but is {bad}"):
            sampling_filters(None, bad)


def _mass_band(z, t, k, p, tol=1e-5):
    """tokens whose float64 softmax mass strictly above them lies within tol * W of top_p * W (among the top-k survivors)"""
    s = (z / t).double()
    if k:
        s = s.masked_fill(s < torch.topk(s, min(k, s.numel()))[0][-1], -float("inf"))
    w = torch.exp(s - s.max())
    W = float(w.sum())
    srt, idx = torch.sort(s, descending=True)
    ws = w[idx]
    inc = torch.cumsum(ws, 0)
    first = torch.searchsorted(-srt, -srt, side="left")          # first sorted position of each token's tie group
    above_sorted = torch.where(first > 0, inc[(first - 1).clamp(min=0)], torch.zeros_like(inc))
    above = torch.empty_like(above_sorted)
    above[idx] = above_sorted
    return (above - p * W).abs() <= tol * W


def _device_mask(m, z, t, k, p):
    B, V = z.shape
    keep = torch.zeros(B, V, dtype=torch.uint8, device="cuda")
    zz = z.cuda().contiguous()
    check(m._lib.vly_test_sample_filter(m._ctx, zz.data_ptr(), B, V, float(t), int(k or 0), float(1.0 if p is None else p),
                                        keep.data_ptr(), None))
    return keep.bool().cpu()


def _check_against(got, want, z, t, k, p, tie_row):
    """top-k exact; top-p exact away from the fp32 summation boundary; a tie group straddling the cut is kept whole"""
    if p is None:
        assert torch.equal(got, want)
        return
    diff = got != want
    if tie_row:
        kept_min = (z / t)[want].min()
        group = (z / t) == kept_min
        diff &= ~(got & group)
    diff &= ~_mass_band(z, t, k, p)
    assert not bool(diff.any()), int(diff.sum())


@pytest.mark.gpu
def test_device_filter_matches_the_hf_warper_masks():
    spec, m = get("tiny")
    cases = _golden()
    by = {}
    for V, name, z, i, setting, want in cases:
        by.setdefault((V, i), []).append((name, z, setting, want))
    for (V, i), rows in by.items():
        t, k, p = rows[0][2]
        got = _device_mask(m, torch.stack([r[1] for r in rows]), t, k, p)
        for r, (name, z, _, want) in enumerate(rows):
            _check_against(got[r], want, z, t, k, p, name in G.TIE_ROWS)


@pytest.mark.gpu
def test_device_filter_reads_rows_too_large_to_stage():
    """rows of more than 51200 scores are read from global memory on every pass: same rule"""
    spec, m = get("tiny")
    V = 70001
    z = (torch.randn(3, V, generator=torch.Generator().manual_seed(3)) * torch.tensor([[0.5], [2.0], [6.0]])).float()
    for t, k, p in [(0.7, 50, None), (1.0, 1, None), (0.7, None, 0.9), (1.0, 200, 0.5), (0.2, V, 0.999)]:
        got = _device_mask(m, z, t, k, p)
        want = torch.isfinite(filter_scores(z / t, *sampling_filters(k, p)))
        for r in range(3):
            _check_against(got[r], want[r], z[r], t, k, p, False)


def _sample_first(m, cache, logits, t, seed, top_k=0, top_p=1.0, eos=-1, pad=0):
    sp = VlySampling(float(t), int(seed), int(eos), int(pad), -1, int(top_k), float(top_p))
    out = torch.empty(cache.batch, dtype=torch.int64, device="cuda")
    lg = logits.reshape(cache.batch, -1).float().contiguous()
    check(m._lib.vly_sample_logits(m._ctx, cache._h, lg.data_ptr(), C.byref(sp), out.data_ptr(), None))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("spec_name", ["tiny", "shape-13b-1l"])
def test_filtered_draws_follow_the_renormalised_filtered_softmax(spec_name):
    """6000 single-seed draws: none outside the kept set, and a chi-square fit against softmax(logits / T) renormalised over the
    kept set (float64), at the same 1e-6 level as the unfiltered sampler's test.  top_k = 1 and a tiny top_p give the arg-max."""
    from scipy import stats
    spec, m = get(spec_name)
    V, T, N = spec.vocab_size, 0.7, 6000
    cache = m.new_cache(1, 128)
    logits = (torch.randn(1, V, generator=torch.Generator().manual_seed(11)) * 1.5).cuda()
    z = logits[0].cpu()
    for k, p in [(20, 1.0), (0, 0.8)]:
        keep = torch.isfinite(filter_scores(z[None] / T, k, p))[0]
        _check_against(_device_mask(m, z[None], T, k, p if p < 1 else None)[0], keep, z, T, k, p if p < 1 else None, False)
        probs = torch.softmax((z.double() / T).masked_fill(~keep, -float("inf")), -1)
        draws = torch.stack([_sample_first(m, cache, logits, T, 1000 + i, k, p) for i in range(N)]).cpu().reshape(-1)
        assert bool(keep[draws].all())
        counts = torch.bincount(draws, minlength=V).double()
        big = probs * N >= 10
        obs = torch.cat([counts[big], counts[~big & keep].sum()[None]])
        exp = torch.cat([probs[big] * N, (probs[~big & keep].sum() * N)[None]])
        if float(exp[-1]) < 5:                       # no tail worth a cell
            obs, exp = obs[:-1], exp[:-1]
        chi2 = float(((obs - exp) ** 2 / exp).sum())
        assert chi2 < stats.chi2.ppf(1 - 1e-6, df=len(obs) - 1), (k, p, chi2, len(obs))
        assert len(obs) >= 10
    amax = int(z.argmax())
    for i in range(50):
        assert int(_sample_first(m, cache, logits, T, 5000 + i, 1, 1.0)) == amax
        assert int(_sample_first(m, cache, logits, T, 6000 + i, 0, 1e-6)) == amax


def _gen(m, ids, px, n, seed, **kw):
    torch.manual_seed(seed)
    return m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=n, **kw)[:, ids.shape[1]:]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 6])
def test_a_filter_that_keeps_everything_draws_the_unfiltered_tokens(B):
    """top_k = V runs the filtered selection and must draw bit for bit what the unfiltered sampler
    draws with the same seed: the first token, the persistent kernel (B <= 4) and the per-op kernels (B = 6)."""
    spec, m = get("tiny")
    V = spec.vocab_size
    ids, px = syn.make_prompt_ids(spec, B, 2, 5), syn.make_pixels(B, 2, 5)
    out = m(input_ids=ids.cuda(), images=px.cuda())
    for seed in range(5):
        a = _sample_first(m, out.past_key_values, out.logits[:, -1], 0.8, 77 + seed)
        b = _sample_first(m, out.past_key_values, out.logits[:, -1], 0.8, 77 + seed, V, 1.0)
        assert torch.equal(a, b)
    plain = _gen(m, ids, px, 12, 4242, do_sample=True, temperature=0.8)
    kept = _gen(m, ids, px, 12, 4242, do_sample=True, temperature=0.8, top_k=V)
    assert torch.equal(plain, kept)
    greedy = _gen(m, ids, px, 12, 0)
    assert not torch.equal(plain, greedy)


@pytest.mark.gpu
@pytest.mark.parametrize("spec_name,B", [("tiny", 1), ("tiny", 2), ("tiny", 6), ("shape-13b-1l", 1), ("shape-13b-1l", 2),
                                         ("shape-13b-1l", 6)])
def test_every_path_draws_the_same_filtered_token(spec_name, B):
    """generate(do_sample=True, T=0.8, top_k=40, top_p=0.9) equals teacher-forcing the drawn ids through forward() and selecting
    each step's logits with vly_sample_logits under the same seed: the fused paths select exactly what the stand-alone one does."""
    spec, m = get(spec_name)
    n, T, K, P = 7, 0.8, 40, 0.9
    ids, px = syn.make_prompt_ids(spec, B, 2, 5), syn.make_pixels(B, 2, 5)
    gen = _gen(m, ids, px, n, 4242, do_sample=True, temperature=T, top_k=K, top_p=P)
    assert gen.shape == (B, n)
    torch.manual_seed(4242)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    out = m(input_ids=ids.cuda(), images=px.cuda())
    cache, toks = out.past_key_values, []
    toks.append(_sample_first(m, cache, out.logits[:, -1], T, seed, K, P))
    for i in range(1, n):
        o = m(input_ids=toks[-1][:, None], past_key_values=cache)
        toks.append(_sample_first(m, cache, o.logits[:, -1], T, seed, K, P))
    assert torch.equal(torch.stack(toks, 1), gen)
    plain = _gen(m, ids, px, n, 4242, do_sample=True, temperature=T)
    assert not torch.equal(plain, gen)                   # the filter changed the draw


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 5])
def test_eos_under_a_filter_stops_and_pads_rows(B):
    """rows are independent and the draw depends only on (logits, seed, row, position): the expected ids are the free-running
    filtered ids, padded after each row's first eos and cut after the last row's"""
    spec, m = get("tiny")
    n, PAD, kw = 10, 7, dict(do_sample=True, temperature=0.8, top_k=30, top_p=0.95)
    ids, px = syn.make_prompt_ids(spec, B, 2, 6), syn.make_pixels(B, 2, 6)
    g = _gen(m, ids, px, n, 99, eos_token_id=None, **kw).cpu()
    i0 = next(i for i in range(2, n) if g[0, i] not in g[0, :i])
    eos = int(g[0, i0])
    exp, stop = g.clone(), []
    for b in range(B):
        hit = (g[b] == eos).nonzero()
        k = int(hit[0]) if len(hit) else n - 1
        exp[b, k + 1:] = PAD
        stop.append(k)
    n_valid = max(stop) + 1
    got = _gen(m, ids, px, n, 99, eos_token_id=eos, pad_token_id=PAD, **kw).cpu()
    assert got.shape[1] == n_valid, (got.shape, n_valid)
    assert torch.equal(got, exp[:, :n_valid])


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 6])
def test_a_filtered_step_adds_a_kernel_only_after_the_persistent_kernel_and_allocates_nothing(B):
    """the persistent kernel (B <= 4) leaves a filtered selection to one more kernel; the per-op path (B > 4) selects in a
    kernel of its own either way"""
    from test_gpu_ownership import held
    spec, m = get("tiny")
    ids, px = syn.make_prompt_ids(spec, B, 2, 3), syn.make_pixels(B, 2, 3)

    def per_step(**kw):
        _gen(m, ids, px, 3, 5, eos_token_id=None, **kw)            # settles the cache's state (and captures its graphs)
        counts = []
        for n in (3, 11):
            before = m.launches()
            _gen(m, ids, px, n, 5, eos_token_id=None, **kw)
            torch.cuda.synchronize()
            counts.append(m.launches() - before)
        return (counts[1] - counts[0]) / 8

    greedy = per_step()
    plain = per_step(do_sample=True, temperature=0.8)
    h0 = held()
    filt = per_step(do_sample=True, temperature=0.8, top_k=40)      # the first filtered generate on this cache captures its graphs
    assert held() == h0
    assert plain == greedy and filt == plain + (1 if B <= 4 else 0), (greedy, plain, filt)
    _gen(m, ids, px, 9, 6, do_sample=True, temperature=0.8, top_p=0.5)
    assert held() == h0


@pytest.mark.gpu
def test_generate_interface_for_the_filters():
    spec, m = get("tiny")
    ids, px = syn.make_prompt_ids(spec, 2, 2, 7), syn.make_pixels(2, 2, 7)
    for kw, msg in [(dict(top_k=-3), "`top_k` has to be a strictly positive integer, but is -3"),
                    (dict(top_p=1.5), "`top_p` has to be a float > 0 and < 1, but is 1.5"),
                    (dict(top_p=-0.1), "`top_p` has to be a float > 0 and < 1, but is -0.1")]:
        with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
            m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=3, do_sample=True, temperature=0.7, **kw)
    greedy = _gen(m, ids, px, 8, 0)
    assert torch.equal(_gen(m, ids, px, 8, 1, do_sample=False, top_k=5, top_p=0.3), greedy)      # not sampling: ignored
    assert torch.equal(_gen(m, ids, px, 8, 1, do_sample=True, temperature=1e-5, top_k=-1), greedy)
    assert torch.equal(_gen(m, ids, px, 8, 2, do_sample=True, temperature=0.7, top_p=0.0), greedy)
    never = lambda seq, scores: False                   # the host-visible loop
    host = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=8, do_sample=True, temperature=0.7, top_k=1,
                      stopping_criteria=[never])[:, ids.shape[1]:]
    assert torch.equal(host, greedy)


@pytest.mark.gpu
def test_completion_and_generate_stream_take_the_filters():
    from test_gpu_dropin import WordTokenizer
    from test_gpu_parity import _FakeTokenizer
    from valley_b200 import serving
    spec, m = get("tiny")
    tok = WordTokenizer(spec)
    clip = syn.make_pixels(1, 8, 3)[0].permute(1, 0, 2, 3).contiguous()            # [3, T, 224, 224]
    message = [{"role": "system", "content": "You are Valley."}, {"role": "user", "content": "Describe it.\n<video>"}]
    want = m.completion(tok, clip, message, dict(do_sample=False, max_new_tokens=12))
    got = m.completion(tok, clip, message, dict(do_sample=True, temperature=0.7, top_k=1, max_new_tokens=12))
    assert got == want
    tk = _FakeTokenizer(spec)
    video = syn.make_pixels(1, 3, 8)[0]
    base = dict(prompt="w5 w9 w33 <video> w77 w78", video=video, max_new_tokens=9)
    greedy = [d["text"] for d in serving.generate_stream(m, tk, dict(base, temperature=0.0), stream_interval=2)]
    top1 = [d["text"] for d in serving.generate_stream(m, tk, dict(base, temperature=0.7, top_k=1), stream_interval=2)]
    assert top1 == greedy and len(greedy) >= 2
