"""GPU (-m gpu): the per-op decode kernels (decode_kernels.cuh) kernel by kernel against float64 references.

These kernels run every decode step of a batch above 4 rows (in groups of at most 4) and the prefill's last-token logits at
any batch size.  Each test drives the production launcher through a test hook (vly_test_gemv / vly_test_decode_attention) on
bf16 inputs and compares with the float64 result of the operation the kernel's comment defines, computed on the GPU from the
same bf16 values.  Every bound is derived from the kernel's arithmetic (see each docstring); each test also applies its bound
to a reference with a plausible defect and asserts that the bound rejects it, so the bound is known to be tight enough to
catch that defect.

Notation: U = 2^-24 (fp32 unit roundoff), BF = 2^-8 (bf16 unit roundoff), S = sum_k |x[b,k] W[n,k]|.
"""
import ctypes as C
import math

import pytest
import torch

import helpers as Hh
from valley_b200 import _lib, synthetic as syn

pytestmark = pytest.mark.gpu

U, BF = 2.0 ** -24, 2.0 ** -8
KC = 2048                                   # columns per ring slice (RingCfg::KC)
QKV_ROPE, RESIDUAL, SWIGLU, LOGITS = 0, 1, 2, 3
ROW_SCALE = (1.0, 1e3, 1e-3, 1e6)           # x rows whose RMS differs by 10^3 from one row to the next
EPS = 1e-5
_state = {}


def _model():
    """any context with LLM weights: the hooks use its RoPE table (theta 10^4, 2048 positions) and its workspace"""
    if "m" not in _state:
        spec = syn.SPECS["tiny"]
        _state["m"] = Hh.build_model(spec, Hh.bf16_weights(spec, 0))
    return _state["m"]


def _num_sms(m):
    n = C.c_int()
    _lib.check(m._lib.vly_num_sms(m._ctx, C.byref(n)))
    return n.value


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _weights(N, K, seed):
    return (torch.randn(N, K, generator=_gen(seed), device="cuda") * 0.02).bfloat16()


def _rows(B, K, seed, extra=0):
    """x [B, K] (or [B, extra + 1, K]: the last of extra + 1 rows per sequence, as the prefill's last-token logits read it)"""
    x = torch.randn(B, extra + 1, K, generator=_gen(seed), device="cuda")
    x *= torch.tensor(ROW_SCALE[:B], device="cuda")[:, None, None]
    x = x.bfloat16()
    return x if extra else x[:, 0]


def _gemv(m, mode, W, x, B, ldx=0, res=None, out=None, kc=None, vc=None, Smax=0, pos=0, logits=None, nxt=None):
    N, K = W.shape
    p = lambda t: None if t is None else t.data_ptr()
    _lib.check(m._lib.vly_test_gemv(m._ctx, mode, W.data_ptr(), x.data_ptr(), N, K, B, ldx, EPS, p(res), p(out), p(kc), p(vc),
                                    Smax, pos, p(logits), p(nxt), None))
    torch.cuda.synchronize()


def _depth(K):
    """fp32 roundings that one product x*w passes through in gemv_ring_kernel: up to 8 FMAs per 2048-column slice in its
    consumer thread, 5 butterfly adds across the warp, 8 adds across the warps and the multiply by rstd"""
    return 8 * -(-K // KC) + 14


def _ref(W, x, norm=True):
    """float64 y = rstd * x W^T and A, the bound on the kernel's fp32 error in y.

    A = (1.5 d + 4) U rstd S with d = _depth(K): the sum itself is off by at most d U rstd S; rstd = rsqrtf(sum x^2 / K + eps)
    sums its squares to the same depth d, which costs d/2 U relative after the square root, and the mean, the + eps and
    rsqrtf (2 ulp) add 4 U more; |y| <= rstd S."""
    K = W.shape[1]
    W64, x64 = W.double(), x.double()
    rstd = torch.rsqrt(x64.pow(2).mean(1, keepdim=True) + EPS) if norm else torch.ones_like(x64[:, :1])
    y = (x64 @ W64.T) * rstd
    A = (x64.abs() @ W64.abs().T) * rstd * (U * (1.5 * _depth(K) + 4))
    return y, A, rstd


def _excess(got, ref, tol):
    """largest amount by which |got - ref| exceeds tol (<= 0: within the bound everywhere)"""
    g = got.double()
    assert torch.isfinite(g).all()
    return float(((g - ref).abs() - tol).max())


def _bf16_ulp(v):
    """spacing of bf16 values at |v| (v bf16-representable): 2^(e - 8) for |v| in [2^(e-1), 2^e)"""
    e = torch.frexp(v).exponent
    return torch.ldexp(torch.ones_like(v), e - 8)


def _dropped_tail(W, x, rstd):
    """the contribution of the last 8 columns of the last (short, where K % 2048 != 0) slice: a kernel that skipped the
    slice's final 16-byte lane would miss exactly this"""
    K = W.shape[1]
    return (x[:, K - 8:].double() @ W[:, K - 8:].double().T) * rstd


RESIDUAL_SHAPES = [(512, 512), (4096, 4096), (4096, 11008), (5120, 5120), (5120, 13824), (4101, 11008)]


@pytest.mark.parametrize("N,K", RESIDUAL_SHAPES, ids=["tiny-o", "7b-o", "7b-down", "13b-o", "13b-down", "n-tail"])
def test_gemv_residual(N, K):
    """GEMV_RESIDUAL (o_proj, down_proj): out = bf16(x W^T + res), no normalisation.  Bound: BF |ref| for the output rounding
    plus (1 + BF) (A + U |ref|) for the accumulation and the fp32 add of the residual.  The down projection at K = 11008 /
    13824 with 3 or 4 rows takes the 225 KB shared-memory budget; N = 4101 ends in a 1-row group.  Negative control: the
    last 8 columns dropped."""
    m = _model()
    W = _weights(N, K, 1)
    for B in (1, 2, 3, 4):
        x = _rows(B, K, 10 + B)
        res = torch.randn(B, N, generator=_gen(20 + B), device="cuda").bfloat16()
        out = torch.empty(B, N, dtype=torch.bfloat16, device="cuda")
        _gemv(m, RESIDUAL, W, x, B, res=res, out=out)
        y, A, rstd = _ref(W, x, norm=False)
        ref = y + res.double()
        tol = BF * ref.abs() + (1 + BF) * (A + U * ref.abs())
        assert _excess(out, ref, tol) <= 0, (B, _excess(out, ref, tol))
        assert _excess(out, ref - _dropped_tail(W, x, rstd), tol) > 0, B
        again = torch.empty_like(out)
        _gemv(m, RESIDUAL, W, x, B, res=res, out=again)
        assert torch.equal(again, out), B
        inplace = res.clone()                                # the decode step adds in place into the residual stream
        _gemv(m, RESIDUAL, W, x, B, res=inplace, out=inplace)
        assert torch.equal(inplace, out), B


@pytest.mark.parametrize("N,K", [(2048, 512), (22016, 4096), (27648, 5120)], ids=["tiny", "7b", "13b"])
def test_gemv_swiglu(N, K):
    """GEMV_SWIGLU (gate/up, rows interleaved (gate j, up j)): out[j] = bf16(bf16(silu(g)) * u) with g = bf16(rstd y[2j]),
    u = bf16(rstd y[2j+1]) -- gate and up are rounded to bf16 before silu(g) * u.  Reference: silu(bf16(g)) * bf16(u) in
    float64.  The kernel's g, u differ from the reference's by their fp32 error A plus, where that error crosses a rounding
    boundary, one bf16 ulp: dg = A_g + ulp(g), du = A_u + ulp(u).  Bound: 1.1 dg |u| (|silu'| < 1.1) + |silu(g)| du
    + 1.1 dg du, plus BF |silu(g) u| for rounding silu to bf16, BF |ref| for the output and 2^-20 |ref| for __expf and the
    fp32 divide and multiply.  Negative controls: another row's rstd; the last 8 columns dropped."""
    m = _model()
    W = _weights(N, K, 2)
    for B in (1, 2, 3, 4):
        x = _rows(B, K, 30 + B)
        out = torch.empty(B, N // 2, dtype=torch.bfloat16, device="cuda")
        _gemv(m, SWIGLU, W, x, B, out=out)
        y, A, rstd = _ref(W, x)

        def swiglu(y):
            g, u = y[:, 0::2].bfloat16().double(), y[:, 1::2].bfloat16().double()
            s = g * torch.sigmoid(g)
            ref = s * u
            dg, du = A[:, 0::2] + _bf16_ulp(g), A[:, 1::2] + _bf16_ulp(u)
            tol = 1.1 * dg * u.abs() + s.abs() * du + 1.1 * dg * du + BF * (s * u).abs() + (BF + 2.0 ** -20) * ref.abs()
            return ref, tol

        ref, tol = swiglu(y)
        assert _excess(out, ref, tol) <= 0, (B, _excess(out, ref, tol))
        assert _excess(out, swiglu(y - _dropped_tail(W, x, rstd))[0], tol) > 0, B
        if B > 1:
            assert _excess(out, swiglu(y / rstd * rstd.roll(1, 0))[0], tol) > 0, B
        again = torch.empty_like(out)
        _gemv(m, SWIGLU, W, x, B, out=again)
        assert torch.equal(again, out), B


def _rope_table(pos):
    """(cos, sin) of pos * 10000^(-2j/128), j < 64, computed in fp32 and rounded to bf16 as rope_table_kernel does"""
    j = torch.arange(64, device="cuda", dtype=torch.float32)
    inv = 1.0 / torch.pow(torch.tensor(10000.0, device="cuda"), 2.0 * j / 128.0)
    fr = float(pos) * inv
    return torch.cos(fr).bfloat16().double(), torch.sin(fr).bfloat16().double()


def _pattern(B, nH, Smax, seed):
    """a cache filled with a bit pattern (any 16-bit value, NaN patterns included): rows the kernel must not touch keep it"""
    bits = torch.randint(-32768, 32768, (B, nH, Smax, 128), generator=_gen(seed), device="cuda", dtype=torch.int32)
    return bits.to(torch.int16).view(torch.bfloat16)


@pytest.mark.parametrize("N,K", [(1536, 512), (12288, 4096), (15360, 5120)], ids=["tiny", "7b", "13b"])
def test_gemv_qkv_rope(N, K):
    """GEMV_QKV_ROPE: rows [q | k | v] of nH heads, each head in the pair-interleaved RoPE order (rows 2j, 2j+1 = dims j,
    j + 64).  z = rstd y; q and k pairs are rotated by the RoPE table at the new token's position pos: (z0 c - z1 s,
    z1 c + z0 s); q goes to out [B, H], k and v to row pos of the caches [B, nH, Smax, 128].  Bound: BF |ref| for the output
    rounding, |c| A0 + |s| A1 + 3 U (|z0 c| + |z1 s|) for the accumulation and the fp32 rotation, and one bf16 ulp of c and
    s on |z0| + |z1| (the table is rounded to bf16; the reference recomputes it).  Every other cache row keeps its bit
    pattern.  Negative control: RoPE at pos - 1 (pos + 1 at pos 0)."""
    m = _model()
    H = N // 3
    nH, Smax = H // 128, 2048
    W = _weights(N, K, 3)

    def rope(z, A, pos):
        c, s = _rope_table(pos)
        z0, z1, A0, A1 = z[..., 0], z[..., 1], A[..., 0], A[..., 1]
        r = torch.stack([z0 * c - z1 * s, z1 * c + z0 * s], -1)
        err = c.abs() * A0 + s.abs() * A1 + 3 * U * ((z0 * c).abs() + (z1 * s).abs()) + \
            (_bf16_ulp(c) + _bf16_ulp(s)) * (z0.abs() + z1.abs())
        return r, torch.stack([err, err], -1)

    for B in (1, 2, 3, 4):
        x = _rows(B, K, 40 + B)
        y, A, _ = _ref(W, x)
        z, Az = y.view(B, 3, nH, 64, 2), A.view(B, 3, nH, 64, 2)
        for pos in (0, 63, 64, 1000, Smax - 1):
            kc, vc = _pattern(B, nH, Smax, 1), _pattern(B, nH, Smax, 2)
            kc0, vc0 = kc.clone(), vc.clone()
            q = torch.empty(B, H, dtype=torch.bfloat16, device="cuda")
            _gemv(m, QKV_ROPE, W, x, B, out=q, kc=kc, vc=vc, Smax=Smax, pos=pos)
            got = torch.stack([q.view(B, nH, 128), kc[:, :, pos], vc[:, :, pos]], 1).view(B, 3, nH, 64, 2)
            rq, eq = rope(z[:, 0], Az[:, 0], pos)
            rk, ek = rope(z[:, 1], Az[:, 1], pos)
            ref = torch.stack([rq, rk, z[:, 2]], 1)
            tol = BF * ref.abs() + torch.stack([eq, ek, Az[:, 2]], 1)
            assert _excess(got, ref, tol) <= 0, (B, pos, _excess(got, ref, tol))
            wrong = pos - 1 if pos > 0 else pos + 1
            bad = torch.stack([rope(z[:, 0], Az[:, 0], wrong)[0], rope(z[:, 1], Az[:, 1], wrong)[0], z[:, 2]], 1)
            assert _excess(got, bad, tol) > 0, (B, pos)
            keep = torch.ones(Smax, dtype=torch.bool, device="cuda")
            keep[pos] = False
            for cache, before in ((kc, kc0), (vc, vc0)):
                assert torch.equal(cache[:, :, keep].view(torch.int16), before[:, :, keep].view(torch.int16)), (B, pos)
            kc2, vc2 = _pattern(B, nH, Smax, 1), _pattern(B, nH, Smax, 2)
            q2 = torch.empty_like(q)
            _gemv(m, QKV_ROPE, W, x, B, out=q2, kc=kc2, vc=vc2, Smax=Smax, pos=pos)
            assert torch.equal(q2, q) and torch.equal(kc2.view(torch.int16), kc.view(torch.int16)) and \
                torch.equal(vc2.view(torch.int16), vc.view(torch.int16)), (B, pos)


def _first_max(lg):
    """lowest index of the maximum of each row"""
    hit = lg == lg.max(-1, keepdim=True).values
    idx = torch.arange(lg.shape[-1], device=lg.device).expand_as(lg)
    return torch.where(hit, idx, lg.shape[-1]).min(-1).values


def _tie_rows(N, grid):
    """(i, j), i < j: two rows of W planted as duplicates, in the same 4-row group, in two groups of the same CTA (g and
    g + grid), and in two CTAs -- the lower index in the lower CTA, and in a higher one (first round vs second round), also
    with both CTAs' partials read by the same lane of the final merge (CTAs c and c + 32)"""
    return [(4 * 7 + 1, 4 * 7 + 3), (4 * 7 + 2, 4 * (7 + grid) + 1), (4 * 3, 4 * 50 + 2), (4 * 100 + 3, 4 * (grid + 5)),
            (4 * 36 + 1, 4 * (grid + 4) + 2)]


@pytest.mark.parametrize("N,K", [(1032, 512), (32008, 4096), (32008, 5120), (32005, 5120)], ids=["tiny", "7b", "13b", "n-tail"])
def test_gemv_logits_and_argmax(N, K):
    """GEMV_LOGITS (lm_head of the decode step and of the prefill's last token): fp32 logits = rstd y, read from rows of
    stride ldx = 3 K (the last of 3 positions per sequence).  Bound: A alone -- no rounding to bf16.  The token is exactly
    the lowest index of the maximum of the kernel's own logits; with two duplicated rows of W made the clear maximum (same
    4-row group, same CTA, different CTAs) their logits are bit-identical and the lower index wins.  Negative controls:
    another row's rstd; the last 8 columns dropped.  Two identical calls give identical bits (the arg-max counter is reset)."""
    m = _model()
    W = _weights(N, K, 4)
    grid = min(-(-N // 4), _num_sms(m))
    ties = _tie_rows(N, grid)
    assert max(j for _, j in ties) < N
    for B in (1, 2, 3, 4):
        xs = _rows(B, K, 50 + B, extra=2)
        x = xs[:, -1]
        lg = torch.empty(B, N, device="cuda")
        nxt = torch.full((B,), -1, dtype=torch.int64, device="cuda")
        _gemv(m, LOGITS, W, xs[:, -1], B, ldx=3 * K, logits=lg, nxt=nxt)
        y, A, rstd = _ref(W, x)
        assert _excess(lg, y, A) <= 0, (B, _excess(lg, y, A))
        assert _excess(lg, y - _dropped_tail(W, x, rstd), A) > 0, B
        if B > 1:
            assert _excess(lg, y / rstd * rstd.roll(1, 0), A) > 0, B
        assert torch.equal(nxt, _first_max(lg)), B
        lg2, nxt2 = torch.empty_like(lg), torch.full_like(nxt, -1)
        _gemv(m, LOGITS, W, xs[:, -1], B, ldx=3 * K, logits=lg2, nxt=nxt2)
        assert torch.equal(lg2.view(torch.int32), lg.view(torch.int32)) and torch.equal(nxt2, nxt), B
        # planted ties: w* points along every row of x, so its logit is the clear maximum of each row
        star = (x.float() / x.float().pow(2).mean(1, keepdim=True).sqrt()).sum(0) * (0.05 / math.sqrt(B))
        for i, j in ties:
            saved = W[[i, j]].clone()
            W[i] = W[j] = star.bfloat16()
            nxt.fill_(-1)
            _gemv(m, LOGITS, W, xs[:, -1], B, ldx=3 * K, logits=lg, nxt=nxt)
            W[[i, j]] = saved
            assert torch.equal(lg[:, i].view(torch.int32), lg[:, j].view(torch.int32)), (B, i, j)
            assert bool((_first_max(lg) == i).all()) and bool((nxt == i).all()), (B, i, j, nxt.tolist())


def _attend(B, L, kind):
    """uint8 mask [B, L] (1 = attend; the newest key L - 1 always) or None"""
    if kind == "none":
        return None
    m = torch.ones(B, L, dtype=torch.uint8, device="cuda")
    if kind.startswith("pad"):                          # left padding: p keys on even rows, p + 1 on odd rows
        for b in range(B):
            m[b, :min(int(kind[3:]) + b % 2, L - 1)] = 0
    elif kind == "mid":                                 # whole 64-key splits 2, 3 and 4
        m[:, 128:320] = 0
    elif kind == "newest":
        m[:, :L - 1] = 0
    return m


def _masks(L):
    kinds = ["none", "newest"] + [f"pad{p}" for p in (1, 64, 130) if p + 1 < L]
    return kinds + (["mid"] if L > 320 else [])


def _attn_ref(q, kc, vc, L, mask, splits=None):
    """float64 softmax(q k^T / sqrt(128)) v over the attended keys below L (below 64 * splits when given) and the bound.

    Score error (natural-log units, fp32): the 128-term dot product (8 products per lane + 4 shuffle adds) and the scale
    give 15 U sum_d |q k| / sqrt(128); s - max adds U (|s| + max |s|).  fast_exp2 (ex2.approx, < 2 ulp) runs twice per
    weight (in the split and in the merge): 8 U.  A relative error e_w on every weight moves the normalised weights by at
    most 2 e_w, and the sums of weights and of p v are 8 + nsplit + 26 roundings deep.  Bound: (2 e_w + (2 nsplit + 26) U)
    sum_i p_i |v_i| plus BF |ref| for the output rounding and one more bf16 ulp (BF |ref|) for fast_exp2."""
    B, H = q.shape
    nH = H // 128
    qd = q.double().view(B, nH, 1, 128)
    k, v = kc[:, :, :L].double(), vc[:, :, :L].double()
    s = (qd @ k.transpose(-1, -2))[:, :, 0] / math.sqrt(128)
    sabs = (qd.abs() @ k.abs().transpose(-1, -2))[:, :, 0] / math.sqrt(128)
    att = torch.ones(B, L, dtype=torch.bool, device="cuda") if mask is None else mask.bool()
    if splits is not None:
        att[:, 64 * splits:] = False
    att = att[:, None, :].expand(B, nH, L)
    if not bool(att.any()):
        return torch.zeros(B, H, dtype=torch.float64, device="cuda"), None
    s = s.masked_fill(~att, -float("inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)                # (a row with nothing attended: 0, as the merge writes)
    ref = (p[:, :, None, :] @ v)[:, :, 0].reshape(B, H)
    pv = (p[:, :, None, :] @ v.abs())[:, :, 0].reshape(B, H)
    fin = s.masked_fill(~att, 0.0)
    smax = fin.abs().amax(-1, keepdim=True)
    dw = (15 * U * sabs + U * (fin.abs() + smax)).masked_fill(~att, 0.0).amax(-1) + 8 * U        # [B, nH]
    nsplit = kc.shape[2] // 64
    tol = (2 * dw[:, :, None].expand(B, nH, 128).reshape(B, H) + (2 * nsplit + 26) * U) * pv + 2 * BF * ref.abs()
    return ref, tol


def _attention(m, q, kc, vc, L, mask):
    B, H = q.shape
    out = torch.empty(B, H, dtype=torch.bfloat16, device="cuda")
    _lib.check(m._lib.vly_test_decode_attention(m._ctx, q.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, H // 128, kc.shape[2], L,
                                                None if mask is None else mask.data_ptr(), out.data_ptr(), None))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("nH", [4, 32, 40])
def test_decode_attention(nH):
    """decode_attention_v2_kernel (fixed 64-key splits, last-arriver merge) for B = 1..4 rows, caches of 128 and 2048 keys,
    lengths at and around the split edges up to a full cache, with left padding, whole masked splits in the middle and every
    key masked but the newest.  Keys at and above len hold 3e4, so reading one would show.  Negative control: the merge
    missing the last split.  Two identical calls give identical bits."""
    m = _model()
    for Smax in (128, 2048):
        for B in (1, 2, 3, 4):
            g = _gen(60 + B)
            q = (torch.randn(B, nH * 128, generator=g, device="cuda") * 2).bfloat16()
            kc0 = torch.randn(B, nH, Smax, 128, generator=g, device="cuda").bfloat16()
            vc0 = torch.randn(B, nH, Smax, 128, generator=g, device="cuda").bfloat16()
            for L in (1, 2, 63, 64, 65, 128, 129, 1000, 2048):
                if L > Smax:
                    continue
                kc, vc = kc0.clone(), vc0.clone()
                kc[:, :, L:] = 3e4
                vc[:, :, L:] = 3e4
                for kind in _masks(L):
                    mask = _attend(B, L, kind)
                    out = _attention(m, q, kc, vc, L, mask)
                    ref, tol = _attn_ref(q, kc, vc, L, mask)
                    assert _excess(out, ref, tol) <= 0, (Smax, B, L, kind, _excess(out, ref, tol))
                    bad, _ = _attn_ref(q, kc, vc, L, mask, splits=-(-L // 64) - 1)
                    assert _excess(out, bad, tol) > 0, (Smax, B, L, kind)
                    if kind == "none":
                        assert torch.equal(_attention(m, q, kc, vc, L, mask), out), (Smax, B, L)


def test_greedy_ties_resolve_to_the_lowest_index_on_every_path():
    """tiny with lm_head rows V/2 + i = rows i: every maximum is tied.  The logits the kernels return through forward()
    come in bit-identical pairs -- the prefill's last-token GEMV_LOGITS, the persistent step (B = 1, 2, 4) and the per-op
    step (B = 6) -- and every selection path picks the lower index of the pair (HF's torch.argmax does): greedy generate on
    the device, greedy with an eos id (the first token through vly_sample_logits) and the host-visible loop."""
    spec = syn.SPECS["tiny"]
    V = spec.vocab_size
    h = V // 2
    sd = Hh.bf16_weights(spec, 0)
    sd["lm_head.weight"][h:] = sd["lm_head.weight"][:h]
    m = Hh.build_model(spec, sd)
    m.logits_all_positions = False
    never = lambda seq, scores: False
    for B in (1, 2, 4, 6):
        ids, px = syn.make_prompt_ids(spec, B, 2, 5), syn.make_pixels(B, 2, 5)
        S = ids.shape[1]
        out = m(input_ids=ids.cuda(), images=px.cuda())
        lg = out.logits[:, -1]
        assert torch.equal(lg[:, :h].view(torch.int32), lg[:, h:].view(torch.int32)), (B, "prefill")
        cache = out.past_key_values
        for i in range(3):
            o = m(input_ids=_first_max(lg)[:, None], past_key_values=cache)
            lg = o.logits[:, -1]
            assert torch.equal(lg[:, :h].view(torch.int32), lg[:, h:].view(torch.int32)), (B, "step", i)
        plain = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=8)[:, S:]
        assert int(plain.max()) < h, (B, plain.tolist())
        with_eos = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=8, eos_token_id=V - 1)[:, S:]
        host = m.generate(input_ids=ids.cuda(), images=px.cuda(), max_new_tokens=8, stopping_criteria=[never])[:, S:]
        assert torch.equal(with_eos, plain) and torch.equal(host, plain), (B, plain.tolist(), with_eos.tolist(), host.tolist())
