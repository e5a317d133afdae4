"""GPU (-m gpu): the prefill / ViT kernels (gemm_tc.cuh, attention_tc.cuh) kernel by kernel against float64 references.

Every ViT frame and every prompt token goes through gemm_tc_kernel (seven fused epilogues) and one of the two flash-attention
kernels.  Each test drives the production launcher through a test hook (vly_test_gemm / vly_test_prefill_attention /
vly_test_vit_attention) on bf16 inputs and compares element-wise with the float64 result of the operation the kernel's comment
defines, computed on the GPU from the same bf16 values.  Every bound is derived from the kernel's arithmetic (see each
docstring); each test also applies its bound to a reference with a plausible defect and asserts that the bound rejects it.
`pytest -s` prints each test's tightness: the largest |got - ref| / tol it met.

Notation: U = 2^-24 (fp32 unit roundoff), BF = 2^-8 (bf16 unit roundoff), Sa = sum_k |a[m,k] w[n,k]|.

Arithmetic the bounds cover:
  * wgmma accumulation.  The tensor cores are not guaranteed to round every FMA to nearest; each k16 step is modelled as at
    most two fp32 roundings of the running sum, so acc is off by at most A = (ceil(K/16) + 4) 2U Sa (_acc_err).
  * Row statistics come from bf16 values: EPI_BIAS_RES_STATS sums the ROUNDED outputs it stores, and the consumers read those
    rows.  The references take mean / rstd from the same bf16 rows (or from the supplied partials), never from an fp32 copy.
  * LayerNorm fold: the kernel forms rstd (acc - mean colsum) + bias from the raw residual stream, so its fp32 error scales
    with rstd (Sa + |mean| |colsum|), not with the output, and var = E[x^2] - mean^2 is one pass in fp32, off by
    ~ depth U (mean^2 + var) / var relative.  Rows with |mean| / std up to 30 exercise both.
  * quick_gelu_f / silu_f compute sigmoid(y) = 1/2 + 1/2 tanh.approx(y/2).  tanh.approx.f32 has a relative error of about
    2^-11 (PTX ISA); after the 1/2 + 1/2 tanh the error is ABSOLUTE: |v| 2^-10.9 / 2 on v sigmoid(.).  For strongly negative
    arguments that exceeds the bf16 rounding of the (tiny) result, so the bounds carry that term and the inputs reach -10.
  * RoPE: rope_table_kernel rounds cos and sin to bf16; the reference uses the same rounded values (_rope_table) plus one bf16
    ulp of each where torch's fp32 cos / sin could round the other way.
  * Attention: P is rounded to bf16 before P V while the row sum adds the unrounded p, so the error is up to about
    BF sum_i p_i |v_i| / sum_i p_i, not BF |ref| (random V cancels in the output).
"""
import math

import pytest
import torch

from valley_b200 import _lib
from test_gpu_decode_per_op import _model, _gen, _excess, _bf16_ulp, _rope_table, _pattern, _attend, ROW_SCALE

pytestmark = pytest.mark.gpu

U, BF = 2.0 ** -24, 2.0 ** -8
TANH = 2.0 ** -10.9                          # |relative error| of tanh.approx.f32, with a little slack over the PTX ISA's 2^-11
BIAS, LN_BIAS, LN_GELU, RES_STATS, QKV_ROPE, SWIGLU, RMS_F32 = range(7)
EPS = 1e-5
_tight = {}


def _note(name, got, ref, tol):
    """assert |got - ref| <= tol everywhere and record max |got - ref| / tol (over tol > 0) for the test's summary line"""
    ex = _excess(got, ref, tol)
    assert ex <= 0, (name, ex)
    d = (got.double() - ref).abs()
    pos = tol > 0
    assert bool((d[~pos] == 0).all()), name                 # a zero bound (an exactly-zero reference) allows no error
    r = float((d[pos] / tol[pos]).max()) if bool(pos.any()) else 0.0
    _tight[name] = max(_tight.get(name, 0.0), r)


def _report(name):
    print(f"\n[tightness] {name}: max |err| / tol = {_tight.pop(name, 0.0):.3f}")


def _ptr(t):
    return None if t is None else t.data_ptr()


def _gemm(epi, A, W, out, bn, bias=None, res=None, colsum=None, stats=None, eps=EPS, stats_out=None, kc=None, vc=None, S=0,
          past=0, Smax=0):
    m = _model()
    M, K = A.shape
    N = W.shape[0]
    nt = 0 if stats is None else stats.shape[1]
    _lib.check(m._lib.vly_test_gemm(m._ctx, A.data_ptr(), W.data_ptr(), M, N, K, epi, _ptr(bias), _ptr(res), out.data_ptr(), bn,
                                    _ptr(colsum), _ptr(stats), nt, eps, _ptr(stats_out), _ptr(kc), _ptr(vc), S, past, Smax, None))
    torch.cuda.synchronize()


def _cdiv(a, b):
    return -(-a // b)


def _acc_err(a64, w64):
    """A = (ceil(K/16) + 4) 2U Sa: the bound on the fp32 error of the wgmma accumulation (two roundings per k16 step)"""
    return (a64.abs() @ w64.abs().T) * ((_cdiv(a64.shape[1], 16) + 4) * 2 * U)


def _last_block(a64, w64):
    """the contribution of the last 64-column K block: a kernel that skipped the final TMA box would miss exactly this"""
    k0 = 64 * (_cdiv(a64.shape[1], 64) - 1)
    return a64[:, k0:] @ w64[:, k0:].T


def _rows(M, K, seed, offset=False):
    """bf16 rows whose scale cycles through ROW_SCALE (a row that read another row's statistics is off by 10^3); with offset,
    a common offset of (0, 30, -10, 3) standard deviations on top"""
    x = torch.randn(M, K, generator=_gen(seed), device="cuda")
    sc = torch.tensor(ROW_SCALE, device="cuda").repeat(_cdiv(M, 4))[:M]
    x = x * sc[:, None]
    if offset:
        x = x + (torch.tensor((0.0, 30.0, -10.0, 3.0), device="cuda").repeat(_cdiv(M, 4))[:M] * sc)[:, None]
    return x.bfloat16()


def _weights(N, K, seed, std):
    return (torch.randn(N, K, generator=_gen(seed), device="cuda") * std).bfloat16()


def _vec(N, seed, std=1.0, mean=0.0):
    return torch.randn(N, generator=_gen(seed), device="cuda") * std + mean


def _partials(x, width, nt=None):
    """[M, nt, 2] fp32 = float2 partial (sum, sumsq) over column tiles of `width` (float64 sums, rounded once to fp32); nt
    beyond the tiles holds zeros -- with width >= K that is copy_rows_stats_kernel's layout (the whole row in partial 0)"""
    M, K = x.shape
    n = _cdiv(K, width)
    x64 = x.double()
    st = torch.zeros(M, nt or n, 2, dtype=torch.float64, device="cuda")
    for i in range(n):
        t = x64[:, i * width:(i + 1) * width]
        st[:, i, 0], st[:, i, 1] = t.sum(1), t.pow(2).sum(1)
    return st.float().contiguous()


def _rms(st, K):
    """rstd = 1 / sqrt(sum sumsq / K + eps) from the float64 sum of the partials, and dr, the bound on the kernel's relative
    error in it: the fp32 sum of nt positive partials and the * (1/K) (nt + 1) U, halved by the square root; + eps and
    rsqrtf (2 ulp) 6 U"""
    nt = st.shape[1]
    rstd = torch.rsqrt(st.double()[..., 1].sum(1) / K + EPS)[:, None]
    return rstd, (nt + 1) * U / 2 + 6 * U


def _ln(st, K):
    """mean, var, rstd of LayerNorm from the float64 sum of the partials, and the kernel's fp32 errors: e_m (absolute, in mean)
    and dr (relative, in rstd).  mean = fl(sum s_i) * fl(1/K): e_m = (nt + 1) U sum |s_i| / K.  var = sumsq/K - mean^2 in fp32:
    e_v = (nt + 1) U sumsq/K + 2 e_m |mean| + e_m^2 + 3 U mean^2 + U var; rstd = rsqrtf(var + eps): dr = e_v / (2 (var + eps))
    + 6 U.  With |mean| = 30 std and nt = 8, dr ~ 1.4e4 U ~ 8e-4: the one-pass variance's cancellation."""
    nt = st.shape[1]
    s = st.double()
    S1, S2 = s[..., 0].sum(1), s[..., 1].sum(1)
    mean = S1 / K
    var = S2 / K - mean * mean
    rstd = torch.rsqrt(var.clamp_min(0) + EPS)
    e_m = (nt + 1) * U * s[..., 0].abs().sum(1) / K
    e_v = (nt + 1) * U * S2 / K + 2 * e_m * mean.abs() + e_m * e_m + 3 * U * mean * mean + U * var.abs()
    dr = e_v / (2 * (var.clamp_min(0) + EPS)) + 6 * U
    return mean[:, None], rstd[:, None], e_m[:, None], dr[:, None]


def _qgelu(v, c=1.702):
    return v * torch.sigmoid(c * v)


def _act_err(v):
    """absolute error of v sigmoid(.) = h + h tanh.approx(.), h = v / 2: |h| (TANH + 4 U) (tanh, the scaled argument, fmaf)"""
    return 0.5 * v.abs() * (TANH + 4 * U)


# ============================================================================================================================
# EPI_BIAS
# ============================================================================================================================
BIAS_SHAPES = [(128, 128, 64, (128,)), (1, 256, 64, (256, 128)), (300, 512, 256, (128, 256)), (1000, 1024, 640, (256, 128)),
               (257, 1024, 640, (128, 256)), (2048, 1024, 640, (256,)), (77, 1032, 512, (128,)), (2056, 1024, 4096, (256, 128)),
               (300, 1024, 1000, (128,))]


@pytest.mark.parametrize("M,N,K,bns", BIAS_SHAPES, ids=["small", "m1", "m300", "m1000", "vit-patch-1f", "vit-patch-8f",
                                                         "n-tail", "m2056-k4096", "k-tail"])
def test_gemm_bias(M, N, K, bns):
    """EPI_BIAS (patch embedding K = 640, projector): out = bf16(acc + bias), with and without bias.  Bound: BF |ref| for the
    output rounding plus (1 + BF) (A + U |ref|) for the accumulation and the fp32 bias add.  N = 1032 ends in a 8-column tile
    (scalar stores); K = 1000 ends in a 40-column block that TMA zero-fills.  Negative control: the last K block dropped.
    Two identical calls give identical bits."""
    name = "gemm_bias"
    A, W = _rows(M, K, 1), _weights(N, K, 2, 0.05)
    a64, w64 = A.double(), W.double()
    y, Aerr = a64 @ w64.T, _acc_err(a64, w64)
    for bn in bns:
        for with_bias in (True, False):
            bias = _vec(N, 3) if with_bias else None
            ref = y + (bias.double() if with_bias else 0)
            tol = BF * ref.abs() + (1 + BF) * (Aerr + U * ref.abs())
            out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
            _gemm(BIAS, A, W, out, bn, bias=bias)
            _note(name, out, ref, tol)
            assert _excess(out, ref - _last_block(a64, w64), tol) > 0, (bn, with_bias)
            again = torch.empty_like(out)
            _gemm(BIAS, A, W, again, bn, bias=bias)
            assert torch.equal(again, out), bn
    _report(name)


# ============================================================================================================================
# EPI_BIAS_RES_STATS
# ============================================================================================================================
RES_SHAPES = [(128, 128, 64, (128,)), (1, 256, 64, (256, 128)), (300, 512, 256, (128, 256)), (1000, 1024, 640, (256,)),
              (2056, 1024, 1024, (256, 128)), (257, 1024, 4096, (128, 256)), (2056, 1024, 4096, (256,)), (300, 4096, 4096, (256, 128)),
              (77, 4096, 11008, (256, 128)), (77, 5120, 13824, (256, 128)), (300, 512, 3776, (128, 256))]


def _res_stats_ref(out, bn):
    """float64 per-tile (sum, sumsq) of the kernel's own bf16 outputs, and the bound: a half-row thread adds n/4 pairs of the
    tile's n columns sequentially, then one shuffle add -- at most (n/2 + 2) U sum |o| (sumsq: + 1 for the squares)"""
    M, N = out.shape
    o = out.double()
    nt = _cdiv(N, bn)
    ref = torch.zeros(M, nt, 2, dtype=torch.float64, device="cuda")
    tol = torch.zeros_like(ref)
    short = torch.zeros_like(ref)                                       # the same without the tile's last 32-column chunk
    for i in range(nt):
        t = o[:, i * bn:(i + 1) * bn]
        n = t.shape[1]
        ref[:, i, 0], ref[:, i, 1] = t.sum(1), t.pow(2).sum(1)
        tol[:, i, 0], tol[:, i, 1] = (n / 2 + 2) * U * t.abs().sum(1), (n / 2 + 3) * U * t.pow(2).sum(1)
        short[:, i, 0], short[:, i, 1] = t[:, :-32].sum(1), t[:, :-32].pow(2).sum(1)
    return ref, tol, short


@pytest.mark.parametrize("M,N,K,bns", RES_SHAPES, ids=["small", "m1", "m300", "m1000", "vit-o", "vit-fc2", "vit-fc2-8f", "7b-o",
                                                        "7b-down", "13b-down", "ragged-down"])
def test_gemm_bias_residual_stats(M, N, K, bns):
    """EPI_BIAS_RES_STATS (ViT out_proj / fc2, LLaMA o_proj / down_proj): out = bf16(acc + bias + residual), also in place,
    and stats_out [M, ceil(N / BN)] = per-tile (sum, sumsq) of the ROUNDED outputs -- what every norm-folded GEMM after it
    reads.  Output bound: BF |ref| + (1 + BF) (A + 2 U (|acc + bias| + |res|)).  Statistics: each partial against the float64
    sum over its tile's columns of the kernel's own bf16 outputs, within (n/2 + 2) U sum |o|.  Negative controls: the last K
    block dropped (output); a tile's last 32-column chunk missing, and another row's partials (statistics).  Two identical
    calls give identical bits; the in-place call gives the same bits as the out-of-place one."""
    name = "gemm_bias_residual_stats"
    A, W = _rows(M, K, 4), _weights(N, K, 5, 0.05)
    a64, w64 = A.double(), W.double()
    y, Aerr = a64 @ w64.T, _acc_err(a64, w64)
    res = _rows(M, N, 6)
    for bn in bns:
        for with_bias in (True, False):
            bias = _vec(N, 7) if with_bias else None
            yb = y + (bias.double() if with_bias else 0)
            ref = yb + res.double()
            tol = BF * ref.abs() + (1 + BF) * (Aerr + 2 * U * (yb.abs() + res.double().abs()))
            out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
            st = torch.full((M, _cdiv(N, bn), 2), float("nan"), device="cuda")
            _gemm(RES_STATS, A, W, out, bn, bias=bias, res=res, stats_out=st)
            _note(name, out, ref, tol)
            assert _excess(out, ref - _last_block(a64, w64), tol) > 0, (bn, with_bias)
            sref, stol, short = _res_stats_ref(out, bn)
            _note(name + " (stats_out)", st, sref, stol)
            assert _excess(st, short, stol) > 0, bn
            if M > 1:
                assert _excess(st, sref.roll(1, 0), stol) > 0, bn
            inplace, st2 = res.clone(), torch.empty_like(st)
            _gemm(RES_STATS, A, W, inplace, bn, bias=bias, res=inplace, stats_out=st2)
            assert torch.equal(inplace, out) and torch.equal(st2, st), bn
            again, st3 = torch.empty_like(out), torch.empty_like(st)
            _gemm(RES_STATS, A, W, again, bn, bias=bias, res=res, stats_out=st3)
            assert torch.equal(again, out) and torch.equal(st3, st), bn
    _report(name)
    _report(name + " (stats_out)")


# ============================================================================================================================
# EPI_LN_BIAS / EPI_LN_BIAS_GELU
# ============================================================================================================================
def _fold(W, gamma, beta, b):
    """what pack_rows_kernel loads: W' = bf16(W gamma), colsum = sum_k W' (fp32), b' = b + W beta (fp32)"""
    w64 = W.double()
    Wf = (W.float() * gamma).bfloat16()
    return Wf, Wf.double().sum(1).float(), (b.double() + w64 @ beta.double()).float()


LN_CASES = [(LN_BIAS, 1, 3072), (LN_BIAS, 77, 1032), (LN_BIAS, 257, 3072), (LN_BIAS, 2056, 3072), (LN_GELU, 1, 4096),
            (LN_GELU, 300, 4096), (LN_GELU, 257, 4096), (LN_GELU, 2056, 4096)]


@pytest.mark.parametrize("epi,M,N", LN_CASES, ids=["qkv-m1", "n-tail-m77", "qkv-1f", "qkv-8f", "fc1-m1", "fc1-m300", "fc1-1f",
                                                    "fc1-8f"])
def test_gemm_layernorm(epi, M, N):
    """EPI_LN_BIAS (ViT q/k/v) and EPI_LN_BIAS_GELU (ViT fc1), K = 1024, against two references on the same data.

    (a) The kernel's stated formula t = rstd (x W'^T - mean colsum) + b' with mean / rstd from the float64 sum of the supplied
    partials.  Bound on t (fp32): rstd A (accumulation over the raw rows -- the LayerNorm fold), dr |t - b'| (rstd's error
    scales the centred term: nm = -mean rstd uses the same rstd), rstd (e_m + 2 U |mean|) |colsum| (mean's error and the
    rounding of nm), U (|b'| + |t|) (the two fmaf); e_m, dr from _ln.  LN_BIAS: out = bf16(t), tol = BF |ref| + (1 + BF)
    tol_t.  GELU: quick_gelu'(.) < 1.1, so tol = BF |ref| + (1 + BF) (1.1 tol_t + _act_err(t) + U |ref|).

    (b) What HF runs: quick_gelu(LN(x) W^T + b) from unfolded W, gamma, beta, with mean / var of the bf16 rows themselves.
    It differs from (a) by what is exactly known: the partials' statistics against the rows' (the change of (a) between the
    two, evaluated in float64), the fold's rounding rstd BF sum_k |x - mean| |W gamma|, colsum's fp32 rounding
    rstd |mean| U |colsum| and b''s U |b'|; GELU multiplies those by 1.1.

    The partials arrive both ways: hand-built (8 tiles of 128 columns; the whole row in partial 0 and zeros in the rest, as
    copy_rows_stats_kernel writes) and from the real chain (an EPI_BIAS_RES_STATS call of width BN feeding stats_in_nt =
    ceil(K / BN)).  Rows have scales 10^{0,3,-3,6} and common offsets of up to 30 standard deviations; W is scaled so that
    t reaches -10.  Negative controls: another row's statistics; only partial 0 of the split; quick_gelu with sigmoid(v) in
    place of sigmoid(1.702 v)."""
    name = "gemm_layernorm"
    K = 1024
    gelu = epi == LN_GELU
    W = _weights(N, K, 10, 4.0 / math.sqrt(K))
    gamma, beta, b = _vec(K, 11, 0.2, 1.0).bfloat16().float(), _vec(K, 12, 0.2).bfloat16().float(), _vec(N, 13, 0.5)
    Wf, colsum, bf = _fold(W, gamma, beta, b)
    w64, wf64, cs64, b64 = W.double(), Wf.double(), colsum.double()[None], bf.double()[None]
    wg64 = w64 * gamma.double()
    act = _qgelu if gelu else (lambda v: v)

    def formula(x64, mean, rstd):
        return rstd * (x64 @ wf64.T - mean * cs64) + b64

    def hf(x64):
        mu = x64.mean(1, keepdim=True)
        var = (x64 - mu).pow(2).mean(1, keepdim=True)
        ln = (x64 - mu) * torch.rsqrt(var + EPS) * gamma.double() + beta.double()
        return act(ln @ w64.T + b.double()[None]), mu, torch.rsqrt(var + EPS)

    # (x, partials, label): hand-built split / single on offset rows, and the chain through EPI_BIAS_RES_STATS
    inputs = []
    x = _rows(M, K, 14, offset=True)
    inputs += [(x, _partials(x, 128), "split"), (x, _partials(x, 2048, nt=_cdiv(K, 256)), "single")]
    a0, w0, r0 = _rows(M, 512, 15).float().mul(1e-3).bfloat16(), _weights(K, 512, 16, 0.02), _rows(M, K, 17, offset=True)
    for bn0 in (128, 256):
        xc = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
        stc = torch.empty(M, _cdiv(K, bn0), 2, device="cuda")
        _gemm(RES_STATS, a0, w0, xc, bn0, res=r0, stats_out=stc)
        inputs.append((xc, stc, f"chain{bn0}"))
    for x, st, label in inputs:
        x64 = x.double()
        mean, rstd, e_m, dr = _ln(st, K)
        t = formula(x64, mean, rstd)
        tol_t = rstd * _acc_err(x64, wf64) + dr * (t - b64).abs() + rstd * (e_m + 2 * U * mean.abs()) * cs64.abs() + \
            U * (b64.abs() + t.abs())
        ref = act(t)
        tol = BF * ref.abs() + (1 + BF) * ((1.1 * tol_t + _act_err(t) + U * ref.abs()) if gelu else tol_t)
        # (b): HF's operation; the known differences from (a) added to its bound
        ref_b, mu_x, rstd_x = hf(x64)
        t_x = formula(x64, mu_x, rstd_x)
        known = (t - t_x).abs() + rstd_x * BF * ((x64 - mu_x).abs() @ wg64.abs().T) + \
            rstd_x * mu_x.abs() * U * cs64.abs() + U * b64.abs()
        tol_b = tol + (1 + BF) * (1.1 if gelu else 1.0) * known
        for bn in ((128, 256) if N % 256 == 0 else (128,)):
            out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
            _gemm(epi, x, Wf, out, bn, bias=bf, colsum=colsum, stats=st)
            _note(name + " (a) kernel formula", out, ref, tol)
            _note(name + " (b) HF operation", out, ref_b, tol_b)
            if M > 1:
                assert _excess(out, act(formula(x64, mean.roll(1, 0), rstd.roll(1, 0))), tol) > 0, (label, bn)
            if label == "split":
                m0, r0_, _, _ = _ln(st[:, :1], K)
                assert _excess(out, act(formula(x64, m0, r0_)), tol) > 0, bn
            if gelu:
                assert _excess(out, _qgelu(t, 1.0), tol) > 0, (label, bn)
            again = torch.empty_like(out)
            _gemm(epi, x, Wf, again, bn, bias=bf, colsum=colsum, stats=st)
            assert torch.equal(again, out), (label, bn)
        if gelu:
            assert float(t.min()) < -8, float(t.min())        # the tanh.approx regime the bound's absolute term is for
    _report(name + " (a) kernel formula")
    _report(name + " (b) HF operation")


# ============================================================================================================================
# EPI_RMS_QKV_ROPE
# ============================================================================================================================
def _rope_rows(positions):
    """bf16-rounded (cos, sin) [len(positions), 64] of every position"""
    cs = [_rope_table(int(p)) for p in positions]
    return torch.stack([c for c, _ in cs]), torch.stack([s for _, s in cs])


@pytest.mark.parametrize("N,K", [(1536, 512), (12288, 4096), (15360, 5120)], ids=["tiny", "7b", "13b"])
def test_gemm_qkv_rope(N, K):
    """EPI_RMS_QKV_ROPE (LLaMA prefill q/k/v): rows [q | k | v] of nH heads in the pair-interleaved RoPE order; row m of A is
    token (b = m / S, s = m % S) at position past + s.  z = rstd acc; q and k pairs are rotated by the RoPE table at that
    position, (z0 c - z1 s, z1 c + z0 s); q goes to out [M, N/3], k and v to row past + s of batch row b of the caches
    [B, nH, Smax, 128].  Bound: BF |ref| + |c| e0 + |s| e1 + 3 U (|z0 c| + |z1 s|) + (ulp(c) + ulp(s)) (|z0| + |z1|) with
    e = rstd A + (dr + U) |z| the error of z (dr from _rms); v: BF |ref| + e.  Every other cache row keeps its bit pattern
    (NaN patterns included).  past in {0, 1, 63, 130}, S in {77, 130} (not multiples of 128), B = 1..3, both tile widths.
    Negative controls: RoPE at position +- 1; K/V rows of the wrong batch row; another row's rstd.  Two identical calls give
    identical bits."""
    name = "gemm_qkv_rope"
    H = N // 3
    nH, Smax = H // 128, 512
    W = _weights(N, K, 20, 0.02)
    w64 = W.double()
    for i, (B, S, past) in enumerate([(1, 77, 0), (2, 77, 1), (3, 130, 63), (2, 130, 130), (1, 130, 1)]):
        M = B * S
        x = _rows(M, K, 21 + i)
        st = _partials(x, 256)
        x64 = x.double()
        rstd, dr = _rms(st, K)
        z = (x64 @ w64.T) * rstd
        ez = rstd * _acc_err(x64, w64) + (dr + U) * z.abs()
        sidx = torch.arange(M, device="cuda") % S                       # row m is token s = m % S at position past + s

        def rope(zz, ee, shift=0):
            c, s = _rope_rows(range(past + shift, past + shift + S))
            c, s = c[sidx][:, None], s[sidx][:, None]
            z0, z1, e0, e1 = zz[..., 0], zz[..., 1], ee[..., 0], ee[..., 1]
            r = torch.stack([z0 * c - z1 * s, z1 * c + z0 * s], -1)
            err = c.abs() * e0 + s.abs() * e1 + 3 * U * ((z0 * c).abs() + (z1 * s).abs()) + \
                (_bf16_ulp(c) + _bf16_ulp(s)) * (z0.abs() + z1.abs())
            return r, torch.stack([err, err], -1)

        zv, ev = z.view(M, 3, nH, 64, 2), ez.view(M, 3, nH, 64, 2)
        rq, eq = rope(zv[:, 0], ev[:, 0])
        rk, ek = rope(zv[:, 1], ev[:, 1])
        ref = torch.stack([rq, rk, zv[:, 2]], 1).reshape(M, 3, H)
        tol = BF * ref.abs() + torch.stack([eq, ek, ev[:, 2]], 1).reshape(M, 3, H)
        shift = -1 if past > 0 else 1
        bad_rope = torch.stack([rope(zv[:, 0], ev[:, 0], shift)[0], rope(zv[:, 1], ev[:, 1], shift)[0], zv[:, 2]], 1).reshape(M, 3, H)
        bad_row = ref.view(B, S, 3, H).roll(1, 0).view(M, 3, H)
        keep = torch.ones(Smax, dtype=torch.bool, device="cuda")
        keep[past:past + S] = False
        for bn in (128, 256):
            kc, vc = _pattern(B, nH, Smax, 1), _pattern(B, nH, Smax, 2)
            kc0, vc0 = kc.clone(), vc.clone()
            q = torch.full((M, H), float("nan"), dtype=torch.bfloat16, device="cuda")
            _gemm(QKV_ROPE, x, W, q, bn, stats=st, kc=kc, vc=vc, S=S, past=past, Smax=Smax)
            rows = lambda c: c[:, :, past:past + S].permute(0, 2, 1, 3).reshape(M, H)
            got = torch.stack([q, rows(kc), rows(vc)], 1)
            _note(name, got, ref, tol)
            assert _excess(got, bad_rope, tol) > 0, (B, S, past, bn)
            if B > 1:
                assert _excess(got[:, 1:], bad_row[:, 1:], tol[:, 1:]) > 0, (B, S, past, bn)
            if M > 1:
                assert _excess(got[:, 2], ref[:, 2] / rstd * rstd.roll(1, 0), tol[:, 2]) > 0, (B, S, past, bn)
            for cache, before in ((kc, kc0), (vc, vc0)):
                assert torch.equal(cache[:, :, keep].view(torch.int16), before[:, :, keep].view(torch.int16)), (B, S, past, bn)
            kc2, vc2 = _pattern(B, nH, Smax, 1), _pattern(B, nH, Smax, 2)
            q2 = torch.empty_like(q)
            _gemm(QKV_ROPE, x, W, q2, bn, stats=st, kc=kc2, vc=vc2, S=S, past=past, Smax=Smax)
            assert torch.equal(q2, q) and torch.equal(kc2.view(torch.int16), kc.view(torch.int16)) and \
                torch.equal(vc2.view(torch.int16), vc.view(torch.int16)), (B, S, past, bn)
    _report(name)


# ============================================================================================================================
# EPI_RMS_SWIGLU / EPI_RMS_F32
# ============================================================================================================================
@pytest.mark.parametrize("N,K", [(2048, 512), (22016, 4096), (27648, 5120)], ids=["tiny", "7b", "13b"])
def test_gemm_swiglu(N, K):
    """EPI_RMS_SWIGLU (LLaMA gate/up, columns (2j, 2j+1) = (gate j, up j)): out [M, N/2] = bf16(silu(g) u) with g = rstd acc[2j],
    u = rstd acc[2j+1] in fp32 -- unlike the decode GEMV, g and u are NOT rounded to bf16, so the reference is silu(g) u on the
    float64 g, u.  With dg, du = rstd A + (dr + U) |.| the errors of g, u: bound BF |ref| + (1 + BF) (1.1 dg |u| +
    |silu(g)| du + 1.1 dg du + _act_err(g) (|u| + du) + 2 U |silu(g) u|) (|silu'| < 1.1; tanh.approx; the fmaf and the
    product).  W is scaled so that g reaches -10.  M in {1, 77, 300}, both tile widths.  Negative controls: another row's
    rstd; the last K block dropped.  Two identical calls give identical bits."""
    name = "gemm_swiglu"
    W = _weights(N, K, 30, 3.5 / math.sqrt(K))
    w64 = W.double()
    for M in (1, 77, 300):
        x = _rows(M, K, 31 + M)
        st = _partials(x, 256)
        x64 = x.double()
        rstd, dr = _rms(st, K)

        def ref_tol(y):
            z = y * rstd
            g, u = z[:, 0::2], z[:, 1::2]
            e = rstd * _acc_err(x64, w64) + (dr + U) * z.abs()
            dg, du = e[:, 0::2], e[:, 1::2]
            sg = g * torch.sigmoid(g)
            ref = sg * u
            tol = BF * ref.abs() + (1 + BF) * (1.1 * dg * u.abs() + sg.abs() * du + 1.1 * dg * du + _act_err(g) * (u.abs() + du) +
                                               2 * U * ref.abs())
            return ref, tol, g

        y = x64 @ w64.T
        ref, tol, g = ref_tol(y)
        assert float(g.min()) < -8, float(g.min())
        for bn in (128, 256):
            out = torch.full((M, N // 2), float("nan"), dtype=torch.bfloat16, device="cuda")
            _gemm(SWIGLU, x, W, out, bn, stats=st)
            _note(name, out, ref, tol)
            assert _excess(out, ref_tol(y - _last_block(x64, w64))[0], tol) > 0, (M, bn)
            if M > 1:
                assert _excess(out, ref_tol(y / rstd * rstd.roll(1, 0))[0], tol) > 0, (M, bn)
            again = torch.empty_like(out)
            _gemm(SWIGLU, x, W, again, bn, stats=st)
            assert torch.equal(again, out), (M, bn)
    _report(name)


@pytest.mark.parametrize("N,K,bns", [(1032, 512, (128,)), (32000, 4096, (256, 128)), (32008, 4096, (256, 128)),
                                     (32008, 5120, (256,)), (32005, 5120, (128, 256))],
                         ids=["tiny", "7b-32000", "7b", "13b", "n-tail"])
def test_gemm_rms_f32(N, K, bns):
    """EPI_RMS_F32 (lm_head over every position): out [M, N] fp32 = rstd acc, no output rounding.  Bound: rstd A + (dr + U) |ref|.
    The prefill launches BN = 256 at V = 32008 although 32008 % 256 != 0: the last tile has 8 live columns; N = 32005 also
    ends mid-chunk (scalar stores).  M in {1, 77, 300}.  Negative controls: another row's rstd; the last K block dropped.
    Two identical calls give identical bits."""
    name = "gemm_rms_f32"
    W = _weights(N, K, 40, 0.02)
    w64 = W.double()
    for M in (1, 77, 300):
        x = _rows(M, K, 41 + M)
        st = _partials(x, 256)
        x64 = x.double()
        rstd, dr = _rms(st, K)
        y = x64 @ w64.T
        ref = y * rstd
        tol = rstd * _acc_err(x64, w64) + (dr + U) * ref.abs()
        for bn in bns:
            out = torch.full((M, N), float("nan"), device="cuda")
            _gemm(RMS_F32, x, W, out, bn, stats=st)
            _note(name, out, ref, tol)
            assert _excess(out, (y - _last_block(x64, w64)) * rstd, tol) > 0, (M, bn)
            if M > 1:
                assert _excess(out, y * rstd.roll(1, 0), tol) > 0, (M, bn)
            again = torch.empty_like(out)
            _gemm(RMS_F32, x, W, again, bn, stats=st)
            assert torch.equal(again.view(torch.int32), out.view(torch.int32)), (M, bn)
    _report(name)


# ============================================================================================================================
# attention
# ============================================================================================================================
def _flash_ref(q, k, v, att, scale, depth_qk, nkv, variants=()):
    """float64 softmax(q k^T * scale) v over the attended keys of each query row and the bound of the flash loop
    (flash_attention_tile).  q [R, Q, d], k / v [R, L, d], att [R or 1, Q, L] bool.

    Score error (relative in log2 units is relative in natural units): the wgmma dot product over d (depth_qk = d/16 + 4
    steps, 2 U each) 2 depth_qk U sum |q k| scale, the fp32 * scale_log2e and the constant's rounding 2 U |s|, s - m
    U (|s| + max |s|); fast_exp2 (ex2.approx, 2 ulp) 4 U: e_w per weight, 2 e_w on the normalised weights.  alpha rescales
    o and the row sum by the same factor, so its ex2 error cancels in the ratio.  P V: every p is rounded to bf16 (BF) while the row sum adds the unrounded p -- BF
    sum p |v| / sum p; the wgmma accumulation over L keys and the per-block alpha rescale (2 ceil(L/16) + 2 nkv + 8) U on the
    same sum; the fp32 row sum, 17 nkv + 4 roundings deep, and the final reciprocal and multiply.  Output: BF |ref|.
    A query row with no attended key is exactly 0 (tol 0).  variants: extra attend masks whose references are returned too."""
    L = k.shape[1]
    s = (q @ k.transpose(1, 2)) * scale
    sabs = (q.abs() @ k.abs().transpose(1, 2)) * scale
    outs = []
    for i, a in enumerate((att,) + tuple(variants)):
        a = a.expand(s.shape)
        sm = s.masked_fill(~a, -float("inf"))
        p = torch.softmax(sm, -1).nan_to_num(0.0)
        ref = p @ v
        if i == 0:
            pv = p @ v.abs()
            fin = s.masked_fill(~a, 0.0)
            smax = fin.abs().amax(-1, keepdim=True)
            e_w = (2 * depth_qk * U * sabs + U * (3 * fin.abs() + smax) + 4 * U).masked_fill(~a, 0.0).amax(-1, keepdim=True)
            tol = (2 * e_w + BF + (2 * _cdiv(L, 16) + 2 * nkv + 8 + 17 * nkv + 4 + 4) * U) * pv + BF * ref.abs()
        outs.append(ref)
    return outs[0], tol, outs[1:]


def _prefill_attention(q, kc, vc, B, S, past, mask):
    m = _model()
    nH, Smax = kc.shape[1], kc.shape[2]
    out = torch.full((B * S, nH * 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    _lib.check(m._lib.vly_test_prefill_attention(m._ctx, q.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, S, past, nH, Smax,
                                                 _ptr(mask), out.data_ptr(), None))
    torch.cuda.synchronize()
    return out


def _prefill_cases(Smax):
    if Smax == 384:
        return [(p, s) for p in (0, 1, 63, 64, 130) for s in (1, 2, 63, 64, 65, 257) if p + s <= Smax]
    return [(p, s) for p in (0, 1, 64, 130, 1000) for s in (65, 257, 700)] + [(1000, s) for s in (1, 2, 63, 64)] + [(63, 700)]


@pytest.mark.parametrize("nH", [4, 32, 40])
def test_prefill_attention(nH):
    """llama_prefill_attention_kernel through vly_test_prefill_attention: query s of batch row b sits at position past + s
    and attends the keys k <= past + s of its row that the mask allows (HF's causal mask AND-ed with the 2-D attention_mask).
    B = 1..3, caches of 384 and 2048 rows, past in {0, 1, 63, 64, 130, 1000} x S in {1, 2, 63, 64, 65, 257, 700}; masks:
    none, left padding of 1 / 64 / 130 keys (whole 64-key blocks, and every key of the first query rows: those rows must be
    exactly 0), everything but the newest key, and keys 128..319 in the middle.  Cache rows at and beyond past + S hold
    3e4 -- finite, as the cache guarantees (P = 0 times V must stay 0).  Bound: _flash_ref with d = 128 (in the kernel's
    interleaved column order on both sides of q k^T, so the dot products are the same).  The reference is computed one
    batch row and a few heads at a time.  Negative controls, each over every (past, S) case: a query that also sees key
    q + 1; every query tile missing the last key block it loads (its diagonal block); the mask ignored.  Two identical calls give identical bits."""
    name = f"prefill_attention[nH={nH}]"
    scale = 1 / math.sqrt(128)
    for Smax in (384, 2048):
        for i, (past, S) in enumerate(_prefill_cases(Smax)):
            B = 1 + (i + nH) % 3
            L = past + S
            g = _gen(100 + i)
            q = (torch.randn(B * S, nH * 128, generator=g, device="cuda") * 2).bfloat16()
            kc = torch.randn(B, nH, Smax, 128, generator=g, device="cuda").bfloat16()
            vc = torch.randn(B, nH, Smax, 128, generator=g, device="cuda").bfloat16()
            kc[:, :, L:] = 3e4
            vc[:, :, L:] = 3e4
            nkv = _cdiv(L, 64)
            keys, rows = torch.arange(L, device="cuda")[None, :], torch.arange(S, device="cuda")[:, None]
            causal = keys <= past + rows                                                           # [S, L]
            # the first key of the last block each query tile loads (its diagonal block)
            diag = (past + torch.clamp((rows // 64 + 1) * 64, max=S) - 1) // 64 * 64
            kinds = ["none", "newest"] + [f"pad{p}" for p in (1, 64, 130) if p + 1 < L] + (["mid"] if L > 320 else [])
            ctrl = [-math.inf] * 3                  # the largest excess of each defective reference over this (past, S)
            for kind in kinds:
                mask = _attend(B, L, kind)
                out = _prefill_attention(q, kc, vc, B, S, past, mask)
                hc = max(1, (1 << 23) // (S * L))                      # heads per reference chunk: <= 8M scores
                for b in range(B):
                    att = causal if mask is None else causal & mask[b].bool()[None, :]
                    variants = [att | (keys == past + rows + 1), att & (keys < diag)] + ([causal] if mask is not None else [])
                    for h0 in range(0, nH, hc):
                        h1 = min(nH, h0 + hc)
                        qq = q[b * S:(b + 1) * S].double().view(S, nH, 128)[:, h0:h1].transpose(0, 1)
                        kk, vv = kc[b, h0:h1, :L].double(), vc[b, h0:h1, :L].double()
                        ref, tol, bad = _flash_ref(qq, kk, vv, att[None], scale, 128 // 16 + 4, nkv, [a[None] for a in variants])
                        got = out[b * S:(b + 1) * S].view(S, nH, 128)[:, h0:h1].transpose(0, 1)
                        _note(name, got, ref, tol)
                        for c, r in enumerate(bad):
                            ctrl[c] = max(ctrl[c], _excess(got, r, tol))
                if kind == kinds[-1]:
                    assert torch.equal(_prefill_attention(q, kc, vc, B, S, past, mask), out), (Smax, past, S, kind)
            # (one masked key among a thousand, or one more, moves the output less than the bound: each control is asked of
            # the case as a whole, whose "newest" mask leaves single keys visible)
            assert S == 1 or ctrl[0] > 0, (Smax, past, S)
            assert ctrl[1] > 0, (Smax, past, S)
            assert L == 1 or ctrl[2] > 0, (Smax, past, S)
    _report(name)
