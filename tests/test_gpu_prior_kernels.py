"""GPU: the diffusion prior's three kernels (csrc/k2_prior.cu) against float64 evaluations of the same fp16 inputs, at the
prior's real geometry (T = 77 + 4 = 81 tokens, 32 heads, width 2048) and at the edges where they go wrong.

Every bound is in fp16 ulps of the float64 reference value (`_ulp16`: 2^-24 in the subnormal range) plus, where the kernel's
fp32 arithmetic can legitimately move a result that cancels to near zero, an absolute term derived next to the assertion.
Each test prints its worst error in ulps (run with -s to see them)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.attention_ref import _ulp16
from tests.attention_ref import check_attention_small as _check_attention
from tests.test_gpu_kernel_bounds import _bits, _Guarded

pytestmark = pytest.mark.gpu

INF = float("inf")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------------
# attention_small
# ------------------------------------------------------------------------------------------------------------------------------
def _qkv(B, T, heads, seed, std=1.0):
    return (torch.randn(B, T, heads * 192, device="cuda", generator=_gen(seed)) * std).half()


def _prefix_keep(lengths, T):
    """keep rows that keep the first `l` tokens of each row (CLIP-style padding at the end)."""
    return (torch.arange(T, device="cuda")[None, :] < torch.tensor(lengths, device="cuda")[:, None]).to(torch.uint8)


@pytest.mark.parametrize("B", [1, 2, 8])
@pytest.mark.parametrize("heads", [1, 3, 32])
@pytest.mark.parametrize("T", [1, 2, 31, 32, 33, 63, 64, 65, 81, 96, 127, 128])
def test_attention_small_lengths_vs_float64(T, heads, B):
    """Every 32-key chunk boundary and the prior's 81 tokens; causal on and off, without a mask, with per-row prefix masks
    (causal) and with masks that have holes (not causal).  Scores of std ~2.3."""
    from kandinsky2 import ops
    qkv = _qkv(B, T, heads, seed=T * 100 + heads * 10 + B, std=1.5)
    g = torch.Generator(device="cuda").manual_seed(T + heads + B)
    prefix = _prefix_keep(torch.randint(1, T + 1, (B,), device="cuda", generator=g).tolist(), T)
    holes = (torch.rand(B, T, device="cuda", generator=g) < 0.6).to(torch.uint8)
    holes[torch.arange(B), torch.randint(0, T, (B,), device="cuda", generator=g)] = 1   # every row keeps at least one key
    ulps, share = 0.0, 0.0
    for causal, keep in ((True, None), (False, None), (True, prefix), (False, holes)):
        out = ops.attention_small(qkv, heads, keep_mask=keep, causal=causal)
        u, s = _check_attention(out, qkv, heads, keep, causal, 0.125, (causal, keep is not None))
        ulps, share = max(ulps, u), max(share, s)
    print(f"attention_small T={T} heads={heads} B={B}: worst {ulps:.2f} ulp, {share:.2f} of the bound")


@pytest.mark.parametrize("B", [1, 2, 4])
@pytest.mark.parametrize("prompt_len", [2, 12, 77])
def test_attention_small_clip_masks_at_prior_geometry(prompt_len, B):
    """The prior's own attention: 77 text tokens + 4 always-kept extension tokens, 32 heads, causal, the keep mask of the
    classifier-free batch [prompt x B | "" x B] (the empty prompt keeps its start and end tokens only)."""
    from kandinsky2 import ops
    T, heads = 81, 32
    text = _prefix_keep([prompt_len] * B + [2] * B, 77)
    keep = F.pad(text, (0, 4), value=1).contiguous()
    qkv = _qkv(2 * B, T, heads, seed=prompt_len * 10 + B, std=1.5)
    out = ops.attention_small(qkv, heads, keep_mask=keep, causal=True)
    ulps, share = _check_attention(out, qkv, heads, keep, True, 0.125, "clip")
    # the same call with a bool mask (what PriorTransformer builds before its uint8 cast) gives the same bits
    assert torch.equal(_bits(ops.attention_small(qkv, heads, keep_mask=keep.bool(), causal=True)), _bits(out))
    print(f"attention_small CLIP mask prompt_len={prompt_len} B={B}: worst {ulps:.2f} ulp, {share:.2f} of the bound")


@pytest.mark.parametrize("causal", [True, False])
def test_attention_small_large_scores_and_masked_maximum(causal):
    """Scores spanning about +-60, and a masked key whose score is the largest of most rows: the row maximum must come from
    the reachable keys only (a maximum taken over a masked key would underflow every weight of the row)."""
    from kandinsky2 import ops
    B, T, heads = 2, 81, 3
    g = _gen(7)
    a = 4.5                                                           # score std 0.125 * 8 * a^2 ~ 20
    common = torch.randn(B, 1, heads, 64, device="cuda", generator=g).sign()
    q = a * (0.5 * common + 0.87 * torch.randn(B, T, heads, 64, device="cuda", generator=g))
    k = a * torch.randn(B, T, heads, 64, device="cuda", generator=g)
    v = torch.randn(B, T, heads, 64, device="cuda", generator=g)
    keep = torch.ones(B, T, dtype=torch.uint8, device="cuda")
    masked = [1, 3, 30] if causal else [5, 40, 70]
    keep[:, masked] = 0
    k[:, masked] = a * common.expand(B, len(masked), heads, 64)          # aligned with every query: score ~ +80
    qkv = torch.cat([q, k, v], -1).reshape(B, T, heads * 192).half()
    s = torch.einsum("bthc,bshc->bhts", *[t.double() for t in qkv.view(B, T, heads, 192).split(64, -1)[:2]]) * 0.125
    unmasked = s[keep[:, None, None, :].expand_as(s).bool()]
    assert unmasked.max().item() > 50 and unmasked.min().item() < -50, (unmasked.min().item(), unmasked.max().item())
    if causal:
        s = s + torch.full((T, T), -INF, dtype=torch.float64, device="cuda").triu(1)
    top_is_masked = (keep[:, None, None, :].expand_as(s).gather(-1, s.argmax(-1, keepdim=True)) == 0).double().mean().item()
    assert top_is_masked > 0.5, top_is_masked
    out = ops.attention_small(qkv, heads, keep_mask=keep, causal=causal)
    ulps, share = _check_attention(out, qkv, heads, keep, causal, 0.125, "large scores")
    print(f"attention_small scores +-60, causal={causal}: worst {ulps:.2f} ulp, {share:.2f} of the bound "
          f"({top_is_masked:.0%} of rows peak on a masked key)")


def test_attention_small_unreachable_rows_are_nan():
    """Contract: a query row with no reachable key is NaN in all its 64 channels, as torch's softmax over an all -inf row is;
    the other rows of the same (batch, head) are unaffected."""
    from kandinsky2 import ops
    B, T, heads = 3, 40, 2
    qkv = _qkv(B, T, heads, seed=11)
    keep = torch.ones(B, T, dtype=torch.uint8, device="cuda")
    keep[0, :3] = 0             # causal: rows 0..2 of image 0 reach nothing
    keep[1, :] = 0              # every row of image 1 reaches nothing
    keep[2, 1::2] = 0
    for causal in (True, False):
        out = ops.attention_small(qkv, heads, keep_mask=keep, causal=causal).view(B, T, heads, 64)
        nan = torch.isnan(out)
        assert nan[1].all()
        assert bool(nan[0, :3].all()) == causal and not nan[0, 3:].any()
        assert not nan[2].any()
        _check_attention(out.view(B, T, heads * 64), qkv, heads, keep, causal, 0.125, "unreachable")


@pytest.mark.parametrize("B,T,heads", [(2, 81, 32), (3, 33, 3), (1, 128, 1)])
def test_attention_small_strided_bounds(B, T, heads):
    """qkv as a channel slice of a wider row (ldq > heads*192, starting 16 channels in), the output into a slice of a wider
    row (ldo > heads*64, 8 channels in); NaN in the gap columns and in guard rows before and after, a fill pattern around
    the output that must survive; the result is the contiguous call's, bit for bit."""
    from kandinsky2 import ops
    qkv = _qkv(B, T, heads, seed=B * T + heads, std=1.5)
    keep = _prefix_keep([min(T, 5 + 3 * b) for b in range(B)], T)
    Cq, Co = heads * 192, heads * 64
    gq = _Guarded((B, T), 16 + Cq, 16 + Cq + 40)
    gq.view[..., 16:] = qkv
    go = _Guarded((B, T), 8 + Co, 8 + Co + 24, out=True)
    go.inside[go.guard:go.guard + B * T * go.ld].view(B * T, go.ld)[:, :8] = False   # the 8 leading columns are not output
    ops.attention_small(gq.view[..., 16:], heads, keep_mask=keep, causal=True, out=go.view[..., 8:])
    y_c = ops.attention_small(qkv, heads, keep_mask=keep, causal=True)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    assert torch.equal(_bits(go.view[..., 8:].contiguous()), _bits(y_c)), "strided result differs from the contiguous call"
    _check_attention(y_c, qkv, heads, keep, True, 0.125, "strided")


# ------------------------------------------------------------------------------------------------------------------------------
# layernorm_f16
# ------------------------------------------------------------------------------------------------------------------------------
def _ln_rows(kind, M, N, seed):
    g = _gen(seed)
    x = torch.randn(M, N, device="cuda", generator=g, dtype=torch.float64)
    sign = torch.where(torch.arange(M, device="cuda") % 2 == 0, 1.0, -1.0).double()[:, None]
    if kind == "offset":        # mean / std in {10, 100, 300, 1000}, both signs: the one-pass fp32 variance cancels
        ratio = torch.tensor([10.0, 100.0, 300.0, 1000.0], device="cuda", dtype=torch.float64)[torch.arange(M, device="cuda") % 4]
        x = x + sign * ratio[:, None]
    elif kind == "constant":    # x - mean = 0 exactly: the output is fp16(beta) whatever eps does
        x = (torch.tensor([0.0, 0.3, -7.5, 1000.0, 65504.0], device="cuda", dtype=torch.float64)[torch.arange(M, device="cuda") % 5])[:, None].expand(M, N)
    elif kind == "massive":     # one channel of +-3e4 in an otherwise O(1) row
        x[torch.arange(M, device="cuda"), torch.arange(M, device="cuda") * 7 % N] = sign[:, 0] * 3e4
    elif kind == "tiny_var":    # variance ~4e-6 < eps = 1e-5: eps decides rstd
        x = 1.0 + 2e-3 * x
    return x.half()


@pytest.mark.parametrize("kind", ["randn", "offset", "constant", "massive", "tiny_var"])
@pytest.mark.parametrize("M", [1, 81, 648])
@pytest.mark.parametrize("N", [1, 128, 200, 768, 2048, 2049])
def test_layernorm_f16_vs_float64(N, M, kind):
    from kandinsky2 import ops
    x = _ln_rows(kind, M, N, seed=N + M)
    g = _gen(N * 3 + 1)
    gamma = torch.randn(N, device="cuda", generator=g)
    beta = torch.randn(N, device="cuda", generator=g)
    y = ops.layernorm_f16(x, gamma, beta).double()
    xd = x.double()
    ref = F.layer_norm(xd, (N,), gamma.double(), beta.double(), eps=1e-5)
    if kind == "constant" or N == 1:
        assert torch.equal(_bits(y.half()), _bits(beta.half().expand(M, N))), "constant rows must give fp16(beta) exactly"
    xhat = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    # The kernel's statistics are float64 (exact mean of fp16 inputs, centred variance); x_hat is rounded to fp32 and
    # gamma * x_hat + beta is one fp32 fma: <= 2^-23 (|gamma x_hat| + |beta|) before the fp16 rounding, which is half an ulp.
    # 2^-20 leaves room for the fp32 gain and bias products without letting a wrong mean or rstd through: a mean off by
    # d * std moves every output by d |gamma|.
    allow = _ulp16(ref) + 2.0 ** -20 * ((gamma.double() * xhat).abs() + beta.double().abs())
    err = (y - ref).abs()
    bad = err > allow
    assert not bad.any(), (kind, int(bad.sum()), err[bad][:4].tolist(), ref[bad][:4].tolist())
    print(f"layernorm_f16 N={N} M={M} {kind}: worst {(err / _ulp16(ref)).max().item():.3f} ulp")


def test_layernorm_f16_in_place():
    """PriorTransformer never does it, but the kernel reads each element before the same thread writes it: y = x is safe."""
    from kandinsky2 import ops
    x = _ln_rows("offset", 81, 2048, seed=5)
    gamma, beta = torch.randn(2048, device="cuda", generator=_gen(6)), torch.randn(2048, device="cuda", generator=_gen(7))
    ref = ops.layernorm_f16(x, gamma, beta)
    ops.layernorm_f16(x, gamma, beta, out=x)
    assert torch.equal(_bits(x), _bits(ref))


# ------------------------------------------------------------------------------------------------------------------------------
# gelu_f16_
# ------------------------------------------------------------------------------------------------------------------------------
def test_gelu_f16_every_fp16_value():
    """All 65536 fp16 bit patterns in one call, against float64 0.5 x erfc(-x / sqrt 2).  Finite inputs: within one ulp of
    the float64 value (correct rounding, or the neighbouring fp16 value when the float64 value sits within fp32 error of a
    rounding tie).  +inf -> +inf, -inf -> NaN and NaN -> NaN, as torch's fp32 GELU gives."""
    from kandinsky2 import ops
    x = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.float16).clone()
    y = ops.gelu_f16_(x.clone())
    fin = torch.isfinite(x)
    t32 = F.gelu(x[~fin].float())
    assert torch.equal(torch.isnan(y[~fin]), torch.isnan(t32)) and torch.equal(y[~fin].float()[~torch.isnan(t32)],
                                                                               t32[~torch.isnan(t32)])
    xd = x[fin].double()
    ref = 0.5 * xd * torch.special.erfc(-xd / math.sqrt(2.0))
    got = y[fin].double()
    err = (got - ref).abs()
    ulps = err / _ulp16(ref)
    worst = ulps.argmax()
    exact = (got == ref.half().double()).double().mean().item()
    print(f"gelu_f16: worst {ulps[worst].item():.3f} ulp at x = {xd[worst].item()!r}; {exact:.4%} correctly rounded")
    assert ulps.max().item() <= 1.0, (xd[ulps > 1][:6].tolist(), got[ulps > 1][:6].tolist(), ref[ulps > 1][:6].tolist())
