"""GPU: the CLIP image tower's two kernels (csrc/k2_clip_vision.cu, csrc/k2_attention.cu at head width 104).

k2_attention_heads against a float64 evaluation of the same fp16 inputs, at the tower's 16 heads and token counts around it
(1, 17, 64, 65, 257, 577), scores up to +-60, on strided views: qkv heads 320 columns apart with NaN in the 8 gap columns of
each head and around the view, the output heads 112 apart inside a pre-filled buffer.  The bound is the one of
tests/test_gpu_prior_kernels.py (one fp16 ulp of the float64 value plus the first-order error of the fp32 scores and
weights) with two terms that recipe adds: P is rounded to fp16 before PV (2^-11 of sum_s p_s |v_s|, plus 2^-25 |v| per key for
weights in fp16's subnormal range), and the PV chain runs over up to 577 keys.

k2_clip_patchify bit for bit against the torch composition (pixels rounded to fp16 in (c, ky, kx) order, the one-hot CLS row,
zero padding to Kp), with guarded gaps around the output rows."""
import pytest
import torch

from tests.test_gpu_kernel_bounds import _Guarded, _bits
from tests.test_gpu_prior_kernels import _ulp16

pytestmark = pytest.mark.gpu

HD = 104


def _ref(qkv, heads, scale):
    """qkv fp16 [B, T, heads, 3 * HD] -> (float64 out [B, T, heads, HD], allowance)."""
    q, k, v = qkv.double().split(HD, -1)
    T = q.shape[1]
    s = torch.einsum("bthc,bshc->bhts", q, k) * scale
    p = torch.softmax(s, -1)
    o = torch.einsum("bhts,bshc->bthc", p, v)
    mx = s.amax(-1, keepdim=True).abs()
    eta = 2.0 ** -17 * scale * torch.einsum("bthc,bshc->bhts", q.abs(), k.abs()) + 2.0 ** -22 * (s.abs() + mx) + 2.0 ** -21
    mag = torch.einsum("bhts,bshc->bthc", p, v.abs())
    allow = (torch.einsum("bhts,bshc->bthc", p * eta, v.abs()) + (p * eta).sum(-1).transpose(1, 2)[..., None] * o.abs()
             + (2.0 ** -11 + (T + 16) * 2.0 ** -24) * mag + T * 2.0 ** -25 * v.abs().amax(1, keepdim=True))
    return o, allow


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 17, 64, 65, 257, 577])
def test_attention_heads_vs_float64(T, B):
    from kandinsky2 import ops
    heads, hs, ohs, scale = 16, 320, 112, HD ** -0.5
    worst = 0.0
    for std in (1.0, 3.2):                      # std 3.2: scores reach +-60
        g = torch.Generator(device="cuda").manual_seed(T * 10 + B + int(std))
        data = torch.randn(B, T, heads, hs, device="cuda", generator=g) * std
        data[..., 2 * HD:] = data[..., 2 * HD:] / std   # values of unit scale
        data[..., 3 * HD:] = float("nan")             # the gap columns of every head
        data = data.half()
        gq = _Guarded.of(data.reshape(B, T, heads * hs), ld=heads * hs + 8)
        go = _Guarded((B, T), heads * ohs, ld=heads * ohs + 16, out=True)
        ops.attention_heads(gq.view, heads, HD, scale, out=go.view, hs=hs, ohs=ohs)
        torch.cuda.synchronize()
        ok, msg = go.untouched()
        assert ok, msg
        got = go.view.reshape(B, T, heads, ohs)
        assert (_bits(got[..., HD:]) == go.bits).all(), "the 8 columns after each output head were written"
        ref, allow = _ref(data[..., :3 * HD], heads, scale)
        got = got[..., :HD].double()
        err = (got - ref).abs()
        bound = _ulp16(ref) + allow
        assert torch.isfinite(got).all()
        assert not (err > bound).any(), (std, int((err > bound).sum()), err.max().item())
        worst = max(worst, (err / bound).max().item())
        if std > 1 and T >= 17:
            q, k = data[..., :HD].double(), data[..., HD:2 * HD].double()
            assert (torch.einsum("bthc,bshc->bhts", q, k) * scale).abs().max() > 40
        # the contiguous call gives the same bits
        flat = ops.attention_heads(data.reshape(B, T, heads * hs), heads, HD, scale, hs=hs)
        assert torch.equal(_bits(flat.reshape(B, T, heads, HD)), _bits(go.view.reshape(B, T, heads, ohs)[..., :HD]))
    print(f"attention_heads T={T} B={B}: {worst:.2f} of the bound")


@pytest.mark.parametrize("B,S,P", [(1, 224, 14), (3, 56, 14), (2, 70, 14), (2, 32, 8)])
def test_clip_patchify_bit_exact(B, S, P):
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(S + B)
    x = torch.randn(B, 3, S, S, device="cuda", generator=g) * 2.5
    x[0, 0, 0, :4] = torch.tensor([65519.0, 1e-7, -3e-5, 0.1], device="cuda")   # overflow edge, subnormals, rounding
    K = 3 * P * P
    kp = (K + 1 + 63) // 64 * 64
    G = S // P
    T = G * G + 1
    go = _Guarded((B, T), kp, ld=kp + 24, out=True)
    ops.clip_patchify(x, P, kp, out=go.view)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    ref = torch.zeros(B, T, kp, dtype=torch.float16, device="cuda")
    ref[:, 0, K] = 1.0
    ref[:, 1:, :K] = x.half().reshape(B, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(B, G * G, K)
    assert torch.equal(_bits(go.view), _bits(ref))
