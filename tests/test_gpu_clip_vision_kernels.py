"""GPU: the CLIP image tower's two kernels (csrc/k2_clip_vision.cu, csrc/k2_attention.cu at head width 104).

k2_attention_heads against a float64 evaluation of the same fp16 inputs, at the tower's 16 heads and token counts around it
(1, 17, 64, 65, 257, 577), scores up to +-60, on strided views: qkv heads 320 columns apart with NaN in the 8 gap columns of
each head and around the view, the output heads 112 apart inside a pre-filled buffer.  The bound is the fused attention
kernels' one (tests/attention_ref.py: one fp16 ulp of the float64 value plus the first-order error of the fp32 scores and
weights, P rounded to fp16 before PV and the PV chain), with a score chain of 104 terms.

k2_clip_patchify bit for bit against the torch composition (pixels rounded to fp16 in (c, ky, kx) order, the one-hot CLS row,
zero padding to Kp), with guarded gaps around the output rows."""
import pytest
import torch

from tests.attention_ref import check, ref_attention
from tests.test_gpu_kernel_bounds import _Guarded, _bits

pytestmark = pytest.mark.gpu

HD = 104


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, 17, 64, 65, 257, 577])
def test_attention_heads_vs_float64(T, B):
    from kandinsky2 import ops
    heads, hs, ohs, scale = 16, 320, 112, HD ** -0.5
    worst = worst_ulps = 0.0
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
        assert torch.isfinite(got[..., :HD]).all()
        for b in range(B):
            q, k, v = data[b, :, :, :3 * HD].split(HD, -1)
            ulps, share = check(got[b, ..., :HD], *ref_attention(q, k, v, scale), (std, b))
            worst, worst_ulps = max(worst, share), max(worst_ulps, ulps)
        if std > 1 and T >= 17:
            q, k = data[..., :HD].double(), data[..., HD:2 * HD].double()
            assert (torch.einsum("bthc,bshc->bhts", q, k) * scale).abs().max() > 40
        # the contiguous call gives the same bits
        flat = ops.attention_heads(data.reshape(B, T, heads * hs), heads, HD, scale, hs=hs)
        assert torch.equal(_bits(flat.reshape(B, T, heads, HD)), _bits(go.view.reshape(B, T, heads, ohs)[..., :HD]))
    print(f"attention_heads T={T} B={B}: worst {worst_ulps:.2f} ulp, {worst:.2f} of the bound")


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
