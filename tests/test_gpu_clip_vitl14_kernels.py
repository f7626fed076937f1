"""GPU: the kernels the Kandinsky 2.1 ViT-L/14 towers add or use at a new geometry (kandinsky2/model/clip_vitl14.py), against
float64 evaluations of the same fp16 inputs:
  - k2_quick_gelu_f16 (csrc/k2_prior.cu) over every fp16 bit pattern, in place and out of place, with guard elements;
  - k2_attention_d64 at the image tower's geometry: 257 tokens (a ragged last key block) and around it, no encoder tokens,
    16 heads of 64, B = 1..4, with tests/attention_ref.py's bound.
Each test prints its worst error (run with -s to see it)."""
import pytest
import torch

from tests.attention_ref import check_d64
from tests.test_gpu_kernel_bounds import _bits, _Guarded
from tests.test_gpu_prior_kernels import _ulp16

pytestmark = pytest.mark.gpu


def _all_fp16():
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.float16).clone()


def test_quick_gelu_f16_every_fp16_value():
    """All 65536 fp16 bit patterns in one call against float64 x sigmoid(1.702 x) = x / (1 + exp(-1.702 x)).  Finite inputs:
    within one ulp of the float64 value.  +inf -> +inf, -inf -> NaN, NaN -> NaN, as torch's fp32 x * sigmoid(1.702 x)."""
    from kandinsky2 import ops
    x = _all_fp16()
    y = ops.quick_gelu_f16_(x.clone())
    fin = torch.isfinite(x)
    xf = x[~fin].float()
    t32 = xf * torch.sigmoid(1.702 * xf)
    nan = torch.isnan(t32)
    assert torch.equal(torch.isnan(y[~fin]), nan) and torch.equal(y[~fin].float()[~nan], t32[~nan])
    xd = x[fin].double()
    ref = xd * torch.sigmoid(1.702 * xd)
    got = y[fin].double()
    ulps = (got - ref).abs() / _ulp16(ref)
    worst = ulps.argmax()
    exact = (got == ref.half().double()).double().mean().item()
    print(f"quick_gelu_f16: worst {ulps[worst].item():.3f} ulp at x = {xd[worst].item()!r}; {exact:.4%} correctly rounded")
    assert ulps.max().item() <= 1.0, (xd[ulps > 1][:6].tolist(), got[ulps > 1][:6].tolist(), ref[ulps > 1][:6].tolist())


@pytest.mark.parametrize("n", [2, 4098, 1 << 20, 77 * 2 * 3072])
def test_quick_gelu_f16_in_and_out_of_place_with_guards(n):
    """Out of place into a guarded buffer: the n outputs equal the in-place result bit for bit, the input is unchanged and no
    element around the output is touched."""
    from kandinsky2 import ops
    x = _all_fp16().repeat(n // 65536 + 1)[:n].view(1, n)
    x = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
    src = x.clone()
    out = _Guarded((1,), n, out=True)
    ops.quick_gelu_f16_(x, out=out.view)
    assert torch.equal(_bits(x), _bits(src))
    out.untouched()
    inplace = ops.quick_gelu_f16_(src.clone())
    assert torch.equal(_bits(out.view.contiguous()), _bits(inplace))


@pytest.mark.parametrize("B", [1, 2, 3, 4])
@pytest.mark.parametrize("T", [255, 256, 257, 258, 129])
def test_attention_d64_image_tower_geometry(B, T):
    """k2_attention_d64 as the ViT-L/14 image tower calls it: qkv [B, T, 16 * 192] per head [q | k | v], no encoder tokens,
    scale 1/8.  T = 257 is the tower's (256 patches + CLS): its last key block holds one key."""
    from kandinsky2 import ops
    heads = 16
    g = torch.Generator(device="cuda").manual_seed(1000 * B + T)
    qkv = (torch.randn(B, T, heads * 192, device="cuda", generator=g) * 1.5).half()
    out = _Guarded((B, T), heads * 64, out=True)
    ops.attention_d64(qkv, heads, None, scale=0.125, out=out.view)
    out.untouched()
    got = out.view.contiguous()
    assert torch.isfinite(got).all()
    ulps, share = check_d64(got, qkv, None, heads, ("vit-l/14", B, T))
    print(f"attention_d64 image tower B={B} T={T}: worst {ulps:.2f} ulp, {share:.3f} of the bound")
