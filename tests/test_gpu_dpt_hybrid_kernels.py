"""GPU: the BiT kernels of the hybrid DPT (csrc/k2_bit.cu).

  - k2_im2col_f16 bit for bit against F.unfold of the zero-padded input plus one fp16 rounding;
  - k2_maxpool_f16 bit for bit against F.pad(value=0) + max_pool2d on finite values, +-0 and +-inf;
  - k2_gn_act_f16 (GroupNorm + ReLU, + an fp16 shortcut, + a second GroupNorm) against float64 at the BiT geometry, rows offset
    by large means, within fp16-ulp bounds in the style of tests/test_gpu_groupnorm_float64.py;
  - all three on strided views with NaN-poisoned gaps: nothing outside the view is written."""
import pytest
import torch
import torch.nn.functional as F

from kandinsky2 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ulp(x):
    """The fp16 spacing at |x| (subnormal spacing below the normal range)."""
    a = x.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


@pytest.mark.parametrize("B,C,H,W,k,s,pt,pl,kp", [(2, 3, 64, 96, 7, 2, 2, 2, 192), (1, 3, 384, 384, 7, 2, 2, 2, 192),
                                                  (1, 5, 17, 11, 3, 1, 1, 1, 64)])
def test_im2col_bit_exact_against_unfold(B, C, H, W, k, s, pt, pl, kp):
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(B, C, H, W, device=DEV, generator=g) * 3
    Ho, Wo = -(-H // s), -(-W // s)
    pb, pr = (Ho - 1) * s + k - H - pt, (Wo - 1) * s + k - W - pl
    ref = F.unfold(F.pad(x, (pl, pr, pt, pb)), k, stride=s)               # [B, C k k, L]
    ref = ref.transpose(1, 2).reshape(B, Ho, Wo, C * k * k).half()
    buf = torch.full((B, Ho, Wo, kp + 24), float("nan"), device=DEV, dtype=torch.float16)
    out = ops.im2col_f16(x, k, s, (pt, pl), (Ho, Wo), kp, out=buf[..., 8:8 + kp])
    torch.cuda.synchronize()
    assert torch.equal(out[..., :C * k * k], ref)
    assert not out[..., C * k * k:].any()
    assert buf[..., :8].isnan().all() and buf[..., 8 + kp:].isnan().all()


def _maxpool_ref(x):
    """BitMaxPool2d on NHWC: F.pad(value=0) (0 before, 1 after on an even side) + max_pool2d(3, 2)."""
    y = F.max_pool2d(F.pad(x.permute(0, 3, 1, 2).float(), (0, 1, 0, 1), value=0.0), 3, 2)
    return y.permute(0, 2, 3, 1).half()


@pytest.mark.parametrize("B,H,W,C", [(2, 96, 96, 64), (1, 128, 192, 64), (3, 6, 4, 16)])
def test_maxpool_bit_exact_with_zero_pad(B, H, W, C):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = (torch.randn(B, H, W, C, device=DEV, generator=g) * 4 - 1).half()
    m = torch.rand(B, H, W, C, device=DEV, generator=g)
    x[m < 0.05] = 0.0
    x[(m >= 0.05) & (m < 0.1)] = -0.0
    x[(m >= 0.1) & (m < 0.12)] = float("inf")
    x[(m >= 0.12) & (m < 0.14)] = float("-inf")
    x[0, :, :, :8] = -1.0      # an all-negative channel block: the zero pad wins at the bottom / right edge
    xb = torch.full((B, H, W, C + 16), float("nan"), device=DEV, dtype=torch.float16)
    xb[..., :C] = x
    Ho, Wo = H // 2, W // 2
    yb = torch.full((B, Ho, Wo, C + 8), float("nan"), device=DEV, dtype=torch.float16)
    y = ops.maxpool_f16(xb[..., :C], (0, 0), (Ho, Wo), out=yb[..., :C])
    ref = _maxpool_ref(x)
    assert torch.equal(y.view(torch.int16), ref.view(torch.int16))   # bits: +0 / -0 included
    assert yb[..., C:].isnan().all()
    assert (y[0, -1, -1, :8] == 0).all()


def _gn64(x, gamma, beta, groups=32, eps=1e-5):
    B, H, W, C = x.shape
    xd = x.double().reshape(B, H * W, groups, C // groups)
    mean = xd.mean((1, 3), keepdim=True)
    var = ((xd - mean) ** 2).mean((1, 3), keepdim=True)
    return ((xd - mean) / torch.sqrt(var + eps)).reshape(B, H, W, C) * gamma.double() + beta.double()


_GEOM = [(1, 192, 192, 64), (1, 256, 256, 64), (2, 96, 96, 64), (2, 96, 96, 256), (1, 48, 48, 128), (2, 48, 48, 512),
         (1, 24, 24, 256), (2, 24, 24, 1024)]


@pytest.mark.parametrize("B,H,W,C", _GEOM)
@pytest.mark.parametrize("mode", ["relu", "shortcut", "norm_shortcut"])
def test_gn_act_against_float64(B, H, W, C, mode):
    g = torch.Generator(device=DEV).manual_seed(C + H)
    offs = torch.randn(1, 1, 1, C, device=DEV, generator=g) * 40       # rows offset by large means
    x = (torch.randn(B, H, W, C, device=DEV, generator=g) * 2 + offs).half()
    ga = 1 + 0.2 * torch.randn(C, device=DEV, generator=g)
    be = 0.2 * torch.randn(C, device=DEV, generator=g)
    st = ops.gn_stats(x, eps=1e-5)
    ref = _gn64(x, ga, be)
    r, r_norm = None, None
    if mode == "shortcut":
        r = torch.randn(B, H, W, C, device=DEV, generator=g).half()
        ref = ref + r.double()
    elif mode == "norm_shortcut":
        r = (torch.randn(B, H, W, C, device=DEV, generator=g) * 3 - offs).half()
        rg, rb = 1 + 0.2 * torch.randn(C, device=DEV, generator=g), 0.2 * torch.randn(C, device=DEV, generator=g)
        r_norm = (ops.gn_stats(r, eps=1e-5), rg, rb)
        ref = ref + _gn64(r, rg, rb)
    ref = ref.clamp_min(0)
    yb = torch.full((B, H, W, C + 8), float("nan"), device=DEV, dtype=torch.float16)
    y = ops.gn_act_f16(x, st, ga, be, r=r, r_norm=r_norm, out=yb[..., :C])
    torch.cuda.synchronize()
    assert yb[..., C:].isnan().all()
    err = (y.double() - ref).abs()
    # the fp32 statistics (mean / rstd rounded to fp32) and the fp32 affine cost a few fp32 ulps of the normalised value;
    # the result is then rounded once: within 1 fp16 ulp of the float64 value plus 1e-3 absolute
    bound = _ulp(ref) + 1e-3
    worst = (err / bound).max().item()
    print(f"gn_act {mode} {B}x{H}x{W}x{C}: worst {worst:.3f} of the bound")
    assert worst <= 1.0


def test_gn_act_into_token_rows_and_no_relu():
    B, gh, gw, C, kp = 2, 4, 6, 64, 128
    T = gh * gw + 1
    g = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(B, gh, gw, C, device=DEV, generator=g).half()
    ga, be = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
    st = ops.gn_stats(x)
    rows = torch.full((B, T, kp), float("nan"), device=DEV, dtype=torch.float16)
    view = rows.as_strided((B, gh, gw, C), (T * kp, gw * kp, kp, 1), kp)
    ops.gn_act_f16(x, st, ga, be, relu=False, out=view)
    want = ops.gn_act_f16(x, st, ga, be, relu=False)
    assert torch.equal(rows[:, 1:, :C].reshape(B, gh, gw, C), want)
    assert rows[:, 0].isnan().all() and rows[:, 1:, C:].isnan().all()
    assert (want < 0).any()
