"""GPU: the DPT neck kernels of csrc/k2_depth.cu.

  - k2_relu_f16 over all 65,536 fp16 bit patterns and k2_relu_f32 on fp32 specials: bit for bit torch.relu on the same
    device, out of place on strided views and in place;
  - k2_bilinear_f16 against float64 (torch's interpolate in double) for x2 and arbitrary sizes, both align_corners, on
    strided views with NaN-poisoned gaps: within one fp16 ulp plus the fp32 index / weight error, and nothing outside the
    output view written;
  - k2_depth_to_space_f16 and k2_readout_rows_f16 bit for bit against the torch composition, on strided views."""
import pytest
import torch

from kandinsky2 import ops

pytestmark = pytest.mark.gpu


def _poisoned(shape, width, dtype=torch.float16):
    """A NaN-filled buffer [..., width] and its [..., shape[-1]] view (a row-strided view with poisoned gaps)."""
    buf = torch.full((*shape[:-1], width), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[..., :shape[-1]]


def test_relu_f16_all_bit_patterns():
    bits = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16)
    x = bits.view(torch.float16).reshape(256, 256)
    ref = torch.relu(x)
    buf, y = _poisoned((256, 256), 264)
    ops.relu_f16(x, out=y)
    assert torch.equal(y.view(torch.int16), ref.view(torch.int16))
    assert torch.isnan(buf[:, 256:]).all()
    xin = x.clone()
    ops.relu_f16(xin)                                                          # in place, 16-byte vectors
    assert torch.equal(xin.view(torch.int16), ref.view(torch.int16))
    odd = x[:, :255]                                                           # width 255: the scalar path
    out = torch.empty(256, 255, device="cuda", dtype=torch.float16)
    ops.relu_f16(odd, out=out)
    assert torch.equal(out.view(torch.int16), ref[:, :255].view(torch.int16))


def test_relu_f32_specials():
    vals = [0.0, -0.0, 1.0, -1.0, float("inf"), -float("inf"), float("nan"), -float("nan"), 1e-45, -1e-45, 3.4e38, -3.4e38]
    x = torch.tensor(vals * 8, device="cuda", dtype=torch.float32).reshape(8, 12)
    x.view(torch.int32)[0, 6] = 0x7fc12345                                      # a NaN with a payload keeps its bits
    ref = torch.relu(x)
    for view_w in (12, 16):
        buf = torch.full((8, view_w), float("nan"), device="cuda")
        y = buf[:, :12]
        ops.relu_f32(x, out=y)
        assert torch.equal(y.view(torch.int32), ref.view(torch.int32))
    xin = torch.randn(4, 1, 24, 24, device="cuda")
    r = torch.relu(xin)
    ops.relu_f32(xin)
    assert torch.equal(xin, r)


def _ulp16(v):
    """fp16 ulp of |v| (subnormal spacing below 2^-14), float64."""
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.pow(2.0, torch.floor(torch.log2(a)) - 10)


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("src,dst", [((5, 7), (10, 14)), ((12, 12), (24, 24)), ((5, 7), (6, 8)), ((12, 9), (7, 13)),
                                     ((1, 3), (4, 5)), ((9, 9), (5, 5)), ((24, 24), (48, 48))])
def test_bilinear_against_float64(src, dst, align):
    g = torch.Generator(device="cuda").manual_seed(src[0] * 100 + dst[1])
    B, C = 2, 40
    xbuf, x = _poisoned((B, *src, C), 48)
    x.copy_(torch.randn(B, *src, C, device="cuda", generator=g).half() * 3)
    ybuf, y = _poisoned((B, *dst, C), 56)
    ops.bilinear_f16(x, dst, align, out=y)
    assert torch.isnan(ybuf[..., C:]).all() and torch.isfinite(y).all()
    x64 = x.double().permute(0, 3, 1, 2)
    ref = torch.nn.functional.interpolate(x64.cpu(), size=dst, mode="bilinear", align_corners=align).cuda()
    ref = ref.permute(0, 2, 3, 1)
    # fp32 index arithmetic moves a source coordinate by a few 2^-24 of the size; the weights move as much, against a
    # corner difference of at most 2 max|x|; plus the fp32 sum of four terms and the fp16 rounding
    amax = x.abs().max().double()
    bound = _ulp16(ref) + 4 * max(src) * 2.0 ** -23 * 2 * amax + 4 * 2.0 ** -24 * amax
    err = (y.double() - ref).abs()
    print(f"bilinear {src}->{dst} align={align}: worst share of the bound {(err / bound).max().item():.3f}")
    assert (err <= bound).all()


def test_bilinear_align_corners_halving_of_an_odd_grid_picks_every_second_pixel():
    x = torch.randn(2, 5, 5, 16, device="cuda").half()
    y = ops.bilinear_f16(x, (3, 3), True)
    assert torch.equal(y, x[:, ::2, ::2])


@pytest.mark.parametrize("s", [4, 2])
def test_depth_to_space_bit_exact(s):
    B, G, C = 2, 5, 24
    gbuf, g = _poisoned((B, G, G, s * s * C), s * s * C + 8)
    g.copy_(torch.randn(B, G, G, s * s * C, device="cuda").half())
    ybuf, y = _poisoned((B, s * G, s * G, C), C + 16)
    ops.depth_to_space_f16(g, s, C, out=y)
    ref = g.reshape(B, G, G, s, s, C).permute(0, 1, 3, 2, 4, 5).reshape(B, s * G, s * G, C)
    assert torch.equal(y, ref) and torch.isnan(ybuf[..., C:]).all()


def test_depth_to_space_matches_conv_transpose():
    """The GEMM + scatter of a ConvTranspose2d(kernel = stride = 2): with exact operands it is torch's conv_transpose2d."""
    B, G, C, s = 1, 3, 16, 2
    x = torch.randint(-4, 5, (B, C, G, G), device="cuda").float()
    w = torch.randint(-4, 5, (C, C, s, s), device="cuda").float()
    b = torch.randint(-4, 5, (C,), device="cuda").float()
    ref = torch.nn.functional.conv_transpose2d(x, w, b, stride=s).permute(0, 2, 3, 1)
    gmat = x.permute(0, 2, 3, 1).reshape(-1, C) @ w.permute(2, 3, 1, 0).reshape(s * s * C, C).T + b.repeat(s * s)
    y = ops.depth_to_space_f16(gmat.reshape(B, G, G, s * s * C).half(), s, C)
    assert torch.equal(y.float(), ref)


def test_readout_rows_bit_exact():
    B, T, H = 3, 26, 64
    hbuf, h = _poisoned((B, T, H), H + 8)
    h.copy_(torch.randn(B, T, H, device="cuda").half())
    ybuf, y = _poisoned((B, T - 1, 2 * H), 2 * H + 24)
    ops.readout_rows_f16(h, out=y)
    ref = torch.cat([h[:, 1:], h[:, :1].expand(-1, T - 1, -1)], -1)
    assert torch.equal(y, ref) and torch.isnan(ybuf[..., 2 * H:]).all()


def test_arguments_are_refused_before_launch():
    from kandinsky2._native import K2Error
    x = torch.zeros(1, 4, 4, 12, device="cuda", dtype=torch.float16)
    with pytest.raises(K2Error, match="bilinear_f16"):
        ops.bilinear_f16(x, (8, 8), True)                                      # C not a multiple of 8
    with pytest.raises(K2Error, match="depth_to_space_f16"):
        ops.depth_to_space_f16(torch.zeros(1, 2, 2, 16, device="cuda", dtype=torch.float16), 2, 8)   # ldg < s^2 C
    with pytest.raises(K2Error, match="readout_rows_f16"):
        ops.readout_rows_f16(torch.zeros(1, 1, 16, device="cuda", dtype=torch.float16))              # no patch token
