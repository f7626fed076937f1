"""GPU: the C-ABI kernels on the strided views the launch plans actually pass, with hostile memory around them.

Every operand lives inside a larger allocation (`_Guarded`): at least one full row and at least 4 KB of guard before and after
it, and a row stride ld > C whose gap columns are part of the allocation too, so a stray access lands in owned memory and cannot
fault.
  - input buffers hold NaN (fp16 0x7E00, fp32 0x7FC00000) everywhere outside the view: a kernel that reads a byte it must not
    depend on produces NaN or a changed result;
  - output buffers are pre-filled with a distinctive bit pattern: after the call every byte outside the view must still hold
    it, and the view must equal the same call on contiguous operands bit for bit (ld changes addresses, never arithmetic);
  - the result is then checked against a float64 evaluation of the operation, with the tolerance each test states.
Shapes are the plans' real ones plus ragged edges: C a multiple of 8 but not of 64, T / H / W that leave partial tiles, Cout
not a multiple of the N tile."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

NAN_BITS = {torch.float16: 0x7E00, torch.float32: 0x7FC00000}
FILL_BITS = {torch.float16: 0x5A3C, torch.float32: 0x5A3C96E1, torch.uint8: 0xA5}
_INT = {torch.float16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}


def _bits(t):
    return t.view(_INT[t.dtype])


class _Guarded:
    """A [*lead, C] view with row stride ld inside one allocation with guards before and after."""

    def __init__(self, lead, C, ld=None, dtype=torch.float16, out=False):
        lead = tuple(lead)
        self.rows = math.prod(lead)
        self.C = C
        self.ld = ld if ld is not None else C
        esz = torch.tensor([], dtype=dtype).element_size()
        self.guard = -(-max(self.ld, 4096 // esz) // 16) * 16        # >= one row, >= 4 KB, keeps 16-byte alignment
        total = 2 * self.guard + self.rows * self.ld
        self.buf = torch.empty(total, dtype=dtype, device="cuda")
        bits = FILL_BITS[dtype] if out else NAN_BITS[dtype]
        if dtype != torch.uint8 and bits >= 1 << (8 * esz - 1):   # as the signed integer of the same width
            bits -= 1 << (8 * esz)
        _bits(self.buf).fill_(bits)
        self.bits = bits
        self.view = self.buf[self.guard:self.guard + self.rows * self.ld].view(*lead, self.ld)[..., :C]
        self.inside = torch.zeros(total, dtype=torch.bool, device="cuda")
        self.inside[self.guard:self.guard + self.rows * self.ld].view(self.rows, self.ld)[:, :C] = True

    @classmethod
    def of(cls, data, ld=None):
        """Input operand: a guarded copy of `data` (last dim = C)."""
        g = cls(data.shape[:-1], data.shape[-1], ld, data.dtype)
        g.view.copy_(data)
        return g

    def untouched(self):
        outside = _bits(self.buf)[~self.inside]
        bad = int((outside != self.bits).sum())
        return bad == 0, f"{bad} elements outside the view were written"


def _assert_untouched(*gs):
    for g in gs:
        ok, msg = g.untouched()
        assert ok, msg


def _same_bits(a, b):
    assert torch.equal(_bits(a.contiguous()), _bits(b.contiguous())), "strided result differs from the contiguous call"


def _rand(*shape, scale=1.0, seed=0, dtype=torch.float16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


# ------------------------------------------------------------------------------------------------------------------------------
# softmax_rows: the MoVQ attention path for widths != 512
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 7, 9, 320, 1027])
@pytest.mark.parametrize("inplace", [False, True])
def test_softmax_rows_bounds(n, inplace):
    from kandinsky2 import ops
    rows = 6
    x = _rand(rows, n, scale=2.0, seed=n)
    x[1] = x[1] * 40                      # large logits: the row maximum must be subtracted first
    x[2] = 0.75                           # a row of equal values: uniform 1/n
    x[3, :] = -30000.0
    x[3, n // 2] = 60000.0                # one dominant logit near the fp16 maximum
    ld8 = (n + 7) // 8 * 8     # the tightest row stride the kernel accepts (a multiple of 8)
    ld = ld8 + 8
    scale = 512 ** -0.5
    gx = _Guarded.of(x, ld)
    xt = torch.zeros(rows, ld8, device="cuda", dtype=torch.float16)
    xt[:, :n] = x
    ref_c = ops.softmax_rows(xt[:, :n], scale, out=torch.empty_like(xt)[:, :n])
    if inplace:
        got = ops.softmax_rows(gx.view, scale, out=gx.view)
        gy = gx
    else:
        gy = _Guarded((rows,), n, ld + 8, out=True)
        got = ops.softmax_rows(gx.view, scale, out=gy.view)
        ok, _ = gx.untouched()  # the input buffer was only read: its NaN guards are still NaN
        assert ok
    torch.cuda.synchronize()
    _assert_untouched(gy)
    _same_bits(got, ref_c)
    ref = torch.softmax(x.double() * scale, dim=-1)
    assert torch.isfinite(got).all()
    # fp16 output: half an ulp is 2^-11 relative (+ 3e-8 absolute in the subnormal range), fp32 exp2 / sum error ~1e-6 relative
    assert ((got.double() - ref).abs() <= 2 ** -11 * ref + 3e-8 + 2e-6 * ref).all(), (got.double() - ref).abs().max().item()


# ------------------------------------------------------------------------------------------------------------------------------
# copies: bit-exact against torch indexing
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("NB,H,W,C", [(2, 5, 7, 72), (1, 12, 12, 512), (3, 3, 1, 8)])
def test_upsample2x_bounds(NB, H, W, C):
    from kandinsky2 import ops
    x = _rand(NB, H, W, C, seed=1)
    gx = _Guarded.of(x, C + 24)
    gy = _Guarded((NB, 2 * H, 2 * W), C, C + 8, out=True)
    ops.upsample2x(gx.view, out=gy.view)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(_bits(gy.view.contiguous()), _bits(ref))


@pytest.mark.parametrize("oy,ox", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("NB,H,W,C", [(2, 6, 10, 72), (1, 32, 32, 128)])
def test_subsample2_bounds(oy, ox, NB, H, W, C):
    from kandinsky2 import ops
    x = _rand(NB, H, W, C, seed=2)
    gx = _Guarded.of(x, C + 8)
    gy = _Guarded((NB, H // 2, W // 2), C, C + 16, out=True)
    ops.subsample2(gx.view, oy, ox, out=gy.view)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    assert torch.equal(_bits(gy.view.contiguous()), _bits(x[:, oy::2, ox::2].contiguous()))


@pytest.mark.parametrize("B,T,C", [(3, 40, 72), (2, 320, 128)])
def test_transpose_f16_bounds(B, T, C):
    from kandinsky2 import ops
    x = _rand(B, T, C, seed=3)
    gx = _Guarded.of(x, C + 40)
    gy = _Guarded((B, C), T, out=True)   # contiguous [B, C, T] output with guards
    ops.transpose_f16(gx.view, out=gy.view)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    assert torch.equal(_bits(gy.view.contiguous()), _bits(x.transpose(1, 2).contiguous()))


def test_nchw_to_nhwc_f32_bounds():
    from kandinsky2 import ops
    x = _rand(3, 4, 7, 9, seed=4, dtype=torch.float32)
    gx = _Guarded.of(x.reshape(-1, 1))
    gy = _Guarded((3 * 7 * 9 * 4,), 1, dtype=torch.float32, out=True)
    ops.nchw_to_nhwc_f32(gx.view.view(3, 4, 7, 9), out=gy.view.view(3, 7, 9, 4))
    torch.cuda.synchronize()
    _assert_untouched(gy)
    assert torch.equal(_bits(gy.view.reshape(3, 7, 9, 4)), _bits(x.permute(0, 2, 3, 1).contiguous()))


@pytest.mark.parametrize("bias", [True, False])
def test_pointwise_nchw_f32_bounds(bias):
    from kandinsky2 import ops
    NB, Ci, Co, H, W = 2, 4, 4, 5, 7
    x = _rand(NB, Ci, H, W, seed=5, dtype=torch.float32)
    w = _rand(Co, Ci, seed=6, dtype=torch.float32)
    b = _rand(Co, seed=7, dtype=torch.float32) if bias else None
    gx = _Guarded.of(x.reshape(-1, 1))
    gy = _Guarded((NB * Co * H * W,), 1, dtype=torch.float32, out=True)
    ops.pointwise_nchw_f32(gx.view.view(NB, Ci, H, W), w, b, out=gy.view.view(NB, Co, H, W))
    torch.cuda.synchronize()
    _assert_untouched(gy)
    ref = torch.einsum("oi,nihw->nohw", w.double(), x.double()) + (b.double()[None, :, None, None] if bias else 0)
    # four fp32 fused multiply-adds: a few fp32 roundings of O(1) terms
    assert (gy.view.view(NB, Co, H, W).double() - ref).abs().max().item() < 4e-6 * max(1.0, ref.abs().max().item())


def test_images_to_u8_bounds():
    """Crop smaller than the image, values outside [-1, 1], and inputs whose (x + 1) * 127.5 is an exact fp32 half-integer, so
    that round-half-to-even (torch.round) is what decides them."""
    from kandinsky2 import ops
    NB, C, H, W, ch, cw = 2, 3, 9, 11, 7, 6
    k = torch.arange(0, 255, dtype=torch.float64, device="cuda")
    cand = ((k + 0.5) / 127.5 - 1).float()
    cand = torch.cat([cand, torch.nextafter(cand, torch.full_like(cand, 2)), torch.nextafter(cand, torch.full_like(cand, -2))])
    v = (cand + 1) * 127.5
    halves = cand[v == torch.floor(v) + 0.5]
    halves = torch.cat([halves, torch.zeros(1, device="cuda")])   # 0 -> exactly 127.5
    kk = ((halves + 1) * 127.5).floor()
    assert halves.numel() >= 10 and (kk % 2 == 0).any() and (kk % 2 == 1).any(), halves.numel()
    x = torch.linspace(-1.3, 1.3, NB * C * H * W, device="cuda")
    x[: halves.numel()] = halves[: x.numel()]
    x = x[torch.randperm(x.numel(), generator=torch.Generator().manual_seed(0)).cuda()].reshape(NB, C, H, W)
    gx = _Guarded.of(x.reshape(-1, 1))
    gy = _Guarded((NB * ch * cw * C,), 1, dtype=torch.uint8, out=True)
    ops.images_to_u8(gx.view.view(NB, C, H, W), ch, cw, out=gy.view.view(NB, ch, cw, C))
    torch.cuda.synchronize()
    _assert_untouched(gy)
    ref = ((x + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)[:, :, :ch, :cw].permute(0, 2, 3, 1).contiguous()
    assert torch.equal(gy.view.view(NB, ch, cw, C), ref)


def test_f32_to_f16_bounds():
    """Odd n, round-to-nearest-even ties, subnormals, +-65504 and overflow to +-inf: bit-exact against Tensor.half()."""
    from kandinsky2 import ops
    ties = torch.tensor([1 + 2 ** -11, 1 + 3 * 2 ** -11, 2049.0, 2051.0, -(1 + 2 ** -11), 2 ** -25, 3 * 2 ** -25],
                        dtype=torch.float64)
    special = torch.tensor([65504.0, -65504.0, 65519.0, 65520.0, -65520.0, 1e6, -1e30, 6e-8, 5.96e-8, 2 ** -24, 2 ** -26,
                            -2 ** -20, 0.0, -0.0, 1e-40], dtype=torch.float64)
    x = torch.cat([ties, special, torch.randn(999, dtype=torch.float64) * 300]).float().cuda()
    assert x.numel() % 2 == 1
    gx = _Guarded.of(x.reshape(-1, 1))
    gy = _Guarded((x.numel(),), 1, out=True)
    ops.f32_to_f16(gx.view.view(-1), out=gy.view.view(-1))
    torch.cuda.synchronize()
    _assert_untouched(gy)
    assert torch.equal(_bits(gy.view.view(-1)), _bits(x.half()))


def test_silu_gelu_f16_in_place_bounds():
    from kandinsky2 import ops
    x = torch.cat([_rand(998, scale=4.0, seed=8), torch.tensor([-65504.0, 65504.0], device="cuda").half()])
    # one fp16 rounding (half an ulp = 2^-11 relative) of an fp32 evaluation: within one ulp (2^-10 relative, 2^-24 in the
    # subnormal range).  SiLU is x sigmoid(x) with ~2^-20 relative fp32 error (k2_common.cuh silu_f); GELU is
    # 0.5 x erfc(-x / sqrt 2) in fp32.  tests/test_gpu_prior_kernels.py and tests/test_gpu_groupnorm_float64.py bound both by
    # one ulp over every fp16 input.
    xd = x.double()
    for name, fn, ref, tol in (("silu", ops.silu_f16_, xd * torch.sigmoid(xd), 6e-8),
                               ("gelu", ops.gelu_f16_, F.gelu(xd), torch.full_like(xd, 5e-7))):
        g = _Guarded.of(x.reshape(-1, 1))
        fn(g.view.view(-1))
        torch.cuda.synchronize()
        _assert_untouched(g)
        err = (g.view.view(-1).double() - ref).abs()
        bad = err > 2 ** -10 * ref.abs() + tol
        assert not bad.any(), (name, xd[bad][:4].tolist(), err[bad][:4].tolist())


def test_layernorm_f16_strided_bounds():
    from kandinsky2 import ops
    M, N = 7, 200
    x = (_rand(M, N, seed=9).float() * 3 + 1).half()
    gamma, beta = _rand(N, seed=10, dtype=torch.float32), _rand(N, seed=11, dtype=torch.float32)
    gx = _Guarded.of(x, N + 16)
    gy = _Guarded((M,), N, N + 8, out=True)
    ops.layernorm_f16(gx.view, gamma, beta, out=gy.view)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    _same_bits(gy.view, ops.layernorm_f16(x, gamma, beta))
    ref = F.layer_norm(x.double(), (N,), gamma.double(), beta.double(), 1e-5)
    # fp16 output of O(3) values: half an ulp is 2^-11 relative; fp32 statistics add ~1e-6
    assert ((gy.view.double() - ref).abs() <= 2 ** -10 * ref.abs() + 1e-4).all()


@pytest.mark.parametrize("K", [100, 64])
@pytest.mark.parametrize("w_half", [True, False])
def test_linear_strided_bounds(K, w_half):
    """ldx / ldy / ldadd larger than the row, K not a multiple of 8, and an fp16 W two bytes off 16-byte alignment (the scalar
    weight path of k2_linear)."""
    from kandinsky2 import ops
    M, N = 5, 37
    x = _rand(M, K, seed=12, dtype=torch.float32)
    W = _rand(N, K, seed=13, dtype=torch.float32) / K ** 0.5
    b = _rand(N, seed=14, dtype=torch.float32)
    add = _rand(M, N, seed=15, dtype=torch.float32)
    Wd = W.half() if w_half else W
    wbuf = torch.full((N * K + 8,), float("nan"), device="cuda", dtype=Wd.dtype)
    Wm = wbuf[1:1 + N * K].view(N, K)        # contiguous, 2 (fp16) / 4 (fp32) bytes off 16-byte alignment
    Wm.copy_(Wd)
    gx, ga = _Guarded.of(x, K + 12), _Guarded.of(add, N + 3)
    gy = _Guarded((M,), N, N + 11, dtype=torch.float32, out=True)
    ops.linear(gx.view, Wm, b, add=ga.view, silu_in=True, out=gy.view)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    _same_bits(gy.view, ops.linear(x, Wm, b, add=add, silu_in=True))   # same (misaligned) W: the same weight path
    ref = F.linear(F.silu(x.double()), Wd.double(), b.double()) + add.double()
    assert torch.allclose(gy.view.double(), ref, atol=2e-4, rtol=1e-4)   # as test_linear_layernorm_temb


# ------------------------------------------------------------------------------------------------------------------------------
# GroupNorm family
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resample", [0, 1, 2])
def test_gn_apply_strided_bounds(resample):
    """Two sources with different ld, y and xres as slices, FiLM rows with film_ld > 2C, every resample mode; statistics from
    k2_gn_stats over the same strided sources."""
    from kandinsky2 import ops
    NB, H, W, C0, C1 = 2, 6, 10, 128, 64
    C = C0 + C1
    x0 = (_rand(NB, H, W, C0, seed=16).float() * 2 + 0.5).half()
    x1 = (_rand(NB, H, W, C1, seed=17).float() - 0.3).half()
    gamma, beta = _rand(C, seed=18, dtype=torch.float32), _rand(C, seed=19, dtype=torch.float32)
    film = _rand(NB, 2 * C, seed=20, dtype=torch.float32) * 0.3
    g0, g1 = _Guarded.of(x0, C0 + 8), _Guarded.of(x1, C1 + 72)
    gf = _Guarded.of(film, 2 * C + 5)
    Ho, Wo = (H, W) if resample == 0 else ((H // 2, W // 2) if resample == 1 else (2 * H, 2 * W))
    gy = _Guarded((NB, Ho, Wo), C, C + 16, out=True)
    gxr = _Guarded((NB, Ho, Wo), C, C + 32, out=True)
    st = ops.gn_stats(g0.view, g1.view)
    st_c = ops.gn_stats(x0, x1)
    ops.gn_apply(g0.view, g1.view, st, gamma, beta, film=gf.view, act=1, resample=resample, y=gy.view, xres=gxr.view)
    y_c, xr_c = ops.gn_apply(x0, x1, st_c, gamma, beta, film=film, act=1, resample=resample, want_xres=True)
    torch.cuda.synchronize()
    _assert_untouched(gy, gxr)
    assert torch.equal(st, st_c)
    _same_bits(gy.view, y_c)
    _same_bits(gxr.view, xr_c)
    xc = torch.cat([x0, x1], -1).double().permute(0, 3, 1, 2)
    ref = F.silu(F.group_norm(xc, 32, gamma.double(), beta.double(), 1e-5) * (1 + film[:, :C, None, None].double()) +
                 film[:, C:, None, None].double())
    ref_x = xc
    if resample == 1:
        ref, ref_x = F.avg_pool2d(ref, 2), F.avg_pool2d(ref_x, 2)
    elif resample == 2:
        ref, ref_x = F.interpolate(ref, scale_factor=2), F.interpolate(ref_x, scale_factor=2)
    # as test_gn_stats_apply: fp16 output of O(3) values (FiLM + SiLU 3e-2, avg-pooled raw x 1e-2, upsampled raw x exact)
    assert (gy.view.double().permute(0, 3, 1, 2) - ref).abs().max().item() < 3e-2
    err_x = (gxr.view.double().permute(0, 3, 1, 2) - ref_x).abs().max().item()
    assert err_x < 1e-2 and (resample != 2 or err_x == 0)


@pytest.mark.parametrize("resample", [0, 1, 2])
def test_gn_apply_fold_and_partials_bounds(resample):
    """Conv-produced partial statistics in a NaN-filled buffer larger than what the epilogue writes; gn_finalize with
    rg = info[6] // NB and gn_apply_fold must read only the row groups that were written, and the conv must not write past
    info[6] * Cout * 2 floats."""
    from kandinsky2 import ops
    NB, H, W, Cin = 2, 12, 20, 72
    outs, parts, rgs, guards = [], [], [], []
    for cout, seed in ((128, 21), (64, 22)):
        x = _rand(NB, H, W, Cin, seed=seed)
        w = _rand(cout, Cin, 3, 3, seed=seed + 1, dtype=torch.float32) / 24
        n = ops.gn_part_floats(NB, H, W, cout)
        gp = _Guarded((n,), 1, dtype=torch.float32)        # NaN everywhere, including the unused tail
        info = [0] * 7
        y = ops.conv_gemm([(_Guarded.of(x, Cin + 8).view, 9)], ops.pack_conv_weight(w), cout, gn_part=gp.view.view(-1),
                          info=info)
        assert info[5] in (1, 2) and info[6] % NB == 0, info   # epilogue partials, or the split-K second pass's
        written = info[6] * cout * 2
        gp.inside.zero_()
        gp.inside[gp.guard:gp.guard + written] = True
        guards.append(gp)
        outs.append(y)
        parts.append(gp.view.view(-1))
        rgs.append(info[6] // NB)
    torch.cuda.synchronize()
    for gp in guards:   # nothing past the row groups the conv reported was written
        _assert_untouched(gp)
        assert torch.isfinite(gp.view.view(-1)[: int(gp.inside.sum())]).all()
    C = 192
    gamma, beta = _rand(C, seed=23, dtype=torch.float32), _rand(C, seed=24, dtype=torch.float32)
    st = torch.empty(NB, 32, 2, device="cuda")
    ops.gn_finalize(parts[0], 128, parts[1], 64, NB, rgs[0], H * W, st, rg1=rgs[1])
    ref_st = ops.gn_stats(outs[0], outs[1])
    torch.cuda.synchronize()
    assert torch.isfinite(st).all()
    # as test_conv_fused_groupnorm_partials: the same fp16 values summed in another order
    assert torch.allclose(st[..., 0], ref_st[..., 0], atol=2e-5) and torch.allclose(st[..., 1], ref_st[..., 1], rtol=2e-5)
    y = ops.gn_apply_fold(outs[0], outs[1], parts[0], rgs[0], parts[1], rgs[1], gamma, beta, act=1, resample=resample)
    y_ref = ops.gn_apply(outs[0], outs[1], st, gamma, beta, act=1, resample=resample)
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    # as test_gn_apply_fold_matches_finalize_plus_apply
    assert (y.float() - y_ref.float()).abs().max().item() <= 2e-3 * max(1.0, y_ref.float().abs().max().item())


def test_sn_apply_strided_bounds():
    from kandinsky2 import ops
    NB, H, W, C = 2, 12, 20, 128
    x = (_rand(NB, H, W, C, seed=25).float() * 1.5 + 0.3).half()
    zq = _rand(NB, 3, 5, 4, seed=26, dtype=torch.float32)
    gamma = 1 + 0.1 * _rand(C, seed=27, dtype=torch.float32)
    beta = 0.1 * _rand(C, seed=28, dtype=torch.float32)
    sn_w = torch.cat([_rand(C, 4, seed=29, dtype=torch.float32) / 2, 1 + _rand(C, 1, seed=30, dtype=torch.float32) / 4,
                      _rand(C, 4, seed=31, dtype=torch.float32) / 2, _rand(C, 1, seed=32, dtype=torch.float32) / 4], 1)
    gx = _Guarded.of(x, C + 24)
    gy = _Guarded((NB, H, W), C, C + 8, out=True)
    st = ops.gn_stats(gx.view, None, eps=1e-6)
    ops.sn_apply(gx.view, st, gamma, beta, zq, sn_w.contiguous(), act=1, y=gy.view)
    y_c = ops.sn_apply(x, ops.gn_stats(x, None, eps=1e-6), gamma, beta, zq, sn_w.contiguous(), act=1)
    torch.cuda.synchronize()
    _assert_untouched(gy)
    _same_bits(gy.view, y_c)
    xn = F.group_norm(x.double().permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), eps=1e-6)
    zu = F.interpolate(zq.double().permute(0, 3, 1, 2), size=(H, W), mode="nearest")
    sw = sn_w.double()
    ref = xn * F.conv2d(zu, sw[:, :4, None, None], sw[:, 4]) + F.conv2d(zu, sw[:, 5:9, None, None], sw[:, 9])
    ref = (ref * torch.sigmoid(ref)).permute(0, 2, 3, 1)
    assert (gy.view.double() - ref).abs().max().item() <= 3e-3 * max(1.0, ref.abs().max().item())   # as test_sn_apply


# ------------------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,heads,T,Tc", [(2, 2, 70, 17), (1, 3, 130, 87)])
def test_attention_d64_strided_bounds(B, heads, T, Tc):
    """ldq > heads*192, lde > heads*128, ldo > heads*64; NaN rows after the last image's T rows and Tc encoder rows."""
    from kandinsky2 import ops
    from tests.attention_ref import check_d64
    qkv = _rand(B, T, heads * 192, seed=33)
    enc = _rand(B, Tc, heads * 128, seed=34)
    gq, ge = _Guarded.of(qkv, heads * 192 + 24), _Guarded.of(enc, heads * 128 + 8)
    go = _Guarded((B, T), heads * 64, heads * 64 + 16, out=True)
    ops.attention_d64(gq.view, heads, ge.view, out=go.view)
    y_c = ops.attention_d64(qkv, heads, enc)
    torch.cuda.synchronize()
    _assert_untouched(go)
    _same_bits(go.view, y_c)
    check_d64(go.view, qkv, enc, heads, "strided")   # tests/attention_ref.py's bound


@pytest.mark.parametrize("T", [320, 64])
def test_attention_d512_strided_bounds(T):
    """ldq > 1536 with non-default offsets (k | v | q), ldo > 512."""
    from kandinsky2 import ops
    B = 2
    q, k, v = _rand(B, T, 512, seed=35, scale=2.0), _rand(B, T, 512, seed=36), _rand(B, T, 512, seed=37)
    ldq = 1600
    gq = _Guarded((B, T), 1576, ldq)
    gq.view[..., 0:512] = k
    gq.view[..., 520:1032] = v
    gq.view[..., 1064:1576] = q
    go = _Guarded((B, T), 512, 520, out=True)
    ops.attention_d512(gq.view, 512 ** -0.5, out=go.view, q_off=1064, k_off=0, v_off=520)
    y_c = ops.attention_d512(torch.cat([q, k, v], -1), 512 ** -0.5)
    torch.cuda.synchronize()
    _assert_untouched(go)
    _same_bits(go.view, y_c)
    from tests.attention_ref import check, ref_attention
    for b in range(B):   # tests/attention_ref.py's bound
        check(go.view[b, :, None], *ref_attention(q[b, :, None], k[b, :, None], v[b, :, None], 512 ** -0.5), b)


# ------------------------------------------------------------------------------------------------------------------------------
# conv / GEMM
# ------------------------------------------------------------------------------------------------------------------------------
def _ref_conv(srcs, ws, bias=None, residual=None):
    """float64 sum over sources of conv(src, w) (3x3 pad 1 or 1x1) + bias + residual; NHWC in, NHWC out."""
    acc = 0
    for (x, taps), w in zip(srcs, ws):
        acc = acc + F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1 if taps == 9 else 0)
    if bias is not None:
        acc = acc + bias.double()[None, :, None, None]
    acc = acc.permute(0, 2, 3, 1)
    if residual is not None:
        acc = acc + residual.double()
    return acc


def _check_conv(got, ref):
    err = (got.double() - ref).abs().max().item()
    rel = ((got.double() - ref).norm() / ref.norm()).item()
    # as test_conv3x3: fp16 output rounding of fp32 sums
    assert err < 2e-2 * max(1.0, ref.abs().max().item()) / 4 and rel < 1e-3, (err, rel)


@pytest.mark.parametrize("Ca,Cb,Cc,Cout", [(72, 200, 64, 320), (64, 72, 8, 136)])
def test_conv_three_source_slices_bounds(Ca, Cb, Cc, Cout):
    """Three sources as channel slices of ONE NaN-guarded buffer (C not multiples of 64), residual and output as slices;
    Cout not a multiple of the N tile."""
    from kandinsky2 import ops
    NB, H, W = 2, 7, 11
    Ct = Ca + Cb + Cc
    xs = _rand(NB, H, W, Ct, seed=38)
    gx = _Guarded.of(xs, Ct + 16)
    a, b, c = gx.view[..., :Ca], gx.view[..., Ca:Ca + Cb], gx.view[..., Ca + Cb:]
    wa = _rand(Cout, Ca, 3, 3, seed=39, dtype=torch.float32) / (9 * Ca) ** 0.5
    wb = _rand(Cout, Cb, 1, 1, seed=40, dtype=torch.float32) / Cb ** 0.5
    wc = _rand(Cout, Cc, 1, 1, seed=41, dtype=torch.float32) / Cc ** 0.5
    wp = torch.cat([ops.pack_conv_weight(wa), ops.pack_conv_weight(wb), ops.pack_conv_weight(wc)], 1).contiguous()
    bias = _rand(Cout, seed=42, dtype=torch.float32)
    res = _rand(NB, H, W, Cout, seed=43)
    gr = _Guarded.of(res, Cout + 24)
    go = _Guarded((NB, H, W), Cout, Cout + 40, out=True)
    srcs = [(a, 9), (b, 1), (c, 1)]
    ops.conv_gemm(srcs, wp, Cout, bias=bias, residual=gr.view, out=go.view)
    y_c = ops.conv_gemm([(a.contiguous(), 9), (b.contiguous(), 1), (c.contiguous(), 1)], wp, Cout, bias=bias, residual=res)
    torch.cuda.synchronize()
    _assert_untouched(go)
    _same_bits(go.view, y_c)
    ref = _ref_conv([(xs[..., :Ca], 9), (xs[..., Ca:Ca + Cb], 1), (xs[..., Ca + Cb:], 1)],
                    [wa.half(), wb.half(), wc.half()], bias, res)
    _check_conv(go.view, ref)


def test_conv_up2_taps4_bounds():
    """taps = 4 (3x3 conv over the nearest-2x upsampled source) from a strided, NaN-guarded source into a strided output."""
    from kandinsky2 import ops
    NB, H, W, C, Cout = 2, 5, 6, 72, 136
    x = _rand(NB, H, W, C, seed=44)
    w = _rand(Cout, C, 3, 3, seed=45, dtype=torch.float32) / (9 * C) ** 0.5
    bias = _rand(Cout, seed=46, dtype=torch.float32)
    gx = _Guarded.of(x, C + 8)
    go = _Guarded((NB, 2 * H, 2 * W), Cout, Cout + 8, out=True)
    wp = ops.pack_conv_weight_up2(w)
    ops.conv_gemm([(gx.view, 4)], wp, Cout, bias=bias, out=go.view)
    y_c = ops.conv_gemm([(x, 4)], wp, Cout, bias=bias)
    torch.cuda.synchronize()
    _assert_untouched(go)
    _same_bits(go.view, y_c)
    up = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    ref = _ref_conv([(up, 9)], [w], bias)
    err = (go.view.double() - ref).abs().max().item()
    rel = ((go.view.double() - ref).norm() / ref.norm()).item()
    # as test_conv3x3_over_nearest_upsample: the pre-summed phase weights are rounded to fp16 once more
    assert rel < 1.5e-3 and err < 1e-2 * max(1.0, ref.abs().max().item()), (rel, err)


def test_conv_out_mode1_nchw_bounds():
    """The fp32 NCHW output head (out_mode 1) with Cout = 3 in a 16-row weight: guards around the output."""
    from kandinsky2 import ops
    NB, H, W, C, Cout = 2, 9, 13, 72, 3
    x = _rand(NB, H, W, C, seed=47)
    w = _rand(Cout, C, 3, 3, seed=48, dtype=torch.float32) / (9 * C) ** 0.5
    bias = _rand(Cout, seed=49, dtype=torch.float32)
    gx = _Guarded.of(x, C + 56)
    go = _Guarded((NB * Cout * H * W,), 1, dtype=torch.float32, out=True)
    wp = ops.pad_rows(ops.pack_conv_weight(w), 16)
    ops.conv_gemm([(gx.view, 9)], wp, Cout, bias=bias, out=go.view.view(NB, Cout, H, W), out_mode=1)
    y_c = ops.conv_gemm([(x, 9)], wp, Cout, bias=bias, out_mode=1)
    torch.cuda.synchronize()
    _assert_untouched(go)
    _same_bits(go.view.view(NB, Cout, H, W), y_c)
    ref = _ref_conv([(x, 9)], [w.half()], bias).permute(0, 3, 1, 2)
    assert (go.view.view(NB, Cout, H, W).double() - ref).abs().max().item() < 2e-3   # as test_head_fp32_nchw (fp32 output)


def test_conv_forced_splitk_bounds():
    """Forced 2-way split-K from strided sources into a strided output with a strided residual; the split reduction is
    deterministic, so the strided call equals the contiguous one bit for bit."""
    from kandinsky2 import ops
    NB, H, W, C, Cout = 1, 4, 12, 512, 200
    x = _rand(NB, H, W, C, seed=50)
    w = _rand(Cout, C, 3, 3, seed=51, dtype=torch.float32) / (9 * C) ** 0.5
    res = _rand(NB, H, W, Cout, seed=52)
    gx, gr = _Guarded.of(x, C + 8), _Guarded.of(res, Cout + 8)
    go = _Guarded((NB, H, W), Cout, Cout + 16, out=True)
    wp = ops.pack_conv_weight(w)
    info, info_c = [0] * 7, [0] * 7
    ops.conv_gemm([(gx.view, 9)], wp, Cout, residual=gr.view, out=go.view, cfg=(0, 0, 2, 0), info=info)
    y_c = ops.conv_gemm([(x, 9)], wp, Cout, residual=res, cfg=(0, 0, 2, 0), info=info_c)
    torch.cuda.synchronize()
    assert info[2] == 2 and info == info_c, (info, info_c)
    _assert_untouched(go)
    _same_bits(go.view, y_c)
    _check_conv(go.view, _ref_conv([(x, 9)], [w.half()], None, res))


def test_batched_attention_gemm_bounds():
    """The MoVQ AttnBlock's batched GEMMs (w_batch_stride, T = 320, B = 3) with NaN rows after the last image's k rows and
    after the last image's transposed values: scores = q k^T, then P v."""
    from kandinsky2 import ops
    B, T, C = 3, 320, 128
    qkv = _rand(B, T, 3 * C, seed=53)
    gq = _Guarded.of(qkv)
    q, k = gq.view[:, :, :C], gq.view[0, :, C:2 * C]
    gs = _Guarded((B, 1, T), T, out=True)
    ops.conv_gemm([(q.unsqueeze(1), 1)], k, T, out=gs.view, w_batch_stride=T * 3 * C)
    s_c = torch.empty(B, T, T, device="cuda", dtype=torch.float16)
    ops.conv_gemm([(qkv[:, :, :C].unsqueeze(1), 1)], qkv[0, :, C:2 * C], T, out=s_c.view(B, 1, T, T), w_batch_stride=T * 3 * C)
    torch.cuda.synchronize()
    _assert_untouched(gs)
    _same_bits(gs.view.view(B, T, T), s_c)
    ref = torch.einsum("btc,bsc->bts", qkv[:, :, :C].double(), qkv[:, :, C:2 * C].double())
    assert ((gs.view.view(B, T, T).double() - ref).norm() / ref.norm()).item() < 1e-3   # as test_transpose_and_batched_gemm
    p = torch.softmax(ref * C ** -0.5, -1).half()
    gv = _Guarded.of(qkv[:, :, 2 * C:].transpose(1, 2).contiguous())     # [B, C, T] values, NaN after the last image
    go = _Guarded((B, 1, T), C, C + 8, out=True)
    ops.conv_gemm([(p.view(B, 1, T, T), 1)], gv.view[0], C, out=go.view, w_batch_stride=C * T)
    torch.cuda.synchronize()
    _assert_untouched(go)
    ref_o = torch.einsum("bts,bsc->btc", p.double(), qkv[:, :, 2 * C:].double())
    assert ((go.view.view(B, T, C).double() - ref_o).norm() / ref_o.norm()).item() < 1e-3
