"""Thin torch-tensor wrappers over the C ABI (include/k2b200.h).

torch is used for device memory, streams and one-off weight re-layout only; every arithmetic op on the
hot path is a kernel of libk2b200.so.  Activations are NHWC fp16 tensors of shape [NB, H, W, C] (a view
may be a channel slice of a wider buffer: stride(-2) is the row stride).
"""
import ctypes

import torch

from . import _native as nat
from ._native import K2ConvSrc, check, ptr, stream_ptr


def _row_stride(t):
    assert t.stride(-1) == 1, "channel dim must be contiguous"
    ld = t.stride(-2)
    # all leading dims must be row-contiguous w.r.t. ld
    n = t.shape[-2]
    for d in range(t.dim() - 3, -1, -1):
        assert t.shape[d] == 1 or t.stride(d) == ld * n, f"not a row-strided NHWC view: {t.shape} {t.stride()}"
        n *= t.shape[d]
    return ld


# ------------------------------------------------------------------------------------------------
# weight packing (host side, once per checkpoint load)
# ------------------------------------------------------------------------------------------------
def _pad64(c):
    return (c + 63) // 64 * 64


def pack_conv_weight(w, split=None):
    """[Cout, Cin, kh, kw] (kh=kw in {1,3}) or [Cout, Cin] / [Cout, Cin, 1] -> fp16 [Cout, taps*pad64(Cin)].

    k = tap * pad64(Cin) + c with tap = ky*3+kx (k2b200.h: k2_conv_gemm).  `split=(C0, C1)` packs a 1x1
    weight whose input is the channel concat of two sources as two independently padded segments.
    """
    w = w.detach()
    if w.dim() == 2:
        w = w[:, :, None, None]
    elif w.dim() == 3:
        w = w[:, :, :, None]
    cout, cin, kh, kw = w.shape
    taps = kh * kw
    assert taps in (1, 9)
    parts = [(0, cin)] if split is None else [(0, split[0]), (split[0], split[0] + split[1])]
    segs = []
    for lo, hi in parts:
        c = hi - lo
        ws = w[:, lo:hi].permute(0, 2, 3, 1).reshape(cout, taps, c)
        if _pad64(c) != c:
            ws = torch.nn.functional.pad(ws, (0, _pad64(c) - c))
        segs.append(ws.reshape(cout, taps * _pad64(c)))
    return torch.cat(segs, dim=1).to(torch.float16).contiguous()


_UP2_TAPS = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}  # output parity a -> 3x3 kernel rows feeding source offsets (a - 1, a)


def pack_conv_weight_up2(w):
    """[Cout, Cin, 3, 3] -> fp16 [Cout, 16 * pad64(Cin)] for a `taps = 4` source of k2_conv_gemm: the 3x3 convolution over the
    nearest-2x upsampled input, as four 2x2 convolutions over the input itself, one per output parity (a, b).  Output pixel
    (2y + a, 2x + b) sees upsampled rows 2y + a + ky - 1, i.e. source rows y + floor((a + ky - 1) / 2): the kernel rows that
    land on the same source row are summed (fp32) before the fp16 rounding.  k = ((a * 2 + b) * 4 + ty * 2 + tx) * pad64(Cin) + c,
    source offset (dy, dx) = (ty + a - 1, tx + b - 1).  2.25x fewer MACs than convolving the upsampled tensor, which is never
    materialised (unet.py:67-77 Upsample + :199-203 h_upd; movq_modules.py:93-97)."""
    w = w.detach().float()
    cout, cin = w.shape[:2]
    blocks = []
    for a in (0, 1):
        for b in (0, 1):
            for ty in (0, 1):
                for tx in (0, 1):
                    acc = torch.zeros(cout, cin, dtype=torch.float32, device=w.device)
                    for ky in _UP2_TAPS[a][ty]:
                        for kx in _UP2_TAPS[b][tx]:
                            acc += w[:, :, ky, kx]
                    if _pad64(cin) != cin:
                        acc = torch.nn.functional.pad(acc, (0, _pad64(cin) - cin))
                    blocks.append(acc)
    return torch.cat(blocks, dim=1).to(torch.float16).contiguous()


def pad_rows(wp, rows):
    if wp.shape[0] >= rows:
        return wp
    return torch.cat([wp, wp.new_zeros(rows - wp.shape[0], wp.shape[1])], 0).contiguous()


# ------------------------------------------------------------------------------------------------
# conv / GEMM
# ------------------------------------------------------------------------------------------------
_CONV_WS_BYTES = 128 << 20  # split-K partial sums; fixed size and address (baked into captured CUDA graphs); conv launches that
# share it must be stream-ordered
_conv_ws = {}


def _workspace(dev):
    buf = _conv_ws.get(dev.index)
    if buf is None:
        buf = torch.empty(_CONV_WS_BYTES, dtype=torch.uint8, device=dev)
        _conv_ws[dev.index] = buf
    return buf


def conv_gemm(srcs, w_packed, cout, bias=None, residual=None, out=None, out_mode=0, geom=None, gn_part=None, info=None,
              cfg=None, w_batch_stride=0, w_map=None, n_slabs=0):
    """srcs: list of (tensor NHWC fp16 [NB,H,W,C], taps); taps = 9 (3x3), 1 (1x1) or 4 (single source: 3x3 over its nearest-2x
    upsampling, weights from pack_conv_weight_up2, output [NB,2H,2W,cout]).  Returns fp16 [NB,H,W,cout] (out_mode 0) or
    fp32 NCHW [NB,cout,H,W] (out_mode 1).  geom=(NB,H,W) overrides the geometry (GEMM on flat rows).
    cfg = (N tile, pair mode, splits, epilogue sets) overrides the library's choice (k2_conv_gemm_cfg; 0 = auto).
    w_batch_stride > 0: batched GEMM, image n uses the weight matrix at w_packed + n * w_batch_stride elements (w_packed is then
    any fp16 tensor whose data_ptr() is matrix 0, shape[0] / shape[1] / stride(0) = rows / K / row stride of ONE matrix).
    w_map (device int32 [NB], with n_slabs >= 1 and w_batch_stride > 0): image n uses slab w_map[n] of the n_slabs matrices
    instead of matrix n (k2_conv_gemm_wmap); the kernel reads the map when it runs, so a captured graph follows its contents."""
    lib = nat.load()
    t0 = srcs[0][0]
    NB, H, W = geom if geom is not None else t0.shape[:3]
    if w_map is not None:
        _check_w_map(w_map, NB, n_slabs)
    if srcs[0][1] == 4:  # 3x3 conv over the nearest-2x upsampling of the source: geometry = the OUTPUT's
        H, W = 2 * H, 2 * W
    arr = (K2ConvSrc * len(srcs))()
    for i, (t, taps) in enumerate(srcs):
        assert t.dtype == torch.float16 and t.is_cuda
        arr[i].ptr = t.data_ptr()
        arr[i].C = t.shape[-1]
        arr[i].ld = _row_stride(t)
        arr[i].taps = taps
    if out is None:
        if out_mode == 0:
            out = torch.empty((NB, H, W, cout), dtype=torch.float16, device=t0.device)
        else:
            out = torch.empty((NB, cout, H, W), dtype=torch.float32, device=t0.device)
    ldo = _row_stride(out) if out_mode == 0 else 0
    ldr = _row_stride(residual) if residual is not None else 0
    assert w_packed.dtype == torch.float16 and w_packed.stride(1) == 1
    ws = _workspace(t0.device)
    _info = (ctypes.c_int * 7)()
    _cfg = (ctypes.c_int * 4)(*cfg) if cfg is not None else None
    args = (arr, len(srcs), NB, H, W, ptr(w_packed), w_packed.shape[0], w_packed.shape[1], w_packed.stride(0), cout,
            ptr(bias), ptr(residual), ldr, ptr(out), ldo, out_mode, ptr(ws), ws.numel(), ptr(gn_part), _info, _cfg,
            int(w_batch_stride))
    if w_map is None:
        check(lib.k2_conv_gemm_cfg(*args, stream_ptr()))
    else:
        check(lib.k2_conv_gemm_wmap(*args, int(n_slabs), ptr(w_map), stream_ptr()))
    if info is not None:
        info[:] = list(_info)
    return out


def _check_w_map(w_map, NB, n_slabs):
    """The weight-slab map of a mapped batched GEMM: a contiguous int32 device tensor of one entry per image."""
    if not torch.is_tensor(w_map) or not w_map.is_cuda:
        raise nat.K2Error("conv_gemm: w_map must be an int32 tensor on a CUDA sm_90 device (the kernel reads it)")
    if w_map.dtype != torch.int32 or not w_map.is_contiguous():
        raise nat.K2Error(f"conv_gemm: w_map must be a contiguous int32 tensor, got {w_map.dtype}"
                          f"{'' if w_map.is_contiguous() else ' (non-contiguous)'}")
    if w_map.numel() != NB:
        raise nat.K2Error(f"conv_gemm: w_map must hold one slab index per image ({NB}), got {tuple(w_map.shape)}")
    if isinstance(n_slabs, bool) or not isinstance(n_slabs, int) or n_slabs < 1:
        raise nat.K2Error(f"conv_gemm: n_slabs must be an int >= 1 with a w_map, got {n_slabs!r}")


def conv_plan(NB, H, W, taps, ktot, cout, out_mode=0, workspace_bytes=_CONV_WS_BYTES, want_gn_partial=True):
    """What k2_conv_gemm would decide for this geometry (host arithmetic only, no GPU): dict of the info[7] fields."""
    lib = nat.load()
    info = (ctypes.c_int * 7)()
    check(lib.k2_conv_plan(NB, H, W, taps, ktot, cout, out_mode, workspace_bytes, int(want_gn_partial), info))
    keys = ("n_tile", "cta_pair", "splits", "m_tiles", "images_per_tile", "gn_partial_mode", "row_groups")
    return dict(zip(keys, list(info)))


def gemm_rows(x, w_packed, cout, bias=None, residual=None, out=None, cfg=None, info=None):
    """x: fp16 [..., K] rows -> fp16 [..., cout]; one 1x1 'conv' over M = prod(leading dims) rows."""
    lead = x.shape[:-1]
    M = 1
    for d in lead:
        M *= d
    x3 = x.reshape(1, 1, M, x.shape[-1]) if x.is_contiguous() else None
    if x3 is None:
        # row-strided view (channel slice): keep stride
        x3 = x.as_strided((1, 1, M, x.shape[-1]), (0, 0, x.stride(-2), 1))
    if out is None:
        out = torch.empty(tuple(lead) + (cout,), dtype=torch.float16, device=x.device)
    o3 = out.as_strided((1, 1, M, cout), (0, 0, out.stride(-2), 1))
    r3 = None
    if residual is not None:
        r3 = residual.as_strided((1, 1, M, cout), (0, 0, residual.stride(-2), 1))
    conv_gemm([(x3, 1)], w_packed, cout, bias=bias, residual=r3, out=o3, geom=(1, 1, M), cfg=cfg, info=info)
    return out


# ------------------------------------------------------------------------------------------------
# GroupNorm
# ------------------------------------------------------------------------------------------------
_gn_scratch = {}


_GN_SCRATCH_FLOATS = 1 << 23  # 32 MB, fixed: its address is baked into captured CUDA graphs


def _scratch(dev, nfloats):
    key = (dev.index, )
    buf = _gn_scratch.get(key)
    if buf is None:
        buf = torch.zeros(_GN_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
        _gn_scratch[key] = buf
    if nfloats > buf.numel():
        raise nat.K2Error(f"gn_stats scratch of {buf.numel()} floats is too small for this geometry ({nfloats})")
    return buf


def gn_stats(x0, x1=None, groups=32, eps=1e-5, stats=None):
    """Per (image, group) [mean, rstd] of the channel concat [x0 | x1]; x*: fp16 NHWC."""
    lib = nat.load()
    NB, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    if stats is None:
        stats = torch.empty((NB, groups, 2), dtype=torch.float32, device=x0.device)
    need = lib.k2_gn_scratch_floats(NB, H * W, C0 + C1)
    scratch = _scratch(x0.device, need)
    check(lib.k2_gn_stats(ptr(x0), C0, _row_stride(x0), ptr(x1), C1, _row_stride(x1) if x1 is not None else 0,
                          NB, H * W, groups, eps, ptr(stats), ptr(scratch), stream_ptr()))
    return stats


def gn_part_floats(NB, H, W, cout):
    """Upper bound of the fp32 count of a conv's fused-statistics partial buffer ([row groups][cout][2], k2b200.h)."""
    tiles = NB * ((H * W + 63) // 64 + 2 * H)  # generous: boxes are >= 64 pixels except at ragged edges
    return max(tiles * 4, (NB * H * W + 15) // 16) * cout * 2


def gn_finalize(part0, C0, part1, C1, NB, rg_per_image, HW, stats, groups=32, eps=1e-5, rg1=None):
    """rg_per_image: row groups per image of source 0 (and of source 1 unless rg1 is given)."""
    lib = nat.load()
    check(lib.k2_gn_finalize(ptr(part0), C0, rg_per_image, ptr(part1), C1, rg1 if rg1 is not None else rg_per_image, NB, HW,
                             groups, eps, ptr(stats), stream_ptr()))
    return stats


def gn_apply(x0, x1, stats, gamma, beta, film=None, act=1, resample=0, groups=32, y=None, want_xres=False,
             zq=None, sn_w=None, xres=None):
    """Fused normalise (+FiLM) (+SiLU) (+2x up / 2x2 avg-pool) (+concat) -> fp16 NHWC. See k2b200.h."""
    lib = nat.load()
    NB, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    C = C0 + C1
    Ho, Wo = (H, W) if resample == 0 else ((H // 2, W // 2) if resample == 1 else (H * 2, W * 2))
    if y is None:
        y = torch.empty((NB, Ho, Wo, C), dtype=torch.float16, device=x0.device)
    if xres is not None:
        want_xres = True
    elif want_xres:
        xres = torch.empty((NB, Ho, Wo, C), dtype=torch.float16, device=x0.device)
    zh = zw = 0
    if zq is not None:
        zh, zw = zq.shape[1], zq.shape[2]
    check(lib.k2_gn_apply(ptr(x0), C0, _row_stride(x0), ptr(x1), C1, _row_stride(x1) if x1 is not None else 0,
                          NB, H, W, groups, ptr(stats), ptr(gamma), ptr(beta), ptr(film),
                          film.stride(0) if film is not None else 0, act, resample,
                          ptr(y), _row_stride(y), ptr(xres), _row_stride(xres) if xres is not None else 0,
                          ptr(zq), zh, zw, ptr(sn_w), stream_ptr()))
    return (y, xres) if want_xres else y


def gn_apply_fold(x0, x1, part0, rg0, part1, rg1, gamma, beta, film=None, act=1, resample=0, groups=32, eps=1e-5, y=None,
                  xres=None):
    """gn_apply that folds the producers' partial sums itself (no gn_finalize launch); round-2 candidate, see k2b200.h."""
    lib = nat.load()
    NB, H, W, C0 = x0.shape
    C1 = x1.shape[-1] if x1 is not None else 0
    Ho, Wo = (H, W) if resample == 0 else ((H // 2, W // 2) if resample == 1 else (H * 2, W * 2))
    if y is None:
        y = torch.empty((NB, Ho, Wo, C0 + C1), dtype=torch.float16, device=x0.device)
    check(lib.k2_gn_apply_fold(ptr(x0), C0, _row_stride(x0), ptr(x1), C1, _row_stride(x1) if x1 is not None else 0,
                               NB, H, W, groups, ptr(part0), rg0, ptr(part1), rg1 if part1 is not None else 0, eps,
                               ptr(gamma), ptr(beta), ptr(film), film.stride(0) if film is not None else 0, act, resample,
                               ptr(y), _row_stride(y), ptr(xres), _row_stride(xres) if xres is not None else 0,
                               stream_ptr()))
    return y


# ------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------
def attention_d64(qkv, heads, enc=None, scale=0.125, out=None, hs=192, q_off=0, k_off=64, v_off=128, ehs=128,
                  ek_off=0, ev_off=64):
    """qkv fp16 [B, T, >=heads*hs]; enc fp16 [B, Tc, heads*ehs] or None -> fp16 [B, T, heads*64]."""
    lib = nat.load()
    B, T = qkv.shape[:2]
    Tc = enc.shape[1] if enc is not None else 0
    if out is None:
        out = torch.empty((B, T, heads * 64), dtype=torch.float16, device=qkv.device)
    check(lib.k2_attention_d64(ptr(qkv), qkv.stride(1), hs, q_off, k_off, v_off, ptr(enc),
                               enc.stride(1) if enc is not None else 0, ehs, ek_off, ev_off, B, heads, T, Tc,
                               scale, ptr(out), out.stride(1), stream_ptr()))
    return out


def attention_d512(qkv, scale, out=None, q_off=0, k_off=512, v_off=1024):
    """qkv fp16 [B, T, >= 1536] (q | k | v of ONE head of width 512) -> fp16 [B, T, 512]; the MoVQ AttnBlock fused."""
    lib = nat.load()
    B, T = qkv.shape[:2]
    if out is None:
        out = torch.empty((B, T, 512), dtype=torch.float16, device=qkv.device)
    check(lib.k2_attention_d512(ptr(qkv), qkv.stride(1), q_off, k_off, v_off, B, T, float(scale), ptr(out), out.stride(1),
                                stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# small dense layers
# ------------------------------------------------------------------------------------------------
def linear(x, W, b=None, add=None, silu_in=False, silu_out=False, out=None):
    """fp32 x [M,K] (row-strided ok) @ W[N,K]^T (+b) (+add) -> fp32 [M,N]."""
    lib = nat.load()
    M, K = x.shape
    N = W.shape[0]
    assert W.shape[1] == K and W.is_contiguous() and x.dtype == torch.float32
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    check(lib.k2_linear(ptr(x), x.stride(0), ptr(W), 1 if W.dtype == torch.float16 else 0, ptr(b), ptr(add),
                        add.stride(0) if add is not None else 0, ptr(out), out.stride(0), M, N, K,
                        int(silu_in), int(silu_out), stream_ptr()))
    return out


def layernorm(x, gamma, beta, eps=1e-5):
    lib = nat.load()
    M, N = x.shape
    y = torch.empty_like(x)
    check(lib.k2_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(y), M, N, eps, stream_ptr()))
    return y


def timestep_embedding(t, dim, max_period=10000.0, out=None):
    lib = nat.load()
    B = t.shape[0]
    if out is None:
        out = torch.empty((B, dim), dtype=torch.float32, device=t.device)
    check(lib.k2_timestep_embedding(ptr(t), ptr(out), B, dim, max_period, stream_ptr()))
    return out


def f32_to_f16(x, out=None):
    lib = nat.load()
    assert x.is_contiguous() and x.dtype == torch.float32
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    check(lib.k2_f32_to_f16(ptr(x), ptr(out), x.numel(), stream_ptr()))
    return out


def silu_f16_(x):
    """SiLU in place on a contiguous fp16 tensor."""
    lib = nat.load()
    assert x.dtype == torch.float16 and x.is_contiguous()
    check(lib.k2_silu_f16(ptr(x), ptr(x), x.numel(), stream_ptr()))
    return x


def stem_im2col(x, x2=None, x3=None, mul23=False, kpad=None, out=None):
    """fp32 NCHW inputs -> fp16 [NB, H, W, kpad] 3x3 patches of cat([x, x2*(x3 if mul23), x3], 1)."""
    lib = nat.load()
    NB, Cx, H, W = x.shape
    C2 = x2.shape[1] if x2 is not None else 0
    C3 = x3.shape[1] if x3 is not None else 0
    cin = Cx + C2 + C3
    if kpad is None:
        kpad = _pad64(9 * cin)
    if out is None:
        out = torch.empty((NB, H, W, kpad), dtype=torch.float16, device=x.device)
    check(lib.k2_stem_im2col(ptr(x), Cx, ptr(x2), C2, ptr(x3), C3, int(mul23), NB, H, W, ptr(out), kpad,
                             stream_ptr()))
    return out


def pack_stem_weight(w):
    """[Cout, Cin, 3, 3] -> fp16 [Cout, pad64(9*Cin)] with k = tap*Cin + c (matches stem_im2col)."""
    cout, cin = w.shape[:2]
    wp = w.detach().permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    k = _pad64(9 * cin)
    if k != 9 * cin:
        wp = torch.nn.functional.pad(wp, (0, k - 9 * cin))
    return wp.to(torch.float16).contiguous()


# ------------------------------------------------------------------------------------------------
# sampler / MoVQ helpers
# ------------------------------------------------------------------------------------------------
def sampler_step(model_out, x, noise, coef, guidance, cond_first, clip=2.0, threshold_mode=0, inpaint_init=None,
                 inpaint_mask=None, work=None, inpaint_noise=None):
    lib = nat.load()
    B, _, H, W = x.shape
    if work is None:
        work = torch.empty(B * 4 * H * W + 4096, dtype=torch.float32, device=x.device)
    check(lib.k2_sampler_step(ptr(model_out), ptr(x), ptr(noise), ptr(coef), B, H, W, float(guidance),
                              int(cond_first), float(clip), int(threshold_mode), ptr(inpaint_init),
                              ptr(inpaint_mask), ptr(inpaint_noise), ptr(work), stream_ptr()))
    return x


def step_begin(x, x_in, t_in, coef_out, ts_seq, coef_seq, noise_seq, noise, counter):
    """k2_step_begin: counter = device int32 [2] = (k, nsteps); see k2b200.h."""
    lib = nat.load()
    n = x.numel()
    assert x_in.numel() == 2 * n and x.is_contiguous() and x_in.is_contiguous()
    check(lib.k2_step_begin(ptr(x), ptr(x_in), n, ptr(t_in), t_in.numel(), ptr(coef_out), ptr(ts_seq), ptr(coef_seq),
                            ptr(noise_seq), ptr(noise), ptr(counter), stream_ptr()))


def step_end(counter):
    check(nat.load().k2_step_end(ptr(counter), stream_ptr()))


def _slot_check(who, S, n, f32=(), state=None, shaped=()):
    """Refuse what the slot kernels would read wrongly: host tensors, fp32 operands that are not contiguous fp32, a state that
    is not a contiguous int32 [2, S], and operands whose element count is not the one the kernel indexes (shaped: (name,
    tensor, expected numel))."""
    tensors = [t for _, t in f32 if t is not None] + ([state] if state is not None else [])
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error(f"{who}: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    for name, t in f32:
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous()):
            raise nat.K2Error(f"{who}: {name} must be a contiguous float32 tensor, got {t.dtype}"
                              f"{'' if t.is_contiguous() else ' (not contiguous)'}")
    if state is not None and (state.dtype != torch.int32 or not state.is_contiguous() or tuple(state.shape) != (2, S)):
        raise nat.K2Error(f"{who}: state must be a contiguous int32 [2, {S}] tensor, got {state.dtype} {tuple(state.shape)}")
    for name, t, numel in shaped:
        if t is not None and t.numel() != numel:
            raise nat.K2Error(f"{who}: {name} must hold {numel} elements for {S} slots of {n}, got {tuple(t.shape)}")


def slot_step_begin(x, x_in, t_in, coef_out, ts_tab, coef_tab, noise_tab, noise, state):
    """k2_slot_step_begin: x fp32 [S, 4, H, W] -> x_in rows s and S + s of every active slot, t_in [2S], coef_out [S, 8] and
    noise [S, 4, H, W] from the slot's row k_s of ts_tab [S, kmax], coef_tab [S, kmax, 8] and noise_tab [S, kmax, 4, H, W]
    (or None); state = device int32 [2, S] = (k_s, steps_s); see k2b200.h."""
    S = x.shape[0]
    n = x[0].numel()
    kmax = ts_tab.shape[-1]
    _slot_check("slot_step_begin", S, n,
                f32=(("x", x), ("x_in", x_in), ("t_in", t_in), ("coef_out", coef_out), ("ts_tab", ts_tab),
                     ("coef_tab", coef_tab), ("noise_tab", noise_tab), ("noise", noise)), state=state,
                shaped=(("x_in", x_in, 2 * S * n), ("t_in", t_in, 2 * S), ("coef_out", coef_out, 8 * S),
                        ("ts_tab", ts_tab, S * kmax), ("coef_tab", coef_tab, 8 * S * kmax),
                        ("noise_tab", noise_tab, S * kmax * n), ("noise", noise, S * n)))
    check(nat.load().k2_slot_step_begin(ptr(x), ptr(x_in), S, n, ptr(t_in), ptr(coef_out), ptr(ts_tab), ptr(coef_tab), kmax,
                                        ptr(noise_tab), ptr(noise), ptr(state), stream_ptr()))


def slot_step_end(state):
    """k2_slot_step_end: k_s += 1 for every active slot of state = device int32 [2, S]."""
    _slot_check("slot_step_end", state.shape[-1], 0, state=state)
    check(nat.load().k2_slot_step_end(ptr(state), state.shape[-1], stream_ptr()))


def _slot_step_operands(who, model_out, x, coef, guidance, state, c2, others):
    S, C, H, W = x.shape
    n = 4 * H * W
    if C != 4:
        raise nat.K2Error(f"{who}: x must be [S, 4, H, W], got {tuple(x.shape)}")
    _slot_check(who, S, n, f32=(("model_out", model_out), ("x", x), ("coef", coef), ("guidance", guidance)) + others,
                state=state, shaped=(("model_out", model_out, 2 * S * c2 * H * W), ("coef", coef, 8 * S),
                                     ("guidance", guidance, S)) + tuple((name, t, S * n) for name, t in others))
    return S, H, W


def slot_sampler_step(model_out, x, noise, coef, guidance, state, work, clip=2.0, *, cond_first=0, threshold_mode=0, sval=None):
    """k2_slot_sampler_step: the DDPM / DDIM step of every active slot of x fp32 [S, 4, H, W] in place, with the slot's row
    of coef [S, 8] and its guidance [S] (device fp32); model_out [2S, 8, H, W], noise and work fp32 [S, 4, H, W].
    cond_first: the row order (0: unconditional row s, conditional row S + s, Kandinsky 2.2; 1: the reverse, Kandinsky 2.1).
    threshold_mode 1 clips each slot's x0 with its own dynamic threshold, written to sval fp32 [S]."""
    S, H, W = _slot_step_operands("slot_sampler_step", model_out, x, coef, guidance, state, 8,
                                  (("noise", noise), ("work", work)))
    _slot_check("slot_sampler_step", S, 1, f32=(("sval", sval),), shaped=(("sval", sval, S),))
    check(nat.load().k2_slot_sampler_step(ptr(model_out), ptr(x), ptr(noise), ptr(coef), ptr(guidance), ptr(state), S, H, W,
                                          float(clip), int(cond_first), int(threshold_mode), ptr(sval), ptr(work),
                                          stream_ptr()))
    return x


def slot_dpm_solver_step(model_out, x, hist, coef, guidance, state, *, cond_first=0):
    """k2_slot_dpm_solver_step: the DPM-Solver++(2M) step of every active slot of x fp32 [S, 4, H, W] in place, hist
    [S, 4, H, W] per slot, model_out [2S, C2, H, W], rows, guidance and cond_first as slot_sampler_step."""
    S, H, W = _slot_step_operands("slot_dpm_solver_step", model_out, x, coef, guidance, state, model_out.shape[1],
                                  (("hist", hist),))
    check(nat.load().k2_slot_dpm_solver_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(hist), ptr(coef),
                                             ptr(guidance), ptr(state), S, H, W, int(cond_first), stream_ptr()))
    return x


def plms_step(model_out, x, out, hist, store, coef, guidance, cond_first):
    """hist: list of up to 3 fp32 [B,4,H,W] tensors, newest first (None entries allowed)."""
    lib = nat.load()
    B, _, H, W = x.shape
    hh = list(hist) + [None] * (3 - len(hist))
    check(lib.k2_plms_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(out), ptr(hh[0]), ptr(hh[1]), ptr(hh[2]), ptr(store),
                           ptr(coef), B, H, W, float(guidance), int(cond_first), stream_ptr()))
    return out


def dpm_solver_step(model_out, x, hist, coef, guidance, cond_first, inpaint_init=None, inpaint_mask=None, inpaint_noise=None,
                    noise=None):
    """k2_dpm_solver_step: x fp32 [B,4,H,W] -> the next DPM-Solver++(2M) iterate in place; hist fp32 [B,4,H,W] -> this step's
    x0 (read only when coef[4] != 0); coef = device fp32 [8] row of DPMSolverSchedule; see k2b200.h.
    noise fp32 [B,4,H,W] selects the SDE step, k2_dpm_solver_sde_step: x' += coef[7] noise (read only when coef[7] != 0)."""
    tensors = (model_out, x, hist, coef, inpaint_init, inpaint_mask, inpaint_noise, noise)
    if not all(t is None or t.is_cuda for t in tensors):
        raise nat.K2Error("dpm_solver_step: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    lib = nat.load()
    B, _, H, W = x.shape
    tail = (ptr(coef), B, H, W, float(guidance), int(cond_first), ptr(inpaint_init), ptr(inpaint_mask), ptr(inpaint_noise),
            stream_ptr())
    if noise is None:
        check(lib.k2_dpm_solver_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(hist), *tail))
    else:
        check(lib.k2_dpm_solver_sde_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(hist), ptr(noise), *tail))
    return x


def unipc_step(model_out, x, last, hist1, hist2, coef, guidance, cond_first, counter=None, inpaint_init=None, inpaint_mask=None,
               inpaint_noise=None):
    """k2_unipc_step: x fp32 [B,4,H,W] -> the next UniPC iterate in place; last -> this step's corrected sample, (hist1, hist2)
    -> (D_k, D_{k-1}).  coef: a device fp32 [16] row of UniPCSchedule, or with counter (device int32 [2] = (k, steps)) the
    staged table [steps, 16] whose row k applies; see k2b200.h."""
    tensors = (model_out, x, last, hist1, hist2, coef, counter, inpaint_init, inpaint_mask, inpaint_noise)
    if not all(t is None or t.is_cuda for t in tensors):
        raise nat.K2Error("unipc_step: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    lib = nat.load()
    B, _, H, W = x.shape
    check(lib.k2_unipc_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(last), ptr(hist1), ptr(hist2), ptr(coef),
                            ptr(counter), B, H, W, float(guidance), int(cond_first), ptr(inpaint_init), ptr(inpaint_mask),
                            ptr(inpaint_noise), stream_ptr()))
    return x


def heun_step(model_out, x, x_prev, d_prev, coef, guidance, cond_first, inpaint_init=None, inpaint_mask=None,
              inpaint_noise=None):
    """k2_heun_step: x fp32 [B,4,H,W] (the latent in the UNet's input scale) -> the next Heun stage in place.  coef = device
    fp32 [8] row of HeunSchedule; its stage column picks the predictor (stores x and d in x_prev / d_prev, which it does not
    read) or the corrector (reads them); see k2b200.h."""
    tensors = (model_out, x, x_prev, d_prev, coef, inpaint_init, inpaint_mask, inpaint_noise)
    if not all(t is None or t.is_cuda for t in tensors):
        raise nat.K2Error("heun_step: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    lib = nat.load()
    B, _, H, W = x.shape
    check(lib.k2_heun_step(ptr(model_out), model_out.shape[1], ptr(x), ptr(x_prev), ptr(d_prev), ptr(coef), B, H, W,
                           float(guidance), int(cond_first), ptr(inpaint_init), ptr(inpaint_mask), ptr(inpaint_noise),
                           stream_ptr()))
    return x


def vq_argmin(z, codebook):
    """z fp32 [n, dim], codebook fp32 [n_embed, dim] -> int64 [n] (ties -> lowest index)."""
    lib = nat.load()
    n, dim = z.shape
    idx = torch.empty((n,), dtype=torch.int64, device=z.device)
    check(lib.k2_vq_argmin(ptr(z), ptr(codebook), ptr(idx), n, codebook.shape[0], dim, stream_ptr()))
    return idx


def pointwise_nchw_f32(x, w, b, out=None):
    lib = nat.load()
    NB, Ci, H, W = x.shape
    Co = w.shape[0]
    y = out if out is not None else torch.empty((NB, Co, H, W), dtype=torch.float32, device=x.device)
    check(lib.k2_pointwise_nchw_f32(ptr(x), ptr(w), ptr(b), ptr(y), NB, Ci, Co, H * W, stream_ptr()))
    return y


def upsample2x(x, out=None):
    """fp16 NHWC [NB,H,W,C] -> nearest 2x [NB,2H,2W,C]."""
    lib = nat.load()
    NB, H, W, C = x.shape
    if out is None:
        out = torch.empty((NB, 2 * H, 2 * W, C), dtype=torch.float16, device=x.device)
    check(lib.k2_upsample2x_nhwc(ptr(x), _row_stride(x), ptr(out), _row_stride(out), NB, H, W, C, stream_ptr()))
    return out


def subsample2(x, oy=1, ox=1, out=None):
    """fp16 NHWC [NB,H,W,C] -> [NB,H/2,W/2,C] taking pixels (2y+oy, 2x+ox)."""
    lib = nat.load()
    NB, H, W, C = x.shape
    if out is None:
        out = torch.empty((NB, H // 2, W // 2, C), dtype=torch.float16, device=x.device)
    check(lib.k2_subsample2_nhwc(ptr(x), _row_stride(x), ptr(out), _row_stride(out), NB, H, W, C, oy, ox, stream_ptr()))
    return out


def softmax_rows(x, scale, out=None):
    """fp16 [rows, n] (row-strided) -> softmax(scale * x) fp16."""
    lib = nat.load()
    rows, n = x.shape
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float16, device=x.device)
    check(lib.k2_softmax_rows(ptr(x), x.stride(0), ptr(out), out.stride(0), rows, n, float(scale), stream_ptr()))
    return out


def sn_apply(x, stats, gamma, beta, zq, sn_w, act=1, groups=32, y=None):
    """MoVQ SpatialNorm (+ swish): x fp16 NHWC [NB,H,W,C], zq fp32 [NB,zh,zw,4], sn_w fp32 [C,10] -> fp16 NHWC (k2_sn_apply)."""
    lib = nat.load()
    NB, H, W, C = x.shape
    if y is None:
        y = torch.empty((NB, H, W, C), dtype=torch.float16, device=x.device)
    check(lib.k2_sn_apply(ptr(x), C, _row_stride(x), NB, H, W, groups, ptr(stats), ptr(gamma), ptr(beta), ptr(zq),
                          zq.shape[1], zq.shape[2], ptr(sn_w), act, ptr(y), _row_stride(y), stream_ptr()))
    return y


def transpose_f16(x, out=None):
    """fp16 [B, T, C] (row-strided) -> contiguous [B, C, T]."""
    lib = nat.load()
    B, T, C = x.shape
    assert x.stride(-1) == 1 and x.stride(0) == T * x.stride(1)
    if out is None:
        out = torch.empty((B, C, T), dtype=torch.float16, device=x.device)
    check(lib.k2_transpose_f16(ptr(x), x.stride(1), ptr(out), B, T, C, stream_ptr()))
    return out


def nchw_to_nhwc_f32(x, out=None):
    lib = nat.load()
    NB, C, H, W = x.shape
    y = out if out is not None else torch.empty((NB, H, W, C), dtype=torch.float32, device=x.device)
    check(lib.k2_nchw_to_nhwc_f32(ptr(x), ptr(y), NB, C, H, W, stream_ptr()))
    return y


def images_to_u8(x, crop_h, crop_w, out=None):
    lib = nat.load()
    NB, C, H, W = x.shape
    if out is None:
        out = torch.empty((NB, crop_h, crop_w, C), dtype=torch.uint8, device=x.device)
    check(lib.k2_images_to_u8(ptr(x), ptr(out), NB, C, H, W, crop_h, crop_w, stream_ptr()))
    return out


def lora_merge(base, up, down, scale, out=None):
    """fp16 base [rows, >= cols] (row-strided) + scale * (fp32 up [rows, rank] @ fp32 down [rank, cols]) -> fp16 [rows, cols],
    fp32 sum in ascending rank order, one rounding (k2_lora_merge).  out may be base itself, or another row-strided fp16
    [rows, >= cols] tensor; its columns from cols on are left alone."""
    lib = nat.load()
    rows, rank = up.shape
    cols = down.shape[1]
    assert up.dtype == down.dtype == torch.float32 and up.is_contiguous() and down.is_contiguous() and down.shape[0] == rank
    assert base.dtype == torch.float16 and base.stride(1) == 1 and base.shape[0] == rows and base.shape[1] >= cols
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.float16, device=base.device)
    assert out.dtype == torch.float16 and out.stride(1) == 1 and out.shape[0] == rows and out.shape[1] >= cols
    check(lib.k2_lora_merge(ptr(base), base.stride(0), ptr(up), ptr(down), rows, cols, rank, float(scale), ptr(out),
                            out.stride(0), stream_ptr()))
    return out


def lora_merge_weights(weights, factors, scale):
    """Merge one LoRA adapter into a model's weights: for each (adapter key, unmerged fp16 weight, out) of `weights`, out =
    the unmerged weight when factors ({adapter key: (up, down)}) has no pair for the key, else lora_merge(base, up, down,
    scale, out=out), which leaves out's columns past the factors' width as they were."""
    for key, base, out in weights:
        f = factors.get(key)
        if f is None:
            out.copy_(base)
        else:
            up, down = (t.to(base.device) for t in f)
            lora_merge(base, up, down, scale, out=out)


def set_tuning(key, value):
    """k2_set_tuning: key 0 = force conv N tile, key 1 = split-K (0 auto, 1 off, n forced)."""
    check(nat.load().k2_set_tuning(int(key), int(value)))


def launch_count():
    return nat.load().k2_launch_count()


def reset_launch_count():
    nat.load().k2_reset_launch_count()


# ------------------------------------------------------------------------------------------------
# diffusion prior helpers (groundwork, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def layernorm_f16(x, gamma, beta, eps=1e-5, out=None):
    """LayerNorm over the last dim of fp16 rows [..., N] (fp32 gain / bias) -> fp16."""
    lib = nat.load()
    N = x.shape[-1]
    M = x.numel() // N
    assert x.dtype == torch.float16 and x.stride(-1) == 1
    if out is None:
        out = torch.empty_like(x)
    check(lib.k2_layernorm_f16(ptr(x), _row_stride(x), ptr(gamma), ptr(beta), ptr(out), _row_stride(out), M, N, eps,
                               stream_ptr()))
    return out


def gelu_f16_(x):
    """Exact GELU in place on a contiguous fp16 tensor."""
    lib = nat.load()
    assert x.dtype == torch.float16 and x.is_contiguous()
    check(lib.k2_gelu_f16(ptr(x), ptr(x), x.numel(), stream_ptr()))
    return x


def quick_gelu_f16_(x, out=None):
    """OpenAI CLIP's QuickGELU, x * sigmoid(1.702 x), on a contiguous fp16 tensor: in place, or into `out` (contiguous fp16
    of the same shape)."""
    if not x.is_cuda or (out is not None and not out.is_cuda):
        raise nat.K2Error("quick_gelu_f16: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    assert x.dtype == torch.float16 and x.is_contiguous(), (x.dtype, x.stride())
    out = x if out is None else out
    assert out.dtype == torch.float16 and out.is_contiguous() and out.shape == x.shape, (out.dtype, tuple(out.shape))
    check(nat.load().k2_quick_gelu_f16(ptr(x), ptr(out), x.numel(), stream_ptr()))
    return out


def attention_small(qkv, heads, keep_mask=None, causal=True, scale=0.125, out=None):
    """qkv fp16 [B, T, heads*192] (per head [q|k|v]), keep_mask uint8 or bool [B, T] (nonzero = key kept) or None -> fp16
    [B, T, heads*64]; T <= 128.  A query row that can reach no key (every key masked, or causal with key 0 masked) is NaN,
    as torch's softmax over an all -inf row is."""
    B, T = qkv.shape[:2]
    assert qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.shape[2] == heads * 192, (qkv.dtype, qkv.shape, heads)
    if keep_mask is not None:
        assert keep_mask.dtype in (torch.uint8, torch.bool), keep_mask.dtype
        assert tuple(keep_mask.shape) == (B, T) and keep_mask.is_contiguous(), (keep_mask.shape, keep_mask.stride(), B, T)
        assert keep_mask.device == qkv.device, (keep_mask.device, qkv.device)
    lib = nat.load()
    if out is None:
        out = torch.empty((B, T, heads * 64), dtype=torch.float16, device=qkv.device)
    assert out.dtype == torch.float16 and tuple(out.shape) == (B, T, heads * 64), (out.dtype, out.shape)
    check(lib.k2_attention_small(ptr(qkv), _row_stride(qkv), ptr(keep_mask), int(causal), ptr(out), _row_stride(out), B, T,
                                 heads, scale, stream_ptr()))
    return out


def _rows_2d(t, dtype, name):
    """(row stride, rows, columns) of a 2-D view with unit column stride; a row stride of 0 (an expanded row) is kept."""
    assert t.dtype == dtype and t.dim() == 2 and t.stride(1) == 1, (name, t.dtype, tuple(t.shape), t.stride())
    return t.stride(0) if t.shape[0] > 1 else t.shape[1], t.shape[0], t.shape[1]


def prior_tokens(x, pos, out):
    """k2_prior_tokens: out fp16 [M, N] (row-strided view) = fp16(fp16(x) + pos) with the eager forward's two roundings.
    x fp32 [M, N] or [1, N] expanded to M rows (row stride 0), pos fp16 likewise."""
    tensors = (x, pos, out)
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error("prior_tokens: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    ldy, M, N = _rows_2d(out, torch.float16, "out")
    ldx, mx, nx = _rows_2d(x, torch.float32, "x")
    ldp, mp, np_ = _rows_2d(pos, torch.float16, "pos")
    assert nx == N and np_ == N and mx == M and mp == M, (tuple(x.shape), tuple(pos.shape), tuple(out.shape))
    check(nat.load().k2_prior_tokens(ptr(x), ldx, ptr(pos), ldp, ptr(out), ldy, M, N, stream_ptr()))
    return out


def f16_to_f32(x, out=None):
    """k2_f16_to_f32: exact widening of fp16 rows [M, N] (row-strided view) -> fp32 [M, N] (out may be row-strided)."""
    if not x.is_cuda or (out is not None and not out.is_cuda):
        raise nat.K2Error("f16_to_f32: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    ldx, M, N = _rows_2d(x, torch.float16, "x")
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    ldy, my, ny = _rows_2d(out, torch.float32, "out")
    assert (my, ny) == (M, N), (tuple(x.shape), tuple(out.shape))
    check(nat.load().k2_f16_to_f32(ptr(x), ldx, ptr(out), ldy, M, N, stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# CLIP image tower (kandinsky2/model/clip_vision.py, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def clip_patchify(x, patch, kp, out=None):
    """k2_clip_patchify: fp32 NCHW pixels [B, 3, S, S] -> fp16 GEMM rows [B, (S / patch)^2 + 1, kp] (out may be row-strided):
    the one-hot CLS row, then each patch's pixels in (c, ky, kx) order, zero-padded to kp columns."""
    if not x.is_cuda or (out is not None and not out.is_cuda):
        raise nat.K2Error("clip_patchify: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    assert x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.shape[2] == x.shape[3] and x.is_contiguous(), \
        (x.dtype, tuple(x.shape))
    B, S = x.shape[0], x.shape[2]
    T = (S // patch) ** 2 + 1
    if out is None:
        out = torch.empty((B, T, kp), dtype=torch.float16, device=x.device)
    assert out.dtype == torch.float16 and tuple(out.shape) == (B, T, kp), (out.dtype, tuple(out.shape))
    check(nat.load().k2_clip_patchify(ptr(x), B, S, patch, ptr(out), _row_stride(out), kp, stream_ptr()))
    return out


def attention_heads(qkv, heads, head_dim, scale, out=None, hs=None, q_off=0, k_off=None, v_off=None, ohs=None):
    """k2_attention_heads: qkv fp16 [B, T, >= heads * hs] with per-head [q | k | v] (hs = 3 head_dim, offsets 0 / head_dim /
    2 head_dim by default: checkpoints.pack_heads) -> fp16 [B, T, heads * head_dim] (out may be a row-strided view whose heads
    are ohs apart).  head_dim 104 only (the library refuses anything else)."""
    hs = 3 * head_dim if hs is None else hs
    k_off = head_dim if k_off is None else k_off
    v_off = 2 * head_dim if v_off is None else v_off
    ohs = head_dim if ohs is None else ohs
    assert qkv.dtype == torch.float16 and qkv.dim() == 3, (qkv.dtype, tuple(qkv.shape))
    B, T = qkv.shape[:2]
    if out is None:
        out = torch.empty((B, T, heads * ohs), dtype=torch.float16, device=qkv.device)
    assert out.dtype == torch.float16 and out.dim() == 3 and tuple(out.shape[:2]) == (B, T), (out.dtype, tuple(out.shape))
    check(nat.load().k2_attention_heads(ptr(qkv), _row_stride(qkv), hs, q_off, k_off, v_off, B, heads, T, head_dim,
                                        float(scale), ptr(out), _row_stride(out), ohs, stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# CLIP text tower (kandinsky2/model/clip_text.py, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def clip_text_embed(ids, tok, pos, out=None):
    """k2_clip_text_embed: int32 ids [B, T] (row-strided view), fp16 tables tok [V, H] and pos [>= T, H] -> fp16 rows
    [B, T, H] (out may be row-strided) = fp16(float(tok[id]) + float(pos[t])); an id outside [0, V) gives a NaN row."""
    tensors = (ids, tok, pos) + ((out,) if out is not None else ())
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error("clip_text_embed: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    ldi, B, T = _rows_2d(ids, torch.int32, "ids")
    assert tok.dtype == torch.float16 and pos.dtype == torch.float16 and tok.is_contiguous() and pos.is_contiguous(), \
        (tok.dtype, pos.dtype)
    V, H = tok.shape
    assert pos.dim() == 2 and pos.shape[1] == H and pos.shape[0] >= T, (tuple(pos.shape), H, T)
    if out is None:
        out = torch.empty((B, T, H), dtype=torch.float16, device=ids.device)
    assert out.dtype == torch.float16 and tuple(out.shape) == (B, T, H), (out.dtype, tuple(out.shape))
    check(nat.load().k2_clip_text_embed(ptr(ids), ldi, B, T, ptr(tok), V, ptr(pos), H, ptr(out), _row_stride(out),
                                        stream_ptr()))
    return out


def clip_text_pool(ids, hidden, eos_id, out=None, index_out=None):
    """k2_clip_text_pool: int32 ids [B, T] (row-strided view), fp16 hidden [B, T, H] (row-strided) -> fp32 [B, H] = the
    hidden row at each sequence's pooled position (eos_id < 0: the first argmax of the ids; else the first position equal to
    eos_id, 0 if none), widened exactly.  index_out: int32 [B] receives the positions."""
    tensors = (ids, hidden) + tuple(t for t in (out, index_out) if t is not None)
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error("clip_text_pool: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    ldi, B, T = _rows_2d(ids, torch.int32, "ids")
    assert hidden.dtype == torch.float16 and hidden.dim() == 3 and tuple(hidden.shape[:2]) == (B, T), \
        (hidden.dtype, tuple(hidden.shape))
    H = hidden.shape[2]
    if out is None:
        out = torch.empty((B, H), dtype=torch.float32, device=ids.device)
    ldo, mo, no = _rows_2d(out, torch.float32, "out")
    assert (mo, no) == (B, H), (tuple(out.shape), B, H)
    if index_out is not None:
        assert index_out.dtype == torch.int32 and tuple(index_out.shape) == (B,) and index_out.is_contiguous()
    check(nat.load().k2_clip_text_pool(ptr(ids), ldi, B, T, int(eos_id), ptr(hidden), _row_stride(hidden), H, ptr(out), ldo,
                                       ptr(index_out), stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# Kandinsky 2.1 text encoder (kandinsky2/model/text_encoders.py, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def xlmr_embed(ids, pad_id, word, pos, type_row, gamma, beta, eps, out=None):
    """k2_xlmr_embed: int32 ids [B, T] (row-strided view) -> fp16 rows [B, T, H] (out may be row-strided) =
    LayerNorm(word[id] + type_row + pos[p]) with the position p computed from the row's ids (pad_id + the count of non-pad
    ids up to t; pad_id on a pad id), fp32 sum, float64 statistics, one rounding.  An id outside [0, V) or a position beyond
    the table gives a NaN row."""
    tensors = (ids, word, pos, type_row, gamma, beta) + ((out,) if out is not None else ())
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error("xlmr_embed: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    ldi, B, T = _rows_2d(ids, torch.int32, "ids")
    assert word.dtype == pos.dtype == type_row.dtype == torch.float16, (word.dtype, pos.dtype, type_row.dtype)
    assert word.is_contiguous() and pos.is_contiguous() and type_row.is_contiguous()
    V, H = word.shape
    P = pos.shape[0]
    assert pos.dim() == 2 and pos.shape[1] == H and type_row.numel() == H, (tuple(pos.shape), tuple(type_row.shape), H)
    for t in (gamma, beta):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == H, (t.dtype, tuple(t.shape), H)
    if out is None:
        out = torch.empty((B, T, H), dtype=torch.float16, device=ids.device)
    assert out.dtype == torch.float16 and tuple(out.shape) == (B, T, H), (out.dtype, tuple(out.shape))
    check(nat.load().k2_xlmr_embed(ptr(ids), ldi, B, T, int(pad_id), ptr(word), V, ptr(pos), P, ptr(type_row), ptr(gamma),
                                   ptr(beta), float(eps), ptr(out), _row_stride(out), H, stream_ptr()))
    return out


def masked_mean_f16(hidden, mask, out=None):
    """k2_masked_mean_f16: fp16 hidden [B, T, H] (row-strided), uint8 / bool mask [B, T] (row-strided, nonzero = kept) -> fp32
    [B, H] (out may be row-strided): the kept rows' fp32 sum in ascending t divided once by their count; NaN for a row with
    no kept token."""
    tensors = (hidden, mask) + ((out,) if out is not None else ())
    if not all(t.is_cuda for t in tensors):
        raise nat.K2Error("masked_mean_f16: tensors must live on a CUDA sm_90 device (no CPU fallback)")
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    ldm, B, T = _rows_2d(mask, torch.uint8, "mask")
    assert hidden.dtype == torch.float16 and hidden.dim() == 3 and tuple(hidden.shape[:2]) == (B, T), \
        (hidden.dtype, tuple(hidden.shape))
    H = hidden.shape[2]
    if out is None:
        out = torch.empty((B, H), dtype=torch.float32, device=hidden.device)
    ldo, mo, no = _rows_2d(out, torch.float32, "out")
    assert (mo, no) == (B, H), (tuple(out.shape), B, H)
    check(nat.load().k2_masked_mean_f16(ptr(hidden), _row_stride(hidden), ptr(mask), ldm, B, T, H, ptr(out), ldo,
                                        stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# DPT depth estimator (kandinsky2/model/depth.py, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def _on_device(name, *tensors):
    if not all(t.is_cuda for t in tensors if t is not None):
        raise nat.K2Error(f"{name}: tensors must live on a CUDA sm_90 device (no CPU fallback)")


def _rows(t, dtype, name):
    """(rows, columns, row stride) of a tensor whose last dimension is contiguous and whose leading dimensions are row-strided
    (_row_stride)."""
    assert t.dtype == dtype and t.dim() >= 2 and t.stride(-1) == 1, (name, t.dtype, tuple(t.shape), t.stride())
    return t.numel() // t.shape[-1] if t.numel() else 0, t.shape[-1], _row_stride(t)


def relu_f16(x, out=None):
    """k2_relu_f16: torch.relu of fp16 rows [..., N] (row-strided views) into out (default: in place)."""
    out = x if out is None else out
    _on_device("relu_f16", x, out)
    M, N, ldx = _rows(x, torch.float16, "x")
    assert tuple(out.shape) == tuple(x.shape), (tuple(out.shape), tuple(x.shape))
    check(nat.load().k2_relu_f16(ptr(x), ldx, ptr(out), _rows(out, torch.float16, "out")[2], M, N, stream_ptr()))
    return out


def relu_f32(x, out=None):
    """k2_relu_f32: torch.relu of fp32 rows [..., N] (row-strided views) into out (default: in place)."""
    out = x if out is None else out
    _on_device("relu_f32", x, out)
    M, N, ldx = _rows(x, torch.float32, "x")
    assert tuple(out.shape) == tuple(x.shape), (tuple(out.shape), tuple(x.shape))
    check(nat.load().k2_relu_f32(ptr(x), ldx, ptr(out), _rows(out, torch.float32, "out")[2], M, N, stream_ptr()))
    return out


def bilinear_f16(x, size, align_corners, out=None):
    """k2_bilinear_f16: fp16 NHWC [NB, Hi, Wi, C] (row-strided) -> [NB, Ho, Wo, C], size = (Ho, Wo); torch's
    interpolate(mode="bilinear", size=size, align_corners=align_corners) on the NCHW view, one rounding per output."""
    NB, Hi, Wi, C = x.shape
    Ho, Wo = size
    if out is None:
        out = torch.empty((NB, Ho, Wo, C), dtype=torch.float16, device=x.device)
    _on_device("bilinear_f16", x, out)
    assert x.dtype == out.dtype == torch.float16 and tuple(out.shape) == (NB, Ho, Wo, C), (x.dtype, out.dtype, tuple(out.shape))
    check(nat.load().k2_bilinear_f16(ptr(x), _row_stride(x), NB, Hi, Wi, C, ptr(out), _row_stride(out), Ho, Wo,
                                     int(bool(align_corners)), stream_ptr()))
    return out


def depth_to_space_f16(g, s, C, out=None):
    """k2_depth_to_space_f16: GEMM rows g fp16 [NB, H, W, >= s^2 C] (column (a s + b) C + c) -> fp16 NHWC [NB, s H, s W, C]."""
    NB, H, W = g.shape[:3]
    if out is None:
        out = torch.empty((NB, s * H, s * W, C), dtype=torch.float16, device=g.device)
    _on_device("depth_to_space_f16", g, out)
    assert g.dtype == out.dtype == torch.float16 and tuple(out.shape) == (NB, s * H, s * W, C), (g.dtype, tuple(out.shape))
    check(nat.load().k2_depth_to_space_f16(ptr(g), _row_stride(g), NB, H, W, C, s, ptr(out), _row_stride(out), stream_ptr()))
    return out


def readout_rows_f16(h, out=None):
    """k2_readout_rows_f16: fp16 [B, T, H] (token 0 = CLS, row-strided) -> fp16 [B, T - 1, 2 H] = cat(token, CLS) rows."""
    B, T, H = h.shape
    if out is None:
        out = torch.empty((B, T - 1, 2 * H), dtype=torch.float16, device=h.device)
    _on_device("readout_rows_f16", h, out)
    assert h.dtype == out.dtype == torch.float16 and tuple(out.shape) == (B, T - 1, 2 * H), (h.dtype, tuple(out.shape))
    check(nat.load().k2_readout_rows_f16(ptr(h), _row_stride(h), B, T, H, ptr(out), _row_stride(out), stream_ptr()))
    return out


# ------------------------------------------------------------------------------------------------
# BiT backbone of the hybrid DPT (kandinsky2/model/depth.py, see k2b200.h)
# ------------------------------------------------------------------------------------------------
def im2col_f16(x, k, s, pad, size, kp, out=None):
    """k2_im2col_f16: fp32 NCHW x [NB, C, H, W] -> fp16 rows [NB, Ho, Wo, kp] (out may be row-strided): the k x k stride-s
    windows with pad = (top, left) zero padding, columns in (c, ky, kx) order, zeros from k^2 C to kp.  size = (Ho, Wo)."""
    NB, C, H, W = x.shape
    Ho, Wo = size
    if out is None:
        out = torch.empty((NB, Ho, Wo, kp), dtype=torch.float16, device=x.device)
    _on_device("im2col_f16", x, out)
    assert x.dtype == torch.float32 and x.is_contiguous(), (x.dtype, x.stride())
    assert out.dtype == torch.float16 and tuple(out.shape) == (NB, Ho, Wo, kp), (out.dtype, tuple(out.shape))
    check(nat.load().k2_im2col_f16(ptr(x), NB, C, H, W, k, s, pad[0], pad[1], Ho, Wo, ptr(out), _row_stride(out), kp,
                                   stream_ptr()))
    return out


def maxpool_f16(x, pad, size, out=None):
    """k2_maxpool_f16: fp16 NHWC [NB, H, W, C] (row-strided) -> [NB, Ho, Wo, C], 3x3 stride 2, pad = (top, left), pad value 0
    (BitMaxPool2d's).  size = (Ho, Wo)."""
    NB, H, W, C = x.shape
    Ho, Wo = size
    if out is None:
        out = torch.empty((NB, Ho, Wo, C), dtype=torch.float16, device=x.device)
    _on_device("maxpool_f16", x, out)
    assert x.dtype == out.dtype == torch.float16 and tuple(out.shape) == (NB, Ho, Wo, C), (x.dtype, tuple(out.shape))
    check(nat.load().k2_maxpool_f16(ptr(x), _row_stride(x), NB, H, W, C, pad[0], pad[1], Ho, Wo, ptr(out), _row_stride(out),
                                    stream_ptr()))
    return out


def gn_act_f16(x, stats, gamma, beta, r=None, r_norm=None, relu=True, groups=32, out=None):
    """k2_gn_act_f16: fp16 NHWC x [NB, H, W, C] (row-strided) -> [relu](GroupNorm(x) + r) fp16, stats fp32 [NB, groups, 2].
    r: None, an fp16 source of x's shape, or with r_norm = (r_stats, r_gamma, r_beta) a second GroupNorm's input.  out may be
    any [NB, H, W, C] view whose pixels are row-strided within an image (its image stride is read from out.stride(0))."""
    NB, H, W, C = x.shape
    if out is None:
        out = torch.empty_like(x, memory_format=torch.contiguous_format)
    rs, rg, rb = r_norm if r_norm is not None else (None, None, None)
    _on_device("gn_act_f16", x, out, r, stats, gamma, beta, rs, rg, rb)
    assert x.dtype == out.dtype == torch.float16 and tuple(out.shape) == (NB, H, W, C), (x.dtype, tuple(out.shape))
    assert r is None or (r.dtype == torch.float16 and tuple(r.shape) == tuple(x.shape)), tuple(r.shape)
    assert out.stride(-1) == 1 and out.stride(1) == W * out.stride(2), (tuple(out.shape), out.stride())
    for t in (stats, gamma, beta, rs, rg, rb):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous()), (t.dtype, t.stride())
    check(nat.load().k2_gn_act_f16(ptr(x), _row_stride(x), ptr(stats), ptr(gamma), ptr(beta), ptr(r),
                                   _row_stride(r) if r is not None else 0, ptr(rs), ptr(rg), ptr(rb), NB, H, W, C, groups,
                                   int(bool(relu)), ptr(out), out.stride(2), out.stride(0) if NB > 1 else H * W * out.stride(2),
                                   stream_ptr()))
    return out
