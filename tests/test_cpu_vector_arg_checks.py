"""CPU: entry points whose kernels move data in 16-byte (uint4 / float4) or 8-byte (float2) vectors refuse row strides, offsets
and pointers that would break those accesses -- before any CUDA call, so the refusal is visible on a machine without a GPU.

Every call below uses fabricated device addresses and carries exactly one defect; the library must return < 0 with the
expected message.  Nothing is launched (on a GPU machine a call that slipped past its checks would dereference the fabricated
addresses, so each case is first proven to be refused here, where no launch can happen)."""
import ctypes

import pytest

A = 0x10000            # a fabricated 16-byte aligned "device" address; never dereferenced
P = ctypes.c_void_p


def _lib():
    from kandinsky2 import _native
    return _native.load()


def _refused(fn, args, msg):
    lib = _lib()
    rc = getattr(lib, fn)(*args)
    err = lib.k2_last_error().decode()
    assert rc < 0, (fn, args)
    assert msg in err, (fn, err)


def _with(base, **change):
    out = dict(base)
    out.update(change)
    return out


# k2_gn_apply(src0, C0, ld0, src1, C1, ld1, NB, H, W, groups, stats, gamma, beta, film, film_ld, act, resample, y, ldy, xres,
#             ldx, zq, zh, zw, sn_w, stream)
GN_APPLY = dict(src0=P(A), C0=64, ld0=64, src1=None, C1=0, ld1=0, NB=1, H=4, W=4, groups=32, stats=P(A), gamma=P(A),
                beta=P(A), film=None, film_ld=0, act=1, resample=0, y=P(A), ldy=64, xres=None, ldx=0, zq=None, zh=0, zw=0,
                sn_w=None, stream=None)
GN_TWO = dict(src1=P(A + 4096), C1=64, ld1=64, ldy=128)   # a second source of 64 channels: the output has 128

GN_APPLY_CASES = [
    (dict(ld0=68), "row strides"),                                 # ld0 not a multiple of 8: row starts lose alignment
    (dict(ld0=32), "row strides"),                                 # ld0 < C0: rows would overlap
    (dict(GN_TWO, ld1=132), "row strides"),
    (dict(ldy=68), "row strides"),
    (dict(ldy=56), "row strides"),
    (dict(xres=P(A), ldx=60), "row strides"),
    (dict(src0=P(A + 8)), "16-byte aligned"),
    (dict(GN_TWO, src1=P(A + 4104)), "16-byte aligned"),
    (dict(y=P(A + 2)), "16-byte aligned"),
    (dict(xres=P(A + 8), ldx=64), "16-byte aligned"),
    (dict(zq=P(A + 4), zh=2, zw=2, sn_w=P(A)), "16-byte aligned"),  # zq is read as float4
]


@pytest.mark.parametrize("change,msg", GN_APPLY_CASES)
def test_gn_apply_refuses_broken_vector_access(change, msg):
    _refused("k2_gn_apply", list(_with(GN_APPLY, **change).values()), msg)


# k2_gn_apply_fold(src0, C0, ld0, src1, C1, ld1, NB, H, W, groups, part0, rg0, part1, rg1, eps, gamma, beta, film, film_ld, act,
#                  resample, y, ldy, xres, ldx, stream)
GN_FOLD = dict(src0=P(A), C0=64, ld0=64, src1=None, C1=0, ld1=0, NB=1, H=4, W=4, groups=32, part0=P(A), rg0=1, part1=None,
               rg1=0, eps=1e-5, gamma=P(A), beta=P(A), film=None, film_ld=0, act=1, resample=0, y=P(A), ldy=64, xres=None,
               ldx=0, stream=None)
GN_FOLD_TWO = dict(GN_TWO, part1=P(A), rg1=1)


@pytest.mark.parametrize("change,msg", [
    (dict(ld0=68), "row strides"),
    (dict(ld0=32), "row strides"),
    (dict(GN_FOLD_TWO, ld1=100), "row strides"),
    (dict(ldy=12), "row strides"),
    (dict(xres=P(A), ldx=66), "row strides"),
    (dict(src0=P(A + 8)), "16-byte aligned"),
    (dict(GN_FOLD_TWO, src1=P(A + 4104)), "16-byte aligned"),
    (dict(y=P(A + 8)), "16-byte aligned"),
    (dict(xres=P(A + 4), ldx=64), "16-byte aligned"),
    (dict(part0=P(A + 4)), "8-byte aligned"),                      # partials are read as float2
    (dict(GN_FOLD_TWO, part1=P(A + 4)), "8-byte aligned"),
])
def test_gn_apply_fold_refuses_broken_vector_access(change, msg):
    _refused("k2_gn_apply_fold", list(_with(GN_FOLD, **change).values()), msg)


# k2_gn_stats(src0, C0, ld0, src1, C1, ld1, NB, HW, groups, eps, stats, scratch, stream)
GN_STATS = dict(src0=P(A), C0=64, ld0=64, src1=None, C1=0, ld1=0, NB=1, HW=16, groups=32, eps=1e-5, stats=P(A),
                scratch=P(A), stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(ld0=76), "row strides"),
    (dict(ld0=56), "row strides"),
    (dict(src1=P(A), C1=64, ld1=36), "row strides"),
    (dict(src0=P(A + 8)), "16-byte aligned"),
    (dict(src1=P(A + 2), C1=64, ld1=64), "16-byte aligned"),
])
def test_gn_stats_refuses_broken_vector_access(change, msg):
    _refused("k2_gn_stats", list(_with(GN_STATS, **change).values()), msg)


def test_gn_finalize_refuses_misaligned_partials():
    # k2_gn_finalize(part0, C0, rg0, part1, C1, rg1, NB, HW, groups, eps, stats, stream)
    _refused("k2_gn_finalize", [P(A + 4), 64, 1, None, 0, 0, 1, 16, 32, 1e-5, P(A), None], "8-byte aligned")
    _refused("k2_gn_finalize", [P(A), 64, 1, P(A + 12), 64, 1, 1, 16, 32, 1e-5, P(A), None], "8-byte aligned")


@pytest.mark.parametrize("x,ldx,y,ldy,n,msg", [
    (A + 8, 64, A, 64, 64, "16-byte aligned"),
    (A, 64, A + 2, 64, 64, "16-byte aligned"),
    (A, 8, A, 64, 64, ">= n"),               # a row stride shorter than the row
    (A, 64, A, 12, 9, "bad arguments"),      # ldy not a multiple of 8 (already refused before this change)
])
def test_softmax_rows_refuses_broken_vector_access(x, ldx, y, ldy, n, msg):
    # k2_softmax_rows(x, ldx, y, ldy, rows, n, scale, stream)
    _refused("k2_softmax_rows", [P(x), ldx, P(y), ldy, 4, n, 1.0, None], msg)


@pytest.mark.parametrize("fn", ["k2_upsample2x_nhwc", "k2_subsample2_nhwc"])
@pytest.mark.parametrize("x,ldx,y,ldy,msg", [
    (A + 8, 64, A, 64, "16-byte aligned"),
    (A, 64, A + 4, 64, "16-byte aligned"),
    (A, 56, A, 64, ">= C"),
    (A, 64, A, 32, ">= C"),
])
def test_resample_copies_refuse_broken_vector_access(fn, x, ldx, y, ldy, msg):
    args = [P(x), ldx, P(y), ldy, 1, 4, 4, 64]
    if fn == "k2_subsample2_nhwc":
        args += [1, 1]
    _refused(fn, args + [None], msg)


@pytest.mark.parametrize("change,msg", [
    (dict(x=P(A + 8)), "16-byte aligned"),
    (dict(y=P(A + 8)), "16-byte aligned"),
    (dict(zq=P(A + 4)), "16-byte aligned"),
    (dict(ldx=32), ">= C"),
])
def test_sn_apply_refuses_broken_vector_access(change, msg):
    # k2_sn_apply(x, C, ldx, NB, H, W, groups, stats, gamma, beta, zq, zh, zw, sn_w, act, y, ldy, stream)
    base = dict(x=P(A), C=64, ldx=64, NB=1, H=4, W=4, groups=32, stats=P(A), gamma=P(A), beta=P(A), zq=P(A), zh=2, zw=2,
                sn_w=P(A), act=1, y=P(A), ldy=64, stream=None)
    _refused("k2_sn_apply", list(_with(base, **change).values()), msg)


def test_vq_argmin_refuses_misaligned_float4_rows():
    # k2_vq_argmin(z, codebook, idx, n, n_embed, dim, stream)
    _refused("k2_vq_argmin", [P(A + 4), P(A), P(A), 16, 16, 4, None], "16-byte aligned")
    _refused("k2_vq_argmin", [P(A), P(A + 8), P(A), 16, 16, 4, None], "16-byte aligned")


def test_existing_vector_checks_still_refuse():
    """Entry points that already refused misaligned vector access keep doing so (attention, transpose, conv sources / output)."""
    # k2_attention_d512(qkv, ldq, q_off, k_off, v_off, B, T, scale, out, ldo, stream)
    _refused("k2_attention_d512", [P(A + 8), 1536, 0, 512, 1024, 1, 64, 1.0, P(A), 512, None], "attention_d512")
    _refused("k2_attention_d512", [P(A), 1536, 4, 512, 1024, 1, 64, 1.0, P(A), 512, None], "attention_d512")
    # k2_transpose_f16(x, ldx, y, B, T, C, stream)
    _refused("k2_transpose_f16", [P(A + 8), 64, P(A), 1, 64, 64, None], "alignment")
    # k2_attention_d64(qkv, ldq, hs, q_off, k_off, v_off, enc, lde, ehs, ek_off, ev_off, B, heads, T, Tc, scale, out, ldo, st)
    _refused("k2_attention_d64", [P(A), 196, 192, 0, 64, 128, None, 0, 128, 0, 64, 1, 1, 64, 0, 0.125, P(A), 64, None],
             "attention_d64")
    from kandinsky2._native import K2ConvSrc
    lib = _lib()

    def conv(src_ptr=A, ld=64, out=A, ldo=64, gn_part=None):
        srcs = (K2ConvSrc * 1)()
        srcs[0].ptr, srcs[0].C, srcs[0].ld, srcs[0].taps = src_ptr, 64, ld, 1
        info = (ctypes.c_int * 7)()
        # k2_conv_gemm_cfg(srcs, nsrc, NB, H, W, w, w_rows, Ktot, ldw, Cout, bias, residual, ldr, out, ldo, out_mode, ws,
        #                  ws_bytes, gn_partial, info, cfg, w_batch_stride, stream)
        return lib.k2_conv_gemm_cfg(srcs, 1, 1, 4, 4, P(A), 64, 64, 64, 64, None, None, 0, P(out), ldo, 0, None, 0,
                                    P(gn_part) if gn_part else None, info, None, 0, None)

    for kw, msg in ((dict(src_ptr=A + 8), "source not 16B aligned"), (dict(ld=68), "bad source C/ld"),
                    (dict(gn_part=A + 4), "gn_partial must be 8-byte aligned")):
        assert conv(**kw) < 0, kw
        assert msg in lib.k2_last_error().decode(), (kw, lib.k2_last_error())
