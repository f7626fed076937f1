"""CPU: what tests/test_gpu_gemm_float64.py and tests/test_gpu_linear_float64.py rest on, checked without a GPU.

  - the GEMM geometry tests/gemm_ref.py derives from the model code and configs is the geometry the models build;
  - the exact-operand checker is sharp: one fp16 ulp, one swapped bias column or one dropped 16-wide K step is refused;
  - k2_conv_gemm_cfg refuses an out_mode other than 0 / 1 and a residual with out_mode 1, and k2_linear refuses K > 5120, all
    before any CUDA call (fabricated device addresses, never dereferenced, as tests/test_cpu_vector_arg_checks.py)."""
import ctypes

import pytest
import torch

from tests import gemm_ref

A = 0x10000
P = ctypes.c_void_p


def _shape(c):
    return (c.geom, c.srcs, c.cout, c.residual, c.out_mode)


def test_tower_gemm_geometry():
    got = {c.name: _shape(c) for c in gemm_ref.tower_gemms()}
    assert len(got) == 57
    rows = lambda M, K, N, res=False: ((1, 1, M), ((K, 1),), N, res, 0)  # noqa: E731
    for r in (1, 2, 8):
        for tower, T, H, I in (("prior", 81, 2048, 8192), ("clip_text", 77, 1280, 5120), ("clip_vision", 257, 1664, 8192),
                               ("xlmr", 77, 1024, 4096)):
            assert got[f"{tower}:attn.qkv:rows{r}"] == rows(r * T, H, 3 * H)
            assert got[f"{tower}:attn.proj:rows{r}"] == rows(r * T, H, H, True)
            assert got[f"{tower}:mlp.fc1:rows{r}"] == rows(r * T, H, I)
            assert got[f"{tower}:mlp.fc2:rows{r}"] == rows(r * T, I, H, True)
        assert got[f"prior2.1:text_enc_proj:rows{r}"] == rows(r * 77, 768, 2048)
        assert got[f"prior2.2:text_enc_proj:rows{r}"] == rows(r * 77, 1280, 2048)
        assert got[f"clip_vision:patch_embed:rows{r}"] == rows(r * 257, 640, 1664, True)


def test_unet_movq_head_stem_geometry():
    got = {c.name: (_shape(c), c.w_rows, c.stem) for c in gemm_ref.unet_gemms() + gemm_ref.movq_gemms() +
           gemm_ref.head_gemms() + gemm_ref.generic_epilogue_gemms() + gemm_ref.stem_gemms()}
    want = {}
    for ds, C in ((2, 768), (4, 1152), (8, 1536)):
        s = 96 // ds
        want[f"unet:qkv:ds{ds}"] = (((1, 1, 8 * s * s), ((C, 1),), 3 * C, False, 0), 0, None)
        want[f"unet:encoder_kv2.1:ds{ds}"] = (((1, 1, 8 * 87), ((768, 1),), 2 * C, False, 0), 0, None)
        want[f"unet:encoder_kv2.2:ds{ds}"] = (((1, 1, 8 * 32), ((768, 1),), 2 * C, False, 0), 0, None)
        want[f"unet:proj_out:ds{ds}"] = (((8, s, s), ((C, 1),), C, True, 0), 0, None)
    want.update({
        "movq:qkv:T9216": (((1, 1, 2 * 9216), ((512, 1),), 1536, False, 0), 0, None),
        "movq:proj:T9216": (((2, 96, 96), ((512, 1),), 512, True, 0), 0, None),
        "movq:encoder_resblock_nin:256to512": (((2, 96, 96), ((512, 9), (256, 1)), 512, False, 0), 0, None),
        "unet:out": (((8, 96, 96), ((384, 9),), 8, False, 1), 16, None),
        "movq:decoder_conv_out": (((2, 768, 768), ((128, 9),), 3, False, 1), 16, None),
        "movq:encoder_conv_out": (((2, 96, 96), ((512, 9),), 4, False, 1), 16, None),
        "hint:conv7": (((2, 96, 96), ((256, 9),), 4, False, 1), 16, None),
        "hint:conv1": (((2, 768, 768), ((16, 9),), 16, False, 0), 16, None),
        "hint:conv2": (((2, 768, 768), ((16, 9),), 32, False, 0), 16, None),
        "hint:conv3": (((2, 384, 384), ((32, 9),), 32, False, 0), 16, None),
        "hint:conv4": (((2, 384, 384), ((32, 9),), 96, False, 0), 16, None),
        "hint:conv5": (((2, 192, 192), ((96, 9),), 96, False, 0), 16, None),
        "abi:splitk_cout72": (((1, 1, 1000), ((2048, 1),), 72, True, 0), 0, None),
        "abi:splitk_cout200": (((1, 1, 1000), ((2048, 1),), 200, True, 0), 0, None),
        "stem:unet": (((8, 96, 96), ((64, 1),), 384, False, 0), 0, (4, 0, 0, 0)),
        "stem:unet_inpaint": (((8, 96, 96), ((128, 1),), 384, False, 0), 0, (4, 4, 1, 1)),
        "stem:unet_controlnet": (((8, 96, 96), ((128, 1),), 384, False, 0), 0, (4, 4, 0, 0)),
        "stem:hint:conv0": (((2, 768, 768), ((64, 1),), 16, False, 0), 0, (3, 0, 0, 0)),
        "stem:movq:decoder_conv_in": (((2, 96, 96), ((64, 1),), 512, False, 0), 0, (4, 0, 0, 0)),
        "stem:movq:encoder_conv_in": (((2, 768, 768), ((64, 1),), 128, False, 0), 0, (3, 0, 0, 0)),
    })
    assert got == want


def test_film_width_and_linear_geometry():
    """The FiLM linear's N (all emb_layers of bench.py's UNet) and the k2_linear shapes the GPU test derives."""
    from tests.test_gpu_linear_float64 import LINEAR, _layernorm_cases, _timesteps
    assert gemm_ref.film_total() == 71424
    got = {(c[0], c[1]): c[2:] for c in LINEAR}
    assert got[("film", 8)] == got[("film", 16)] == (1536, 71424, True, True, True, False, False)
    assert got[("2.1:to_model_dim_n", 616)] == (1024, 768, False, True, False, False, False)
    assert got[("2.2:image_embeds", 8)] == (1280, 24576, False, True, False, False, False)
    assert got[("prior2.1:out_proj", 8)] == (2048, 768, False, True, False, False, False)
    assert got[("prior2.2:clip_img_proj", 2)] == (1280, 2048, False, True, False, False, False)
    assert got[("clip_vision:visual_projection", 8)] == (1664, 1280, False, False, False, False, False)
    assert got[("xlmr:proj", 2)] == (1024, 768, False, True, False, False, False)
    assert got[("abi:k5120", 9)][0] == 5120
    assert _layernorm_cases() == [(8, 1536), (256, 768)]
    ts = _timesteps()
    assert ts[0] == 0 and ts[-1] == 999 and 1 in ts and len(ts) >= 50


# ------------------------------------------------------------------------------------------------------------------------------
# the exact checker is sharp
# ------------------------------------------------------------------------------------------------------------------------------
def _exact_case():
    g = torch.Generator().manual_seed(3)
    M, K, N = 64, 256, 96
    x = gemm_ref.ints(g, (M, K))
    w = gemm_ref.scale_odd_rows(gemm_ref.ints(g, (N, K)), gemm_ref.exact_scale(K))
    b = gemm_ref.ints(g, (N,), lim=64, dtype=torch.float32)
    r = gemm_ref.ints(g, (M, N), lim=64)
    out = lambda x, b: gemm_ref.exact_expected(x.double() @ w.double().T + b.double() + r.double(), torch.float16)  # noqa: E731
    return x, b, out


def test_exact_checker_accepts_the_exact_result():
    x, b, out = _exact_case()
    want = out(x, b)
    assert (want.float().abs() > 2048).any()
    gemm_ref.check_exact(want.clone(), want, "exact")


def test_exact_checker_refuses_one_ulp():
    x, b, out = _exact_case()
    want = out(x, b)
    y = want.clone()
    y.view(torch.int16)[17, 33] += 1
    with pytest.raises(AssertionError, match="1 of"):
        gemm_ref.check_exact(y, want, "one ulp")


def test_exact_checker_refuses_swapped_bias_columns():
    x, b, out = _exact_case()
    j = int((b != b[5]).nonzero()[0])
    sw = b.clone()
    sw[5], sw[j] = b[j], b[5]
    with pytest.raises(AssertionError, match="differ from the exact result"):
        gemm_ref.check_exact(out(x, sw), out(x, b), "swapped bias")


@pytest.mark.parametrize("step", [0, 7, 15])
def test_exact_checker_refuses_a_dropped_k_step(step):
    x, b, out = _exact_case()
    dropped = x.clone()
    dropped[:, 16 * step:16 * step + 16] = 0
    with pytest.raises(AssertionError, match="differ from the exact result"):
        gemm_ref.check_exact(out(dropped, b), out(x, b), "dropped K step")


# ------------------------------------------------------------------------------------------------------------------------------
# ABI refusals, before any CUDA call
# ------------------------------------------------------------------------------------------------------------------------------
def _lib():
    from kandinsky2 import _native
    return _native.load()


def _conv(out_mode, residual):
    from kandinsky2._native import K2ConvSrc
    lib = _lib()
    srcs = (K2ConvSrc * 1)()
    srcs[0].ptr, srcs[0].C, srcs[0].ld, srcs[0].taps = A, 64, 64, 1
    info = (ctypes.c_int * 7)()
    # k2_conv_gemm_cfg(srcs, nsrc, NB, H, W, w, w_rows, Ktot, ldw, Cout, bias, residual, ldr, out, ldo, out_mode, ws, ws_bytes,
    #                  gn_partial, info, cfg, w_batch_stride, stream)
    rc = lib.k2_conv_gemm_cfg(srcs, 1, 1, 4, 4, P(A), 64, 64, 64, 64, P(A), P(residual) if residual else None, 64, P(A), 64,
                              out_mode, P(A), 1 << 20, None, info, None, 0, None)
    return rc, lib.k2_last_error().decode()


@pytest.mark.parametrize("out_mode", [2, 3, -1])
def test_conv_gemm_refuses_unknown_out_mode(out_mode):
    rc, err = _conv(out_mode, None)
    assert rc < 0 and "out_mode must be 0" in err, (rc, err)


def test_conv_gemm_refuses_residual_with_fp32_nchw_output():
    rc, err = _conv(1, A)
    assert rc < 0 and "takes no residual" in err, (rc, err)


def test_linear_refuses_k_beyond_the_shared_memory_tile():
    lib = _lib()
    # k2_linear(x, ldx, W, w_is_half, b, add, ldadd, y, ldy, M, N, K, silu_in, silu_out, stream)
    rc = lib.k2_linear(P(A), 5121, P(A), 1, None, None, 0, P(A), 64, 8, 64, 5121, 0, 0, None)
    assert rc < 0 and "K too large" in lib.k2_last_error().decode()
