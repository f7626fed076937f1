"""GPU: the conditioning path's fp32 layers against float64 at the geometry the models build -- k2_linear (fp16 and fp32
weights, SiLU on the input or the output, the added row), k2_layernorm and k2_timestep_embedding.

k2_linear in two modes:
  exact   integer x, W, bias and add (tests/gemm_ref.py), no SiLU: every partial sum is an integer below 2^24, so the fp32 FMA
          chains are exact in any order and the output must equal the float64 sum bit for bit;
  random  Gaussian data, bound of fp32 FMA accumulation: 1.01 (K + 8) 2^-24 (sum_k |x_k W_nk| + |b_n|) (K FMAs per lane chain,
          five butterfly adds, the bias), with SiLU's own error on each input (silu_in) or on the output (silu_out, slope at
          most 1.1; tests/test_gpu_groupnorm_float64.py) and one rounding of the added row.
Shapes: the UNet's FiLM linear (all emb_layers as one fp16 weight; its N puts the kernel on the ni = LIN_NI path) at M = 8 and
16 (two row tiles), time_embed.0 / .2, the 2.1 and 2.2 conditioning heads (unet.py get_text_emb), the priors' time, image,
text and output projections, the towers' final projections, a K that is not a multiple of 8 and K = 5120, the largest the
shared-memory x tile takes.  Each case prints its worst share of the bound (run with -s)."""
import inspect

import pytest
import torch

from tests.gemm_ref import UNET_GEOM, check_exact, exact_expected, exact_scale, film_total, ints, scale_odd_rows
from tests.test_gpu_groupnorm_float64 import SILU_SLOPE, _silu64, _silu_allow

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -140


def _linear_cases():
    """[(name, M, K, N, w_is_half, bias, silu_in, silu_out, add)] derived from the model code and configs."""
    import bench
    from kandinsky2 import configs
    from kandinsky2.model.clip_text import text_tower_config
    from kandinsky2.model.clip_vision import tower_config
    from kandinsky2.model.text_encoders import XLMRobertaTokenizer, xlmr_config
    from oracle.prior_oracle import CONFIG_PRIOR
    from tests import clip_text_oracle, clip_vision_oracle, xlmr_oracle
    from tests.gemm_ref import _prior_meta
    from tests.prior22_oracle import CONFIG_PRIOR22
    N = UNET_GEOM[0]
    u22 = bench.UNET_CFG
    mc = u22["model_channels"]
    temb = 4 * mc
    out = [("film", m, temb, film_total(), True, True, True, False, False) for m in (N, 2 * N)]
    out += [("time_embed.0", N, mc, temb, False, True, False, True, False),
            ("time_embed.2", N, temb, temb, False, True, False, False, True)]
    u21 = configs.CONFIG_2_1["model_config"]
    md = u21["model_dim"]
    text_len = inspect.signature(XLMRobertaTokenizer).parameters["model_max_length"].default
    out += [("2.1:clip_to_seq", N, u21["image_encoder_in_dim"], md * u21["num_image_embs"], False, True, False, False, False),
            ("2.1:to_model_dim_n", N * text_len, u21["text_encoder_in_dim1"], md, False, True, False, False, False),
            ("2.1:proj_n", N, u21["text_encoder_in_dim2"], temb, False, True, False, False, False),
            ("2.1:img_layer", N, u21["image_encoder_in_dim"], temb, False, True, False, False, True),
            ("2.2:image_embeds", N, u22["image_encoder_in_dim"], u22["model_dim"] * u22["num_image_embs"], False, True, False,
             False, False),
            ("2.2:image_proj", N, u22["image_encoder_in_dim"], temb, False, True, False, False, False)]
    for ver, cfg in (("2.1", CONFIG_PRIOR), ("2.2", CONFIG_PRIOR22)):
        p = _prior_meta(cfg)
        W, D = p.xf_width, p.clip_dim
        for m in (2, 8):   # 2B CFG rows, B = 1 and 4
            out += [(f"prior{ver}:time_embed.0", m, W, W, False, True, False, False, False),
                    (f"prior{ver}:time_embed.2", m, W, W, False, True, True, False, False),
                    (f"prior{ver}:clip_img_proj", m, D, W, False, True, False, False, False),
                    (f"prior{ver}:text_emb_proj", m, D, W, False, True, False, False, False),
                    (f"prior{ver}:out_proj", m, W, D, False, True, False, False, False)]
    ct = text_tower_config(clip_text_oracle.CONFIG_BIGG)
    cv = tower_config(clip_vision_oracle.CONFIG_BIGG)
    cx = xlmr_config(xlmr_oracle.CONFIG_LARGE)
    for m in (2, 8):
        out += [("clip_text:text_projection", m, ct["hidden_size"], ct["projection_dim"], False, False, False, False, False),
                ("clip_vision:visual_projection", m, cv["hidden_size"], cv["projection_dim"], False, False, False, False,
                 False),
                ("xlmr:proj", m, cx["hidden_size"], xlmr_oracle.OUT_LARGE, False, True, False, False, False)]
    out += [("abi:k77_half", 5, 77, 96, True, True, True, False, True),     # K % 8 != 0: the scalar K loop
            ("abi:k77_f32", 5, 77, 96, False, True, False, True, False),
            ("abi:k5120", 9, 5120, 64, True, True, False, False, True)]     # the largest K of the shared-memory x tile
    seen, cases = set(), []
    for c in out:
        if c[1:] not in seen:
            seen.add(c[1:])
            cases.append(c)
    return cases


LINEAR = _linear_cases()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("name,M,K,N,w_half,has_b,silu_in,silu_out,has_add", LINEAR, ids=[f"{c[0]}:M{c[1]}" for c in LINEAR])
def test_linear_vs_float64(name, M, K, N, w_half, has_b, silu_in, silu_out, has_add, mode):
    from kandinsky2 import ops
    if name == "film":
        # k2_misc.cu: ni = LIN_NI when N >= 8 warps x LIN_CB x LIN_NI x 2 x SMs = 256 x SMs
        assert N >= 256 * _sms(), (N, _sms())
    g = torch.Generator(device="cuda").manual_seed(M * 131 + K * 7 + N)
    wdt = torch.float16 if w_half else torch.float32
    if mode == "exact":
        silu_in = silu_out = False
        x = ints(g, (M, K), device="cuda", dtype=torch.float32)
        W = scale_odd_rows(ints(g, (N, K), device="cuda", dtype=wdt), exact_scale(K))
        b = ints(g, (N,), lim=64, device="cuda", dtype=torch.float32) if has_b else None
        add = ints(g, (M, N), lim=64, device="cuda", dtype=torch.float32) if has_add else None
    else:
        x = torch.randn(M, K, device="cuda", generator=g) * 2
        W = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).to(wdt)
        b = torch.randn(N, device="cuda", generator=g) * 0.5 if has_b else None
        add = torch.randn(M, N, device="cuda", generator=g) if has_add else None
    y = ops.linear(x, W, b, add=add, silu_in=silu_in, silu_out=silu_out)
    torch.cuda.synchronize()
    xd, Wd = x.double(), W.double()
    xin = _silu64(xd) if silu_in else xd
    v = xin @ Wd.T + (b.double() if b is not None else 0)
    what = f"linear {name} M={M} K={K} N={N} {mode}"
    if mode == "exact":
        want = v + (add.double() if add is not None else 0)
        check_exact(y, exact_expected(want, torch.float32), what)
        print(f"{what}: bit-exact")
        return
    acc = 1.01 * (K + 8) * U * (xin.abs() @ Wd.abs().T + (b.double().abs() if b is not None else 0))
    if silu_in:
        acc = acc + _silu_allow(xd) @ Wd.abs().T
    ref, bound = v, acc
    if silu_out:
        ref, bound = _silu64(v), SILU_SLOPE * acc + _silu_allow(v)
    if add is not None:
        ref = ref + add.double()
        bound = bound + U * ref.abs()
    bound = bound + TINY
    share = ((y.double() - ref).abs() / bound).max().item()
    assert share <= 1.0, f"{what}: {share:.3f} of the bound"
    print(f"{what}: worst {share:.2e} of the bound")


# ------------------------------------------------------------------------------------------------------------------------------
# k2_layernorm (fp32) and k2_timestep_embedding
# ------------------------------------------------------------------------------------------------------------------------------
def _layernorm_cases():
    """(rows, width) of the conditioning heads' fp32 LayerNorms: 2.1 ln_model_n and 2.2 image_norm over the time-embedding
    width, 2.2 encoder_hid_proj.norm over the image tokens."""
    import bench
    N, u = UNET_GEOM[0], bench.UNET_CFG
    temb = 4 * u["model_channels"]
    return sorted({(N, temb), (N * u["num_image_embs"], u["model_dim"])})


@pytest.mark.parametrize("M,N", _layernorm_cases())
def test_layernorm_vs_float64(M, N):
    """y = (x - fmean) rstd g + b in fp32 with float64 statistics rounded once: 2^-24 |g| rstd |mean| from fmean, then at most
    four roundings of the product chain (2^-24 each, of |g (x - mean) rstd|) and one of the sum (2^-24 |y|)."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(M + N)
    worst = 0.0
    for mean in (0.0, 0.5, 3.0):
        x = torch.randn(M, N, device="cuda", generator=g) * 1.5 + mean
        gam = torch.randn(N, device="cuda", generator=g) * 0.2 + 1.0
        bet = torch.randn(N, device="cuda", generator=g) * 0.1
        y = ops.layernorm(x, gam, bet)
        torch.cuda.synchronize()
        xd = x.double()
        mu = xd.mean(-1, keepdim=True)
        d = xd - mu
        r = 1.0 / torch.sqrt((d * d).mean(-1, keepdim=True) + 1e-5)
        t = d * r * gam.double()
        ref = t + bet.double()
        bound = 1.01 * (U * gam.double().abs() * r * mu.abs() + 4 * U * t.abs() + U * ref.abs()) + TINY
        share = ((y.double() - ref).abs() / bound).max().item()
        assert share <= 1.0, (M, N, mean, share)
        worst = max(worst, share)
    print(f"layernorm M={M} N={N}: worst {worst:.3f} of the bound")


TS_C = 21   # arg error of k2_timestep_embedding in units of |t f| 2^-23, derived in test_timestep_embedding_vs_float64


def _timesteps():
    """t = 0, 1, 999 and the timesteps of a 50-step respaced schedule (the UNet's and the prior's sampling loops feed integer
    timesteps of such schedules)."""
    from kandinsky2.model.gaussian_diffusion import space_timesteps
    return sorted({0, 1, 999} | set(space_timesteps(1000, "50")))


@pytest.mark.parametrize("dim", [384, 2048])
def test_timestep_embedding_vs_float64(dim):
    """out[b, j] = cos / sin(t_b f_j), f_j = expf(-logf(P) j / half) in fp32, against float64 of the same formula.  The fp32
    argument t f carries, relative to |t f|: logf's 1 ulp (2^-23) and the product and quotient (2^-24 each) make the exponent
    a = -ln(P) j / half wrong by 2^-22 |a| <= 2^-22 ln(10^4), i.e. 18.42 2^-23 relative in exp(a); expf's 2 ulps add 2 2^-23
    and t f its own rounding 0.5 2^-23: c = 20.92 -> 21 (TS_C).  cosf / sinf (slope <= 1) add 2 ulps of the result."""
    from kandinsky2 import ops
    ts = torch.tensor(_timesteps(), dtype=torch.float32, device="cuda")
    y = ops.timestep_embedding(ts, dim)
    torch.cuda.synchronize()
    half = dim // 2
    f = torch.exp(-torch.log(torch.tensor(10000.0, dtype=torch.float64)) * torch.arange(half, dtype=torch.float64) / half)
    arg = ts.double().cpu()[:, None] * f[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    bound = 1.01 * (TS_C * 2.0 ** -23 * torch.cat([arg, arg], 1).abs() + 2 * 2.0 ** -23 * ref.abs()) + 2.0 ** -140
    share = ((y.double().cpu() - ref).abs() / bound).max().item()
    assert share <= 1.0, (dim, share)
    print(f"timestep_embedding dim={dim} over {ts.numel()} timesteps: worst {share:.3f} of the bound")
