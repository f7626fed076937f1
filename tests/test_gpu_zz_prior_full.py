"""GPU: the full-size Kandinsky 2.1 diffusion prior (oracle/prior_oracle.py CONFIG_PRIOR: 20 layers, width 2048, 32 heads,
77 text tokens + 4) on synthetic weights, against the oracle on the same GPU.

Which reference?  Kandinsky2_1 runs the reference prior halved under use_fp16 (kandinsky2_1_model.py:58-59).  The forward is
calibrated as tests/test_gpu_unet.py::test_unet_full_size_fp16_calibration does: the product must be at least as close to
the fp32 oracle as the oracle in the reference's fp16 mode is, in max-abs AND relative L2.  Both oracles get the weights as
the product stores them (fp16 GEMM matrices), so the comparison measures arithmetic, not weight quantisation.  About 12 GB of
device memory."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# the GEMM matrices PriorTransformer.finalize packs in fp16; every other parameter stays fp32 in the product
_FP16_STORED = ("attn.c_qkv.weight", "attn.c_proj.weight", "mlp.c_fc.weight", "mlp.c_proj.weight")


@pytest.fixture(scope="module")
def full():
    from kandinsky2.model.prior import PriorTransformer
    from oracle import prior_oracle as po, synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = po.CONFIG_PRIOR
    sd = {k: v.cuda() for k, v in synth.synth_state_dict(po.prior_param_spec(cfg)).items()}
    m = PriorTransformer(**cfg, device="cuda")
    m.load_state_dict(sd, strict=True)
    m.finalize()
    stored = {k: (v.half().float() if k.endswith(_FP16_STORED) or k == "text_enc_proj.weight" else v) for k, v in sd.items()}
    del sd
    yield dict(cfg=cfg, m=m, sd32=stored)
    torch.cuda.empty_cache()


def _inputs(B, prompt_len, seed):
    """Classifier-free batch [prompt x B | "" x B]: the text features of one prompt repeated B times, then those of the
    empty prompt, whose CLIP mask keeps its start and end tokens only."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    D, L, X = 768, 77, 768
    text_emb = torch.randn(2, D, device="cuda", generator=g).repeat_interleave(B, 0)
    text_enc = torch.randn(2, L, X, device="cuda", generator=g).repeat_interleave(B, 0)
    lens = torch.tensor([prompt_len] * B + [2] * B, device="cuda")
    mask = torch.arange(L, device="cuda")[None, :] < lens[:, None]
    return text_emb, text_enc, mask, g


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


@pytest.mark.parametrize("B,prompt_len", [(1, 12), (4, 77)])
def test_prior_full_size_fp16_calibration(full, B, prompt_len, monkeypatch):
    from kandinsky2 import ops
    from oracle import prior_oracle as po
    cfg, m, sd32 = full["cfg"], full["m"], full["sd32"]
    text_emb, text_enc, mask, g = _inputs(B, prompt_len, seed=B)
    N = 2 * B
    x = torch.randn(N, 768, device="cuda", generator=g)
    t = torch.tensor([999.0, 500.0, 120.0, 0.0] * B, device="cuda")[:N]
    # the residual stream is the output of every GEMM that adds the residual: record that each is finite and its magnitude
    peaks, gemm_rows = [], ops.gemm_rows

    def recording_gemm_rows(*a, **kw):
        y = gemm_rows(*a, **kw)
        if kw.get("residual") is not None:
            peaks.append(y.abs().amax())          # inf / NaN propagate into the recorded value
        return y

    monkeypatch.setattr(ops, "gemm_rows", recording_gemm_rows)
    y = m(x, t, text_emb=text_emb, text_enc=text_enc, mask=mask)
    monkeypatch.undo()
    assert len(peaks) == 2 * cfg["xf_layers"]
    peak = torch.stack(peaks).max().item()
    assert torch.isfinite(torch.stack(peaks)).all() and torch.isfinite(y).all(), peak
    with torch.no_grad():
        ref32 = po.prior_forward(sd32, cfg, x, t, text_emb, text_enc, mask)
        sd16 = {k: v.half() for k, v in sd32.items()}
        ref16 = po.prior_forward(sd16, cfg, x, t, text_emb, text_enc, mask, fp16=True)
        del sd16
    k_abs, k_rel = _dev(y, ref32)
    r_abs, r_rel = _dev(ref16, ref32)
    print(f"prior full size B={B}: residual stream peak |h| {peak:.1f}; output rms {ref32.pow(2).mean().sqrt().item():.3f}; "
          f"k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | reference-fp16 vs fp32 max-abs {r_abs:.3e} rel-L2 {r_rel:.3e}")
    assert k_rel <= r_rel and k_abs <= r_abs, (k_abs, k_rel, r_abs, r_rel)
    # an fp16 residual stream over 20 layers: a few fp16 half-ulps (2^-11 = 4.9e-4) of accumulated relative error
    # (H100, 400 W: 1.3e-3 to 1.4e-3 measured, against 1.5e-3 to 1.7e-3 for the reference's fp16 mode)
    assert k_rel < 5e-3, k_rel


def test_prior_full_size_sampling(full):
    """PriorDiffusionModel's 25-step guided sampling (guidance 4) with the same x_T and per-step noise, the product's forward
    against the fp32 oracle's."""
    from kandinsky2.model.gaussian_diffusion import space_timesteps
    from kandinsky2.model.prior import sample_prior
    from oracle import prior_oracle as po
    cfg, m, sd32 = full["cfg"], full["m"], full["sd32"]
    B = 2
    text_emb, text_enc, mask, g = _inputs(B, 12, seed=9)
    use_steps = sorted(space_timesteps(1000, [25]))
    assert len(use_steps) == 25
    x_T = torch.randn(B, 768, device="cuda", generator=g)
    noise = torch.randn(25, B, 768, device="cuda", generator=g)
    clip_mean = 0.1 * torch.randn(768, device="cuda", generator=g)
    clip_std = 0.5 + torch.rand(768, device="cuda", generator=g)
    s = sample_prior(m, text_emb, text_enc, mask, use_steps, 4.0, clip_mean, clip_std, x_T, noise)
    with torch.no_grad():
        ref = po.prior_sample(lambda xx, tt: po.prior_forward(sd32, cfg, xx, tt, text_emb, text_enc, mask), x_T, noise, use_steps,
                              4.0, clip_mean, clip_std)
    err, rel = _dev(s, ref)
    print(f"prior full size 25-step sampling, guidance 4: rel-L2 {rel:.3e} max-abs {err:.3e} (sample rms "
          f"{ref.pow(2).mean().sqrt().item():.3f})")
    assert torch.isfinite(s).all()
    # 25 forwards of ~1.4e-3 relative deviation each (H100: 1.7e-3 measured); each x0-prediction step mostly replaces x, so
    # the deviations do not compound.  Three times tighter than the tiny golden's 3e-2 (tests/test_gpu_zz_prior.py).
    assert rel < 1e-2, rel
