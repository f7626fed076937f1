"""CPU: the Kandinsky 2.2 prior's host side -- the diffusers state-dict remap (checkpoints.diffusers_prior_to_k2), the UnCLIP
schedule rows (model.prior.UnCLIPSchedule) and the argument checks of k2_prior_tokens / k2_f16_to_f32."""
import math

import numpy as np
import pytest
import torch

from tests import prior22_oracle as p22
from tests.test_cpu_vector_arg_checks import A, P, _refused, _with


def _diffusers_sd(cfg, device="cpu", seed=0):
    from oracle import synth
    spec = p22.diffusers_prior_spec(cfg)
    if device == "meta":
        return {k: torch.empty(s, device="meta") for k, s in spec}
    return synth.synth_state_dict(spec, seed=seed)


@pytest.mark.parametrize("cfg,device", [(p22.CONFIG_PRIOR22_TINY, "cpu"), (p22.CONFIG_PRIOR22, "meta")])
def test_remap_lands_on_the_prior_keys(cfg, device):
    from kandinsky2.checkpoints import diffusers_prior_to_k2, unpack_heads
    from kandinsky2.model.prior import PriorTransformer
    dsd = _diffusers_sd(cfg, device)
    dsd["causal_attention_mask"] = torch.zeros(1)      # a non-persistent buffer some exports carry: ignored
    sd, mean, std = diffusers_prior_to_k2(dsd)
    want = PriorTransformer(**cfg, device="meta").state_dict()
    assert sorted(sd) == sorted(want)
    assert all(tuple(sd[k].shape) == tuple(want[k].shape) for k in want)
    assert tuple(mean.shape) == tuple(std.shape) == (cfg["clip_dim"],)
    if device == "cpu":   # the round trip: the packed rows split back into the diffusers projections bit for bit
        for i in range(cfg["xf_layers"]):
            for suffix in ("weight", "bias"):
                parts = unpack_heads(sd[f"transformer.resblocks.{i}.attn.c_qkv.{suffix}"], 3)
                for c, part in zip("qkv", parts):
                    assert torch.equal(part, dsd[f"transformer_blocks.{i}.attn1.to_{c}.{suffix}"])
        assert torch.equal(sd["prd_emb"], dsd["prd_embedding"]) and torch.equal(sd["final_ln.weight"], dsd["norm_out.weight"])
        assert torch.equal(mean, dsd["clip_mean"][0]) and torch.equal(std, dsd["clip_std"][0])


def test_remap_refuses_unknown_and_missing_keys():
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import diffusers_prior_to_k2
    dsd = _diffusers_sd(p22.CONFIG_PRIOR22_TINY)
    extra = dict(dsd, **{"norm_in.weight": torch.zeros(128)})
    with pytest.raises(K2Error, match=r"unknown keys \['norm_in.weight'\]"):
        diffusers_prior_to_k2(extra)
    lacking = {k: v for k, v in dsd.items() if k != "transformer_blocks.1.attn1.to_k.bias"}
    with pytest.raises(K2Error, match=r"missing keys \['transformer_blocks.1.attn1.to_k.bias'\]"):
        diffusers_prior_to_k2(lacking)
    with pytest.raises(K2Error, match="clip_std"):
        diffusers_prior_to_k2({k: v for k, v in dsd.items() if k != "clip_std"})


def _text_inputs(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    N, D, X, L = len(lens), cfg["clip_dim"], cfg["clip_xf_width"], cfg["text_ctx"]
    x = torch.randn(N, D, generator=g)
    t = torch.tensor([999.0, 500.0, 42.0, 0.0] * N)[:N]
    text_emb = torch.randn(N, D, generator=g)
    text_enc = torch.randn(N, L, X, generator=g)
    mask = torch.arange(L)[None, :] < torch.tensor(lens)[:, None]
    return x, t, text_emb, text_enc, mask


@pytest.mark.parametrize("lens", [[5, 5], [1, 3, 5, 2]])
def test_remapped_reference_forward_equals_diffusers_form(lens):
    """Head interleaving and every renamed key, checked through the network: the reference's forward (oracle/prior_oracle.py,
    pinned to the reference's classes) on the remapped weights against the diffusers-form forward on the original ones.
    Padded masks included: the start token is always kept, so -10000 and -inf masks give the same softmax in fp32."""
    from kandinsky2.checkpoints import diffusers_prior_to_k2
    from oracle import prior_oracle as po
    cfg = p22.CONFIG_PRIOR22_TINY
    dsd = _diffusers_sd(cfg, seed=3)
    sd, _, _ = diffusers_prior_to_k2(dsd)
    x, t, te, tenc, mask = _text_inputs(cfg, lens, seed=len(lens))
    with torch.no_grad():
        ref = po.prior_forward(sd, cfg, x, t, te, tenc, mask)
        dif = p22.diffusers_prior_forward(dsd, cfg, x, t, te, tenc, mask)
    rel = ((dif - ref).norm() / ref.norm()).item()
    assert rel <= 1e-5, rel
    # a wrong interleave is caught: q and k of the heads swapped
    sd_bad = dict(sd)
    w = sd["transformer.resblocks.0.attn.c_qkv.weight"].view(2, 3, 64, -1)
    sd_bad["transformer.resblocks.0.attn.c_qkv.weight"] = w[:, [1, 0, 2]].reshape(w.shape[0] * 192, -1)
    with torch.no_grad():
        bad = po.prior_forward(sd_bad, cfg, x, t, te, tenc, mask)
    assert ((bad - dif).norm() / dif.norm()).item() > 1e-3


def _apply_rows(rows, model_fn, x_T, noise, guidance, clip_mean, clip_std):
    """The rows through k2_sampler_step's formula (include/k2b200.h), in float64: x0 = r0 x - r1 eps, clamp +-10,
    x' = r2 x0 + r3 x + r6 exp(0.5 (0.5 r4 + 0.5 r5)) z."""
    x = x_T.double()
    B = x.shape[0]
    for k, r in enumerate(rows):
        out = model_fn(torch.cat([x, x]).float(), None).double()
        eps = out[:B] + guidance * (out[B:] - out[:B])
        x0 = (r[0] * x - r[1] * eps).clamp(-10, 10)
        mean = r[2] * x0 + r[3] * x
        logvar = 0.5 * r[5] + 0.5 * r[4]
        x = mean + (r[6] * math.exp(0.5 * logvar) * noise[k].double() if r[6] != 0 else 0.0)
    return x * clip_std.double() + clip_mean.double()


@pytest.mark.parametrize("N", [2, 5, 10, 25, 50])
def test_unclip_rows_reproduce_the_scheduler_loop(N):
    from kandinsky2.model.prior import UnCLIPSchedule
    sched = UnCLIPSchedule(N)
    rows = sched.rows()
    assert rows.shape == (N, 8) and rows.dtype == np.float64
    g = torch.Generator().manual_seed(N)
    B, D = 3, 16
    x_T = torch.randn(B, D, generator=g, dtype=torch.float64)
    noise = torch.randn(N, B, D, generator=g, dtype=torch.float64)
    mean, std = 0.1 * torch.randn(D, generator=g, dtype=torch.float64), 0.5 + torch.rand(D, generator=g, dtype=torch.float64)
    # a prediction that depends on the sample, reaches past the +-10 clamp, and differs between the CFG halves
    w = torch.randn(D, D, generator=g, dtype=torch.float64)
    fn = lambda xx, tt: (8 * torch.tanh(xx.double() @ w) + torch.linspace(-6, 6, xx.shape[0], dtype=torch.float64)[:, None])  # noqa: E731
    got = _apply_rows(rows, fn, x_T, noise, 4.0, mean, std)
    ref = p22.unclip_sample(fn, x_T, noise, N, 4.0, mean, std)
    assert ((got - ref).abs().max() / ref.abs().max()).item() <= 1e-12
    assert np.array_equal(sched.timesteps, p22.unclip_timesteps(N))


def test_unclip_timesteps_and_last_row():
    from kandinsky2.model.prior import UnCLIPSchedule
    assert UnCLIPSchedule(2).timesteps.tolist() == [999, 0]
    ts = UnCLIPSchedule(25).timesteps
    assert ts.tolist() == (np.arange(25) * (999 / 24)).round()[::-1].astype(int).tolist()
    assert ts[:3].tolist() == [999, 957, 916] and ts[-2:].tolist() == [42, 0]
    for N in (2, 25, 50):
        last = UnCLIPSchedule(N).rows()[-1]
        # x' = 1 * x0 + 0 * x, no noise: the last step lands on x0 exactly
        assert last[2] == 1.0 and last[3] == 0.0 and last[6] == 0.0, last
        assert UnCLIPSchedule(N).coef_table().dtype == np.float32
    with pytest.raises(ValueError):
        UnCLIPSchedule(1)


# k2_prior_tokens(x, ldx, pos, ldp, y, ldy, M, N, stream)
TOK = dict(x=P(A), ldx=2048, pos=P(A), ldp=0, y=P(A), ldy=81 * 2048, M=2, N=2048, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(x=None), "bad arguments"),
    (dict(pos=None), "bad arguments"),
    (dict(y=None), "bad arguments"),
    (dict(M=0), "bad arguments"),
    (dict(N=0), "bad arguments"),
    (dict(ldx=2047), "row strides"),
    (dict(ldp=100), "row strides"),
    (dict(ldy=2047), "row strides"),
    (dict(ldx=-1), "row strides"),
    (dict(x=P(A + 2)), "alignment"),
    (dict(pos=P(A + 1)), "alignment"),
    (dict(y=P(A + 1)), "alignment"),
])
def test_prior_tokens_refuses(change, msg):
    _refused("k2_prior_tokens", list(_with(TOK, **change).values()), msg)


# k2_f16_to_f32(x, ldx, y, ldy, M, N, stream)
WIDEN = dict(x=P(A), ldx=81 * 2048, y=P(A), ldy=2048, M=2, N=2048, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(x=None), "bad arguments"),
    (dict(y=None), "bad arguments"),
    (dict(M=0), "bad arguments"),
    (dict(N=-4), "bad arguments"),
    (dict(ldx=0), "row strides"),
    (dict(ldy=2047), "row strides"),
    (dict(x=P(A + 1)), "alignment"),
    (dict(y=P(A + 2)), "alignment"),
])
def test_f16_to_f32_refuses(change, msg):
    _refused("k2_f16_to_f32", list(_with(WIDEN, **change).values()), msg)


def test_prior_embedder22_refuses_text_emb_and_one_step():
    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder22, sample_prior22
    emb = PriorEmbedder22(prior=None, clip_text=None, clip_mean=torch.zeros(4), clip_std=torch.ones(4))
    with pytest.raises(K2Error):
        emb.text_emb("a cat", 1)
    with pytest.raises(ValueError):   # refused before anything touches a device
        sample_prior22(None, None, None, None, 1, 4.0, None, None, torch.zeros(1, 4), torch.zeros(1, 1, 4))
