"""CPU: LoRA adapters of the Kandinsky 2.2 diffusion prior in diffusers' attention-processor format -> (up', down') factors of
the packed c_qkv / c_proj weights (kandinsky2/checkpoints.py: prior_lora_to_k2), checked against the per-projection deltas and
through the network against the unfused processor arithmetic (tests/prior_lora_oracle.py); the refusals, and load_lora's
CPU-only failure."""
import pytest
import torch

from tests import prior22_oracle as p22
from tests import prior_lora_oracle as plo


def _key(i, proj, which):
    return f"transformer_blocks.{i}.attn1.processor.{proj}_lora.{which}.weight"


def test_full_size_adapter_fully_consumed():
    """The notebook's adapter on the full 2.2 prior: 20 layers x 4 projections x (down, up) = 160 tensors, every layer gets
    both packed targets, with factors [3W, 3r] / [3r, W] for c_qkv and [W, r] / [r, W] for c_proj."""
    from kandinsky2.checkpoints import prior_lora_to_k2
    cfg = p22.CONFIG_PRIOR22
    W, L, r = cfg["xf_width"], cfg["xf_layers"], 4
    lora = plo.synth_prior_lora(cfg, rank=r, dtype=torch.float16)
    assert len(lora) == 160
    packed = prior_lora_to_k2(lora, W, L)
    want = {f"transformer.resblocks.{i}.attn.{t}.weight" for i in range(L) for t in ("c_qkv", "c_proj")}
    assert set(packed) == want
    for key, (up, down) in packed.items():
        assert up.dtype == down.dtype == torch.float32 and up.is_contiguous() and down.is_contiguous()
        n = 3 if key.endswith("c_qkv.weight") else 1
        assert up.shape == (n * W, n * r) and down.shape == (n * r, W), (key, up.shape, down.shape)
    # every factor element came from the adapter: c_qkv's down stacks q | k | v, c_proj's pair is to_out's as stored
    up, down = packed["transformer.resblocks.7.attn.c_qkv.weight"]
    assert torch.equal(down, torch.cat([lora[_key(7, p, "down")].float() for p in ("to_q", "to_k", "to_v")]))
    up, down = packed["transformer.resblocks.19.attn.c_proj.weight"]
    assert torch.equal(up, lora[_key(19, "to_out", "up")].float()) and torch.equal(down, lora[_key(19, "to_out", "down")].float())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_factors_equal_the_packed_per_projection_deltas(dtype):
    """In float64, up' @ down' is pack_heads of (delta q, delta k, delta v) for c_qkv (zero for a missing projection) and
    delta out for c_proj, where delta = up @ down; layers without any q / k / v (or to_out) factor have no c_qkv (c_proj) entry."""
    from kandinsky2.checkpoints import pack_heads, prior_lora_to_k2
    cfg = dict(p22.CONFIG_PRIOR22_TINY, xf_width=192, xf_heads=3, xf_layers=4)
    W = cfg["xf_width"]
    lora = plo.synth_prior_lora(cfg, rank=3, seed=2, dtype=dtype)
    dropped = {(0, "to_k"), (1, "to_q"), (1, "to_v"), (1, "to_out"), (2, "to_q"), (2, "to_k"), (2, "to_v")}
    lora = {k: v for k, v in lora.items() if (int(k.split(".")[1]), k.split(".processor.")[1].split("_lora.")[0]) not in dropped}
    packed = prior_lora_to_k2(lora, W, cfg["xf_layers"])

    def delta(i, proj):
        if _key(i, proj, "down") not in lora:
            return torch.zeros(W, W, dtype=torch.float64)
        return lora[_key(i, proj, "up")].double() @ lora[_key(i, proj, "down")].double()

    assert set(packed) == {f"transformer.resblocks.{i}.attn.c_qkv.weight" for i in (0, 1, 3)} | \
        {f"transformer.resblocks.{i}.attn.c_proj.weight" for i in (0, 2, 3)}
    for key, (up, down) in packed.items():
        i = int(key.split(".")[2])
        want = pack_heads([delta(i, p) for p in ("to_q", "to_k", "to_v")]) if "c_qkv" in key else delta(i, "to_out")
        got = up.double() @ down.double()
        assert got.shape == want.shape
        assert ((got - want).norm() / want.norm()).item() < 1e-12, key
    assert packed["transformer.resblocks.1.attn.c_qkv.weight"][0].shape == (3 * W, 3)   # only to_k: rank 3, not 9


def _inputs(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    N, D, X, L = len(lens), cfg["clip_dim"], cfg["clip_xf_width"], cfg["text_ctx"]
    x = torch.randn(N, D, generator=g)
    t = torch.tensor([999.0, 500.0, 42.0, 0.0] * N)[:N]
    mask = torch.arange(L)[None, :] < torch.tensor(lens)[:, None]
    return x, t, torch.randn(N, D, generator=g), torch.randn(N, L, X, generator=g), mask


def test_oracle_without_adapter_is_the_diffusers_forward():
    from oracle import synth
    cfg = p22.CONFIG_PRIOR22_TINY
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=4)
    args = _inputs(cfg, [5, 2], seed=1)
    with torch.no_grad():
        assert torch.equal(plo.lora_prior_forward(dsd, cfg, {}, 1.0, *args), p22.diffusers_prior_forward(dsd, cfg, *args))


@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("lens", [[5, 5], [1, 3, 5, 2]])
def test_merged_reference_forward_equals_unfused_processors(scale, lens):
    """The network check: the reference's forward (oracle/prior_oracle.py) on diffusers_prior_to_k2's weights with
    scale * up' @ down' merged into c_qkv / c_proj in fp32, against the diffusers-form forward with LoRAAttnProcessor run
    unfused on the original weights: within 1e-5 relative, the bound of the plain remap (tests/test_cpu_prior22.py), while the
    adapter moves the output by far more than that."""
    from kandinsky2.checkpoints import diffusers_prior_to_k2, prior_lora_to_k2
    from oracle import prior_oracle as po
    from oracle import synth
    cfg = p22.CONFIG_PRIOR22_TINY
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=3)
    lora = plo.synth_prior_lora(cfg, rank=4, seed=6)
    sd, _, _ = diffusers_prior_to_k2(dsd)
    merged = dict(sd)
    for key, (up, down) in prior_lora_to_k2(lora, cfg["xf_width"], cfg["xf_layers"]).items():
        merged[key] = sd[key] + scale * (up @ down)
    args = _inputs(cfg, lens, seed=len(lens))
    with torch.no_grad():
        ref = po.prior_forward(merged, cfg, *args)
        dif = plo.lora_prior_forward(dsd, cfg, lora, scale, *args)
        plain = p22.diffusers_prior_forward(dsd, cfg, *args)
    rel = ((dif - ref).norm() / ref.norm()).item()
    assert rel <= 1e-5, rel
    assert ((plain - dif).norm() / dif.norm()).item() > 1e-2


def _rejects(lora, match, width=128, layers=2):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import prior_lora_to_k2
    with pytest.raises(K2Error, match=match):
        prior_lora_to_k2(lora, width, layers)


def test_rejections_name_the_offending_key():
    cfg = p22.CONFIG_PRIOR22_TINY
    W = cfg["xf_width"]
    base = plo.synth_prior_lora(cfg, rank=2, seed=1)
    p = "transformer_blocks.1.attn1.processor."

    # unknown projection, a layer the prior does not have, another attention, a stray key
    _rejects(dict(base, **{p + "to_z_lora.down.weight": torch.zeros(2, W)}), r"to_z_lora")
    _rejects(dict(base, **{_key(2, "to_q", "down"): torch.zeros(2, W)}), r"transformer_blocks\.2\.attn1")
    _rejects(dict(base, **{"transformer_blocks.0.attn2.processor.to_q_lora.down.weight": torch.zeros(2, W)}), r"attn2")
    _rejects(dict(base, **{"transformer_blocks.0.attn1.to_q.weight": torch.zeros(W, W)}), r"attn1\.to_q\.weight")
    # the decoder's added K / V projections are not the prior's
    _rejects(dict(base, **{p + "add_k_proj_lora.down.weight": torch.zeros(2, W)}), r"add_k_proj_lora")
    # a down without its up (and the reverse)
    d = dict(base)
    del d[p + "to_k_lora.up.weight"]
    _rejects(d, r"to_k_lora\.down\.weight.*no matching up")
    d = dict(base)
    del d[p + "to_out_lora.down.weight"]
    _rejects(d, r"to_out_lora\.up\.weight.*no matching down")
    # rank mismatch within a pair, wrong in / out dimensions
    _rejects(dict(base, **{p + "to_v_lora.up.weight": torch.zeros(W, 3)}), r"to_v_lora.*rank mismatch")
    _rejects(dict(base, **{p + "to_q_lora.down.weight": torch.zeros(2, W + 64)}), r"to_q_lora.*down \[rank, 128\]")
    _rejects(dict(base, **{p + "to_out_lora.up.weight": torch.zeros(2 * W, 2)}), r"to_out_lora.*up \[128, rank\]")
    _rejects(base, r"to_q_lora.*down \[rank, 256\]", width=256)
    # PEFT keys and alpha entries
    _rejects(dict(base, **{"transformer_blocks.0.attn1.to_q.lora_A.weight": torch.zeros(2, W)}), r"lora_A.*PEFT")
    _rejects(dict(base, **{"transformer_blocks.0.attn1.to_q.lora_B.weight": torch.zeros(W, 2)}), r"lora_B.*PEFT")
    _rejects(dict(base, **{p + "to_q_lora.network_alpha": torch.tensor(4.0)}), r"to_q_lora\.network_alpha.*alpha")
    _rejects(dict(base, **{p + "to_q_lora.alpha": torch.tensor(4.0)}), r"to_q_lora\.alpha.*alpha")
    # not a floating 2-D tensor
    _rejects(dict(base, **{p + "to_q_lora.down.weight": torch.zeros(2, W, dtype=torch.int32)}), r"to_q_lora\.down")
    _rejects(dict(base, **{p + "to_q_lora.down.weight": torch.zeros(2, W, 1)}), r"to_q_lora\.down.*2-D")
    _rejects(dict(base, **{p + "to_q_lora.down.weight": [[0.0] * W] * 2}), r"to_q_lora\.down.*2-D")


def test_load_lora_without_gpu_raises():
    """Like every op, merging needs the GPU: load_lora raises K2Error on a CPU prior and leaves it without an adapter and with
    its state dict unchanged.  A malformed adapter is refused before that, naming its key."""
    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorTransformer
    from oracle import synth
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only failure mode")
    from kandinsky2.checkpoints import diffusers_prior_to_k2
    cfg = p22.CONFIG_PRIOR22_TINY
    m = PriorTransformer(**cfg, device="cpu")
    m.load_state_dict(diffusers_prior_to_k2(synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=1))[0], strict=True)
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    lora = plo.synth_prior_lora(cfg, rank=2)
    with pytest.raises(K2Error):
        m.load_lora(lora)
    assert m.lora_scale is None
    with pytest.raises(K2Error, match="to_x_lora"):
        m.load_lora(dict(lora, **{"transformer_blocks.0.attn1.processor.to_x_lora.up.weight": torch.zeros(128, 2)}))
    assert m.lora_scale is None
    m.unload_lora()
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())
