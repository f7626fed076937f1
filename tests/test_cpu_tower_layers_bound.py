"""CPU: the bounds of tests/tower_layers_ref.py are neither too tight nor vacuous, on the oracles' tiny towers: the CLIP text
and image towers (ViT-bigG/14's layout), the OpenAI ViT-L/14 text and image towers (QuickGELU), XLM-R (post-LN, key masks),
DPT and DPT-Hybrid (LayerNorm eps 1e-12) and the 2.1 and 2.2 priors (causal, the keep mask with the extension tokens).

Each tower's layers run as an emulated plan (fp16 weights, fp16 rounding at every storage point, float64 elsewhere) from a
unit-normal fp16 embedding; every launch of every layer is then restated in float64 on the emulation's own fp16 input and must
hold the emulation inside its bound.  Every mutation that applies to the tower must leave the bound by at least 4x on some
element of some launch.  The median share of the bound is printed (run with -s), so that a bound gone loose shows.  The
layers start from a unit-normal embedding rather than the oracles' own; test_stack_restatement_equals_the_oracles pins the
restatement's layer semantics to the independent fp32 oracles instead, and the embeds are checked on their own."""
import pytest
import torch

from tests import tower_layers_ref as R

MIN_REJECT = 4.0


def _towers():
    from tests import clip_text_oracle as cto
    from tests import clip_vision_oracle as cvo
    from tests import dpt_oracle as do
    from tests import openai_clip_oracle as oo
    from tests import xlmr_oracle as xo
    from tests import dpt_hybrid_oracle as ho
    from tests import prior22_oracle as p22
    from oracle import prior_oracle as po
    from oracle import synth
    g = oo.GEO_TINY
    dcfg = do.TINY[0][1]
    return {
        "clip_text": (lambda: cto.synth_weights(cto.tiny_config(1000, 999), 3), "clip_text", 2, 16,
                      dict(heads=2, hd=64, eps=1e-5, act="gelu", post_ln=False, attn="small", causal=True)),
        "clip_vision": (lambda: cvo.synth_weights(cvo.CONFIG_TINY, 3), "clip_vision", 2, 17,
                        dict(heads=2, hd=104, eps=1e-5, act="gelu", post_ln=False, attn="fused", causal=False)),
        "openai_text": (lambda: oo.synth_weights(g, 3), "openai_text", g["text_layers"], g["context"],
                        dict(heads=2, hd=64, eps=1e-5, act="quick_gelu", post_ln=False, attn="small", causal=True)),
        "openai_vision": (lambda: oo.synth_weights(g, 3), "openai_vision", g["vision_layers"], 17,
                          dict(heads=2, hd=64, eps=1e-5, act="quick_gelu", post_ln=False, attn="fused", causal=False)),
        "xlmr": (lambda: xo.synth_weights(xo.tiny_config(1000), 32, 3), "mclip", 2, 20,
                 dict(heads=2, hd=64, eps=1e-5, act="gelu", post_ln=True, attn="small", causal=False, masked=True)),
        "dpt": (lambda: do.synth_weights(dcfg, 3), "dpt", dcfg["num_hidden_layers"], 17,
                dict(heads=2, hd=64, eps=1e-12, act="gelu", post_ln=False, attn="fused", causal=False)),
        "dpt_hybrid": (lambda: ho.synth_weights(ho.CFG_TINY, 3), "dpt", ho.CFG_TINY["num_hidden_layers"], 17,
                       dict(heads=2, hd=64, eps=1e-12, act="gelu", post_ln=False, attn="fused", causal=False)),
        "prior21": (lambda: synth.synth_state_dict(po.prior_param_spec(po.CONFIG_PRIOR_TINY), seed=3), "prior21",
                    po.CONFIG_PRIOR_TINY["xf_layers"], po.CONFIG_PRIOR_TINY["text_ctx"] + 4,
                    dict(heads=2, hd=64, eps=1e-5, act="gelu", post_ln=False, attn="small", causal=True, masked=True)),
        "prior22": (lambda: synth.synth_state_dict(p22.diffusers_prior_spec(p22.CONFIG_PRIOR22_TINY), seed=3), "prior22",
                    p22.CONFIG_PRIOR22_TINY["xf_layers"], p22.CONFIG_PRIOR22_TINY["text_ctx"] + 4,
                    dict(heads=2, hd=64, eps=1e-5, act="gelu", post_ln=False, attn="small", causal=True, masked=True)),
    }


TOWERS = ["clip_text", "clip_vision", "openai_text", "openai_vision", "xlmr", "dpt", "dpt_hybrid", "prior21", "prior22"]


@pytest.mark.parametrize("name", TOWERS)
def test_emulated_plan_inside_and_mutations_outside(name):
    make, fmt, L, T, t = _towers()[name]
    sd = make()
    Ps = [R.layer_params(fmt, sd, i) for i in range(L)]
    H = Ps[0]["q"][0].shape[0]
    t = dict(t, scale=t["hd"] ** -0.5)
    B = 2
    g = torch.Generator().manual_seed(7)
    h = R.V(torch.randn(B, T, H, generator=g).half().double())
    keep = None
    if t.get("masked"):   # padded prompts; the prior keeps its 4 extension tokens after the text
        ext = 4 if fmt.startswith("prior") else 0
        keep = (torch.arange(T)[None] < torch.tensor([T - ext - 2, 2])[:, None]).to(torch.uint8)
        keep[:, T - ext:] = 1
    stages = R.POST_LN if t["post_ln"] else R.PRE_LN
    worst, meds, rejected = 0.0, [], {}
    for i in range(L):
        P, Pn = Ps[i], Ps[i + 1] if i + 1 < L else Ps[i - 1]
        em = R.layer(P, Pn, h, t, R.Mode(em=True), keep=keep)
        snap = {k: R.V(v.v, torch.zeros_like(v.v)) for k, v in em.items()}
        ref = R.layer(P, Pn, h, t, R.EXACT, snap=snap, keep=keep)
        assert tuple(ref) == stages
        per = R.stage_shares({k: v.v for k, v in em.items()}, ref)
        for k, (w, m) in per.items():
            assert w <= 1.0, (name, i, k, w)
            worst = max(worst, w)
            meds.append(m)
        for mut in R.mutations(t):
            got = R.layer(P, Pn, h, t, R.Mode(mut=mut), snap=snap, keep=keep)
            rejected[mut] = max(rejected.get(mut, 0.0), R.rejection(got, ref))
        h = em[stages[-1]]
    med = sorted(meds)[len(meds) // 2]
    print(f"{name}: emulated plan worst {worst:.3f} of the bound, median {med:.3f}; mutations "
          + ", ".join(f"{k} {v:.3g}x" for k, v in rejected.items()))
    for mut, w in rejected.items():
        assert w >= MIN_REJECT, (name, mut, w)
    assert 1e-4 < med < 0.5, (name, med)   # a bound far above the emulation's error would let wiring errors through


def test_embeds_inside_and_their_mutations_outside():
    """xlmr_embed (its positions shifted by one must leave the bound) and the prior's token rows (the time token written to
    the image-token row must leave the image row's bound), emulated plans inside, on the tiny configs' tables."""
    from oracle import prior_oracle as po
    from oracle import synth
    from tests import xlmr_oracle as xo
    cfg = xo.tiny_config(1000)
    sd = xo.synth_weights(cfg, 32, 3)
    p = "transformer.embeddings."
    ids = torch.full((2, 20), xo.PAD_ID, dtype=torch.long)
    ids[0, :17] = torch.randint(3, 1000, (17,), generator=torch.Generator().manual_seed(2))
    ids[1, :5] = torch.randint(3, 1000, (5,), generator=torch.Generator().manual_seed(3))
    args = (sd[p + "word_embeddings.weight"], sd[p + "position_embeddings.weight"], sd[p + "token_type_embeddings.weight"][0],
            sd[p + "LayerNorm.weight"], sd[p + "LayerNorm.bias"], xo.PAD_ID, 1e-5)
    ref = R.xlmr_embed(ids, *args)
    w, med = R.share(R.xlmr_embed(ids, *args, M=R.Mode(em=True)).v, ref)
    rej = R.share(R.xlmr_embed(ids, *args, M=R.Mode(mut="pos_shift")).v, ref)[0]
    assert torch.equal(R.xlmr_positions(ids, xo.PAD_ID), xo.position_ids(ids, xo.PAD_ID))   # the oracle's positions
    print(f"xlmr_embed: emulated worst {w:.3f}, median {med:.3f}; pos_shift {rej:.3g}x")
    assert w <= 1.0 and rej >= MIN_REJECT
    psd = synth.synth_state_dict(po.prior_param_spec(po.CONFIG_PRIOR_TINY), seed=3)
    g = torch.Generator().manual_seed(4)
    pos, ctx = psd["positional_embedding"][0], po.CONFIG_PRIOR_TINY["text_ctx"]
    tok_t, tok_x = (R.V(torch.randn(2, pos.shape[1], generator=g).double()) for _ in range(2))
    ref = R.prior_token(tok_x, pos[ctx + 2][None])
    em = (tok_x.v.float().half().float() + pos[ctx + 2].half().float()).half().double()
    w = R.share(em, ref)[0]
    rej = R.share(R.prior_token(tok_t, pos[ctx + 2][None]).v, ref)[0]
    print(f"prior tokens: emulated worst {w:.3f}; time_token_to_image_row {rej:.3g}x")
    assert w <= 1.0 and rej >= MIN_REJECT


def test_stack_restatement_equals_the_oracles():
    """The restatement's layer semantics (residual order, which LayerNorm is ln_1 in the post-LN stack, q / k / v layout) are
    the independent oracles': R.stack in float64 against xlmr_oracle._tower and openai_clip_oracle._resblocks in fp32."""
    from tests import openai_clip_oracle as oo
    from tests import xlmr_oracle as xo
    g = torch.Generator().manual_seed(5)
    cfg = xo.tiny_config(1000)
    sd = xo.synth_weights(cfg, 32, 3)
    h = torch.randn(2, 20, 128, generator=g).half().float()
    mask = (torch.arange(20)[None] < torch.tensor([17, 5])[:, None]).long()
    Ps = [R.layer_params("mclip", sd, i) for i in range(2)]
    layers = [tuple(P[r] for r in ("q", "k", "v", "proj", "ln_1", "fc1", "fc2", "ln_2")) for P in Ps]
    want = xo._tower(h, mask, layers, (sd["LinearTransformation.weight"], sd["LinearTransformation.bias"]), cfg,
                     torch.float32)[0]
    t = dict(heads=2, hd=64, scale=0.125, eps=1e-5, act="gelu", post_ln=True, attn="small", causal=False)
    got = R.stack(Ps, R.V(h.double()), t, keep=mask.to(torch.uint8))
    assert R.rel_l2(got, want.double()) < 1e-5, R.rel_l2(got, want.double())
    osd = oo.synth_weights(oo.GEO_TINY, 3)
    for fmt, prefix, causal, T in (("openai_text", "transformer.", True, 16), ("openai_vision", "visual.transformer.", False, 17)):
        x = torch.randn(2, T, 128, generator=g).half().float()
        want = oo._resblocks(x, oo._openai_layers(osd, prefix, 2, torch.float32), 2, causal, torch.float32)
        t = dict(heads=2, hd=64, scale=0.125, eps=1e-5, act="quick_gelu", post_ln=False,
                 attn="small" if causal else "fused", causal=causal)
        got = R.stack([R.layer_params(fmt, osd, i) for i in range(2)], R.V(x.double()), t)
        assert R.rel_l2(got, want.double()) < 1e-5, (fmt, R.rel_l2(got, want.double()))


def test_every_mutation_applies_somewhere():
    seen = {"pos_shift", "time_token_to_image_row"}   # test_embeds_inside_and_their_mutations_outside
    seen_layers = set()
    for name in TOWERS:
        t = _towers()[name][4]
        seen_layers.update(R.mutations(dict(t, scale=t["hd"] ** -0.5)))
    assert seen | seen_layers == set(R.MUTATIONS), set(R.MUTATIONS) - seen - seen_layers


def test_qkv_weight_is_the_kernel_layout():
    """The reference's qkv layout is checkpoints.pack_heads' (the layout the attention kernels read), from q / k / v alone."""
    from kandinsky2.checkpoints import pack_heads
    g = torch.Generator().manual_seed(1)
    P = {r: (torch.randn(208, 16, generator=g), torch.randn(208, generator=g)) for r in "qkv"}
    w, b = R.qkv_weight(P, 104)
    assert torch.equal(w, pack_heads([P[r][0] for r in "qkv"], 104))
    assert torch.equal(b, pack_heads([P[r][1] for r in "qkv"], 104))
