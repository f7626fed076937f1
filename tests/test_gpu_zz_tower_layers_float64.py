"""GPU: every launch of the transformer towers as each tower's launch plan runs it, at the geometry the product runs, against the
float64 restatements of tests/tower_layers_ref.py on the plan's own inputs, with the weights read from the state dicts the
towers were loaded from.  Synthetic weights (the oracles' synth_weights / specs) at full size:
  ViT-bigG/14 text     32 x 1280, attention_small causal, n = 2 (6 and 77 tokens)
  ViT-bigG/14 image    48 x 1664, attention_heads at head width 104, B = 2
  ViT-L/14 text        12 x 768, QuickGELU, attention_small causal
  ViT-L/14 image       24 x 1024, QuickGELU, attention_d64
  XLM-R-large          24 x 1024, post-LN, padded key masks, n = 2 (9 and 77 tokens)
  dpt-large ViT        24 x 1024, 577 tokens (384^2), eps 1e-12
  DPT-Hybrid ViT       12 x 768, 577 tokens after the BiT stages
  2.1 and 2.2 priors   20 x 2048, 81 tokens, attention_small causal with the CFG keep mask: one _PriorStepPlan step, B = 2
                       (4 rows, prompts of 12 and 40 tokens and two empty ones), final_ln
Before the stack the embeds (clip_text_embed, xlmr_embed, clip_patchify and the patch-embedding GEMM with its position
residual, the prior's time-embedding chain and token rows) are restated, after it the final LayerNorms, clip_text_pool,
masked_mean_f16, the fp32 widening and the linear projections.

Harness: the plan is built as usual, with the ops entry points its steps call (and encoder.ACTIVATIONS, bound at import)
wrapped.  Its steps are then run one at a time, eagerly; each wrapped call snapshots its inputs before it runs and its output
after.  Four things are asserted:
  1. bit identity: the step-wise outputs equal one CUDA graph replay of the same plan, so the snapshots are of what the graph
     computes;
  2. wiring: every launch read exactly the bits its producer wrote (snapshots compared, so a buffer overwritten between
     producer and consumer fails too): inside every layer, from the embeds into layer 0, and from the last layer into the
     launches after the stack;
  3. float64 agreement: every launch of every layer and every restated launch around the stack within its bound, all rows;
  4. completeness: the plan's wrapped calls, counted per entry point, are exactly the checked ones plus the tower's explicit
     exempt list, and its other step kinds are the tower's listed ones, each with its reason -- a launch added to a tower later
     fails here until it is checked or exempted.
Every tower runs under the tuner's default choice and under forced N tile 256 + split-K 2 where the library takes them.

Output (run with -s): the worst and median share of the bound per launch kind and tower; each wiring error of
tower_layers_ref.MUTATIONS that applies, at layer L/2 (or at the launch it concerns), with its rejection share.  For the layer
mutations also how far the mutation moves the layer stack's output (float64, relative L2 over all rows, padded ones included)
next to how far the plan's own fp16 arithmetic leaves that output from float64."""
import collections
import contextlib
import time

import pytest
import torch

from tests import tower_layers_ref as R

pytestmark = pytest.mark.gpu

MIN_REJECT = 4.0
SETTINGS = ("default", "forced-tiles")

# inputs snapshotted for each wrapped entry point: (positional index or keyword) -> snapshot name
_INPUTS = {"layernorm_f16": {0: "x"}, "gemm_rows": {0: "x", "residual": "res"}, "attention_small": {0: "qkv"},
           "attention_heads": {0: "qkv"}, "attention_d64": {0: "qkv"}, "gelu_f16_": {0: "x"}, "quick_gelu_f16_": {0: "x"},
           "clip_text_embed": {0: "ids"}, "clip_text_pool": {1: "x"}, "xlmr_embed": {0: "ids"}, "masked_mean_f16": {0: "x"},
           "clip_patchify": {0: "pix"}, "linear": {0: "x"}, "f16_to_f32": {0: "x"}, "readout_rows_f16": {0: "x"},
           "prior_tokens": {0: "x"}, "timestep_embedding": {0: "t"}}

_NECK = "the DPT neck and head (readout, convolutions, resampling): test_gpu_zz_depth_blocks_float64.py"
_NECK_KINDS = {"conv", "relu", "bilinear", "depth_to_space", "subsample"}
_BIT_KINDS = {"im2col", "conv", "conv_stride2_at_1", "conv_gemm", "gn_stats", "gn_finalize", "gn_act", "maxpool", "subsample",
              "relu"}


# ------------------------------------------------------------------------------------------------------------------------------
# recording
# ------------------------------------------------------------------------------------------------------------------------------
class _Rec:
    def __init__(self):
        self.on, self.calls, self.step = False, [], -1


def _wrap(ops, name, rec):
    fn = getattr(ops, name)
    ins = _INPUTS[name]

    def f(*a, **k):
        if not rec.on:
            return fn(*a, **k)
        snap = {}
        for key, sname in ins.items():
            t = a[key] if isinstance(key, int) and key < len(a) else k.get(key) if isinstance(key, str) else None
            if t is not None:
                snap[sname] = t.clone()
        out = fn(*a, **k)
        o = k.get("out") if k.get("out") is not None else out
        rec.calls.append(dict(name=name, step=rec.step, ins=snap, out=o.clone()))
        return out
    return f


@contextlib.contextmanager
def _recording(setting, rec):
    from kandinsky2 import launch_plan as lp
    from kandinsky2 import ops
    from kandinsky2.model import encoder
    from tests.test_gpu_plan_blocks_float64 import _forced_tune
    mp = pytest.MonkeyPatch()
    try:
        for name in _INPUTS:
            mp.setattr(ops, name, _wrap(ops, name, rec))
        mp.setattr(encoder, "ACTIVATIONS", {"gelu": ops.gelu_f16_, "quick_gelu": ops.quick_gelu_f16_})
        if setting == "forced-tiles":
            mp.setattr(lp, "tune", _forced_tune)
        yield
    finally:
        mp.undo()


def _stepwise(plan, rec):
    rec.calls, rec.on = [], True
    try:
        for i, (fn, _, _) in enumerate(plan.steps):
            rec.step = i
            fn()
    finally:
        rec.on = False
    torch.cuda.synchronize()
    return rec.calls


# ------------------------------------------------------------------------------------------------------------------------------
# the launches around the stack: each handler checks one call's wiring and returns [(label, got, V ref, {mutation: V})]
# ------------------------------------------------------------------------------------------------------------------------------
def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), what


def _f32(sd, k):
    return sd[k].float()


def _clip_text_embed(c, d, prev):
    sd, (tok, pos) = d["sd"], d["embed"]
    ids = c["ins"]["ids"].long()
    x = R.V(_f32(sd, tok)[ids].double())
    return [("embed", c["out"], R.prior_token(x, _f32(sd, pos)[:ids.shape[1]][None]), {})]


def _xlmr_embed(c, d, prev):
    sd, p, cfg = d["sd"], "transformer.embeddings.", d["cfg"]
    ids = c["ins"]["ids"].long()
    args = (_f32(sd, p + "word_embeddings.weight"), _f32(sd, p + "position_embeddings.weight"),
            _f32(sd, p + "token_type_embeddings.weight")[0], _f32(sd, p + "LayerNorm.weight"), _f32(sd, p + "LayerNorm.bias"),
            cfg["pad_token_id"], cfg["layer_norm_eps"])
    ref = R.xlmr_embed(ids, *args)
    return [("embed", c["out"], ref, {"pos_shift": R.xlmr_embed(ids, *args, M=R.Mode(mut="pos_shift"))})]


def _patchify(c, d, prev):
    P, kp = d["patch"]
    return [("patchify", c["out"], R.patchify(c["ins"]["pix"], P, kp), {})]


def _patch_embed(c, d, prev):
    sd, (w, cls, pos, bias) = d["sd"], d["patch_embed"]
    _eq(c["ins"]["x"], prev["out"], f"{d['name']}: the patch-embedding GEMM does not read the patch rows")
    pv = _f32(sd, pos).reshape(-1, _f32(sd, w).shape[0])
    ref = R.patch_embed(R.V(c["ins"]["x"].double()), _f32(sd, w), _f32(sd, cls), pv, d["patch"][1],
                        bias=_f32(sd, bias) if bias else None)
    return [("patch embed", c["out"], ref, {})]


def _layernorm(name):
    def f(c, d, prev, src=None):
        sd = d["sd"]
        _eq(c["ins"]["x"], src if src is not None else prev["out"], f"{d['name']}: {name} does not read its producer")
        return [(name, c["out"], R.layernorm(R.V(c["ins"]["x"].double()), _f32(sd, name + ".weight"), _f32(sd, name + ".bias"),
                                             d["eps"]), {})]
    return f


def _pool(c, d, prev):
    _eq(c["ins"]["x"], prev["out"], f"{d['name']}: the pool does not read the final LayerNorm")
    return [("pool", c["out"], R.pool_rows(R.V(c["ins"]["x"].double()), d["pool_index"]), {})]


def _masked_mean(c, d, prev):
    x = R.V(c["ins"]["x"].double())
    return [("masked mean", c["out"], R.masked_mean(x, d["keep"]), {"mask_one_longer": R.masked_mean(
        x, d["keep"], R.Mode(mut="mask_one_longer"))})]


def _widen(c, d, prev):
    _eq(c["ins"]["x"], prev["out"], f"{d['name']}: the widening does not read the LayerNorm output")
    x = c["ins"]["x"].double()
    return [("widen", c["out"], R.V(x, torch.zeros_like(x)), {})]


def _projection(key):
    def f(c, d, prev):
        sd = d["sd"]
        if prev is not None:
            _eq(c["ins"]["x"], prev["out"], f"{d['name']}: the projection does not read its producer")
        w, b, t = key
        W = _f32(sd, w).t() if t else _f32(sd, w)
        return [("projection", c["out"], R.projection(R.V(c["ins"]["x"].double()), W, _f32(sd, b) if b else None), {})]
    return f


def _prior_pre(cs, d):
    """The prior's time-embedding chain and token rows: timestep_embedding, linear, linear (SiLU in), prior_tokens (time
    row), linear (image embedding), prior_tokens (image-token row)."""
    sd, (te0, te2, img) = d["sd"], d["prior_names"]
    ts, l0, l1, tk_t, li, tk_x = cs
    W = l0["out"].shape[1]
    ctx = d["ctx"]
    pos = _f32(sd, "positional_embedding")[0]
    out = [("timestep embedding", ts["out"], R.timestep_embedding(ts["ins"]["t"], W), {})]
    _eq(l0["ins"]["x"], ts["out"], "time linear 0 does not read the timestep embedding")
    out.append(("time linear", l0["out"], R.projection(R.V(l0["ins"]["x"].double()), _f32(sd, te0 + ".weight"),
                                                      _f32(sd, te0 + ".bias")), {}))
    _eq(l1["ins"]["x"], l0["out"], "time linear 2 does not read time linear 0")
    out.append(("time linear", l1["out"], R.projection(R.V(l1["ins"]["x"].double()), _f32(sd, te2 + ".weight"),
                                                      _f32(sd, te2 + ".bias"), silu_in=True), {}))
    _eq(tk_t["ins"]["x"], l1["out"], "the time token does not read the time embedding")
    out.append(("tokens", tk_t["out"], R.prior_token(R.V(tk_t["ins"]["x"].double()), pos[ctx + 1][None]), {}))
    out.append(("image linear", li["out"], R.projection(R.V(li["ins"]["x"].double()), _f32(sd, img + ".weight"),
                                                       _f32(sd, img + ".bias")), {}))
    _eq(tk_x["ins"]["x"], li["out"], "the image token does not read the image linear")
    mut = R.prior_token(R.V(tk_t["ins"]["x"].double()), pos[ctx + 2][None])
    out.append(("tokens", tk_x["out"], R.prior_token(R.V(tk_x["ins"]["x"].double()), pos[ctx + 2][None]),
                {"time_token_to_image_row": mut}))
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# towers
# ------------------------------------------------------------------------------------------------------------------------------
def _text_ids(n_lengths, bos, eos, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(len(n_lengths), 77, dtype=torch.long)
    for r, n in enumerate(n_lengths):
        ids[r, 0], ids[r, n - 1] = bos, eos
        ids[r, 1:n - 1] = torch.randint(1, bos, (n - 2,), generator=g)
    return ids


def _bigg_text():
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower
    from tests import clip_text_oracle as cto
    cfg = cto.CONFIG_BIGG
    sd = {k: v.cuda() for k, v in cto.synth_weights(cfg, 21).items()}
    tower = CLIPTextTower(transformers_clip_text_to_k2(sd), cfg, device="cuda").finalize()
    V = cfg["vocab_size"]
    ids = _text_ids((6, 77), V - 2, V - 1, V, 5)
    return dict(name="bigG text", sd=sd, fmt="clip_text", L=cfg["num_hidden_layers"], obj=tower, eps=1e-5,
                run=lambda g: tower.forward(ids, use_graph=g), plan=lambda: tower._plan(*ids.shape),
                t=dict(heads=20, hd=64, scale=0.125, eps=1e-5, act="gelu", post_ln=False, attn="small", causal=True),
                embed=("text_model.embeddings.token_embedding.weight", "text_model.embeddings.position_embedding.weight"),
                pool_index=cto.pooled_index(ids, cfg["eos_token_id"]).cuda(),
                pre=[("clip_text_embed", _clip_text_embed)],
                post=[("layernorm_f16", _layernorm("text_model.final_layer_norm")), ("clip_text_pool", _pool),
                      ("linear", _projection(("text_projection.weight", None, False)))])


def _bigg_image():
    from kandinsky2.model.clip_vision import CLIPVisionTower
    from tests import clip_vision_oracle as cvo
    cfg = cvo.CONFIG_BIGG
    sd = {k: v.cuda() for k, v in cvo.synth_weights(cfg, 21).items()}
    tower = CLIPVisionTower.from_transformers(sd, cfg, device="cuda")
    pix = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda()
    e = "vision_model.embeddings."
    return dict(name="bigG image", sd=sd, fmt="clip_vision", L=cfg["num_hidden_layers"], obj=tower, eps=1e-5,
                run=lambda g: tower.forward(pix, use_graph=g), plan=lambda: tower._plan(2),
                t=dict(heads=16, hd=104, scale=104 ** -0.5, eps=1e-5, act="gelu", post_ln=False, attn="fused", causal=False),
                patch=(14, tower.cfg["kp"]),
                patch_embed=(e + "patch_embedding.weight", e + "class_embedding", e + "position_embedding.weight", None),
                pre=[("clip_patchify", _patchify), ("gemm_rows", _patch_embed),
                     ("layernorm_f16", _layernorm("vision_model.pre_layrnorm"))],
                post=[("layernorm_f16", _layernorm("vision_model.post_layernorm")), ("f16_to_f32", _widen),
                      ("linear", _projection(("visual_projection.weight", None, False)))], cls_post=True)


_L14 = {}


def _l14():
    if not _L14:
        from kandinsky2.model.clip_vitl14 import load_openai_clip
        from tests import openai_clip_oracle as oo
        sd = {k: v.cuda() for k, v in oo.synth_weights(oo.GEO_L14, 31).items()}
        _L14.update(sd=sd, towers=load_openai_clip(sd, "cuda"))
    return _L14


def _l14_text():
    d = _l14()
    tower = d["towers"][0]
    ids = _text_ids((5, 77), 49406, 49407, 49408, 8)
    return dict(name="ViT-L/14 text", sd=d["sd"], fmt="openai_text", L=12, obj=tower, eps=1e-5,
                run=lambda g_: tower.forward(ids, use_graph=g_), plan=lambda: tower._plan(*ids.shape),
                t=dict(heads=12, hd=64, scale=0.125, eps=1e-5, act="quick_gelu", post_ln=False, attn="small", causal=True),
                embed=("token_embedding.weight", "positional_embedding"), pool_index=ids.argmax(-1).cuda(),
                pre=[("clip_text_embed", _clip_text_embed)],
                post=[("layernorm_f16", _layernorm("ln_final")), ("clip_text_pool", _pool),
                      ("linear", _projection(("text_projection", None, True)))])


def _l14_image():
    d = _l14()
    tower = d["towers"][1]
    pix = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(4)).cuda()
    return dict(name="ViT-L/14 image", sd=d["sd"], fmt="openai_vision", L=24, obj=tower, eps=1e-5,
                run=lambda g: tower.forward(pix, use_graph=g), plan=lambda: tower._plan(2),
                t=dict(heads=16, hd=64, scale=0.125, eps=1e-5, act="quick_gelu", post_ln=False, attn="fused", causal=False),
                patch=(14, tower.cfg["kp"]),
                patch_embed=("visual.conv1.weight", "visual.class_embedding", "visual.positional_embedding", None),
                pre=[("clip_patchify", _patchify), ("gemm_rows", _patch_embed), ("layernorm_f16", _layernorm("visual.ln_pre"))],
                post=[("layernorm_f16", _layernorm("visual.ln_post")), ("f16_to_f32", _widen),
                      ("linear", _projection(("visual.proj", None, True)))], cls_post=True)


def _xlmr():
    from kandinsky2.model.text_encoders import MultilingualCLIP
    from tests import xlmr_oracle as xo
    from tests.test_gpu_zz_text_encoder import large_ids
    cfg = xo.CONFIG_LARGE
    sd = {k: v.cuda() for k, v in xo.synth_weights(cfg, xo.OUT_LARGE, 21).items()}
    tower = MultilingualCLIP.from_state_dict(sd, cfg, device="cuda")
    ids, mask = large_ids(2, seed=6, lengths=(9, 77))
    return dict(name="XLM-R-large", sd=sd, fmt="mclip", L=cfg["num_hidden_layers"], obj=tower, cfg=cfg,
                eps=cfg["layer_norm_eps"], run=lambda g: tower.forward(ids, mask, use_graph=g), plan=lambda: tower._plan(*ids.shape),
                t=dict(heads=16, hd=64, scale=0.125, eps=cfg["layer_norm_eps"], act="gelu", post_ln=True, attn="small",
                       causal=False, masked=True),
                keep=mask.to(torch.uint8).cuda(), pre=[("xlmr_embed", _xlmr_embed)],
                post=[("masked_mean_f16", _masked_mean),
                      ("linear", _projection(("LinearTransformation.weight", "LinearTransformation.bias", False)))])


def _dpt():
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_oracle as do
    cfg = do.CFG_LARGE
    sd = {k: v.cuda() for k, v in do.synth_weights(cfg, 31).items()}
    est = DPTDepthEstimator.from_transformers(sd, cfg)
    pix = torch.randn(1, 3, 384, 384, generator=torch.Generator().manual_seed(2)).cuda()
    e = "dpt.embeddings."
    return dict(name="DPT-large ViT", sd=sd, fmt="dpt", L=24, obj=est, eps=1e-12,
                run=lambda g: (est.predicted_depth(pix, use_graph=g),), plan=lambda: est._plan(1),
                t=dict(heads=16, hd=64, scale=0.125, eps=1e-12, act="gelu", post_ln=False, attn="fused", causal=False),
                patch=(16, est.cfg["kp"]),
                patch_embed=(e + "patch_embeddings.projection.weight", e + "cls_token", e + "position_embeddings",
                             e + "patch_embeddings.projection.bias"),
                pre=[("clip_patchify", _patchify), ("gemm_rows", _patch_embed)], post=None,
                exempt_kinds=dict.fromkeys(_NECK_KINDS, _NECK))


def _dpt_hybrid():
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_hybrid_oracle as ho
    cfg = ho.CFG_HYBRID
    sd = {k: v.cuda() for k, v in ho.synth_weights(cfg, 31, last_bias=ho.REAL_LAST_BIAS).items()}
    est = DPTDepthEstimator.from_transformers(sd, cfg)
    pix = torch.randn(1, 3, 384, 384, generator=torch.Generator().manual_seed(2)).cuda()
    bit = "the BiT backbone (convolutions, GroupNorm, pooling): test_gpu_zz_depth_blocks_float64.py"
    return dict(name="DPT-Hybrid ViT", sd=sd, fmt="dpt", L=12, obj=est, eps=1e-12,
                run=lambda g: (est.predicted_depth(pix, use_graph=g),), plan=lambda: est._plan(1, 384, 384),
                t=dict(heads=12, hd=64, scale=0.125, eps=1e-12, act="gelu", post_ln=False, attn="fused", causal=False),
                pre=[], pre_exempt={"gemm_rows": "the token projection of the BiT features: part of " + bit}, post=None,
                exempt_kinds={**dict.fromkeys(_NECK_KINDS, _NECK), **dict.fromkeys(_BIT_KINDS - _NECK_KINDS, bit)})


def _prior(kind):
    from kandinsky2.model.prior import PriorTransformer, UnCLIPSchedule
    from oracle import synth
    if kind == "2.1":
        from oracle import prior_oracle as po
        cfg = po.CONFIG_PRIOR
        sd = {k: v.cuda() for k, v in synth.synth_state_dict(po.prior_param_spec(cfg)).items()}
        m = PriorTransformer(**cfg, device="cuda")
        m.load_state_dict(sd, strict=True)
        names, fmt, fin, outp = ("time_embed.0", "time_embed.2", "clip_img_proj"), "prior21", "final_ln", "out_proj"
    else:
        from kandinsky2.checkpoints import diffusers_prior_to_k2
        from tests import prior22_oracle as p22
        cfg = p22.CONFIG_PRIOR22
        sd = {k: v.cuda() for k, v in synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=11).items()}
        m = PriorTransformer(**cfg, device="cuda")
        m.load_state_dict(diffusers_prior_to_k2(sd)[0], strict=True)
        names = ("time_embedding.linear_1", "time_embedding.linear_2", "proj_in")
        fmt, fin, outp = "prior22", "norm_out", "proj_to_clip_embeddings"
    m.finalize()
    B, D, L, X = 2, cfg["clip_dim"], cfg["text_ctx"], cfg["clip_xf_width"]
    g = torch.Generator(device="cuda").manual_seed(17)
    te = torch.randn(2 * B, D, device="cuda", generator=g)
    tenc = torch.randn(2 * B, L, X, device="cuda", generator=g)
    lens = torch.tensor([12, 40, 2, 2], device="cuda")
    mask = torch.arange(L, device="cuda")[None] < lens[:, None]
    keep = torch.nn.functional.pad(mask, (0, 4), value=True).to(torch.uint8)
    st = {}

    def run(use_graph):
        plan = m._step_plan(B)
        if "x" not in st:
            plan.bind(te, tenc, mask)
            plan.set_schedule(UnCLIPSchedule(5), torch.randn(B, D, device="cuda", generator=g),
                              torch.randn(5, B, D, device="cuda", generator=g), 4.0, use_graph=True)
            st.update(x=plan.x.clone(), counter=plan.counter.clone())
        plan.run(use_graph)
        return plan.model_out.clone(), plan.x.clone()

    def reset():
        plan = m._step_plan(B)
        plan.x.copy_(st["x"])
        plan.counter.copy_(st["counter"])

    def new_plans():
        m._step_plans = {}
        st.clear()

    step = "k2_step_begin / k2_sampler_step / k2_step_end: test_gpu_sampler_kernels.py and the prior sampling tests"
    return dict(name=f"{kind} prior", sd=sd, fmt=fmt, L=cfg["xf_layers"], obj=m, new_plans=new_plans, eps=1e-5, run=run,
                reset=reset, plan=lambda: m._step_plan(B), ctx=L, prior_names=names, keep=keep,
                t=dict(heads=cfg["xf_heads"], hd=64, scale=0.125, eps=1e-5, act="gelu", post_ln=False, attn="small",
                       causal=True, masked=True),
                pre=[("timestep_embedding", None), ("linear", None), ("linear", None), ("prior_tokens", None),
                     ("linear", None), ("prior_tokens", None)], prior_pre=True,
                post=[("layernorm_f16", _layernorm(fin)), ("f16_to_f32", _widen),
                      ("linear", _projection((outp + ".weight", outp + ".bias", False)))], last_row=True,
                exempt_kinds={"step": step, "sampler_step": step}, outputs=lambda p: [p.model_out, p.x])


TOWERS = {"bigg_text": _bigg_text, "bigg_image": _bigg_image, "l14_text": _l14_text, "l14_image": _l14_image,
          "xlmr": _xlmr, "dpt_large": _dpt, "dpt_hybrid": _dpt_hybrid, "prior21": lambda: _prior("2.1"),
          "prior22": lambda: _prior("2.2")}


# ------------------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------------------
def _ops(t):
    act = "quick_gelu_f16_" if t["act"] == "quick_gelu" else "gelu_f16_"
    attn = {"small": "attention_small"}.get(t["attn"], "attention_heads" if t["hd"] == 104 else "attention_d64")
    return act, attn


def _split(calls, plan, d):
    """-> (pre calls, {stage: call} per layer, post calls, calls after the stack the tower exempts)."""
    t, L = d["t"], d["L"]
    stages = R.POST_LN if t["post_ln"] else R.PRE_LN
    act, attn = _ops(t)
    op = dict(ln_1="layernorm_f16", ln_2="layernorm_f16", qkv="gemm_rows", proj="gemm_rows", fc1="gemm_rows",
              fc2="gemm_rows", att=attn, act=act)
    pre_names = [n for n, _ in d["pre"]] + list(d.get("pre_exempt", {}))
    p0 = len(pre_names)
    assert [c["name"] for c in calls[:p0]] == pre_names, (d["name"], [c["name"] for c in calls[:p0 + 1]])
    layers = []
    for i in range(L):
        cs = calls[p0 + 8 * i:p0 + 8 * i + 8]
        assert [c["name"] for c in cs] == [op[s] for s in stages], (d["name"], i, [c["name"] for c in cs])
        layers.append(dict(zip(stages, cs)))
    rest = calls[p0 + 8 * L:]
    if d["post"] is not None:
        assert [c["name"] for c in rest] == [n for n, _ in d["post"]], (d["name"], [c["name"] for c in rest])
        return calls[:p0], layers, rest, []
    return calls[:p0], layers, [], rest


def _completeness(plan, calls, neck, d):
    """Every wrapped call is a checked one or on the tower's exempt list; every other step kind is listed with its reason."""
    L = d["L"]
    act, attn = _ops(d["t"])
    checked = collections.Counter({"layernorm_f16": 2 * L, "gemm_rows": 4 * L, attn: L, act: L})
    checked.update(n for n, _ in d["pre"])
    checked.update(n for n, _ in (d["post"] or []))
    exempt = collections.Counter(list(d.get("pre_exempt", {})))
    reasons = dict(d.get("pre_exempt", {}))
    if neck:
        assert {c["name"] for c in neck} <= {"gemm_rows", "readout_rows_f16", "gelu_f16_"}, [c["name"] for c in neck]
        exempt.update(c["name"] for c in neck)
        reasons.update(dict.fromkeys((c["name"] for c in neck), _NECK))
    got = collections.Counter(c["name"] for c in calls)
    assert got == checked + exempt, (d["name"], got, checked, exempt)
    assert len({c["step"] for c in calls}) == len(calls), "more than one wrapped call in one step"
    stepped = {c["step"] for c in calls}
    unwrapped = collections.Counter(k for i, (_, k, _) in enumerate(plan.steps) if i not in stepped)
    kinds = d.get("exempt_kinds", {})
    assert set(unwrapped) <= set(kinds), (d["name"], unwrapped)
    reasons.update({k: kinds[k] for k in unwrapped})
    print(f"  completeness: checked {dict(checked)}; exempt calls {dict(exempt)}, other step kinds {dict(unwrapped)}")
    for k, r in reasons.items():
        print(f"    exempt {k}: {r}")


def _around(pre, layers, post, d, stack_out):
    """Wiring and float64 restatements of the launches before and after the stack -> [(label, got, ref, {mutation: V})]."""
    out = []
    first = R.POST_LN[0] if d["t"]["post_ln"] else R.PRE_LN[0]
    stack_in = layers[0][first]["ins"]["x"]
    if d.get("prior_pre"):
        out += _prior_pre(pre, d)
        ctx = d["ctx"]
        _eq(stack_in[:, ctx + 1], pre[3]["out"], f"{d['name']}: layer 0 does not read the time token")
        _eq(stack_in[:, ctx + 2], pre[5]["out"], f"{d['name']}: layer 0 does not read the image token")
    else:
        prev = None
        for c, (_, fn) in zip(pre, d["pre"]):
            out += fn(c, d, prev)
            prev = c
        if pre:
            _eq(stack_in, pre[-1]["out"], f"{d['name']}: layer 0 does not read the embedding")
    if d["post"] is not None:
        src = stack_out[:, 0] if d.get("cls_post") else stack_out[:, -1] if d.get("last_row") else None
        prev = None
        for j, (c, (name, fn)) in enumerate(zip(post, d["post"])):
            if j == 0:
                _eq(c["ins"]["x"], stack_out if src is None else src, f"{d['name']}: {name} does not read the last layer")
                out += fn(c, d, None) if name != "layernorm_f16" else fn(c, d, None, src=c["ins"]["x"])
            else:
                out += fn(c, d, prev)
            prev = c
    return out


def _float64(layers, d, per_kind):
    """Every layer within the bound, all rows."""
    sd, t, L = d["sd"], d["t"], d["L"]
    keep = d.get("keep")
    for i, c in enumerate(layers):
        P = R.layer_params(d["fmt"], sd, i)
        Pn = R.layer_params(d["fmt"], sd, i + 1 if i + 1 < L else i - 1)
        first = R.POST_LN[0] if t["post_ln"] else R.PRE_LN[0]
        h = R.V(c[first]["ins"]["x"].double())
        snap = {s: R.V(cc["out"].double()) for s, cc in c.items()}
        ref = R.layer(P, Pn, h, t, R.EXACT, snap=snap, keep=keep)
        for s, (w, m) in R.stage_shares({s: cc["out"] for s, cc in c.items()}, ref).items():
            kind = s if s in ("att", "act") else ("layernorm" if s.startswith("ln") else "gemm " + s)
            per_kind[kind].append((w, m, i))
            assert w <= 1.0, (d["name"], i, s, w)


def _mutations(layers, d, stack_out):
    """Each applicable layer mutation at layer L/2: rejection share, and its float64 effect on the stack's output."""
    sd, t, L = d["sd"], d["t"], d["L"]
    keep = d.get("keep")
    i = L // 2
    c = layers[i]
    P, Pn = R.layer_params(d["fmt"], sd, i), R.layer_params(d["fmt"], sd, i + 1)
    first = R.POST_LN[0] if t["post_ln"] else R.PRE_LN[0]
    h = R.V(c[first]["ins"]["x"].double())
    snap = {s: R.V(cc["out"].double()) for s, cc in c.items()}
    ref = R.layer(P, Pn, h, t, R.EXACT, snap=snap, keep=keep)
    Ps = [R.layer_params(d["fmt"], sd, j) for j in range(L)]
    h0 = R.V(layers[0][first]["ins"]["x"].double())
    exact = R.stack(Ps, h0, t, keep=keep)
    plan_dev = R.rel_l2(stack_out.double(), exact)
    for mut in R.mutations(t):
        w = R.rejection(R.layer(P, Pn, h, t, R.Mode(mut=mut), snap=snap, keep=keep), ref)
        moved = R.rel_l2(R.stack(Ps, h0, t, keep=keep, at=i, mut=mut), exact)
        print(f"  mutation {mut} ({R.MUTATIONS[mut]}) at layer {i}: {w:.3g} x the bound; moves the layer stack's output by "
              f"rel L2 {moved:.2e}, the plan's own fp16 arithmetic by {plan_dev:.2e}")
        assert w >= MIN_REJECT, (d["name"], mut, w)


@pytest.mark.parametrize("tower", list(TOWERS))
def test_tower_layers_float64(tower):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    d = TOWERS[tower]()
    rec = _Rec()
    for setting in SETTINGS:
        if "new_plans" in d:
            d["new_plans"]()
        else:
            d["obj"]._plans = {}
        with _recording(setting, rec):
            graph = [x.clone() for x in d["run"](True)]
            plan = d["plan"]()
            if "reset" in d:
                d["reset"]()
            torch.cuda.synchronize()
            calls = _stepwise(plan, rec)
        outs = d["outputs"](plan) if "outputs" in d else [plan.out] + ([plan.hidden] if hasattr(plan, "hidden") else [])
        for g in graph:   # 1. the step-wise run equals the graph replay, bit for bit
            assert any(o.shape == g.shape and torch.equal(o, g) for o in outs), (d["name"], setting, "step-wise != graph")
        pre, layers, post, neck = _split(calls, plan, d)
        stack_out = R.check_wiring(layers, d["t"]["post_ln"], d["name"])   # 2. inside the stack
        print(f"{d['name']} [{setting}]:")
        _completeness(plan, calls, neck, d)                                 # 4.
        per_kind = collections.defaultdict(list)
        _float64(layers, d, per_kind)                                       # 3.
        for label, got, ref, muts in _around(pre, layers, post, d, stack_out):   # 2. and 3. around the stack
            w, m = R.share(got, ref)
            per_kind[label].append((w, m, -1))
            assert w <= 1.0, (d["name"], label, w)
            for mut, v in muts.items():
                r = R.share(v.v, ref)[0]
                if setting == "default":
                    print(f"  mutation {mut} ({R.MUTATIONS[mut]}) at the {label}: {r:.3g} x the bound")
                assert r >= MIN_REJECT, (d["name"], mut, r)
        for kind, v in per_kind.items():
            w = max(v)
            at = f" (layer {w[2]})" if w[2] >= 0 else ""
            print(f"  {kind}: worst {w[0]:.3f} of the bound{at}, median {sorted(x[1] for x in v)[len(v) // 2]:.3f}")
        if setting == "default":
            _mutations(layers, d, stack_out)
        del calls, layers, pre, post, neck
        torch.cuda.empty_cache()
    print(f"{d['name']}: {time.time() - t0:.1f} s")
