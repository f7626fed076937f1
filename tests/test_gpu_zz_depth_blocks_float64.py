"""GPU: every launch of the depth estimators outside the ViT layers -- the DPT neck, fusion and head, the hybrid's BiT backbone
and token GEMM -- and of the ControlNet hint stem, as the launch plans (and UNet.hint_features) run them, against the float64
restatements of tests/depth_blocks_ref.py on the launches' own inputs, with the weights read from the transformers / diffusers
state dicts the models were loaded from.  Synthetic weights at the real widths:
  DPT-large    dpt_oracle.CFG_LARGE, seed 31: 384^2, B = 1 (even 24 x 24 grid, factors 4 / 2 / 1 / 0.5), and 400^2, B = 2
               (preprocessor size 400: a 25 x 25 grid, the odd 0.5 path, the fusion resize at three stages, 416^2 output)
  DPT-Hybrid   dpt_hybrid_oracle.CFG_HYBRID, REAL_LAST_BIAS: 384^2, B = 1, and 208 x 336, B = 2 (a 13 x 21 grid)
  hint stem    the ControlNet UNet's input_hint_block: 768^2, N = 2, and 360 x 536, N = 1

Harness (test_gpu_zz_tower_layers_float64.py's): the ops entry points the plans call are wrapped; while a plan is built,
kandinsky2.model.depth.record_layers / record_patch_embed are wrapped to note their step ranges (the tower test checks those).
The plan's steps are then run one at a time; each wrapped call snapshots its inputs before it runs and its output after.
Asserted:
  1. bit identity: the step-wise output equals a CUDA graph replay of the same plan;
  2. wiring: every launch read exactly the bits its producer wrote (the hybrid's token rows: the last BiT block's output, a 1
     in column C3 of the CLS row and zeros elsewhere);
  3. float64: every launch, every element, within its bound;
  4. completeness: every step outside the layer ranges holds exactly one wrapped call, and the calls are the restatement's
     launches in order -- a launch added to a plan later fails here until it is restated.
Every geometry runs under the tuner's default choice and under forced N tile 256 + split-K 2 (the hint stem calls the library
directly, without the tuner: both settings run the same launches there).

Output (run with -s): the worst and median share of the bound per launch kind, the largest mean / std of any BiT GroupNorm,
and each mutation of depth_blocks_ref.MUTATIONS that applies, at the site where it falls furthest outside, with its
rejection share."""
import collections
import contextlib
import time

import pytest
import torch

from tests import depth_blocks_ref as D

pytestmark = pytest.mark.gpu

SETTINGS = ("default", "forced-tiles")
_OPS = ("conv_gemm", "gemm_rows", "readout_rows_f16", "gelu_f16_", "depth_to_space_f16", "subsample2", "bilinear_f16",
        "relu_f16", "relu_f32", "im2col_f16", "maxpool_f16", "gn_stats", "gn_finalize", "gn_act_f16", "silu_f16_",
        "stem_im2col")


class _Rec:
    def __init__(self):
        self.on, self.calls, self.step, self.ranges, self.depth = False, [], -1, [], 0


def _clone(t):
    return None if t is None else t.clone()


def _ins(name, a, k):
    if name == "conv_gemm":
        return {"srcs": [t.clone() for t, _ in a[0]], "res": _clone(k.get("residual"))}
    if name == "gemm_rows":
        return {"x": a[0].clone(), "res": _clone(k.get("residual"))}
    if name == "gn_act_f16":
        return {"x": a[0].clone(), "r": _clone(k.get("r"))}
    if name == "gn_finalize":
        return {}
    return {"x": a[0].clone()}


def _wrap(ops, name, rec):
    fn = getattr(ops, name)

    def f(*a, **k):
        if not rec.on or rec.depth:   # an entry point another one calls (gemm_rows -> conv_gemm) is that launch
            return fn(*a, **k)
        ins = _ins(name, a, k)
        rec.depth += 1
        try:
            out = fn(*a, **k)
        finally:
            rec.depth -= 1
        o = k.get("out") if k.get("out") is not None else out
        rec.calls.append(dict(name=name, step=rec.step, ins=ins, out=o.clone()))
        return out
    return f


def _ranged(fn, rec):
    def f(plan, *a, **k):
        s = len(plan.steps)
        out = fn(plan, *a, **k)
        rec.ranges.append((s, len(plan.steps)))
        return out
    return f


@contextlib.contextmanager
def _recording(setting, rec):
    from kandinsky2 import launch_plan as lp
    from kandinsky2 import ops
    from kandinsky2.model import depth
    from tests.test_gpu_plan_blocks_float64 import _forced_tune
    mp = pytest.MonkeyPatch()
    try:
        for name in _OPS:
            mp.setattr(ops, name, _wrap(ops, name, rec))
        for name in ("record_layers", "record_patch_embed"):
            mp.setattr(depth, name, _ranged(getattr(depth, name), rec))
        if setting == "forced-tiles":
            mp.setattr(lp, "tune", _forced_tune)
        yield
    finally:
        mp.undo()


# ------------------------------------------------------------------------------------------------------------------------------
# geometries: each returns (name, run(rec, setting) -> (calls outside the layer ranges, walk builder))
# ------------------------------------------------------------------------------------------------------------------------------
def _plan_calls(est, pix, plan_of, rec, setting):
    """Build the plan (recording its layer ranges), replay it as a graph, then run its steps one by one under the wrappers."""
    est._plans = {}
    rec.ranges = []
    with _recording(setting, rec):
        graph = est.predicted_depth(pix, use_graph=True).clone()
        plan = plan_of()
        torch.cuda.synchronize()
        rec.calls, rec.on = [], True
        try:
            for i, (fn, _, _) in enumerate(plan.steps):
                rec.step = i
                fn()
        finally:
            rec.on = False
        torch.cuda.synchronize()
    assert torch.equal(plan.out, graph), "step-wise != graph replay"                                  # 1.
    inside = {i for s, e in rec.ranges for i in range(s, e)}
    calls = [c for c in rec.calls if c["step"] not in inside]
    steps = collections.Counter(c["step"] for c in calls)
    assert all(n == 1 for n in steps.values()), "more than one wrapped call in one step"
    missing = collections.Counter(plan.steps[i][1] for i in range(len(plan.steps)) if i not in inside and i not in steps)
    assert not missing, f"steps outside the layers that no wrapped call checks: {dict(missing)}"     # 4.
    return calls, len(inside)


def _dpt_large(B, size):
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_oracle as do
    cfg = do.CFG_LARGE
    sd = {k: v.cuda() for k, v in do.synth_weights(cfg, 31).items()}
    est = DPTDepthEstimator.from_transformers(sd, cfg, preprocessor_config=None if size == 384 else {"size": size})
    pix = torch.randn(B, 3, size, size, generator=torch.Generator().manual_seed(2)).cuda()
    G = size // 16

    def run(rec, setting):
        calls, n_in = _plan_calls(est, pix, lambda: est._plan(B), rec, setting)
        hidden = [D.V(c["ins"]["x"].double()) for c in calls if c["name"] == "readout_rows_f16"]

        def walk(wk):
            D.dpt(wk, sd, cfg, hidden, (G, G))
        return calls, walk, n_in
    return run


def _dpt_hybrid(B, h, w):
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_hybrid_oracle as ho
    cfg = ho.CFG_HYBRID
    sd = {k: v.cuda() for k, v in ho.synth_weights(cfg, 31, last_bias=ho.REAL_LAST_BIAS).items()}
    est = DPTDepthEstimator.from_transformers(sd, cfg)
    pix = torch.randn(B, 3, h, w, generator=torch.Generator().manual_seed(2)).cuda()

    def run(rec, setting):
        calls, n_in = _plan_calls(est, pix, lambda: est._plan(B, h, w), rec, setting)
        hidden = [D.V(c["ins"]["x"].double()) for c in calls if c["name"] == "readout_rows_f16"]

        def walk(wk):
            D.hybrid(wk, sd, cfg, pix, est.cfg["kp"], lambda emb: hidden)
        return calls, walk, n_in
    return run


def _hint(N, h, w):
    from kandinsky2.model.unet import Text2ImUNet
    from oracle import controlnet_oracle as co
    from oracle import synth
    cfg = dict(co.CONFIG_2_2_HINT, model_channels=128, num_res_blocks=2, model_dim=256)   # test_gpu_unet.py's ControlNet UNet
    sd = synth.synth_state_dict(co.param_spec(cfg), seed=21)
    m = Text2ImUNet(model_dim=256, image_encoder_in_dim=1280, num_image_embs=32, pooling_type="from_model", in_channels=8,
                    model_channels=128, out_channels=8, num_res_blocks=2, attention_resolutions=(2, 4, 8),
                    channel_mult=(1, 2, 3, 4), use_fp16=True, num_head_channels=64, use_scale_shift_norm=True,
                    resblock_updown=True, cond_version="2.2", hint_channels=4)
    m.load_state_dict(sd, strict=True)
    m.to("cuda")
    m.finalize()
    sdc = {k: v.cuda() for k, v in sd.items() if k.startswith("add_embedding.input_hint_block.")}
    hint = torch.rand(N, 3, h, w, generator=torch.Generator().manual_seed(4)).cuda()

    def run(rec, setting):
        plain = m.hint_features(hint).clone()
        with _recording(setting, rec):
            rec.calls, rec.on = [], True
            try:
                got = m.hint_features(hint)
            finally:
                rec.on = False
            torch.cuda.synchronize()
        assert torch.equal(got, plain), "the recorded run differs from a plain run"

        def walk(wk):
            wk.hint(sdc, hint)
        return rec.calls, walk, 0
    return run


GEOMETRIES = {"dpt_large_384": lambda: _dpt_large(1, 384), "dpt_large_400_b2": lambda: _dpt_large(2, 400),
              "dpt_hybrid_384": lambda: _dpt_hybrid(1, 384, 384), "dpt_hybrid_208x336_b2": lambda: _dpt_hybrid(2, 208, 336),
              "hint_768_n2": lambda: _hint(2, 768, 768), "hint_360x536": lambda: _hint(1, 360, 536)}


# ------------------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------------------
def _same(got, want, what):
    assert got is not None and got.numel() == want.numel() and torch.equal(got.reshape(-1), want.to(got).reshape(-1)), what


def _wiring(calls, launches, name):
    """2.: each launch's input snapshots equal its producers' output snapshots (or the tensor the restatement builds)."""
    for i, (c, lau) in enumerate(zip(calls, launches)):
        for key, src in lau["reads"].items():
            what = f"{name}: launch {i} ({lau['label']}) does not read its producer's output as {key}"
            if c["name"] == "gn_finalize":   # reads partials: its statistics are restated from the producer's output
                continue
            if key == "srcs":
                assert len(c["ins"]["srcs"]) == len(src), what
                for t, j in zip(c["ins"]["srcs"], src):
                    _same(t, calls[j]["out"], what)
            elif isinstance(src, int):
                _same(c["ins"][key], calls[src]["out"], what)
            else:
                _same(c["ins"][key], src, what)


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_depth_blocks_float64(geometry):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    run = GEOMETRIES[geometry]()
    rec = _Rec()
    for setting in SETTINGS:
        calls, walk, n_in = run(rec, setting)
        wk = D.Walk(D.EXACT, snap=[c["out"].double() for c in calls], muts=setting == "default")
        walk(wk)
        names = [c["name"] for c in calls]
        ops = [l["op"] for l in wk.launches]
        assert len(names) == len(ops) and all(n in (o if isinstance(o, set) else {o}) for n, o in zip(names, ops)), \
            (geometry, [(n, o) for n, o in zip(names, ops) if n not in (o if isinstance(o, set) else {o})][:3],
             len(names), len(ops))                                                                    # 4.
        _wiring(calls, wk.launches, geometry)                                                         # 2.
        per, first_mut, ratio = collections.defaultdict(list), {}, 0.0
        for i, (c, lau) in enumerate(zip(calls, wk.launches)):
            got = c["out"]
            for label, ref, muts in lau["checks"]:
                if isinstance(ref, D.Stats):
                    w, m = ref.share(got)
                    ratio = max(ratio, ref.ratio.max().item())
                else:
                    w, m = D.share(got.reshape(ref.v.shape), ref)
                per[label].append((w, m))
                assert w <= 1.0, (geometry, setting, i, label, w)                                     # 3.
                for mut, v in muts.items():
                    r = D.share(v, ref)[0]
                    first_mut[mut] = max(first_mut.get(mut, (0.0, -1, "")), (r, i, label))
        print(f"{geometry} [{setting}]: {len(calls)} launches checked, {n_in} steps in the layer ranges (the tower test's)")
        print(f"  completeness: {dict(collections.Counter(names))}; no exempt kinds")
        for label, v in per.items():
            print(f"  {label}: worst {max(x[0] for x in v):.3f} of the bound, median "
                  f"{sorted(x[1] for x in v)[len(v) // 2]:.3f} ({len(v)} launches)")
        if ratio:
            print(f"  largest |mean| / std of a BiT GroupNorm group: {ratio:.3g}")
        for mut, (r, i, label) in first_mut.items():
            print(f"  mutation {mut} ({D.MUTATIONS[mut]}): {r:.3g} x the bound at launch {i} ({label})")
            assert r >= D.MIN_REJECT, (geometry, mut, r)
        del calls, wk
        torch.cuda.empty_cache()
    print(f"{geometry}: {time.time() - t0:.1f} s")
