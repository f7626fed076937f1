"""GPU: every UNet and MoVQ block as its launch plan runs it, against float64 restatements from the oracle's fp32 state dict,
fed the plan's own fp16 inputs and side inputs (FiLM rows, encoder K / V, zq), with the term-by-term bounds of
tests/plan_blocks_ref.py.

Harness: while a plan is built, _Plan._layer (UNet), _MovqPlan._res / _attn and every norm launch are wrapped to record each
block's inputs, output, norm outputs and [start, end) range in plan.steps.  The steps are then run one at a time, eagerly:
a block's inputs are cloned before its first step, each norm output after its step, the block's scratch intermediates and
output after its last step (`_tmp` buffers are reused by later blocks).  The step-wise output must equal the CUDA graph's bit
for bit, so the snapshots are of the computation the graph replays.  Stems, up / down convolutions and heads are the step
ranges between blocks.  What the block checks take as given is checked too: each block reads the previous block's output
(or the section's), each up-path skip is the output of its matching input block, and every FiLM row is restated from t_in and
xf_proj through the plan's time-embedding buffers (e0, e1, emb).

Every geometry runs under settings that force both sides of each plan decision: the autotuner off / forced to N tile 256,
two epilogue sets and split-K 2 where the library accepts them (the launches that ran two epilogue sets are counted); GroupNorm statistics folded into the apply (FOLD_MAX_RG
large) / from k2_gn_finalize (0); the forked side stream on / off; the MoVQ's fused attention on / off.  Step kinds are
counted to show each path ran.  Each block prints its worst share of the bound over its stages and the median share of its
output (run with -s); each wiring error of plan_blocks_ref.MUTATIONS prints its rejection share and how far it moves the
whole model's output against the end-to-end tolerances (UNet rel L2 2e-3, MoVQ 8e-3)."""
import collections
import contextlib
import time

import pytest
import torch
import torch.nn.functional as F

from tests import plan_blocks_ref as R

pytestmark = pytest.mark.gpu

SETTINGS = {
    "default": dict(tune="auto", fold=None, fork=True, fused=True),
    "untuned/finalize/serial/unfused": dict(tune="none", fold=0, fork=False, fused=False),
    "forced-tiles/fold/fork": dict(tune="forced", fold=1 << 30, fork=True, fused=True),
}
MIN_REJECT = 4.0
_FORCED = ((256, 1, 2, 2), (256, 1, 2, 1), (128, 1, 2, 1), (256, 1, 1, 2), (128, 1, 1, 2))


def _forced_tune(key, run, m_rows=0):
    """N tile 256, two epilogue sets and split-K 2 where the library takes them (info reports what it used)."""
    for cfg in _FORCED:
        info = [0] * 7
        try:
            run(cfg, info)
        except Exception:
            continue
        if info[0] == cfg[0] and info[2] == cfg[2]:
            return cfg
    return None


@contextlib.contextmanager
def _building(name, rec):
    """Plan construction under setting `name`, recording blocks, norm outputs and each conv step's split factor into rec."""
    from kandinsky2 import launch_plan as lp
    from kandinsky2 import ops
    from kandinsky2.model import unet as um
    from kandinsky2.vqgan import autoencoder as ae
    s = SETTINGS[name]
    mp = pytest.MonkeyPatch()
    o_layer, o_res, o_attn = um._Plan._layer, ae._MovqPlan._res, ae._MovqPlan._attn
    o_norm, o_sn, o_add, o_conv = lp.LaunchPlan._norm, ae._MovqPlan._sn, lp.LaunchPlan._add, ops.conv_gemm
    o_ts, o_lin = ops.timestep_embedding, ops.linear

    def blk(plan, kind, name, start, a, out):
        rec["blocks"].append(dict(kind=kind, name=name, start=start, end=len(plan.steps), a=a, out=out, b=None))
        return rec["blocks"][-1]

    def layer(self, p, layer, a, b):
        s0 = len(self.steps)
        o = o_layer(self, p, layer, a, b)
        blk(self, layer[0], p, s0, a, o).update(b=b, layer=layer)
        return o

    def movq(orig, kind):
        def f(self, x, zq, d):
            s0 = len(self.steps)
            o = orig(self, x, zq, d)
            names = {id(v): k for k, v in self.m._packed.items()}
            blk(self, kind, _MOVQ_NAMES.get(names[id(d)], names[id(d)] + "."), s0, x, o)
            return o
        return f

    def norm(self, a, b, gamma, beta, y, *args, **kw):
        o_norm(self, a, b, gamma, beta, y, *args, **kw)
        rec["norms"].append((len(self.steps), y))

    def sn(self, x, zq, n, act, y):
        o_sn(self, x, zq, n, act, y)
        rec["norms"].append((len(self.steps), y))

    def conv_gemm(*a, **k):
        out = o_conv(*a, **k)
        if k.get("info") is not None:
            rec["last"] = (list(k["info"]), k.get("cfg"))
        return out

    def add(self, fn, kind="misc", flops=0):
        rec["last"] = None
        o_add(self, fn, kind, flops)
        if rec["last"] is not None:
            info, cfg = rec["last"]
            rec["splits"].append(info[2])
            # k2_api.cu plan_conv / launch_conv_gemm: cfg[3] = 2 runs both consumer warpgroups' epilogues at N tiles 128 / 256
            rec["es2"] += bool(cfg and cfg[3] == 2 and info[0] in (128, 256))

    def chain_out(orig):
        """The forked conditioning branch's fp32 buffers (e0, e1, emb, film), in the order the plan writes them."""
        def f(*a, **k):
            out = orig(*a, **k)
            o = k.get("out")
            if o is not None and all(o is not c for c in rec["chain"]):
                rec["chain"].append(o)
            return out
        return f

    try:
        mp.setattr(um._Plan, "_layer", layer)
        mp.setattr(ae._MovqPlan, "_res", movq(o_res, "res"))
        mp.setattr(ae._MovqPlan, "_attn", movq(o_attn, "attn"))
        mp.setattr(lp.LaunchPlan, "_norm", norm)
        mp.setattr(ae._MovqPlan, "_sn", sn)
        mp.setattr(lp.LaunchPlan, "_add", add)
        mp.setattr(ops, "conv_gemm", conv_gemm)
        mp.setattr(ops, "timestep_embedding", chain_out(o_ts))
        mp.setattr(ops, "linear", chain_out(o_lin))
        if s["tune"] == "none":
            mp.setattr(lp, "tune", lambda key, run, m_rows=0: None)
        elif s["tune"] == "forced":
            mp.setattr(lp, "tune", _forced_tune)
        if s["fold"] is not None:
            mp.setattr(lp, "FOLD_MAX_RG", s["fold"])
        mp.setattr(lp, "FORK", s["fork"])
        mp.setattr(ae, "_FUSED_ATTN", s["fused"])
        yield
    finally:
        mp.undo()


_MOVQ_NAMES = {"mid1": "decoder.mid.block_1.", "mida": "decoder.mid.attn_1.", "mid2": "decoder.mid.block_2.",
               "e_mid1": "encoder.mid.block_1.", "e_mida": "encoder.mid.attn_1.", "e_mid2": "encoder.mid.block_2."}


def _new_rec():
    return dict(blocks=[], norms=[], splits=[], es2=0, chain=[], last=None)


def _scratch(plan, slot, *shape):
    return plan._scratch[(slot, torch.float16) + tuple(shape)]


def _stepwise(plan, rec, scratch_of):
    """Runs plan.steps once, one at a time, and returns per-block snapshots {a, b, out, norms: [...], <scratch slot>: ...}."""
    starts, ends, norm_at = {}, {}, {}
    for j, b in enumerate(rec["blocks"]):
        starts.setdefault(b["start"], []).append(j)
        ends.setdefault(b["end"], []).append(j)
    for n, y in rec["norms"]:
        norm_at.setdefault(n, []).append(y)
    snaps = [dict(norms=[]) for _ in rec["blocks"]]
    norm_snaps = {}
    torch.cuda.synchronize()
    for i, (fn, _, _) in enumerate(plan.steps):
        for j in starts.get(i, ()):
            torch.cuda.synchronize()
            b = rec["blocks"][j]
            snaps[j]["a"] = b["a"].clone()
            snaps[j]["b"] = b["b"].clone() if b["b"] is not None else None
        fn()
        if i + 1 in norm_at or i + 1 in ends:
            torch.cuda.synchronize()
        for y in norm_at.get(i + 1, ()):
            norm_snaps.setdefault(i + 1, []).append(y.clone())
        for j in ends.get(i + 1, ()):
            b = rec["blocks"][j]
            snaps[j]["out"] = b["out"].clone()
            for k, t in scratch_of(plan, b).items():
                snaps[j][k] = t.clone()
    torch.cuda.synchronize()
    for j, b in enumerate(rec["blocks"]):
        for n in sorted(norm_snaps):
            if b["start"] < n <= b["end"]:
                snaps[j]["norms"] += norm_snaps[n]
    return snaps


def _nchw(t, H=None, W=None):
    if t.dim() == 3:
        t = t.reshape(t.shape[0], H, W, t.shape[-1])
    return t.double().permute(0, 3, 1, 2)


def _counts(plan, rec):
    k = collections.Counter(kind for _, kind, _ in plan.steps)
    return dict(fold=k["gn_apply"] + k["sn_apply"] - k["gn_finalize"] - k["gn_stats"], gn_finalize=k["gn_finalize"],
                gn_stats=k["gn_stats"], split_k=sum(s > 1 for s in rec["splits"]), epilogue_sets_2=rec["es2"],
                attention=k["attention"],
                softmax=k["softmax"], join=k["join"])


def _report(what, worst, med, per=None):
    extra = " (" + " ".join(f"{k} {v:.2f}" for k, v in per.items()) + ")" if per else ""
    print(f"  {what}: worst {worst:.3f} of the bound, median {med:.3f}{extra}")
    assert worst <= 1.0, (what, per)


def _stage_check(run, got):
    """got {stage: NCHW float64 of the plan}; run(M, snap) the restatement.  -> (ref, snap V, worst, median, per stage)."""
    snap = {k: R.V(v, torch.zeros_like(v)) for k, v in got.items() if k != "out"}
    ref = run(R.EXACT, snap)
    worst, med, per = R.check_stages(got, ref)
    return ref, snap, worst, med, per


def _mutation(label, run, snap, ref, mut, e2e=None, tol=None):
    got = run(R.Mode(mut=mut), snap)
    w, _, _ = R.check_stages({k: v.v for k, v in got.items()}, ref)
    e = f", end to end rel L2 {e2e:.2e} against the {tol:g} tolerance" if e2e is not None else ""
    print(f"  mutation {mut} ({R.MUTATIONS[mut]}) at {label}: {w:.3g} x the bound{e}")
    assert w >= MIN_REJECT, (label, mut, w)


# ------------------------------------------------------------------------------------------------------------------------------
# UNet
# ------------------------------------------------------------------------------------------------------------------------------
def _unet_scratch(plan, b):
    N = plan.N
    Ho, Wo, C = b["out"].shape[1:]
    if b["kind"] == "res":
        out = dict(h2=_scratch(plan, "h2", N, Ho, Wo, C))
        if b["layer"][3] is not None:
            out["xres"] = _scratch(plan, "xres", N, Ho, Wo, b["layer"][1])
        return out
    T = Ho * Wo
    return dict(qkv=_scratch(plan, "qkv", N, T, 3 * C), att=_scratch(plan, "att", N, T, C))


def _unet_inputs(cfg, B, H, W, seed=11):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, H, W, generator=g).cuda()
    t = torch.tensor([981.0, 40.0] * (B // 2)).cuda()
    kw = dict(image_emb=torch.randn(B, cfg["image_encoder_in_dim"], generator=g).cuda())
    if cfg.get("cond", "2.1") == "2.1":
        kw.update(full_emb=torch.randn(B, 77, 1024, generator=g).cuda(), pooled_emb=torch.randn(B, 768, generator=g).cuda())
    if cfg.get("inpainting"):
        kw.update(inpaint_image=torch.randn(B, 4, H, W, generator=g).cuda(),
                  inpaint_mask=(torch.rand(B, 1, H, W, generator=g) > 0.5).float().cuda())
    return x, t, kw


def _unet_run(m, sd, cfg, setting, x, t, kw, idx, mutate=False):
    """Builds the plan under `setting`, checks graph == step-wise bit for bit and every block / section against float64 on
    images idx.  -> step-kind counts."""
    m._plans, m.cache = {}, None
    rec = _new_rec()
    with _building(setting, rec):
        y = m(x, t, **kw)
    plan = next(iter(m._plans.values()))
    torch.cuda.synchronize()
    snaps = _stepwise(plan, rec, _unet_scratch)
    assert torch.equal(plan.out, y), "step-wise run differs from the CUDA graph"
    counts = _counts(plan, rec)
    print(f"{setting}: {counts}")
    lay = R.film_layout(cfg)
    cond = m.cache
    sel = lambda t_: t_[idx]  # noqa: E731
    # side inputs: the encoder K / V of every attention layer
    for p, enc in plan.enc_kv.items():
        ref = R.unet_enc_kv(sd, p, cond["xf_out"][idx])
        _report(f"enc_kv {p}", *R.share(enc[idx].double().permute(0, 2, 1)[..., None], ref))
    # stem
    xs = plan.x_in
    if m._inpainting:
        xs = torch.cat([plan.x_in, plan.img_in * plan.mask_in, plan.mask_in], 1)
    _report("stem", *R.share(_nchw(sel(snaps[0]["a"])), R.unet_stem(sd, sel(xs))))
    # the forked conditioning branch: every FiLM row from t_in and xf_proj, split at its fp32 buffers
    e0, e1, emb, film_all = rec["chain"]
    assert film_all is plan.film
    got = {"e0": sel(e0).double(), "e1": sel(e1).double(), "emb": sel(emb).double(), "out": sel(plan.film).double()}
    run = lambda M, snap: R.film_chain(sd, lay, sel(plan.t_in), sel(plan.xf_proj), M, snap)  # noqa: E731
    ref, snapv, worst, med, per = _stage_check(run, got)
    _report("film chain", worst, med, per)
    if mutate:
        for mut in ("film_packed_neighbour", "emb_no_xf_proj", "film_no_silu_in"):
            _mutation("the FiLM chain", run, snapv, ref, mut)
    _check_wiring(rec["blocks"], snaps)
    done = set()
    for j, (b, sn) in enumerate(zip(rec["blocks"], snaps)):
        p, layer = b["name"], b["layer"]
        a = R.inp(sel(sn["a"]))
        bb = R.inp(sel(sn["b"])) if sn["b"] is not None else None
        Ho, Wo = sn["out"].shape[1:3]
        got = {k: _nchw(sel(v), Ho, Wo) for k, v in sn.items() if k not in ("a", "b", "norms")}
        if layer[0] == "res":
            ud = layer[3]
            got["h1s" if ud == "up" else "h1"] = _nchw(sel(sn["norms"][0]))
            got["h3"] = _nchw(sel(sn["norms"][1]))
            off, cout = lay[p]
            nb_off = lay[R.film_neighbour(lay, p)][0]
            film, film_nb = plan.film[idx, off:off + 2 * cout], plan.film[idx, nb_off:nb_off + 2 * cout]

            def run(M, snap, p=p, a=a, bb=bb, ud=ud, film=film, film_nb=film_nb):
                return R.unet_res(sd, p, a, bb, film_nb if M.mut == "film_neighbour" else film, ud, M, snap)
        else:
            got["xn"] = _nchw(sel(sn["norms"][0]))
            enc = plan.enc_kv[p][idx]
            run = lambda M, snap, p=p, a=a, enc=enc: R.unet_attn(sd, p, a, enc, M, snap)  # noqa: E731
        ref, snapv, worst, med, per = _stage_check(run, got)
        _report(f"{p} {layer[0]}{'/' + layer[3] if layer[0] == 'res' and layer[3] else ''}", worst, med, per)
        if mutate:
            muts = ["film_neighbour", "film_scale"] if layer[0] == "res" else ["no_enc"]
            if layer[0] == "res" and bb is not None:
                muts.append("gn_first_source")
            if layer[0] == "res" and layer[3] is not None:
                muts.append("res_unresampled")
            if layer[0] == "res" and layer[3] == "up":
                muts.append("up2_plain")
            for mut in muts:
                if mut in done:
                    continue
                done.add(mut)
                e2e = _unet_e2e(sd, cfg, x, t, kw, p, mut, lay)
                _mutation(p, run, snapv, ref, mut, e2e, 2e-3)
    if mutate:
        assert done == {"film_neighbour", "film_scale", "gn_first_source", "res_unresampled", "up2_plain", "no_enc"}, done
    # head: GroupNorm + SiLU + conv3x3 -> fp32 NCHW
    _report("head", *R.share(sel(plan.out).double(), R.unet_head(sd, R.inp(sel(snaps[-1]["out"])))))
    return counts


def _check_wiring(blocks, snaps):
    """What the per-block checks take as given: every block reads the previous block's output, and the up path's skip is the
    output of the matching input block (the stem's for the last), as unet_oracle.unet_forward pops them."""
    hs = [snaps[0]["a"]]
    for j, b in enumerate(blocks):
        if j:
            assert torch.equal(snaps[j]["a"], snaps[j - 1]["out"]), f"{b['name']} does not read {blocks[j - 1]['name']}"
        nxt = blocks[j + 1]["name"] if j + 1 < len(blocks) else ""
        if b["name"].startswith("input_blocks.") and not nxt.startswith(b["name"].rsplit(".", 2)[0] + "."):
            hs.append(snaps[j]["out"])
    for b, sn in zip(blocks, snaps):
        if b["name"].startswith("output_blocks.") and b["name"].endswith(".0."):
            assert sn["b"] is not None and torch.equal(sn["b"], hs.pop()), f"{b['name']} reads the wrong skip"
    assert not hs


def _unet_e2e(sd, cfg, x, t, kw, target, mut, lay):
    """Relative L2 change of the fp32 oracle's output when block `target` carries mutation `mut`."""
    from oracle import unet_oracle as uo
    table = {p: c0 for p, _, c0 in R.unet_block_table(cfg)}
    o_res, o_attn = uo._res, uo._attn
    M = R.Mode(bound=False, mut=None if mut == "film_neighbour" else mut)

    def res(xx, emb, sd_, p, ud):
        if p != target:
            return o_res(xx, emb, sd_, p, ud)
        q = R.film_neighbour(lay, p) if mut == "film_neighbour" else p
        film = F.linear(F.silu(emb.double()), sd_[q + "emb_layers.1.weight"].double(), sd_[q + "emb_layers.1.bias"].double())
        c0 = table[p]
        a = R.V(xx[:, :c0].double())
        b = R.V(xx[:, c0:].double()) if c0 < xx.shape[1] else None
        return R.unet_res(sd_, p, a, b, film, ud, M)["out"].v.to(xx.dtype)

    def attn(xx, xf, sd_, p, hc):
        if p != target:
            return o_attn(xx, xf, sd_, p, hc)
        enc = (F.conv1d(xf.double(), sd_[p + "encoder_kv.weight"].double(), sd_[p + "encoder_kv.bias"].double())
               .permute(0, 2, 1))
        return R.unet_attn(sd_, p, R.V(xx.double()), enc, M)["out"].v.to(xx.dtype)

    kwo = {k: v for k, v in kw.items()}
    with torch.no_grad():
        ref = uo.unet_forward(sd, cfg, x, t, **kwo)
        mp = pytest.MonkeyPatch()
        mp.setattr(uo, "_res", res)
        mp.setattr(uo, "_attn", attn)
        try:
            y = uo.unet_forward(sd, cfg, x, t, **kwo)
        finally:
            mp.undo()
    return ((y - ref).norm() / ref.norm()).item()


def _unet_model(cfg, seed=3):
    from oracle import synth
    from oracle import unet_oracle as uo
    from tests.test_gpu_unet import _build
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=seed)
    m = _build(cfg, sd)
    return m, {k: v.cuda() for k, v in sd.items()}


def _assert_both_sides(all_counts, what, fold=True, attention=False):
    """Both sides of each decision ran: folded statistics (UNet; the MoVQ always finalizes) and gn_finalize, split-K, the side
    stream forked and not, fused attention and softmax_rows."""
    un = all_counts["untuned/finalize/serial/unfused"]
    if fold:
        assert all_counts["default"]["fold"] > 0 and all_counts["forced-tiles/fold/fork"]["fold"] > 0, (what, all_counts)
    assert un["fold"] == 0 and un["gn_finalize"] > 0 and un["join"] == 0, (what, un)
    forced = all_counts["forced-tiles/fold/fork"]
    assert forced["split_k"] > 0 and forced["epilogue_sets_2"] > 0, (what, all_counts)
    assert all_counts["default"]["join"] > 0 or "movq" in what, (what, all_counts)
    if attention:
        assert all_counts["default"]["attention"] > 0 and un["softmax"] > 0 and un["attention"] == 0, (what, all_counts)


def _mid_cfg(kind):
    from oracle import unet_oracle as uo
    base = uo.CONFIG_2_2 if kind == "2.2" else uo.CONFIG_2_1
    return dict(base, model_channels=128, num_res_blocks=2, model_dim=256, inpainting=kind == "inpaint")


@pytest.mark.parametrize("kind", ["2.1", "2.2", "inpaint"])
def test_unet_mid_blocks(kind):
    """test_unet_mid_vs_oracle's geometry (128 channels, 2 ResBlocks per level, B = 2, 32 x 48): 2.1 head, 2.2 head and the
    9-channel inpainting stem, every block in every setting; the mutations on the 2.1 head."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    cfg = _mid_cfg(kind)
    m, sd = _unet_model(cfg)
    x, t, kw = _unet_inputs(cfg, 2, 32, 48)
    counts = {}
    for setting in SETTINGS:
        counts[setting] = _unet_run(m, sd, cfg, setting, x, t, kw, [0, 1], mutate=kind == "2.1" and setting == "default")
    _assert_both_sides(counts, f"unet {kind}")
    print(f"unet mid {kind}: {time.time() - t0:.1f} s")


def test_unet_full_size_blocks():
    """CONFIG_2_1 at cfg-2: N = 8 (4 conditional + 4 unconditional rows), 96 x 96 latents, every setting; float64 on one
    conditional and one unconditional image."""
    from oracle import unet_oracle as uo
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    cfg = dict(uo.CONFIG_2_1)
    m, sd = _unet_model(cfg, seed=4)
    x, t, kw = _unet_inputs(cfg, 8, 96, 96)
    counts = {s: _unet_run(m, sd, cfg, s, x, t, kw, [0, 4]) for s in SETTINGS}
    c = counts["default"]
    assert c["fold"] > 0 and c["gn_finalize"] > 0, c   # level 0 (72 row groups) finalizes, the rest fold
    _assert_both_sides(counts, "unet full size")
    print(f"unet full size: {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------------------------------------
# MoVQ
# ------------------------------------------------------------------------------------------------------------------------------
def _movq_scratch(plan, b):
    B = plan.B
    H, W, C = b["out"].shape[1:]
    if b["kind"] == "res":
        return dict(h=_scratch(plan, "h", B, H, W, C))
    return dict(qkv=_scratch(plan, "qkv", B, H * W, 3 * C), att=_scratch(plan, "att", B, H * W, C))


def _movq_model(dd, n_embed, seed):
    from kandinsky2.vqgan import MOVQ
    from oracle import movq_oracle as mo
    from oracle import synth
    sd = synth.synth_state_dict(mo.movq_param_spec(dd, 4, n_embed), seed=seed)
    m = MOVQ(dd, n_embed, 4)
    m.load_state_dict(sd)
    m.to("cuda")
    return m, {k: v.cuda() for k, v in sd.items()}


def _movq_run(m, sd, mode, setting, x, idx, mutate=False):
    """-> (step-kind counts, plan, per-block snapshots)."""
    m._plans = {}
    rec = _new_rec()
    with _building(setting, rec):
        y = (m.decode(x) if mode == "decode" else m.encode(x)).clone()
    plan = next(iter(m._plans.values()))
    torch.cuda.synchronize()
    snaps = _stepwise(plan, rec, _movq_scratch)
    assert torch.equal(plan.out, y), "step-wise run differs from the CUDA graph"
    counts = _counts(plan, rec)
    print(f"movq {mode} {setting}: {counts}")
    sel = lambda t_: t_[idx]  # noqa: E731
    zq = sel(plan.x_in) if mode == "decode" else None
    blocks = rec["blocks"]
    stem = R.movq_dec_stem(sd, zq) if mode == "decode" else R.movq_enc_stem(sd, sel(plan.x_in))
    _report("stem", *R.share(_nchw(sel(snaps[0]["a"])), stem))
    done = set()
    for j, (b, sn) in enumerate(zip(blocks, snaps)):
        p = b["name"]
        a = R.inp(sel(sn["a"]))
        H, W = sn["out"].shape[1:3]
        got = {k: _nchw(sel(v), H, W) for k, v in sn.items() if k not in ("a", "b", "norms")}
        got["hn"] = _nchw(sel(sn["norms"][0]))
        if b["kind"] == "res":
            got["hn2"] = _nchw(sel(sn["norms"][1]))
            run = lambda M, snap, p=p, a=a: R.movq_res(sd, p, a, zq, M, snap)  # noqa: E731
            muts = ["zq_offset"] if zq is not None else []
        else:
            fused = any(k == "attention" for _, k, _ in plan.steps[b["start"]:b["end"]])
            assert fused == (any(k == "softmax" for _, k, _ in plan.steps[b["start"]:b["end"]]) is False)
            run = lambda M, snap, p=p, a=a, fused=fused: R.movq_attn(sd, p, a, zq, fused, M, snap)  # noqa: E731
            muts = ["no_scale"]
        ref, snapv, worst, med, per = _stage_check(run, got)
        _report(f"{p} {b['kind']}{' fused' if b['kind'] == 'attn' and fused else ''}", worst, med, per)
        if mutate:
            for mut in muts:
                if mut not in done:
                    done.add(mut)
                    _mutation(p, run, snapv, ref, mut, _movq_e2e(sd, m.ddconfig, x, p, mut), 8e-3)
        if j + 1 < len(blocks) and blocks[j + 1]["start"] == b["end"]:
            assert torch.equal(snaps[j + 1]["a"], sn["out"]), f"{blocks[j + 1]['name']} does not read {p}"
        # the section up to the next block: an up conv (decode) or a down conv + subsample2(1, 1) (encode)
        if j + 1 < len(blocks) and blocks[j + 1]["start"] > b["end"]:
            lvl = p.split(".")[2] + "."
            pre = ("decoder.up." if mode == "decode" else "encoder.down.") + lvl
            fn = R.movq_upconv if mode == "decode" else R.movq_downconv
            ref = fn(sd, pre, R.inp(sel(sn["out"])))
            got_s = _nchw(sel(snaps[j + 1]["a"]))
            _report(f"{pre} {'up' if mode == 'decode' else 'down'}conv", *R.share(got_s, ref))
            if mutate and mode == "decode" and "up2_plain" not in done:
                done.add("up2_plain")
                w, _ = R.share(fn(sd, pre, R.inp(sel(sn["out"])), R.Mode(mut="up2_plain")).v, ref)
                e2e = _movq_up2_e2e(sd, m.ddconfig, x, pre)
                print(f"  mutation up2_plain ({R.MUTATIONS['up2_plain']}) at {pre}: {w:.3g} x the bound, end to end rel L2 "
                      f"{e2e:.2e} against the 0.008 tolerance")
                assert w >= MIN_REJECT, w
    last = R.inp(sel(snaps[-1]["out"]))
    head = R.movq_dec_head(sd, last, zq) if mode == "decode" else R.movq_enc_head(sd, last)
    _report("head", *R.share(sel(plan.out).double(), head))
    if mutate:
        assert done == {"zq_offset", "no_scale", "up2_plain"}, done
    return counts, plan, snaps


def _movq_e2e(sd, dd, z, target, mut):
    from oracle import movq_oracle as mo
    o_res, o_attn = mo._res, mo._attn
    M = R.Mode(bound=False, mut=mut)

    def res(x, zq, sd_, p):
        return R.movq_res(sd_, p, R.V(x.double()), zq, M)["out"].v.float() if p == target else o_res(x, zq, sd_, p)

    def attn(x, zq, sd_, p):
        return R.movq_attn(sd_, p, R.V(x.double()), zq, True, M)["out"].v.float() if p == target else o_attn(x, zq, sd_, p)

    with torch.no_grad():
        ref = mo.movq_decode(sd, dd, z)
        mp = pytest.MonkeyPatch()
        mp.setattr(mo, "_res", res)
        mp.setattr(mo, "_attn", attn)
        try:
            y = mo.movq_decode(sd, dd, z)
        finally:
            mp.undo()
    return ((y - ref).norm() / ref.norm()).item()


class _UpConvMutated:
    """torch.nn.functional for oracle.movq_oracle with one Upsample's conv2d replaced by the up2_plain restatement over the
    low-resolution input (every second pixel of the nearest-2x upsampling)."""
    def __init__(self, sd, pre):
        self.sd, self.pre, self.w = sd, pre, sd[pre + "upsample.conv.weight"]

    def __getattr__(self, name):
        return getattr(F, name)

    def conv2d(self, x, w, *a, **k):
        if w is not self.w:
            return F.conv2d(x, w, *a, **k)
        low = R.V(x[:, :, ::2, ::2].double())
        return R.movq_upconv(self.sd, self.pre, low, R.Mode(bound=False, mut="up2_plain")).v.to(x.dtype)


def _movq_up2_e2e(sd, dd, z, pre):
    from oracle import movq_oracle as mo
    with torch.no_grad():
        ref = mo.movq_decode(sd, dd, z)
        mp = pytest.MonkeyPatch()
        mp.setattr(mo, "F", _UpConvMutated(sd, pre))
        try:
            y = mo.movq_decode(sd, dd, z)
        finally:
            mp.undo()
    return ((y - ref).norm() / ref.norm()).item()


def _latent(B, h, seed):
    return torch.randn(B, 4, h, h, generator=torch.Generator().manual_seed(seed)).cuda()


def test_movq_decoder_blocks_32():
    """DDCONFIG_2_1 on a 32 x 32 latent, B = 2, every setting (C = 512 attention fused and unfused); the mutations."""
    from oracle import movq_oracle as mo
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    m, sd = _movq_model(dict(mo.DDCONFIG_2_1), 16384, seed=10)
    z = _latent(2, 32, 2)
    counts = {s: _movq_run(m, sd, "decode", s, z, [0, 1], mutate=s == "default")[0] for s in SETTINGS}
    _assert_both_sides(counts, "movq decode", fold=False, attention=True)
    print(f"movq decode 32: {time.time() - t0:.1f} s")


def test_movq_decoder_blocks_96():
    """DDCONFIG_2_1 on a 96 x 96 latent (768 x 768 image, T = 9216 attention tokens), B = 1, every setting."""
    from oracle import movq_oracle as mo
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    m, sd = _movq_model(dict(mo.DDCONFIG_2_1), 16384, seed=10)
    z = _latent(1, 96, 3)
    counts = {s: _movq_run(m, sd, "decode", s, z, [0])[0] for s in SETTINGS}
    _assert_both_sides(counts, "movq decode 96", fold=False, attention=True)
    print(f"movq decode 96: {time.time() - t0:.1f} s")


def test_movq_decoder_blocks_unfused_width():
    """A C = 256 attention config (ch 64, mult (1, 2, 4), 32 x 32 latent): the unfused route at its native width."""
    from oracle import movq_oracle as mo
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m, sd = _movq_model(dict(mo.DDCONFIG_2_1, ch=64, ch_mult=(1, 2, 4), resolution=128), 128, seed=9)
    z = _latent(2, 32, 1)
    for s in SETTINGS:
        c = _movq_run(m, sd, "decode", s, z, [0, 1])[0]
        assert c["softmax"] > 0 and c["attention"] == 0, c


def test_movq_encoder_blocks():
    """DDCONFIG_2_1's encoder on 256 x 256 images, B = 2, every setting: plain GroupNorm (gn_stats after each subsample2)."""
    from oracle import movq_oracle as mo
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.time()
    m, sd = _movq_model(dict(mo.DDCONFIG_2_1), 16384, seed=10)
    img = (torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(5)) * 2 - 1).cuda()
    counts = {s: _movq_run(m, sd, "encode", s, img, [0, 1])[0] for s in SETTINGS}
    assert all(c["gn_stats"] > 0 for c in counts.values()), counts
    _assert_both_sides(counts, "movq encode", fold=False, attention=True)
    print(f"movq encode: {time.time() - t0:.1f} s")


def test_movq_batch2_blocks_bit_identical_across_plans():
    """The full-size decode's open item: per-block snapshots of the batch-2 96 x 96 decode plan, then -- in the same process --
    a batch-1 MoVQ plan and a UNet plan are built and run, then the batch-2 plan runs step-wise again: every block must be
    bit-identical, and the first one that is not is named.  Run once."""
    from oracle import movq_oracle as mo
    m, _ = _movq_model(dict(mo.DDCONFIG_2_1), 16384, seed=10)
    z = _latent(2, 96, 2)
    rec = _new_rec()
    with _building("default", rec):
        m.decode(z)
    plan = m._plans[("decode", 2, 96, 96)]
    first = _stepwise(plan, rec, _movq_scratch)
    out1 = plan.out.clone()
    m.decode(z[:1])
    cfg = _mid_cfg("2.1")
    um, _ = _unet_model(cfg)
    x, t, kw = _unet_inputs(cfg, 2, 32, 48)
    um(x, t, **kw)
    torch.cuda.synchronize()
    second = _stepwise(plan, rec, _movq_scratch)
    for b, s1, s2 in zip(rec["blocks"], first, second):
        for k in s1:
            if k == "norms":
                same = all(torch.equal(u, v) for u, v in zip(s1[k], s2[k]))
            else:
                same = s1[k] is None or torch.equal(s1[k], s2[k])
            assert same, f"first block that differs after other plans ran: {b['name']} ({k})"
    assert torch.equal(plan.out, out1)
    plan.run(True)
    assert torch.equal(plan.out, out1), "graph replay differs from the step-wise run"
