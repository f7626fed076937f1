"""CPU, float64: the restatements and bounds of tests/depth_blocks_ref.py are neither too tight nor vacuous, on the tiny DPT
configs (dpt_oracle.TINY: the even 4 x 4 and the odd 5 x 5 patch grid), the tiny DPT-Hybrid (dpt_hybrid_oracle.CFG_TINY at
64 x 64 and 80 x 80) and the ControlNet hint stem.

  - the restatement composed end to end in exact arithmetic equals dpt_oracle.forward, dpt_hybrid_oracle.forward (the depth
    and the BiT stage maps) and controlnet_oracle.hint_features, all in float64 (the two DPT oracles round their outputs to
    fp32, so those are compared within 2^-24 relative), which ties the restatement to oracles pinned to transformers;
  - an emulated plan (fp16 weights, fp16 rounding at every storage point, float64 elsewhere) stays inside every bound;
  - every wiring error of MUTATIONS applies somewhere and falls outside the bound by at least MIN_REJECT.
Printed (run with -s): the worst and median share of the bound per launch kind, and each mutation's rejection share."""
import collections

import pytest
import torch

from tests import depth_blocks_ref as D
from tests import tower_layers_ref as R
from tests.plan_blocks_ref import V

PURE = D.Mode(bound=False)
EM = D.Mode(em=True)


def _pure(M):
    return not M.em and not M.bound


def _vit_hidden(sd, cfg, emb, keep, M):
    """The pre-LN DPT layers (tower_layers_ref.layer, fused attention) over emb (V [B, T, H]) -> the hidden states after the
    layers in keep."""
    H = cfg["hidden_size"]
    t = dict(heads=H // 64, hd=64, scale=0.125, eps=cfg.get("layer_norm_eps", 1e-12), act="gelu", post_ln=False,
             attn="fused", causal=False)
    out, h = [], V(emb.v)
    for i in range(max(keep) + 1):
        P = R.layer_params("dpt", sd, i)
        h = V(R.layer(P, P, h, t, M)["fc2"].v)
        if M.em:
            h = V(h.v.half().double())
        if i in keep:
            out.append(h)
    return out


def _dpt_case(name):
    from tests import dpt_oracle as do
    cfg, proc = {n: (c, p) for n, c, p in do.TINY}[name]
    sd = {k: v.double() for k, v in do.synth_weights(cfg, 11).items()}
    S, P = proc["size"]["height"], cfg["patch_size"]
    G = S // P
    pix = torch.randn(2, 3, S, S, generator=torch.Generator().manual_seed(3)).double()
    e = "dpt.embeddings."
    kp = (3 * P * P + 1 + 63) // 64 * 64
    pos = torch.cat([sd[e + "position_embeddings"][0, :1], resize_pos_embed_64(sd[e + "position_embeddings"][0], G)])

    def hidden(M):
        emb = R.patch_embed(R.patchify(pix, P, kp), sd[e + "patch_embeddings.projection.weight"], sd[e + "cls_token"], pos,
                            kp, PURE, bias=sd[e + "patch_embeddings.projection.bias"])
        hs = _vit_hidden(sd, cfg, emb, cfg["backbone_out_indices"], PURE)
        return hs if _pure(M) else [V(h.v.half().double()) for h in hs]

    def run(wk, M):
        return D.dpt(wk, sd, cfg, hidden(M), (G, G))[0]
    oracle = do.forward(sd, cfg, pix, dtype=torch.float64)
    return run, lambda out: _close32(out.v[:, 0], oracle, "dpt " + name)


def resize_pos_embed_64(pos, G):
    """DPTViTEmbeddings._resize_pos_embed in float64: the grid rows resized bilinearly (align_corners=False)."""
    g0 = int(round((pos.shape[0] - 1) ** 0.5))
    p = pos[1:].reshape(1, g0, g0, -1).permute(0, 3, 1, 2)
    p = torch.nn.functional.interpolate(p, size=(G, G), mode="bilinear")
    return p.permute(0, 2, 3, 1).reshape(G * G, -1)


def _hybrid_case(size):
    from tests import dpt_hybrid_oracle as ho
    cfg = ho.CFG_TINY
    sd = {k: v.double() for k, v in ho.synth_weights(cfg, 5).items()}
    pix = ho.sample_pixels(*size, seed=7, B=2).double()
    idx = cfg["backbone_out_indices"]

    em_hidden = []

    def run(wk, M):
        def vit(emb):   # the bound walk reads the emulated plan's hidden states, as the GPU test reads the plan's
            if M.bound:
                return em_hidden
            hs = _vit_hidden(sd, cfg, V(emb.v), idx[2:], EM if M.em else PURE)
            if M.em:
                em_hidden[:] = hs
            return hs
        (out, _), maps = D.hybrid(wk, sd, cfg, pix, _kp(cfg), vit)
        return out, maps
    oracle, omaps = ho.forward(sd, cfg, pix, dtype=torch.float64, with_maps=True)

    def tie(res):
        out, maps = res
        _close32(out.v[:, 0], oracle, f"hybrid {size}")
        for (m, _), om in zip(maps, omaps):
            _close32(m.v.permute(0, 3, 1, 2), om, f"hybrid {size} BiT map")
    return run, tie


def _kp(cfg):
    from kandinsky2.model.depth import dpt_hybrid_config
    return dpt_hybrid_config(cfg)["kp"]


def _hint_case():
    from oracle import controlnet_oracle as co
    from oracle import synth
    sd = {k: v.double() for k, v in synth.synth_state_dict(co.hint_param_spec(), seed=21).items()}
    hint = torch.rand(2, 3, 64, 48, generator=torch.Generator().manual_seed(4)).double()
    ref = co.hint_features(sd, hint)

    def tie(out):
        rel = ((out.v - ref).norm() / ref.norm()).item()
        assert rel < 1e-10, ("hint stem", rel)
    return (lambda wk, M: wk.hint(sd, hint)[0]), tie


def _close32(got, oracle, what):
    """got float64 vs an oracle evaluated in float64 and returned rounded to fp32."""
    err = (got - oracle.double()).abs()
    tol = 2.0 ** -24 * oracle.double().abs() + 1e-10 * oracle.double().abs().max()
    assert (err <= tol).all(), (what, (err / tol).max().item())


CASES = {"dpt_even": lambda: _dpt_case("even"), "dpt_odd": lambda: _dpt_case("odd"),
         "hybrid_64": lambda: _hybrid_case((64, 64)), "hybrid_80": lambda: _hybrid_case((80, 80)), "hint": _hint_case}
_REJECT = collections.defaultdict(float)


@pytest.mark.parametrize("case", list(CASES))
def test_restatement_matches_oracle_and_emulation_within_bound(case):
    torch.manual_seed(0)
    run, tie = CASES[case]()
    tie(run(D.Walk(PURE), PURE))                        # exact composition == the oracle
    em = D.Walk(EM)
    run(em, EM)                                         # the emulated plan
    snap = [v.v.float().double() if isinstance(v, D.Stats) else v.v for v in em.vals]
    wk = D.Walk(D.EXACT, snap=snap)
    run(wk, D.EXACT)
    assert [l["op"] for l in wk.launches] == [l["op"] for l in em.launches]
    per = collections.defaultdict(list)
    for lau, got in zip(wk.launches, snap):
        for label, ref, muts in lau["checks"]:
            w, m = ref.share(got) if isinstance(ref, D.Stats) else D.share(got, ref)
            per[label].append((w, m))
            assert w <= 1.0, (case, label, w)
            for mut, v in muts.items():
                r = D.share(v, ref)[0]
                _REJECT[mut] = max(_REJECT[mut], r)
    print(f"{case}:")
    for label, v in per.items():
        print(f"  {label}: worst {max(x[0] for x in v):.3f} of the bound, median {sorted(x[1] for x in v)[len(v) // 2]:.3f}")


def test_every_mutation_is_rejected():
    """Runs after the cases above (module order); every MUTATIONS entry applied somewhere, each at >= MIN_REJECT."""
    if len(_REJECT) < len(D.MUTATIONS):
        for case in CASES:
            test_restatement_matches_oracle_and_emulation_within_bound(case)
    for mut, what in D.MUTATIONS.items():
        print(f"  mutation {mut} ({what}): {_REJECT[mut]:.3g} x the bound")
        assert _REJECT[mut] >= D.MIN_REJECT, (mut, _REJECT[mut])
