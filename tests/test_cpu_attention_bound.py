"""CPU: the fused attention kernels' allowance (tests/attention_ref.py) is neither vacuous nor too tight.

Both kernel recipes are emulated in float32 on CPU tensors:
  flash   flash_attention_kernel (head widths 104 / 512): 16-key blocks, the score scaled (s c) and then max-subtracted in
          two roundings;
  d64     attention_d64_kernel: 128-key blocks, encoder keys in blocks of their own before the spatial keys, ex2(fmaf(s, c,
          -m)) with one rounding.
Both keep a running maximum, rescale l and O by alpha = 2^(m_old - m_new), sum l from the unrounded weights, round P to fp16
before P V and O / l once to fp16.  Each emulation must stay inside the allowance; each mutant -- a plausible kernel defect --
must leave it somewhere.  Inputs plant dominant keys (first and last key of a block, T - 1, the last encoder key) so that a
defect touching one key is visible."""
import math

import pytest
import torch

from tests.attention_ref import check, ref_attention
from tests.test_gpu_prior_kernels import _ulp16

LOG2E = 1.4426950408889634
MUTANTS = ("l_not_rescaled", "last_key_dropped", "tail_scored_zero", "scale_fp16", "halves_swapped")


def _f32(x):
    return torch.tensor(x, dtype=torch.float32)


def _emulate(q, k, v, scale, recipe, segments, mutant=None):
    """q [T, D], k / v [Tkv, D] fp16 (one head) -> fp16 [T, D] as the kernel computes it.  segments: key counts of the
    sources that start their own blocks (d64: [Tc, T]; flash: [Tkv])."""
    bkv = 16 if recipe == "flash" else 128
    sc = _f32(scale) if mutant != "scale_fp16" else torch.tensor(scale, dtype=torch.float16).float()
    c = sc * _f32(LOG2E)
    qf, kf, vf = q.float(), k.float(), v.float()
    T, D = qf.shape
    m = torch.full((T,), -math.inf)
    l = torch.zeros(T)
    o = torch.zeros(T, vf.shape[1])
    start = 0
    for n in segments:
        for j0 in range(0, n, bkv):
            valid = min(bkv, n - j0)
            kb = torch.zeros(bkv, D)
            vb = torch.zeros(bkv, vf.shape[1])
            kb[:valid] = kf[start + j0:start + j0 + valid]     # rows past the source's end arrive zero-filled
            vb[:valid] = vf[start + j0:start + j0 + valid]
            s = qf @ kb.T
            keep = valid - 1 if mutant == "last_key_dropped" and valid < bkv else valid
            if mutant != "tail_scored_zero":
                s[:, keep:] = -math.inf
            if recipe == "flash":
                s = s * c
                m_new = torch.maximum(m, s.amax(1))
                p = torch.exp2(s - m_new[:, None])
            else:
                m_new = torch.maximum(m, s.amax(1) * c)
                p = torch.exp2((s.double() * c.double() - m_new.double()[:, None]).float())   # fmaf: one rounding
            alpha = torch.exp2(m - m_new)
            m = m_new
            l = (l if mutant == "l_not_rescaled" else l * alpha) + p.sum(1)
            o = o * alpha[:, None] + p.half().float() @ vb
        start += n
    out = (o * (1.0 / l)[:, None]).half()
    if mutant == "halves_swapped":
        out = torch.cat([out[:, 256:], out[:, :256]], 1)
    return out


def _inputs(T, Tc, D, std, seed, bkv):
    """fp16 q [T, D], k / v [Tc + T, D]: keys are the Tc encoder keys then the T spatial keys.  V's channel halves are drawn
    differently (means +-1, scales 1 and 2), so an exchange of the two 256-channel halves shows.  Query rows 0, 1, ... each
    get one dominant key (score 24 above its copy's own scale) at the first and last key of a block, the last encoder key
    and the last key: the row's maximum then sits at that key, and for the last key it arrives in the last block."""
    g = torch.Generator().manual_seed(seed)
    Tkv = Tc + T
    q = torch.randn(T, D, generator=g) * std
    k = torch.randn(Tkv, D, generator=g) * std
    v = torch.randn(Tkv, D, generator=g)
    v[:, :D // 2] += 1.0
    v[:, D // 2:] = 2.0 * v[:, D // 2:] - 1.0
    planted = {Tkv - 1, 0, min(bkv - 1, Tkv - 1)}
    if Tc:
        planted |= {Tc - 1, Tc, Tc + min(bkv - 1, T - 1)}
    mid = (Tkv // 2) // bkv * bkv
    planted |= {mid, max(mid - 1, 0)}
    planted = sorted(planted)
    for r, key in enumerate(planted[:T]):
        q[r] = k[key] * (24.0 / (k[key].norm() ** 2 * D ** -0.5))
    return q.half(), k.half(), v.half(), planted


def _check(q, k, v, out, scale, what):
    ref, allow = ref_attention(q[:, None], k[:, None], v[:, None], scale)
    return check(out[:, None], ref, allow, what)


def _share(q, k, v, out, scale):
    """Largest share of the bound (> 1: outside it)."""
    ref, allow = ref_attention(q[:, None], k[:, None], v[:, None], scale)
    return ((out[:, None].double() - ref).abs() / (_ulp16(ref) + allow)).max().item()


_CASES = [   # (recipe, D, T, Tc)
    ("flash", 512, 100, 0), ("flash", 512, 1000, 0), ("flash", 512, 1024, 0), ("flash", 64, 301, 0),
    ("d64", 64, 300, 87), ("d64", 64, 1000, 32), ("d64", 64, 129, 200), ("d64", 512, 1000, 0),
]


@pytest.mark.parametrize("std", [1.0, 2.2])
@pytest.mark.parametrize("recipe,D,T,Tc", _CASES)
def test_emulated_recipe_inside_allowance(recipe, D, T, Tc, std):
    """std 2.2: scores up to about +-60 besides the planted keys."""
    q, k, v, _ = _inputs(T, Tc, D, std, seed=T + Tc + D, bkv=16 if recipe == "flash" else 128)
    scale = D ** -0.5
    segs = [Tc, T] if recipe == "d64" and Tc else [Tc + T]
    out = _emulate(q, k, v, scale, recipe, segs)
    assert torch.isfinite(out).all()
    ulps, share = _check(q, k, v, out, scale, (recipe, D, T, Tc, std))
    print(f"{recipe} D={D} T={T} Tc={Tc} std={std}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


def _mutant_cases():
    cases = []
    for recipe, D, T, Tc in _CASES:
        for mut in MUTANTS:
            if mut == "scale_fp16":
                continue     # test_scale_rounded_to_fp16_breaks_allowance
            if mut == "halves_swapped" and (recipe, D) != ("flash", 512):
                continue     # only the head width 512 splits its output channels over two CTAs
            if mut in ("last_key_dropped", "tail_scored_zero") and all(n % (16 if recipe == "flash" else 128) == 0
                                                                      for n in ([Tc, T] if Tc else [T])):
                continue     # no partial block
            cases.append((recipe, D, T, Tc, mut))
    return cases


@pytest.mark.parametrize("recipe,D,T,Tc,mutant", _mutant_cases())
def test_mutant_breaks_allowance(recipe, D, T, Tc, mutant):
    """std 1: a tail key scored 0 adds 2^-m to l, visible where the row maximum m is small."""
    q, k, v, _ = _inputs(T, Tc, D, 1.0, seed=T + Tc + D, bkv=16 if recipe == "flash" else 128)
    scale = D ** -0.5
    segs = [Tc, T] if recipe == "d64" and Tc else [Tc + T]
    share = _share(q, k, v, _emulate(q, k, v, scale, recipe, segs, mutant), scale)
    print(f"{recipe} D={D} T={T} Tc={Tc} {mutant}: {share:.1f} of the bound")
    assert share > 1.0, (mutant, share)


def test_scale_rounded_to_fp16_breaks_allowance():
    """A scale rounded to fp16 multiplies every score by 1 + e, which moves a weight by e times its score's distance from the
    row's weighted mean: only a weight far below the maximum that still carries the output shows it.  At head width 104,
    fp16(104^-0.5) is 2^-11.9 off; one query over two keys, scores 12.55 and 7.6 lower (weight just below 2^-11, values 0
    and 1), puts the mutant at about 1.7 of the bound.  At width 512, fp16(512^-0.5) is 2^-13.2 off: no row the allowance
    admits moves by more than its 2^-11 for P's own fp16 rounding, so a per-element bound cannot see this defect there."""
    D, scale = 104, 104 ** -0.5
    q = torch.zeros(2, D)
    k = torch.zeros(2, D)
    v = torch.zeros(2, D)
    q[0, 0], k[0, 0] = 8.0, 16.0
    s_a = 8.0 * 16.0 * scale
    s_b = s_a - math.log((1 - 0.99 * 2.0 ** -11) / (0.99 * 2.0 ** -11))      # p_b = 0.99 * 2^-11
    k[1, 0] = s_b / (8.0 * scale)
    v[1] = 1.0
    q, k, v = q.half(), k.half(), v.half()
    e = (torch.tensor(scale, dtype=torch.float16).double().item() - scale) / scale
    assert 2.0 ** -12 < e < 2.0 ** -11.5
    inside = _share(q, k, v, _emulate(q, k, v, scale, "flash", [2]), scale)
    share = _share(q, k, v, _emulate(q, k, v, scale, "flash", [2], "scale_fp16"), scale)
    print(f"flash D=104 scale rounded to fp16: {share:.2f} of the bound (the recipe: {inside:.2f})")
    assert inside <= 1.0 < share, (inside, share)


def test_every_mutant_is_exercised():
    assert {c[-1] for c in _mutant_cases()} | {"scale_fp16"} == set(MUTANTS)
    # the partial-block mutants reach the encoder tail of the d64 recipe
    assert ("d64", 64, 300, 87, "last_key_dropped") in _mutant_cases()
