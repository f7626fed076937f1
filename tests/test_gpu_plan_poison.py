"""GPU: launch plans built over NaN-poisoned buffers.

Every buffer a LaunchPlan allocates (`_new`, `_tmp`) starts filled with NaN here, and so does the shared split-K workspace and
the shared GroupNorm-statistics scratch (except its first 1024 words: the self-resetting arrival counters must be zero).  A plan
whose kernels read only what an earlier launch of the same plan wrote computes exactly what it computes over fresh buffers:
the outputs must be finite and bit-identical to an unpoisoned build of the same plan, eagerly and as a CUDA graph.  A read of an
uninitialised byte -- a partial-statistics buffer read past what its producer wrote, a stale `_parts` entry, a kernel reading
the gap columns of a row-strided view -- turns into NaN or a changed bit, on the first run and independent of allocator state.

Each case then builds a second, poisoned plan for another batch size and replays the first plan's graph once: building a plan
must not disturb a plan that already exists (the shared workspaces are the only state they have in common)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

NAN16 = 0x7E00        # fp16 quiet NaN
NAN32 = 0x7FC00000    # fp32 quiet NaN
GN_COUNTERS = 1024    # words of ops._gn_scratch that hold the gn_stats arrival counters (k2b200.h: zeroed, self-resetting)


def _fill_nan_(t):
    if t.dtype == torch.float16:
        t.view(torch.int16).fill_(NAN16)
    elif t.dtype == torch.float32:
        t.view(torch.int32).fill_(NAN32)
    elif t.dtype == torch.uint8 and t.numel() % 4 == 0:
        t.view(torch.int32).fill_(NAN32)
    else:
        t.fill_(0xFF if t.dtype == torch.uint8 else -1)
    return t


class _Poison:
    """Switchable NaN fill of every buffer a LaunchPlan creates, plus the process-wide workspaces while switched on."""

    def __init__(self, monkeypatch):
        from kandinsky2.launch_plan import LaunchPlan
        self.on = False
        new, tmp = LaunchPlan._new, LaunchPlan._tmp
        poison = self

        def _new(plan, *shape, dtype=torch.float16):
            t = new(plan, *shape, dtype=dtype)
            return _fill_nan_(t) if poison.on else t

        def _tmp(plan, slot, *shape, dtype=torch.float16):
            fresh = ((slot, dtype) + tuple(shape)) not in plan._scratch
            t = tmp(plan, slot, *shape, dtype=dtype)
            return _fill_nan_(t) if poison.on and fresh else t

        monkeypatch.setattr(LaunchPlan, "_new", _new)
        monkeypatch.setattr(LaunchPlan, "_tmp", _tmp)

    def workspaces(self):
        from kandinsky2 import ops
        dev = torch.device("cuda", torch.cuda.current_device())
        ws = ops._workspace(dev)
        ops._scratch(dev, 0)
        return ws, ops._gn_scratch[(dev.index,)]

    def __enter__(self):
        ws, gs = self.workspaces()
        _fill_nan_(ws)
        _fill_nan_(gs[GN_COUNTERS:])
        self.on = True
        return self

    def __exit__(self, *exc):
        self.on = False
        ws, gs = self.workspaces()
        torch.cuda.synchronize()
        ws.zero_()
        gs.zero_()
        return False


@pytest.fixture
def poison(monkeypatch):
    p = _Poison(monkeypatch)
    yield p
    p.on = False
    torch.cuda.synchronize()


def _same(a, b, what):
    assert torch.isfinite(a).all(), f"{what}: {int((~torch.isfinite(a)).sum())} non-finite outputs of {a.numel()}"
    assert torch.equal(a, b), f"{what}: max abs difference {(a - b).abs().max().item():.3e}"


def _check_plan(poison, run, other, drop_plans):
    """run(graph) -> output of the model's plan for the primary geometry (built on first use); other() builds and runs a plan
    for a second batch size; drop_plans() forgets the model's plans (the tuning cache stays, so a rebuild takes the same
    launch configurations)."""
    ref_eager = run(False)
    ref_graph = run(True)
    assert torch.equal(ref_eager, ref_graph)
    drop_plans()
    with poison:
        _same(run(False), ref_eager, "poisoned plan, eager")
        _same(run(True), ref_eager, "poisoned plan, graph")
        other()
        _same(run(True), ref_eager, "replay after building a plan for another batch size")
    drop_plans()


def _movq(dd, n_embed, seed):
    from kandinsky2.vqgan import MOVQ
    from oracle import movq_oracle as mo, synth
    sd = synth.synth_state_dict(mo.movq_param_spec(dd, 4, n_embed), seed=seed)
    m = MOVQ(dd, n_embed, 4)
    m.load_state_dict(sd)
    return m.to("cuda")


def _movq_case(m, fn, x, x_other):
    def run(graph):
        m.use_cuda_graph = graph
        return getattr(m, fn)(x)

    def drop():
        m._plans = {}

    return run, (lambda: getattr(m, fn)(x_other)), drop


def _golden_movq():
    fx = torch.load(os.path.join(GOLD, "movq_tiny.pt"), weights_only=False)
    return fx, _movq(fx["dd"], fx["n_embed"], fx["weight_seed"])


def test_movq_decode_tiny_poisoned(poison):
    """Golden tiny decoder (C = 64 attention: q k^T and P v as batched GEMMs around softmax_rows), batch 2, then batch 3."""
    fx, m = _golden_movq()
    z = fx["z"].cuda()
    _check_plan(poison, *_movq_case(m, "decode", z, torch.cat([z, z[:1]])))


def test_movq_encode_tiny_poisoned(poison):
    """Golden tiny encoder (Downsample = stride-1 conv + subsample2), batch 2, then batch 1."""
    fx, m = _golden_movq()
    img = fx["image"].cuda()
    _check_plan(poison, *_movq_case(m, "encode", img, img[1:]))


@pytest.mark.parametrize("name,dd,hw", [
    ("mid", dict(ch=64, ch_mult=(1, 2, 4), resolution=128), 32),           # test_movq_decode_mid_vs_oracle: C = 256, T = 1024
    ("fused512", dict(ch=128, ch_mult=(1, 4), resolution=64, attn_resolutions=()), 16),  # C = 512: k2_attention_d512, T = 256
])
def test_movq_decode_poisoned(poison, name, dd, hw):
    from oracle import movq_oracle as mo
    m = _movq(dict(mo.DDCONFIG_2_1, **dd), 128, 9)
    z = torch.randn(2, 4, hw, hw, generator=torch.Generator().manual_seed(1)).cuda()
    _check_plan(poison, *_movq_case(m, "decode", z, z[1:]))


@pytest.mark.parametrize("variant", ["2.1", "2.2", "inpaint"])
def test_unet_tiny_poisoned(poison, variant):
    """Tiny UNet (every layer kind: forked FiLM branch, up / down ResBlocks, attention with encoder tokens, skip concat), batch
    2, then batch 3."""
    from oracle import synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    if variant == "2.2":
        cfg = dict(uo.CONFIG_TINY, cond="2.2")
        g = torch.Generator().manual_seed(5)
        inp = dict(x=torch.randn(2, 4, 16, 16, generator=g), t=torch.tensor([981.0, 40.0]),
                   image_emb=torch.randn(2, cfg["image_encoder_in_dim"], generator=g))
        seed = 5
    else:
        fx = torch.load(os.path.join(GOLD, "unet_tiny.pt" if variant == "2.1" else "unet_tiny_inpaint.pt"))
        cfg, inp, seed = fx["cfg"], fx["inputs"], fx["weight_seed"]
    m = _build(cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=seed))
    inp = {k: v.cuda() for k, v in inp.items()}
    other = {k: torch.cat([v, v[:1]]) for k, v in inp.items()}

    def call(d):
        m.del_cache()   # the conditioning cache is per batch (reference behaviour); recomputing it is deterministic
        return m(d["x"], d["t"], **{k: v for k, v in d.items() if k not in ("x", "t")})

    def run(graph):
        m.use_cuda_graph = graph
        return call(inp)

    def drop():
        m._plans = {}

    _check_plan(poison, run, lambda: call(other), drop)
