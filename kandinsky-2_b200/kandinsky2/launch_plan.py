"""Static launch plans: a forward pass at a fixed geometry as a list of C-ABI launches over pre-allocated buffers, built once by
running it eagerly (so data-dependent decisions -- did a conv emit GroupNorm partials? which tile shape is fastest? -- are
known when the next launch is recorded) and then replayed eagerly or as ONE CUDA graph.  Shared by the UNet
(kandinsky2/model/unet.py) and the MoVQ encoder / decoder (kandinsky2/vqgan/autoencoder.py)."""
import gc
import os

import torch

from . import ops

# GroupNorm statistics are folded inside k2_gn_apply_fold when an image has at most this many partial row groups per source.
# The per-block fold costs L2 latency x row groups; a separate k2_gn_finalize launch costs one more launch per GroupNorm, so the
# fold pays where an image has few row groups (UNet levels 1-3, up to 18) and not at level 0 (72).  The threshold has not been
# re-measured on the H100.
FOLD_MAX_RG = int(os.environ.get("K2_GN_FOLD_MAX_RG", "18"))
TUNE = os.environ.get("K2_AUTOTUNE", "1") != "0"
FORK = os.environ.get("K2_FORK", "1") != "0"
# Layers with at most this many output rows (UNet levels 2-3: 4608 / 1152 rows at cfg-2) also try split-K factors 2..4: their
# tile counts leave a large part of the machine idle in the configuration the cycle model picks.  A K split changes the fp32
# summation order: deterministic per configuration, not bit-identical across configurations (the choice is cached per process
# and shape).
TUNE_SMALL_M = int(os.environ.get("K2_TUNE_SMALL_M", "8192"))
_tune_cache = {}


def tune(key, run, m_rows=0):
    """Launch configuration of one conv / GEMM layer shape: (N tile, pair mode, splits, epilogue warp sets = 1) for
    k2_conv_gemm_cfg, picked by timing candidates with CUDA events on the current stream: N tiles (bit-identical results) for
    layers of more than 64 output channels, plus split-K variants for layers of at most TUNE_SMALL_M output rows
    (m_rows; see above).  Cached per shape and device; None = the library's own choice.  key = (kind, Cout, ...); run(cfg, info)
    must enqueue the launch and report the configuration the library actually used in info."""
    if not TUNE:
        return None
    key = (torch.cuda.current_device(), TUNE_SMALL_M) + key
    if key in _tune_cache:
        return _tune_cache[key]
    info = [0] * 7
    run(None, info)
    bn0, splits = info[0], info[2]
    cout = key[3]
    best = None
    if cout > 64:
        bns = [bn0] if splits > 1 else [bn for bn in (128, 192, 256) if bn - 64 < cout or bn == bn0]
        cands = [(bn0, 0, splits, 1)] + [(bn, 0, splits, 1) for bn in bns if bn != bn0]
        if 0 < m_rows <= TUNE_SMALL_M and splits == 1:
            for bn in (128, 192, 256):
                if bn - 64 >= cout:
                    continue
                for sp in (2, 3, 4):
                    probe = [0] * 7
                    try:
                        run((bn, 1, sp, 1), probe)
                    except Exception:
                        continue
                    if probe[0] == bn and probe[2] == sp:  # else: the library refused
                        cands.append((bn, 1, sp, 1))

        def timed(cfg, reps=6):
            run(cfg)
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
            evs[0].record()
            for i in range(reps):
                run(cfg)
                evs[i + 1].record()
            torch.cuda.synchronize()
            return min(evs[i].elapsed_time(evs[i + 1]) for i in range(reps))

        t0 = tb = timed(cands[0])
        for cfg in cands[1:]:
            t = timed(cfg)
            if t < tb and t < 0.97 * t0:  # a candidate must beat the cycle model's choice by > 3 % ...
                t = max(t, timed(cfg))    # ... twice (event timing of a ~20 us launch is noisy)
                if t < tb and t < 0.97 * t0:
                    best, tb = cfg, t
    _tune_cache[key] = best
    return best


class LaunchPlan:
    def __init__(self, dev, nb):
        self.dev = dev
        self.NB = nb          # images per launch (GroupNorm statistics are per image)
        self._parts = {}      # tensor data_ptr -> (partial buffer, row groups per image) written by the producing conv
        self._scratch = {}
        self.steps = []
        self.graph = None
        self._side_stream = None   # forked branch of the launch DAG (see _side)
        self._side_open = False
        self._serial = False       # profile passes run the side branch in line so that every launch is timed on one stream

    # buffers -----------------------------------------------------------------------------------
    def _tmp(self, slot, *shape, dtype=torch.float16):
        """Scratch reused by every block that asks for the same (slot, shape): all launches are stream-ordered
        and a block's temporaries are dead when the next block starts."""
        key = (slot, dtype) + tuple(shape)
        if key not in self._scratch:
            self._scratch[key] = torch.empty(*shape, device=self.dev, dtype=dtype)
        return self._scratch[key]

    def _new(self, *shape, dtype=torch.float16):
        return torch.empty(*shape, device=self.dev, dtype=dtype)

    # recording ---------------------------------------------------------------------------------
    def _add(self, fn, kind="misc", flops=0):
        """Record a launch AND run it once now (build = eager trace)."""
        fn()
        self.steps.append((fn, kind, flops))

    # A second stream for launches that are off the critical path (the step's time / FiLM linears next to the stem conv, the
    # up ResBlocks' skip upsampling next to norm -> conv): _side() forks after the launches recorded so far, _join() makes
    # everything recorded afterwards wait for the branch.  Under graph capture the branch becomes a parallel chain of the
    # CUDA graph.  FORK = os.environ K2_FORK (default on).
    def _side(self, fn, kind="misc", flops=0):
        if not FORK:
            return self._add(fn, kind, flops)
        first = not self._side_open
        self._side_open = True

        def step():
            if self._serial:
                return fn()
            if self._side_stream is None:
                self._side_stream = torch.cuda.Stream(device=self.dev)
            if first:
                ev = torch.cuda.Event()
                ev.record()
                self._side_stream.wait_event(ev)
            with torch.cuda.stream(self._side_stream):
                fn()
        self._add(step, kind, flops)

    def _join(self):
        if not self._side_open:
            return
        self._side_open = False

        def step():
            if self._serial:
                return
            ev = torch.cuda.Event()
            ev.record(self._side_stream)
            torch.cuda.current_stream().wait_event(ev)
        self._add(step, "join", 0)

    def _conv(self, srcs, w, cout, out, flops, bias=None, residual=None, want_stats=True, part_slot=None, out_mode=0,
              geom=None, w_batch_stride=0, w_map=None, n_slabs=0, kind="conv_gemm"):
        """conv_gemm step; with want_stats the epilogue also writes GroupNorm partial statistics of `out` (when the
        launch geometry allows it: k2b200.h), remembered in self._parts for the consumer's norm.  The launch
        configuration (N tile, epilogue warp sets) is timed once per distinct layer shape (tune) and baked in."""
        part = None
        if want_stats and out_mode == 0:
            g = geom if geom is not None else tuple(out.shape[:3])
            n = ops.gn_part_floats(g[0], g[1], g[2], cout)
            part = self._tmp(part_slot, n, dtype=torch.float32) if part_slot else self._new(n, dtype=torch.float32)
        info = [0] * 7
        run = lambda cfg, info=None: ops.conv_gemm(srcs, w, cout, bias=bias, residual=residual, out=out, gn_part=part,
                                                   info=info, cfg=cfg, out_mode=out_mode, geom=geom,
                                                   w_batch_stride=w_batch_stride, w_map=w_map, n_slabs=n_slabs)
        # a mapped layer (one weight slab chosen per image) never shares an unmapped layer's configuration
        key = ("conv", cout, tuple(out.shape), geom, tuple((t.shape[-1], taps) for t, taps in srcs), residual is not None,
               part is not None, out_mode, w_batch_stride > 0, w_map is not None)
        cfg = tune(key, run, m_rows=out.shape[0] * out.shape[1] * out.shape[2] if out_mode == 0 and geom is None else 0)
        self._add(lambda: run(cfg, info), kind, flops)
        if part is not None and info[5]:
            self._parts[out.data_ptr()] = (part, info[6] // (geom[0] if geom is not None else out.shape[0]))
        else:
            self._parts.pop(out.data_ptr(), None)

    def _gemm(self, x, w, cout, out, flops, bias=None, residual=None):
        """Flat-row GEMM step (no per-image structure, no statistics), tuned like _conv."""
        run = lambda cfg, info=None: ops.gemm_rows(x, w, cout, bias=bias, residual=residual, out=out, cfg=cfg, info=info)
        cfg = tune(("gemm", cout, tuple(x.shape), residual is not None), run, m_rows=x.shape[0] * x.shape[1])
        self._add(lambda: run(cfg), "conv_gemm", flops)
        self._parts.pop(out.data_ptr(), None)

    def _stats(self, a, b, eps):
        """-> fp32 [NB, 32, 2] (mean, rstd) of the channel concat [a | b] via one launch: k2_gn_finalize over the producers'
        fused partials when every source has them, else a k2_gn_stats read pass."""
        pa = self._parts.get(a.data_ptr())
        pb = self._parts.get(b.data_ptr()) if b is not None else None
        st = self._new(self.NB, 32, 2, dtype=torch.float32)
        HW = a.shape[1] * a.shape[2]
        if pa is not None and (b is None or pb is not None):
            c1 = b.shape[-1] if b is not None else 0
            self._add(lambda: ops.gn_finalize(pa[0], a.shape[-1], pb[0] if pb else None, c1, self.NB, pa[1], HW, st,
                                              rg1=pb[1] if pb else None, eps=eps), "gn_finalize")
        else:
            self._add(lambda: ops.gn_stats(a, b, stats=st, eps=eps), "gn_stats")
        return st

    def _norm(self, a, b, gamma, beta, y, film=None, act=1, resample=0, xres=None, eps=1e-5):
        """GroupNorm32 (+FiLM) (+SiLU) (+resample) of the channel concat [a | b] -> y.  Statistics: folded inside the apply
        kernel from the producing convs' fused partial sums when every source has them and an image has few row groups (one
        launch per GroupNorm); otherwise a statistics launch (_stats) + k2_gn_apply."""
        pa = self._parts.get(a.data_ptr())
        pb = self._parts.get(b.data_ptr()) if b is not None else None
        have = pa is not None and (b is None or pb is not None)
        cpg = (a.shape[-1] + (b.shape[-1] if b is not None else 0)) // 32
        if have and cpg >= 2 and max(pa[1], pb[1] if pb else 0) <= FOLD_MAX_RG:
            self._add(lambda: ops.gn_apply_fold(a, b, pa[0], pa[1], pb[0] if pb else None, pb[1] if pb else 0, gamma, beta,
                                                film=film, act=act, resample=resample, y=y, xres=xres, eps=eps), "gn_apply")
            return
        st = self._stats(a, b, eps)
        self._add(lambda: ops.gn_apply(a, b, st, gamma, beta, film=film, act=act, resample=resample, y=y, xres=xres),
                  "gn_apply")

    # execution ---------------------------------------------------------------------------------
    def launch(self):
        for fn, _, _ in self.steps:
            fn()

    def _timed_pass(self):
        evs = []
        self._serial = True
        torch.cuda.synchronize()
        torch.cuda._sleep(int(4e7))  # the host runs ahead: events are not skewed by launch latency
        for fn, kind, flops in self.steps:
            s = torch.cuda.Event(enable_timing=True)
            e = torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            evs.append((s, e))
        torch.cuda.synchronize()
        self._serial = False
        return [s.elapsed_time(e) for s, e in evs]

    def profile_detail(self, reps=3):
        """[(kind, flops, ms)] per launch, averaged over `reps` eager passes (CUDA events around every launch)."""
        acc = [0.0] * len(self.steps)
        for _ in range(reps):
            for i, ms in enumerate(self._timed_pass()):
                acc[i] += ms / reps
        return [(k, f, ms) for (_, k, f), ms in zip(self.steps, acc)]

    def profile(self, reps=3):
        """Per-kernel-family device time of one eager pass -> {kind: dict(ms=..., launches=..., flops=...)}."""
        agg = {}
        for kind, flops, ms in self.profile_detail(reps):
            if kind == "join":
                continue
            a = agg.setdefault(kind, dict(ms=0.0, launches=0, flops=0))
            a["ms"] += ms
            a["launches"] += 1
            a["flops"] += flops
        return agg

    def run(self, use_graph):
        if not use_graph:
            self.launch()
            return
        if self.graph is None:
            self.launch()  # warm-up: one-time cudaFuncSetAttribute calls are not capturable
            torch.cuda.synchronize()
            self.graph = capture_graph(self.launch)
        self.graph.replay()


def capture_graph(launch):
    """launch() recorded into a new CUDA graph, with Python's cyclic garbage collector paused for the capture.  A launch plan
    is a reference cycle (its launch closures hold it), so the CUDA graph of a plan nobody holds any more is destroyed whenever
    the collector next runs; if that happens while a stream captures, the destruction invalidates the capture."""
    g = torch.cuda.CUDAGraph()
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(g):
            launch()
    finally:
        if enabled:
            gc.enable()
    return g
