"""Continuous batching of Kandinsky 2.2 text2img requests: one CFG-doubled UNet batch of S slots, every slot a request at its
own denoising step, refilled from a FIFO queue as requests finish.

Rows follow the 2.2 layout, unconditional s and conditional S + s for slot s.  The device keeps per slot its step index, its
timestep / coefficient / per-step noise tables and its guidance scale (k2b200.h: k2_slot_step_begin); one step of the whole
batch is ONE captured CUDA graph (k2_slot_step_begin, the UNet plan, the slot form of the sampler step, k2_slot_step_end)
whose buffers never move, so admitting a request is a handful of copies into them and the host loop reads nothing back from
the device: it knows from its own bookkeeping which slot finishes at which step.

A request computes what generate_text2img(batch_size=1) computes on a pipeline whose base_seed is the request's seed: the same
start latent and per-step noise draws, the same tables (create_ddpm_v22 / the SCHEDULE_SAMPLERS builders), the same
conditioning and step kernels.  Its result does not depend on the other slots: the UNet's normalisation, attention and
convolutions are per image, the conditioning is written per row (Text2ImUNet.bind_slot) and the slot step kernels read and
write only the rows of active slots.  An idle slot still costs a full row of UNet compute.

With max_loras = L > 0 each request may name a LoRA adapter registered with add_lora.  The attention layers' qkv and proj_out
weights then live in slab tables of 1 + L fp16 copies per layer (slab 0: the pipeline's packed weights when the batcher was
made, slabs 1 .. L: base + scale * up @ down of a registered adapter, merged by k2_lora_merge as load_lora merges), and both
GEMMs run batched, rows s and S + s of slot s multiplying the slab a device map names (k2_conv_gemm_wmap).  A slot's encoder
K/V rows are computed at admission with its adapter's merged encoder_kv weights.  Registering, removing and admitting write
slabs, the map and conditioning rows in place, so the step graph never changes.
"""
import collections

import torch

from . import ops, parallel
from ._native import K2Error
from .launch_plan import capture_graph
from .model.gaussian_diffusion import create_ddpm_v22
from .model.unet import _Plan

BATCHER_SAMPLERS = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")


def check_batcher_args(max_batch, h, w, sampler, max_steps, max_loras=0):
    """Refuse what a Batcher cannot serve, before any work: ValueError naming the argument."""
    if sampler not in BATCHER_SAMPLERS:
        raise ValueError(f"batcher: sampler {sampler!r} is not served; use one of {', '.join(BATCHER_SAMPLERS)}")
    for name, v in (("max_batch", max_batch), ("h", h), ("w", w), ("max_steps", max_steps)):
        if isinstance(v, bool) or not isinstance(v, int) or v < 1:
            raise ValueError(f"batcher: {name} must be a positive int, got {v!r}")
    if isinstance(max_loras, bool) or not isinstance(max_loras, int) or max_loras < 0:
        raise ValueError(f"batcher: max_loras must be an int >= 0, got {max_loras!r}")


def request_tables(sampler, steps):
    """(model timesteps fp32 [steps], coefficient rows fp32 [steps, 8]) of one request in loop order: the rows the sampling
    loop of generate_text2img stages for `sampler` at decoder_steps = steps, from the same schedule builders."""
    from .pipelines import _solver_schedule
    diffusion = create_ddpm_v22(steps)
    sched = diffusion if sampler == "ddpm_sampler" else _solver_schedule(sampler, diffusion, steps)
    coef, ts = sched._tables("cpu")
    order = torch.arange(sched.num_timesteps - 1, -1, -1)
    return ts[order].contiguous(), coef[order].contiguous()


class SlotQueue:
    """The host bookkeeping of a Batcher: a FIFO of waiting requests, which request holds which slot, and how many steps each
    slot has left."""

    def __init__(self, slots):
        self.waiting = collections.deque()
        self.holder = [None] * slots
        self.left = [0] * slots

    def submit(self, handle, steps):
        self.waiting.append((handle, steps))

    def admit(self, limit=None):
        """Move waiting requests, oldest first, into the free slots, lowest first (at most `limit` of them) -> [(slot,
        handle)]."""
        out = []
        for s in range(len(self.holder)):
            if not self.waiting or (limit is not None and len(out) == limit):
                break
            if self.holder[s] is None:
                handle, steps = self.waiting.popleft()
                self.holder[s], self.left[s] = handle, steps
                out.append((s, handle))
        return out

    def release(self, slot):
        """Free `slot` without finishing its request (an admission that failed)."""
        self.holder[slot], self.left[slot] = None, 0

    def advance(self):
        """One step of every occupied slot -> [(slot, handle)] of the requests it finished, whose slots are free again."""
        done = []
        for s, handle in enumerate(self.holder):
            if handle is None:
                continue
            self.left[s] -= 1
            if self.left[s] == 0:
                self.holder[s] = None
                done.append((s, handle))
        return done

    def busy(self):
        return any(h is not None for h in self.holder)


class _Request:
    __slots__ = ("steps", "guidance", "seed", "ts", "coef", "negative", "positive", "lora")


class Batcher:
    """Requests of one geometry and one sampler served from max_batch slots (Kandinsky2_2.batcher builds it)."""

    RUN_AHEAD = 2   # replayed steps the host may have in flight on the GPU when it admits (2: the GPU never waits on admission)

    def __init__(self, pipe, max_batch, h, w, sampler="ddpm_sampler", max_steps=100, max_loras=0):
        check_batcher_args(max_batch, h, w, sampler, max_steps, max_loras)
        if pipe.task_type != "text2img":
            raise ValueError(f"batcher: serves text2img pipelines only, this one is {pipe.task_type!r}")
        self.pipe, self.sampler, self.max_steps = pipe, sampler, max_steps
        self.h, self.w = pipe.get_new_h_w(h, w)
        S, H, W = max_batch, self.h // 8, self.w // 8
        model = pipe.model
        if model._packed is None:
            model.finalize()
        self._packed = model._packed
        dev = pipe.device
        self.max_loras = max_loras
        self._loras = {}   # adapter name -> (slab index, {attention layer -> merged encoder_kv weight})
        self.w_map = None
        slabs = None
        if max_loras:
            # allocated once, so the graph's addresses never change; slab 0 and its encoder_kv weights are copies, so
            # load_lora / unload_lora on the pipeline leave this batcher's weights as they were
            self.w_map = torch.zeros(2 * S, device=dev, dtype=torch.int32)
            layers, self._wenc0 = {}, {}
            for name, a in model._packed["attn"].items():
                tabs = []
                for key in ("wqkv", "wproj"):
                    t = torch.zeros((1 + max_loras,) + tuple(a[key].shape), device=dev, dtype=torch.float16)
                    t[0].copy_(a[key])
                    tabs.append(t)
                layers[name] = tuple(tabs)
                self._wenc0[name] = a["wenc"].clone()
            slabs = dict(map=self.w_map, layers=layers)
        # a plan of its own: another call on the pipeline at the same geometry must not rebind these rows
        self.plan = p = _Plan(model, 2 * S, H, W, model.num_image_embs, attn_slabs=slabs)
        p.xf_proj.zero_()
        for buf in p.enc_kv.values():
            buf.zero_()
        f32 = dict(device=dev, dtype=torch.float32)
        self.x = torch.zeros(S, 4, H, W, **f32)
        self.state = torch.tensor([[-1] * S, [0] * S], device=dev, dtype=torch.int32)
        self.ts_tab = torch.zeros(S, max_steps, **f32)
        self.coef_tab = torch.zeros(S, max_steps, 8, **f32)
        self.coef = torch.zeros(S, 8, **f32)
        self.guidance = torch.zeros(S, **f32)
        ddpm = sampler == "ddpm_sampler"
        # the DDPM step's noise for every step of every slot, drawn at admission: S x max_steps x 4 H W floats
        self.noise_tab = torch.zeros(S, max_steps, 4, H, W, **f32) if ddpm else None
        self.noise = torch.zeros(S, 4, H, W, **f32) if ddpm else None
        self.work = torch.zeros(S, 4, H, W, **f32) if ddpm else None
        self.hist = None if ddpm else torch.zeros(S, 4, H, W, **f32)
        self.queue = SlotQueue(S)
        self._requests = {}
        self._next_handle = 0
        self._emb_dim = pipe.config["model_config"]["image_encoder_in_dim"]
        # one event per replayed step, the newest RUN_AHEAD of them: step() waits for the oldest before it admits, so the host
        # stays at most RUN_AHEAD steps ahead of the GPU and a request that arrives while a slot is free joins the batch at the
        # next step on the GPU's clock, not after everything already enqueued
        self._events = collections.deque()
        self._launch()  # warm-up with every slot idle (changes nothing): one-time cudaFuncSetAttribute calls are not capturable
        torch.cuda.synchronize()
        self.graph = capture_graph(self._launch)

    def _launch(self):
        p = self.plan
        ops.slot_step_begin(self.x, p.x_in, p.t_in, self.coef, self.ts_tab, self.coef_tab, self.noise_tab, self.noise,
                            self.state)
        p.launch()
        if self.sampler == "ddpm_sampler":
            ops.slot_sampler_step(p.out, self.x, self.noise, self.coef, self.guidance, self.state, self.work)
        else:
            ops.slot_dpm_solver_step(p.out, self.x, self.hist, self.coef, self.guidance, self.state)
        ops.slot_step_end(self.state)

    def add_lora(self, name, state_dict, scale=1.0):
        """Register a LoRA adapter of the decoder's attention blocks under `name` (the format Text2ImUNet.load_lora takes):
        merged into a free slab from the UNet's unmerged weights, as load_lora(state_dict, scale) would merge it, so the
        slab's bits are those load_lora writes.  Adapters do not stack with one the pipeline has loaded.  Requests submitted
        with lora=name use it."""
        if not self.max_loras:
            raise ValueError("add_lora: this batcher was made with max_loras=0; make one with max_loras > 0")
        if name in self._loras:
            raise ValueError(f"add_lora: an adapter named {name!r} is already registered")
        used = {k for k, _ in self._loras.values()}
        free = [k for k in range(1, self.max_loras + 1) if k not in used]
        if not free:
            raise ValueError(f"add_lora: all {self.max_loras} adapter slabs are in use; remove_lora one first")
        model = self.pipe.model
        if model._packed is not self._packed:
            raise K2Error("batcher: the UNet's weights were reloaded after the batcher was made; make a new one")
        factors, scale = model.lora_factors(state_dict), float(scale)
        k, wenc = free[0], {}
        for p, a in self._packed["attn"].items():
            base = model._lora_base[p] if model._lora_base is not None else a
            wqkv, wproj = self.plan.attn_slabs["layers"][p]
            wenc[p] = torch.empty_like(base["wenc"])
            targets = {"wqkv": wqkv[k], "wproj": wproj[k], "wenc": wenc[p]}
            for key, proj in model._LORA_WEIGHTS:   # what Text2ImUNet._merge_lora writes into the packed weights
                f = factors.get(p + proj + ".weight")
                targets[key].copy_(base[key])
                if f is not None:
                    up, down = (t.to(base[key].device) for t in f)
                    ops.lora_merge(base[key], up, down, scale, out=targets[key])
        self._loras[name] = (k, wenc)

    def remove_lora(self, name):
        """Unregister adapter `name`, freeing its slab; refused while a waiting or active request uses it."""
        if name not in self._loras:
            raise ValueError(f"remove_lora: no adapter named {name!r} is registered")
        if any(r.lora == name for r in self._requests.values()):
            raise ValueError(f"remove_lora: adapter {name!r} is used by a waiting or active request")
        del self._loras[name]

    def submit(self, prompt=None, *, image_embeds=None, negative_image_embeds=None, decoder_steps=50, decoder_guidance_scale=4,
               seed=None, prior_steps=25, prior_guidance_scale=4, negative_prior_prompt="", negative_decoder_prompt="",
               lora=None):
        """Queue one image -> its handle (the key of its image in what step() / run() return).  Either a prompt, whose image
        embeddings the pipeline's embedder makes now at batch 1 as generate_text2img does (the prior keywords as there), or
        image_embeds and negative_image_embeds ([1, D] or [D]) as diffusers' KandinskyV22Pipeline takes them.  seed plays the
        part of the pipeline's base_seed for global sample 0 (default: the pipeline's base_seed).  lora: the name of an
        adapter registered with add_lora, or None for the weights slab 0 holds."""
        pipe = self.pipe
        if (prompt is None) == (image_embeds is None):
            raise ValueError("submit: pass either a prompt or image_embeds")
        if image_embeds is not None and negative_image_embeds is None:
            raise ValueError("submit: image_embeds needs negative_image_embeds")
        for name, e in (("image_embeds", image_embeds), ("negative_image_embeds", negative_image_embeds)):
            if e is not None and (not torch.is_tensor(e) or e.numel() != self._emb_dim or e.dim() not in (1, 2)
                                  or not e.is_floating_point()):
                raise ValueError(f"submit: {name} must be one floating-point image embedding, [1, {self._emb_dim}] or "
                                 f"[{self._emb_dim}], got {tuple(e.shape) if torch.is_tensor(e) else type(e).__name__}")
        if isinstance(decoder_steps, bool) or not isinstance(decoder_steps, int) or not 1 <= decoder_steps <= self.max_steps:
            raise ValueError(f"submit: decoder_steps must be an int in [1, {self.max_steps}] (the batcher's max_steps), "
                             f"got {decoder_steps!r}")
        if lora is not None and lora not in self._loras:
            raise ValueError(f"submit: no adapter named {lora!r} is registered (Batcher.add_lora)")
        r = _Request()
        r.lora = lora
        r.steps, r.guidance = decoder_steps, float(decoder_guidance_scale)
        r.seed = pipe.base_seed if seed is None else int(seed)
        r.ts, r.coef = request_tables(self.sampler, decoder_steps)
        if prompt is not None:
            pk = pipe._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
            r.positive, r.negative = pipe._embeds(prompt, 1, negative_decoder_prompt, pk)
        else:
            r.positive, r.negative = image_embeds, negative_image_embeds
        handle = self._next_handle
        self._next_handle += 1
        self._requests[handle] = r
        self.queue.submit(handle, decoder_steps)
        return handle

    def _admit(self):
        """Stage waiting requests into free slots, one at a time: a request holds its slot in the host bookkeeping only once
        its conditioning, tables, latent and noise are written, so a failed admission leaves no slot that would be stepped
        and decoded from another request's buffers."""
        while True:
            got = self.queue.admit(limit=1)
            if not got:
                return
            s, handle = got[0]
            try:
                self._stage(s, self._requests[handle])
            except BaseException:
                self.queue.release(s)
                self.state[:, s] = torch.tensor([-1, 0], dtype=torch.int32)
                del self._requests[handle]
                raise

    def _stage(self, s, r):
        pipe, H, W = self.pipe, self.x.shape[2], self.x.shape[3]
        if self.w_map is None:
            pipe.model.bind_slot(self.plan, s, r.negative, r.positive)
        else:
            k, wenc = self._loras[r.lora] if r.lora is not None else (0, self._wenc0)
            pipe.model.bind_slot(self.plan, s, r.negative, r.positive, wenc=wenc)
            self._set_slab(s, k)
        k = r.steps
        self.ts_tab[s, :k].copy_(r.ts)
        self.coef_tab[s, :k].copy_(r.coef)
        # the draws of generate_text2img(batch_size=1) with base_seed = r.seed (_DecoderBase._decode, _sampling_loop)
        self.x[s].copy_(parallel.sample_noise(range(1), (4, H, W), base_seed=r.seed, device=pipe.device)[0])
        if self.noise_tab is not None:
            gen = pipe._generators(0, 1, base_seed=r.seed)[0]
            self.noise_tab[s, :k].copy_(torch.randn(k, 4, H, W, device=pipe.device, generator=gen))
        else:
            self.hist[s].zero_()
        self.guidance[s] = r.guidance
        self.state[:, s] = torch.tensor([0, k], dtype=torch.int32)

    def step(self):
        """Admit waiting requests into free slots, run one denoising step of every occupied slot (one graph replay), decode
        the requests that step finished -> {handle: PIL image}."""
        if self.pipe.model._packed is not self._packed:
            raise K2Error("batcher: the UNet's weights were reloaded after the batcher was made; make a new one")
        if len(self._events) >= self.RUN_AHEAD:
            self._events.popleft().synchronize()   # waits for a step to end; reads nothing back
        self._admit()
        if not self.queue.busy():
            return {}
        self.graph.replay()
        ev = torch.cuda.Event()
        ev.record()
        self._events.append(ev)
        done = {}
        for s, handle in self.queue.advance():
            done[handle] = self.pipe._finish(self.x[s:s + 1], self.h, self.w)[0]
            del self._requests[handle]
            if self.w_map is not None:
                self._set_slab(s, 0)   # idle slots use slab 0, so a removed adapter's slab is read by no slot
        return done

    def _set_slab(self, s, k):
        S = self.x.shape[0]
        self.w_map[s] = k
        self.w_map[S + s] = k

    def run(self):
        """step() until every submitted request is finished -> {handle: PIL image} of all of them."""
        out = {}
        while self.queue.waiting or self.queue.busy():
            out.update(self.step())
        return out
