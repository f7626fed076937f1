"""Continuous batching of Kandinsky 2.2 (Batcher) and 2.1 (Batcher21) text2img and img2img requests, and of Kandinsky 2.2
ControlNet-depth requests: one CFG-doubled UNet batch of S slots, every slot a request at its own denoising step, refilled from
a FIFO queue as requests finish.

Rows follow the version's layout: for slot s, unconditional s and conditional S + s in 2.2, the reverse in 2.1.  The device
keeps per slot its step index, its timestep / coefficient / per-step noise tables and its guidance scale (SlotSteps, k2b200.h:
k2_slot_step_begin); one step of the whole batch is ONE captured CUDA graph (SlotSteps.begin, the UNet plan, SlotSteps.step,
SlotSteps.end) whose buffers never move, so admitting a request is a handful of copies into them and the host loop
(_SlotBatcher) reads nothing back from the device: it knows from its own bookkeeping which slot finishes at which step.

A request computes what generate_text2img(batch_size=1) computes on a pipeline whose base_seed is the request's seed: the same
start latent and per-step noise draws, the same tables (request_tables: the rows of the schedule the pipeline's sampling loop
runs), the same conditioning, and the step that loop runs, set as the loop sets it from the schedule and the pipeline (step
kernel, noise, clamp of x0, dynamic threshold, row order).  Its result does not depend on the other slots: the UNet's
normalisation, attention and convolutions are per image, the conditioning is written per row (Text2ImUNet.bind_slot) and the
slot step kernels read and write only the rows of active slots.  2.1's p_sampler clips x0 with the 99.5 percentile of the
request's own x0 (at batch 1 the reference's "sample 0" is the request itself): the slot step computes one percentile per
slot.  An idle slot still costs a full row of UNet compute.

An img2img request (submit(image=, strength=)) computes what generate_img2img(batch_size=1) computes: its image is encoded at
submit, the pipeline's _img2img_start noises it to the first step its rule keeps, and the request runs only the rows that
step keeps (request_tables(..., init_step)), so requests of different lengths share the batch.  Its start latent replaces the
fresh draw when it is admitted; the solvers' history is zeroed as for any request, and their tables make the first kept step
first order.  A batcher of a ControlNet-depth pipeline gives every request its own depth hint: the hint stem runs at admission
(Text2ImUNet.bind_slot(hint=)) and writes the slot's rows of the plan's hint_in, which the step graph's stem reads.

With max_loras = L > 0 each request may name a LoRA adapter registered with add_lora.  The attention layers' qkv and proj_out
weights then live in slab tables of 1 + L fp16 copies per layer (slab 0: the pipeline's packed weights when the batcher was
made, slabs 1 .. L: base + scale * up @ down of a registered adapter, merged by ops.lora_merge_weights as load_lora merges),
and both GEMMs run batched, rows s and S + s of slot s multiplying the slab a device map names (k2_conv_gemm_wmap).  A
slot's encoder K/V rows are computed at admission with its adapter's merged encoder_kv weights.  Registering, removing and
admitting write slabs, the map and conditioning rows in place, so the step graph never changes.

PriorBatcher serves the Kandinsky 2.2 prior the same way: S slots, each an image_emb(prompt, 1) or emb2emb(prompt, image, 1)
request at its own UnCLIP step of its own tables, one graph replay per step (SlotSteps around the prior network of
model.prior._PriorSlotPlan), results left on the device.  A decoder Batcher made with prior_slots = P > 0 runs the
pipeline's embedding rules against prior requests instead of prior calls at submit; a request waits until its embeddings
are done and then joins the decoder queue (requests ready at the same prior step in submit order).  step() replays one
prior step before the decoder step while the prior batch has work, and prior steps back to back until a prior request
finishes when a decoder slot is free and no ready request can take it.
"""
import collections
import inspect

import numpy as np
import torch

from . import ops, parallel
from ._native import K2Error
from .launch_plan import capture_graph
from .model.gaussian_diffusion import SpacedDiffusion
from .model.prior import UnCLIPSchedule, _PriorSlotPlan
from .model.unet import _Plan
from .pipelines import _sampler_schedule

BATCHER_SAMPLERS = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
# Kandinsky 2.1's: PLMS is not among them, its first step evaluates the UNet twice and it keeps its epsilon history on the host
BATCHER_SAMPLERS_21 = ("p_sampler", "ddim_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")


def _check_int(who, name, v, lo, hi=None):
    """Refuse v unless it is an int (a bool is not) in [lo, hi], hi None for no upper bound: ValueError naming the argument."""
    if isinstance(v, bool) or not isinstance(v, int) or v < lo or (hi is not None and v > hi):
        bounds = f">= {lo}" if hi is None else f"in [{lo}, {hi}]"
        raise ValueError(f"{who}: {name} must be an int {bounds}, got {v!r}")


def check_batcher_args(max_batch, h, w, sampler, max_steps, max_loras=0, samplers=BATCHER_SAMPLERS):
    """Refuse what a Batcher cannot serve, before any work: ValueError naming the argument."""
    if sampler not in samplers:
        raise ValueError(f"batcher: sampler {sampler!r} is not served; use one of {', '.join(samplers)}")
    for name, v, lo in (("max_batch", max_batch, 1), ("h", h, 1), ("w", w, 1), ("max_steps", max_steps, 1),
                        ("max_loras", max_loras, 0)):
        _check_int("batcher", name, v, lo)


def request_tables(pipe, sampler, steps, init_step=None):
    """(model timesteps fp32 [n], coefficient rows fp32 [n, 8]) of one request in loop order: the rows the sampling loop of
    pipe.generate_text2img stages for `sampler` at `steps` steps, from the schedule it runs (n = steps, except for DDIM, whose
    timesteps range(0, 1000, 1000 // steps) are more than steps when steps does not divide 1000).  init_step: the one
    pipe._img2img_start returns, for the rows of generate_img2img's loop -- the solver schedules and DDIM cut their own tables
    to it, the loop over a SpacedDiffusion runs its rows init_step - 1 .. 0."""
    sched = _sampler_schedule(sampler, pipe._diffusion(sampler, steps), steps, init_step)
    return _loop_rows(sched, init_step if isinstance(sched, SpacedDiffusion) else None)


def _loop_rows(sched, init_step=None):
    """(timesteps, coefficient rows) of a schedule in the order _sampling_loop runs them: the rows [:init_step], last first."""
    coef, ts = sched._tables("cpu")
    order = torch.arange(sched.num_timesteps)[:init_step].flip(0)
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


class SlotSteps:
    """The device side of S slots, each at its own step of its own tables of max_steps rows: state int32 [2, S] = (k_s, steps_s)
    of k2b200.h (idle: [-1, 0]), the latents x [S, *shape] and the step kernels' operands.  begin, step and end launch one
    step of every active slot around the network; stage and idle are the only writers of state."""

    def __init__(self, S, shape, max_steps, device, kind="ddpm", draws_noise=True, clip=10.0, cond_first=0,
                 threshold_mode=0):
        ddpm = kind == "ddpm"
        self.S, self.clip, self.cond_first, self.threshold_mode = S, clip, cond_first, threshold_mode
        f32 = dict(device=device, dtype=torch.float32)
        self.x = torch.zeros(S, *shape, **f32)
        self.state = torch.tensor([[-1] * S, [0] * S], device=device, dtype=torch.int32)
        self.ts_tab = torch.zeros(S, max_steps, **f32)
        self.coef_tab = torch.zeros(S, max_steps, 8, **f32)
        self.coef = torch.zeros(S, 8, **f32)
        self.guidance = torch.zeros(S, **f32)
        self.noise_tab = torch.zeros(S, max_steps, *shape, **f32) if draws_noise else None
        self.noise = torch.zeros(S, *shape, **f32) if ddpm else None
        self.work = torch.zeros(S, *shape, **f32) if ddpm else None
        self.sval = torch.zeros(S, **f32) if threshold_mode else None   # each slot's dynamic threshold
        self.hist = None if ddpm else torch.zeros(S, *shape, **f32)

    def begin(self, x_in, t_in):
        ops.slot_step_begin(self.x, x_in, t_in, self.coef, self.ts_tab, self.coef_tab, self.noise_tab, self.noise, self.state)

    def step(self, model_out):
        if self.hist is None:
            ops.slot_sampler_step(model_out, self.x, self.noise, self.coef, self.guidance, self.state, self.work, self.clip,
                                  cond_first=self.cond_first, threshold_mode=self.threshold_mode, sval=self.sval)
        else:
            ops.slot_dpm_solver_step(model_out, self.x, self.hist, self.coef, self.guidance, self.state,
                                     cond_first=self.cond_first)

    def end(self):
        ops.slot_step_end(self.state)

    def stage(self, s, ts, coef, x, guidance, noise=None):
        """Slot s starts a request of k = len(ts) steps from latent x, with its k rows of tables and, when the step draws
        noise, its k steps' noise (x and noise reshaped to the slot's latents); its solver history is zeroed."""
        k = ts.shape[0]
        self.ts_tab[s, :k].copy_(ts)
        self.coef_tab[s, :k].copy_(coef)
        self.x[s].copy_(x.reshape(self.x.shape[1:]))
        if noise is not None:
            self.noise_tab[s, :k].copy_(noise.reshape((k,) + self.x.shape[1:]))
        if self.hist is not None:
            self.hist[s].zero_()
        self.guidance[s] = guidance
        self.state[:, s] = torch.tensor([0, k], dtype=torch.int32)

    def idle(self, s):
        self.state[:, s] = torch.tensor([-1, 0], dtype=torch.int32)


class _SlotBatcher:
    """The host loop of a batcher: requests registered under handles, a SlotQueue, and one step of every occupied slot per
    graph replay.  A subclass makes plan and slots (SlotSteps), calls _capture, and gives _stage(s, r) (bind r's conditioning,
    then slots.stage) and _weights() (once they change, a step raises K2Error(WEIGHTS_CHANGED))."""

    def __init__(self, S):
        self.queue = SlotQueue(S)
        self._requests = {}
        self._next_handle = 0

    def _capture(self, model_out):
        self._model_out = model_out   # the plan's output, as the step kernel reads it
        self._weights0 = self._weights()
        self._launch()  # warm-up with every slot idle (changes nothing): one-time cudaFuncSetAttribute calls are not capturable
        torch.cuda.synchronize()
        self.graph = capture_graph(self._launch)

    def _launch(self):
        self.slots.begin(self.plan.x_in, self.plan.t_in)
        self.plan.launch()
        self.slots.step(self._model_out)
        self.slots.end()

    def _check_weights(self):
        if any(a is not b for a, b in zip(self._weights(), self._weights0)):
            raise K2Error(self.WEIGHTS_CHANGED)

    def _enqueue(self, r, ready=True):
        """Register request r -> its handle; a ready request joins the queue for its r.steps steps."""
        handle = self._next_handle
        self._next_handle += 1
        self._requests[handle] = r
        if ready:
            self.queue.submit(handle, r.steps)
        return handle

    def pending(self):
        """Whether a request is waiting or being sampled."""
        return bool(self.queue.waiting) or self.queue.busy()

    def _admit(self):
        """Stage waiting requests into free slots, one at a time: a request holds its slot in the host bookkeeping only once
        its conditioning, tables, latent and noise are written, so a failed admission leaves no slot that would be stepped
        and finished from another request's buffers."""
        while True:
            got = self.queue.admit(limit=1)
            if not got:
                return
            s, handle = got[0]
            try:
                self._stage(s, self._requests[handle])
            except BaseException:
                self.queue.release(s)
                self.slots.idle(s)
                del self._requests[handle]
                raise

    def _before_admit(self):
        pass

    def _step_slots(self):
        """Admit waiting requests into free slots and run one step of every occupied slot (one graph replay) -> [(slot,
        handle)] of the requests it finished, no longer registered, or None when no slot was occupied (no replay)."""
        self._check_weights()
        self._before_admit()
        self._admit()
        if not self.queue.busy():
            return None
        self.graph.replay()
        done = self.queue.advance()
        for _, handle in done:
            del self._requests[handle]
        return done

    def run(self):
        """step() until every submitted request is finished -> {handle: result} of all of them."""
        out = {}
        while self.pending():
            out.update(self.step())
        return out


class _Request:
    __slots__ = ("steps", "guidance", "seed", "ts", "coef", "negative", "positive", "lora", "full", "pooled", "start", "hint")


def _check_embedding(name, e, dim):
    if e is not None and (not torch.is_tensor(e) or e.numel() != dim or e.dim() not in (1, 2) or not e.is_floating_point()):
        raise ValueError(f"submit: {name} must be one floating-point image embedding, [1, {dim}] or [{dim}], got "
                         f"{tuple(e.shape) if torch.is_tensor(e) else type(e).__name__}")


def _check_img2img(image, strength):
    if image is None and strength is not None:
        raise ValueError("submit: strength without image; strength is the noise level an img2img request's image starts at")
    if strength is not None and (isinstance(strength, bool) or not isinstance(strength, (int, float)) or
                                 not 0 <= strength <= 1):
        raise ValueError(f"submit: strength must be a number in [0, 1], got {strength!r}")


class Batcher(_SlotBatcher):
    """Kandinsky 2.2 requests of one geometry and one sampler served from max_batch slots (Kandinsky2_2.batcher builds it).
    What differs between the versions is a class attribute or one of the methods Batcher21 overrides: the sampler set, the
    tasks, the geometry and context length, submit's keywords, the image latent and the conditioning a slot is bound to.  The
    tables, the img2img start, the step and the row order are the pipeline's."""

    RUN_AHEAD = 2   # replayed steps the host may have in flight on the GPU when it admits (2: the GPU never waits on admission)
    SAMPLERS = BATCHER_SAMPLERS
    TASKS = ("text2img", "controlnet")
    WEIGHTS_CHANGED = "batcher: the UNet's weights were reloaded after the batcher was made; make a new one"
    hinted = False   # True on a ControlNet pipeline's batcher: every request brings its own depth hint
    prior = None     # the PriorBatcher of a batcher made with prior_slots > 0

    def __init__(self, pipe, max_batch, h, w, sampler="ddpm_sampler", max_steps=100, max_loras=0, prior_slots=0):
        self._check_args(max_batch, h, w, sampler, max_steps, max_loras)
        if pipe.task_type not in self.TASKS:
            raise ValueError(f"batcher: serves {' and '.join(self.TASKS)} pipelines only, this one is {pipe.task_type!r}")
        _check_int("batcher", "prior_slots", prior_slots, 0)
        if prior_slots and not hasattr(pipe.embedder, "batcher"):
            raise ValueError("batcher: prior_slots > 0 needs an embedder that samples the prior in a batch (batcher(max_batch), "
                             f"e.g. model.prior.PriorEmbedder22); this pipeline's is a {type(pipe.embedder).__name__}")
        self.pipe, self.sampler, self.max_steps = pipe, sampler, max_steps
        self.hinted = pipe.task_type == "controlnet"
        self.h, self.w, H, W = self._geometry(h, w)
        self._latent_hw = (H, W)
        S = max_batch
        model = pipe.model
        if model._packed is None:
            model.finalize()
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
        self.plan = p = _Plan(model, 2 * S, H, W, self._context(), attn_slabs=slabs)
        p.xf_proj.zero_()
        for buf in p.enc_kv.values():
            buf.zero_()
        # the step settings the sampling loop reads from its schedule and the pipeline, read from the schedule at two steps
        # (the fewest a DDPM schedule has; the settings do not depend on the count)
        sched = _sampler_schedule(sampler, pipe._diffusion(sampler, 2), 2)
        self.slots = SlotSteps(S, (4, H, W), max_steps, dev, sched.step_kind, sched.draws_noise, sched.clip_range,
                               int(pipe.cond_first), int(isinstance(sched, SpacedDiffusion) and pipe.dynamic_threshold))
        super().__init__(S)
        # prompt requests' image embeddings sampled in a batch of prior slots: a decoder request waits in _held (handle ->
        # embeddings still missing) until the prior requests in _waiting_on (prior handle -> (handle, "positive" /
        # "negative")) are done
        self.prior = pipe.embedder.batcher(prior_slots) if prior_slots else None
        self._held, self._waiting_on = {}, {}
        self._emb_dim = pipe.config["model_config"]["image_encoder_in_dim"]
        # one event per replayed step, the newest RUN_AHEAD of them: step() waits for the oldest before it admits, so the host
        # stays at most RUN_AHEAD steps ahead of the GPU and a request that arrives while a slot is free joins the batch at the
        # next step on the GPU's clock, not after everything already enqueued
        self._events = collections.deque()
        self._capture(p.out)

    def _weights(self):
        return (self.pipe.model._packed,)

    def _check_args(self, max_batch, h, w, sampler, max_steps, max_loras):
        check_batcher_args(max_batch, h, w, sampler, max_steps, max_loras, self.SAMPLERS)

    def _geometry(self, h, w):
        """-> (decoded image height, width, latent height, width): 2.2 rounds the image up to multiples of 64."""
        h, w = self.pipe.get_new_h_w(h, w)
        return h, w, h // 8, w // 8

    def _context(self):
        return self.pipe.model.num_image_embs

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
        self._check_weights()
        model = self.pipe.model
        factors = model.lora_factors(state_dict)
        k, wenc, out = free[0], {}, {}   # out: id(packed weight) -> where this adapter's merge of it goes
        for p, a in model._packed["attn"].items():
            wqkv, wproj = self.plan.attn_slabs["layers"][p]
            wenc[p] = a["wenc"].clone()   # so its padding columns, which a merge leaves alone, are the packed weight's
            out.update({id(a["wqkv"]): wqkv[k], id(a["wproj"]): wproj[k], id(a["wenc"]): wenc[p]})
        ops.lora_merge_weights([(key, base, out[id(w)]) for key, base, w in model.lora_weights()], factors, float(scale))
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
               lora=None, image=None, strength=None, hint=None, prior_strength=None):
        """Queue one image -> its handle (the key of its image in what step() / run() return).  Either a prompt, whose image
        embeddings the pipeline's embedder makes now at batch 1 as generate_text2img does (the prior keywords as there), or
        image_embeds and negative_image_embeds ([1, D] or [D]) as diffusers' KandinskyV22Pipeline takes them.  seed plays the
        part of the pipeline's base_seed for global sample 0 (default: the pipeline's base_seed).  lora: the name of an
        adapter registered with add_lora, or None for the weights slab 0 holds.
        image (a PIL image, an image tensor or an encoded latent, as generate_img2img takes it) makes the request img2img, the
        image encoded now: generate_img2img(batch_size=1), strength defaulting to its default.  On a ControlNet batcher hint
        (a [1, 3, h, w] / [3, h, w] depth map, or a PIL image with the pipeline's depth_estimator) is required: the request
        is generate_controlnet(batch_size=1), or with an image generate_controlnet_img2img(batch_size=1, strength=,
        prior_strength=) -- prior_strength runs the prior from the image's embedding as that method does."""
        pipe = self.pipe
        if (prompt is None) == (image_embeds is None):
            raise ValueError("submit: pass either a prompt or image_embeds")
        if image_embeds is not None and negative_image_embeds is None:
            raise ValueError("submit: image_embeds needs negative_image_embeds")
        for name, e in (("image_embeds", image_embeds), ("negative_image_embeds", negative_image_embeds)):
            _check_embedding(name, e, self._emb_dim)
        _check_int("submit", "decoder_steps", decoder_steps, 1, self.max_steps)
        if lora is not None and lora not in self._loras:
            raise ValueError(f"submit: no adapter named {lora!r} is registered (Batcher.add_lora)")
        _check_img2img(image, strength)
        self._check_hint(hint)
        if prior_strength is not None and (not self.hinted or prompt is None or image is None):
            raise ValueError("submit: prior_strength (generate_controlnet_img2img's) needs a ControlNet batcher, a prompt and "
                             "an image")
        pk = pipe._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt) if prompt is not None else None
        if prior_strength is not None:
            pipe._check_prior_strength(prior_strength, pk)
        # with prior slots the pipeline's embedding rules run against _PriorQueue: prior requests, checked, queued by _enqueue
        embedder = _PriorQueue(self.prior, pipe.embedder) if self.prior is not None else None
        r = self._request(decoder_guidance_scale, seed, image, strength, decoder_steps, lora, self._slot_hint(hint))
        if prompt is None:
            r.positive, r.negative = image_embeds, negative_image_embeds
        elif prior_strength is None:
            r.positive, r.negative = pipe._embeds(prompt, 1, negative_decoder_prompt, pk, embedder)
        else:
            r.positive, r.negative = pipe._controlnet_img2img_embeds(prompt, image, 1, negative_decoder_prompt, pk,
                                                                     prior_strength, embedder)
        return self._enqueue(r)

    def _check_hint(self, hint):
        if self.hinted and hint is None:
            raise ValueError("submit: a ControlNet batcher needs hint= (the request's depth map)")
        if not self.hinted and hint is not None:
            raise ValueError("submit: hint is taken by the batcher of a task_type='controlnet' pipeline only")

    def _slot_hint(self, hint):
        """The request's depth map as generate_controlnet takes it -> fp32 [1, 3, h, w] on the device (None: no hint)."""
        if hint is None:
            return None
        pipe = self.pipe
        hint = pipe._depth_hint(hint)
        if not (torch.is_tensor(hint) and hint.dim() in (3, 4) and hint.shape[-3] == 3 and (hint.dim() == 3 or
                                                                                             hint.shape[0] == 1)):
            raise ValueError("submit: hint must be one depth map, a [1, 3, h, w] or [3, h, w] tensor (or a PIL image when the "
                             f"pipeline has a depth_estimator), got {tuple(hint.shape) if torch.is_tensor(hint) else type(hint)}")
        return pipe._hint(hint, self.h, self.w).to(pipe.device)

    def _image_latent(self, image):
        """The latent generate_img2img starts from: the MoVQ encoding of image at the batcher's h x w."""
        return self.pipe._encode_image(image, self.h, self.w)

    def _request(self, guidance, seed, image, strength, steps, lora=None, hint=None):
        """A request with its guidance, seed (default: the pipeline's base_seed), img2img start latent and tables."""
        r = _Request()
        r.lora, r.hint = lora, hint
        r.guidance = float(guidance)
        r.seed = self.pipe.base_seed if seed is None else int(seed)
        r.start, init_step = self._img2img_start(image, strength, steps, r.seed)
        r.ts, r.coef = request_tables(self.pipe, self.sampler, steps, init_step)
        return r

    def _img2img_start(self, image, strength, steps, seed):
        """-> (start latent [1, 4, H, W], init_step) of the pipeline's img2img rule with base_seed = seed, or (None, None) for
        a request without an image.  Refuses an image whose latent is not the batcher's grid and a strength whose rule keeps
        no step."""
        if image is None:
            return None, None
        pipe = self.pipe
        if strength is None:   # the default of the method the request stands for
            method = pipe.generate_controlnet_img2img if self.hinted else pipe.generate_img2img
            strength = inspect.signature(method).parameters["strength"].default
        lat = self._image_latent(image)
        grid = (1, 4) + tuple(self._latent_hw)
        if tuple(lat.shape) != grid:
            raise ValueError(f"submit: the image's latent is {list(lat.shape)}, the batcher's latent grid is {list(grid)}: pass "
                             f"an image of the batcher's {self.h} x {self.w}, or a PIL image")
        x, start = pipe._img2img_start(lat, pipe._diffusion(self.sampler, steps), steps, strength, self.sampler,
                                       base_seed=seed)
        if start < 1:
            raise ValueError(f"submit: strength {strength} keeps no denoising step of {self.sampler} at {steps} steps")
        return x, start

    def _enqueue(self, r):
        """Queue a request whose tables are set -> its handle; it runs one step per row of its tables.  An embedding that is
        a prior request (_PriorRequest) is queued on the prior batcher, and the request waits for it in _held."""
        r.steps = r.ts.shape[0]
        if r.steps > self.max_steps:
            raise ValueError(f"submit: the request's schedule has {r.steps} steps, more than the batcher's max_steps "
                             f"{self.max_steps}")
        waits = [name for name in ("positive", "negative") if isinstance(getattr(r, name), _PriorRequest)]
        handle = super()._enqueue(r, ready=not waits)
        if waits:
            self._held[handle] = len(waits)
        for name in waits:
            self._waiting_on[self.prior.enqueue(getattr(r, name))] = (handle, name)
        return handle

    def _prior_step(self):
        """One step of the prior batch; the embeddings it finished go to their requests, and the requests that now have all
        of theirs join the decoder queue in submit order -> whether a prior request finished.  A prior request whose
        admission failed is gone from the prior batcher: its decoder request is dropped too (and the result of its other
        prior request, if any, discarded), then the error propagates, as for a failed decoder admission."""
        try:
            done = self.prior.step()
        except BaseException:
            lost = {self._waiting_on[ph][0] for ph in self._waiting_on if ph not in self.prior._requests}
            for ph in [ph for ph, (handle, _) in self._waiting_on.items() if handle in lost]:
                del self._waiting_on[ph]
            for handle in lost:
                del self._held[handle], self._requests[handle]
            raise
        ready = []
        for ph, emb in done.items():
            if ph not in self._waiting_on:   # the other embedding of a dropped request
                continue
            handle, name = self._waiting_on.pop(ph)
            setattr(self._requests[handle], name, emb)
            self._held[handle] -= 1
            if not self._held[handle]:
                del self._held[handle]
                ready.append(handle)
        for handle in sorted(ready):
            self.queue.submit(handle, self._requests[handle].steps)
        return bool(done)

    def _run_prior(self):
        """The prior steps of one step(): while a decoder slot is free and no ready request can take it, prior steps back to
        back until a prior request finishes; otherwise one prior step while the prior batch has work."""
        if not self.prior.pending():
            return
        if None in self.queue.holder and not self.queue.waiting:
            while self.prior.pending() and not self._prior_step():
                pass
        else:
            self._prior_step()

    def _bind(self, s, r):
        """Write request r's conditioning into slot s's rows of the plan."""
        if self.w_map is None:
            self.pipe.model.bind_slot(self.plan, s, r.negative, r.positive, hint=r.hint)
        else:
            k, wenc = self._loras[r.lora] if r.lora is not None else (0, self._wenc0)
            self.pipe.model.bind_slot(self.plan, s, r.negative, r.positive, wenc=wenc, hint=r.hint)
            self._set_slab(s, k)

    def _stage(self, s, r):
        pipe, (H, W) = self.pipe, self._latent_hw
        self._bind(s, r)
        # the draws of generate_text2img(batch_size=1) with base_seed = r.seed (_DecoderBase._decode, _sampling_loop), or the
        # img2img start latent made at submit; the DDPM noise below is drawn for the rows the request runs
        x = r.start if r.start is not None else parallel.sample_noise(range(1), (4, H, W), base_seed=r.seed, device=pipe.device)
        noise = None
        if self.slots.noise_tab is not None:
            gen = pipe._generators(0, 1, base_seed=r.seed)[0]
            noise = torch.randn(r.steps, 4, H, W, device=pipe.device, generator=gen)
        self.slots.stage(s, r.ts, r.coef, x, r.guidance, noise)

    def _before_admit(self):
        if len(self._events) >= self.RUN_AHEAD:
            self._events.popleft().synchronize()   # waits for a step to end; reads nothing back
        if self.prior is not None:
            self._run_prior()

    def step(self):
        """Admit waiting requests into free slots, run one denoising step of every occupied slot (one graph replay), decode
        the requests that step finished -> {handle: PIL image}."""
        finished = self._step_slots()
        if finished is None:
            return {}
        ev = torch.cuda.Event()
        ev.record()
        self._events.append(ev)
        done = {}
        for s, handle in finished:
            done[handle] = self.pipe._finish(self.slots.x[s:s + 1], self.h, self.w)[0]
            if self.w_map is not None:
                self._set_slab(s, 0)   # idle slots use slab 0, so a removed adapter's slab is read by no slot
        return done

    def _set_slab(self, s, k):
        self.w_map[s] = k
        self.w_map[self.slots.S + s] = k

    def pending(self):
        """Whether a request is waiting for its embeddings, waiting for a slot or being denoised."""
        return super().pending() or bool(self._held)


class Batcher21(Batcher):
    """Kandinsky 2.1 requests of one geometry and one sampler served from max_batch slots (Kandinsky2_1.batcher builds it).
    Slot s owns the conditional row s and the unconditional row S + s.  Each row is conditioned on the text encoder's
    full_emb / pooled_emb and an image embedding, so the plan's context is num_image_embs + the text length.  Decoded images
    are cropped to h x w from the latent grid _new_h_w_latent_21(h, w), as generate_text2img crops them.  p_sampler's step
    clips each slot's x0 with that slot's own 99.5 percentile."""

    SAMPLERS = BATCHER_SAMPLERS_21
    TASKS = ("text2img",)

    def __init__(self, pipe, max_batch, h, w, sampler="ddim_sampler", max_steps=100, max_loras=0):
        super().__init__(pipe, max_batch, h, w, sampler=sampler, max_steps=max_steps, max_loras=max_loras)

    def _check_args(self, max_batch, h, w, sampler, max_steps, max_loras):
        super()._check_args(max_batch, h, w, sampler, max_steps, max_loras)
        if max_loras:
            raise ValueError("batcher: max_loras must be 0 for Kandinsky 2.1; per-request LoRA adapters serve 2.2 only")

    def _geometry(self, h, w):
        return (h, w) + tuple(self.pipe.get_new_h_w(h, w))

    def _image_latent(self, image):
        return super()._image_latent(image) * self.pipe.scale   # as generate_img2img scales it

    def _context(self):
        # the text rows' length is the embedder's: read it once from the embedding of ""
        self._text_len = self.pipe.embedder.text_emb("", 1)[0].shape[1]
        return self.pipe.model.num_image_embs + self._text_len

    def submit(self, prompt, *, image_embeds=None, negative_image_embeds=None, num_steps=100, guidance_scale=7,
               negative_decoder_prompt="", seed=None, image=None, strength=None):
        """Queue one image of Kandinsky2_1.generate_text2img(prompt, batch_size=1, ...) -> its handle (the key of its image in
        what step() / run() return).  The text rows are the embedder's text_emb(prompt, 1); the image rows those
        generate_text2img makes (the prior's embedding of prompt, and the zero image embedding or, with
        negative_decoder_prompt, the prior's embedding of that).  image_embeds / negative_image_embeds ([1, D] or [D]) replace
        either: prompt="" with image_embeds=embedder.interpolate(items, weights, 1) is mix_images(items, weights,
        batch_size=1).  seed plays the part of the pipeline's base_seed (default: the pipeline's base_seed).  image (a PIL image,
        an image tensor or an encoded latent) makes it Kandinsky2_1.generate_img2img(prompt, image, strength, batch_size=1),
        the image encoded now, strength defaulting to that method's default."""
        pipe = self.pipe
        if not isinstance(prompt, str):
            raise ValueError(f"submit: prompt must be a str, got {type(prompt).__name__}")
        for name, e in (("image_embeds", image_embeds), ("negative_image_embeds", negative_image_embeds)):
            _check_embedding(name, e, self._emb_dim)
        _check_int("submit", "num_steps", num_steps, 1, self.max_steps)
        _check_img2img(image, strength)
        r = self._request(guidance_scale, seed, image, strength, num_steps)
        r.full, r.pooled = pipe.embedder.text_emb(prompt, 1)
        if r.full.shape[1] != self._text_len:
            raise ValueError(f"submit: the embedder's text rows have length {r.full.shape[1]}, the batcher's {self._text_len}")
        r.positive = image_embeds if image_embeds is not None else pipe.embedder.image_emb(prompt, 1)
        r.negative = (negative_image_embeds if negative_image_embeds is not None
                      else pipe._negative_image_emb(1, negative_decoder_prompt))
        return self._enqueue(r)

    def _bind(self, s, r):
        self.pipe.model.bind_slot(self.plan, s, r.negative, r.positive, full_emb=r.full, pooled_emb=r.pooled)


# ------------------------------------------------------------------------------------------------------------------------------
# the Kandinsky 2.2 prior in continuously refilled slots
# ------------------------------------------------------------------------------------------------------------------------------
def prior_request_tables(steps, keep=None):
    """(timesteps fp32 [n], coefficient rows fp32 [n, 8]) of one prior request in loop order, n = keep or steps: the rows
    _PriorStepPlan.set_schedule stages from UnCLIPSchedule(steps, keep=keep)."""
    sched = UnCLIPSchedule(steps, keep=keep)
    return torch.from_numpy(sched.timesteps.astype(np.float32)), torch.from_numpy(sched.coef_table())


class _PriorRequest:
    __slots__ = ("steps", "guidance", "rows", "ts", "coef", "x", "noise")


class PriorBatcher(_SlotBatcher):
    """Kandinsky 2.2 prior requests served from max_batch slots (PriorEmbedder22.batcher builds it): one UnCLIP sampling step of
    every slot is ONE graph replay (SlotSteps around the prior network of a _PriorSlotPlan), each slot at its own step of its
    own tables, refilled from a FIFO queue as requests finish.  A request computes what the embedder's image_emb(prompt, 1,
    ...) -- or with an image emb2emb(prompt, image, 1, strength, ...) -- computes: the CLIP rows, guidance and generator of its
    _call_args, the same draws in the same order, UnCLIPSchedule's tables, and a slot step that runs the batch step's kernels
    on the slot's rows alone.  Its result stays on the device.  The host reads nothing back: it knows from its own
    bookkeeping which slot finishes at which step."""

    MAX_STEPS = 1000   # table rows per slot, _PriorStepPlan's limit
    WEIGHTS_CHANGED = ("prior batcher: the prior's packed weights changed after the batcher was made (load_lora, unload_lora "
                       "or a reload); make a new one")

    def __init__(self, embedder, max_batch):
        _check_int("prior batcher", "max_batch", max_batch, 1)
        self.embedder = embedder
        prior = embedder.prior
        if prior._packed is None:
            prior.finalize()
        # a plan of its own: a batch-1 image_emb call between steps must not rebind these rows
        self.plan = _PriorSlotPlan(prior, max_batch)
        # a slot's clip_dim floats as the step kernels see them, [4, 1, clip_dim / 4]; SlotSteps' defaults are the prior's
        self.slots = SlotSteps(max_batch, (4, 1, prior.clip_dim // 4), self.MAX_STEPS, self.plan.dev)
        super().__init__(max_batch)
        self._capture(self.plan.model_out.view((2 * max_batch, 8) + self.slots.x.shape[2:]))

    def _weights(self):
        return self.embedder.prior._packed, self.embedder.prior._lora

    def submit(self, prompt, *, prior_steps=None, prior_guidance_scale=None, negative_prior_prompt=None, image=None,
               strength=None):
        """Queue one image embedding -> its handle (the key of its embedding in what step() / run() return).  Without image:
        image_emb(prompt, 1, prior_steps, prior_guidance_scale, negative_prior_prompt); with one (a CLIP image embedding [1, D]
        / [D], or a PIL image for the embedder's clip_image): emb2emb(prompt, image, 1, strength, ...), strength defaulting to
        emb2emb's.  Unset keywords are the embedder's defaults."""
        return self.enqueue(self.request(prompt, prior_steps=prior_steps, prior_guidance_scale=prior_guidance_scale,
                                         negative_prior_prompt=negative_prior_prompt, image=image, strength=strength))

    def request(self, prompt, *, prior_steps=None, prior_guidance_scale=None, negative_prior_prompt=None, image=None,
                strength=None):
        """The request submit queues, checked and drawn but not queued (enqueue queues it)."""
        emb = self.embedder
        steps = emb.prior_steps if prior_steps is None else prior_steps
        _check_int("submit", "prior_steps", steps, 2, self.MAX_STEPS)
        keep = None
        if image is None and strength is not None:
            raise ValueError("submit: strength without image; strength is how much of the prior an image request runs")
        if image is not None:
            if strength is None:   # emb2emb's default
                strength = inspect.signature(type(emb).emb2emb).parameters["strength"].default
            if isinstance(strength, bool) or not isinstance(strength, (int, float)):
                raise ValueError(f"submit: strength must be a number in [0, 1], got {strength!r}")
            keep = emb._emb2emb_keep(steps, strength, who="submit")
            D = emb.prior.clip_dim
            if torch.is_tensor(image) and tuple(image.shape) not in ((D,), (1, D)):
                raise ValueError(f"submit: image must be one CLIP image embedding, [1, {D}] or [{D}], or a PIL image; got "
                                 f"{list(image.shape)}")
            start = emb._image_embedding(image, 1, who="submit: image")
        steps, g, rows, gen = emb._call_args(prompt, 1, steps, prior_guidance_scale, negative_prior_prompt)
        dev, D = emb.clip_mean.device, emb.prior.clip_dim
        r = _PriorRequest()
        # image_emb's draws: x_T, then the step noise; emb2emb's: z, then the noise of the kept steps
        x = torch.randn(1, D, device=dev, generator=gen)
        r.noise = torch.randn(steps if keep is None else keep, 1, D, device=dev, generator=gen)
        r.x = x if keep is None else UnCLIPSchedule(steps, keep=keep).start_latent(start, x)
        r.ts, r.coef = prior_request_tables(steps, keep)
        r.steps, r.guidance, r.rows = r.ts.shape[0], g, rows
        return r

    def enqueue(self, r):
        """Queue a request made by request() -> its handle."""
        return self._enqueue(r)

    def _stage(self, s, r):
        self.plan.bind_slot(s, *r.rows)
        self.slots.stage(s, r.ts, r.coef, r.x, r.guidance, r.noise)

    def step(self):
        """Admit waiting requests into free slots, run one UnCLIP step of every occupied slot (one graph replay) -> {handle:
        fp32 [1, clip_dim] on the device} of the requests it finished, each a tensor of its own (x * clip_std + clip_mean,
        as sample_prior22 finishes)."""
        emb = self.embedder
        return {handle: self.slots.x[s:s + 1].view(1, -1) * emb.clip_std + emb.clip_mean
                for s, handle in self._step_slots() or ()}


class _PriorQueue:
    """The embedder calls of the pipeline's embedding rules (Kandinsky2_2._embeds, _negative, _controlnet_img2img_embeds) at
    batch 1 as prior requests: image_emb and emb2emb return a PriorBatcher request, checked but not queued (Batcher._enqueue
    queues it once the whole decoder request is checked); zero_image_emb is the embedder's own."""

    def __init__(self, prior, embedder):
        self.prior, self.embedder = prior, embedder

    def image_emb(self, prompt, batch_size, **prior_kw):
        return self.prior.request(prompt, **prior_kw)

    def emb2emb(self, prompt, image, batch_size, strength, **prior_kw):
        return self.prior.request(prompt, image=image, strength=strength, **prior_kw)

    def zero_image_emb(self, batch_size):
        return self.embedder.zero_image_emb(batch_size)
