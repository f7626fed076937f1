"""CPU: the host side of the continuously refilled batch (kandinsky2/batching.py) -- admission order and slot reuse, the
per-request tables against the schedule builders the sampling loop uses, what a batcher refuses, and the argument checks of
the slot entry points without a GPU."""
import ctypes

import pytest
import torch


def test_admission_is_fifo_into_the_lowest_free_slot_and_slots_are_reused():
    from kandinsky2.batching import SlotQueue
    q = SlotQueue(3)
    for name, steps in (("a", 2), ("b", 4), ("c", 1), ("d", 3), ("e", 2)):
        q.submit(name, steps)
    assert q.admit() == [(0, "a"), (1, "b"), (2, "c")] and [h for h, _ in q.waiting] == ["d", "e"]
    assert q.advance() == [(2, "c")]
    assert q.admit() == [(2, "d")]
    assert q.advance() == [(0, "a")]
    assert q.admit() == [(0, "e")] and not q.waiting
    assert q.advance() == []
    assert q.holder == ["e", "b", "d"] and q.left == [1, 1, 1] and q.busy()
    assert q.advance() == [(0, "e"), (1, "b"), (2, "d")] and not q.busy() and q.admit() == []


@pytest.mark.parametrize("sampler", ["ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler"])
@pytest.mark.parametrize("steps", [2, 7, 50, 100])
def test_request_tables_of_a_22_pipeline_are_its_sampling_loops(sampler, steps):
    """A request's staged tables, built from the pipeline (request_tables(pipe, ...)), are the rows _sampling_loop stages for
    Kandinsky2_2.generate_text2img(decoder_steps=steps): the schedule's coefficient table and model timesteps, last table row
    first."""
    import numpy as np
    from kandinsky2.batching import request_tables
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22
    from kandinsky2.pipelines import SCHEDULE_SAMPLERS, Kandinsky2_2
    ts, coef = request_tables(Kandinsky2_2.__new__(Kandinsky2_2), sampler, steps)
    d = create_ddpm_v22(steps)
    if sampler == "ddpm_sampler":
        sched = d
    else:
        cls, kw = SCHEDULE_SAMPLERS[sampler]
        sched = cls(d.base_alphas_cumprod, steps, **kw)
    want_coef = sched.coef_table()[::-1]
    want_ts = np.asarray(sched.model_timesteps(), dtype=np.float32)[::-1]
    assert ts.dtype == coef.dtype == torch.float32 and coef.shape == (steps, 8) and ts.shape == (steps,)
    assert np.array_equal(coef.numpy(), want_coef) and np.array_equal(ts.numpy(), want_ts)
    if sampler == "ddpm_sampler":
        assert ts[0].item() == (steps - 1) * (1000 // steps) and ts[-1].item() == 0 and coef[-1, 6].item() == 0


@pytest.mark.parametrize("kw,what", [(dict(sampler="unipc_sampler"), "unipc_sampler"),
                                     (dict(sampler="euler_ancestral_sampler"), "euler_ancestral_sampler"),
                                     (dict(sampler="p_sampler"), "p_sampler"),
                                     (dict(max_batch=0), "max_batch"), (dict(max_batch=2.0), "max_batch"),
                                     (dict(h=0), "h"), (dict(w=-64), "w"), (dict(h=512.5), "h"),
                                     (dict(max_steps=0), "max_steps")])
def test_batcher_refuses_sampler_and_geometry(kw, what):
    """Kandinsky2_2.batcher refuses a sampler it does not serve and a geometry that is not positive, naming it, before any work
    (the bare object below has no model)."""
    from kandinsky2.pipelines import Kandinsky2_2
    args = dict(max_batch=4, h=512, w=512, sampler="ddpm_sampler", max_steps=50)
    args.update(kw)
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    with pytest.raises(ValueError, match=what):
        pipe.batcher(args.pop("max_batch"), args.pop("h"), args.pop("w"), **args)


def test_batcher_refuses_other_tasks():
    from kandinsky2.pipelines import Kandinsky2_2
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    pipe.task_type = "inpainting"
    with pytest.raises(ValueError, match="inpainting"):
        pipe.batcher(2, 512, 512)


P = ctypes.c_void_p(256)   # never dereferenced: every call below fails its checks first
# entry point -> (its arguments before the stream, all valid; [(the changed arguments, the message)]); each message
# names the entry point without its k2_ prefix
SLOT_ARGUMENTS = {
    "k2_slot_step_begin": (
        [P, P, 4, 64, P, P, P, P, 10, P, P, P],
        [({0: None}, "null pointer"), ({1: None}, "null pointer"), ({4: None}, "null pointer"), ({5: None}, "null pointer"),
         ({6: None}, "null pointer"), ({7: None}, "null pointer"), ({11: None}, "null pointer"), ({2: 0}, "S in"),
         ({2: 70000}, "S in"), ({3: 0}, "n and kmax"), ({8: 0}, "n and kmax"), ({10: None}, "noise_tab without")]),
    "k2_slot_step_end": ([P, 4], [({0: None}, "null state"), ({1: 0}, "S must be")]),
    "k2_slot_sampler_step": (
        [P, P, P, P, P, P, 4, 8, 8, 2.0, 1, 1, P, P],
        [({i: None}, "null pointer") for i in (0, 1, 2, 3, 4, 5, 13)]
        + [({6: 0}, "must be >= 1"), ({7: 0}, "must be >= 1"), ({8: -2}, "must be >= 1"),
           ({10: 2}, "cond_first must be 0 or 1"), ({10: -1}, "cond_first must be 0 or 1"),
           ({11: 2}, "threshold_mode must be 0 or 1"), ({11: 3}, "threshold_mode must be 0 or 1"),
           ({11: -1}, "threshold_mode must be 0 or 1"), ({12: None}, "threshold_mode 1 needs sval")]),
    "k2_slot_dpm_solver_step": (
        [P, 8, P, P, P, P, P, 4, 8, 8, 1],
        [({i: None}, "null pointer") for i in (0, 2, 3, 4, 5, 6)]
        + [({1: 3}, "C2 >= 4"), ({7: 0}, "must be >= 1"), ({9: 0}, "must be >= 1"), ({10: 2}, "cond_first must be 0 or 1"),
           ({10: -1}, "cond_first must be 0 or 1")]),
}


SLOT_CASES = [(name, changes, msg) for name, (_, cases) in sorted(SLOT_ARGUMENTS.items()) for changes, msg in cases]


@pytest.mark.parametrize("name,changes,msg", SLOT_CASES,
                         ids=[f"{n}-{','.join(f'{i}={v}' for i, v in c.items())}" for n, c, _ in SLOT_CASES])
def test_slot_entry_point_refuses_each_bad_argument_without_a_gpu(name, changes, msg):
    """Each bad argument alone makes the entry point fail before any CUDA call, with a message that names the entry point."""
    from kandinsky2 import _native
    lib = _native.load()
    args = list(SLOT_ARGUMENTS[name][0])
    for i, v in changes.items():
        args[i] = v
    assert getattr(lib, name)(*args, None) != 0
    err = lib.k2_last_error().decode()
    assert msg in err and f"{name[3:]}: " in err, err


@pytest.mark.parametrize("op,args", [("slot_step_end", lambda t: (t,)),
                                     ("slot_sampler_step", lambda t: (t, t, t, t, t, t, t)),
                                     ("slot_dpm_solver_step", lambda t: (t, t, t, t, t, t))])
def test_slot_ops_refuse_host_tensors(op, args):
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    with pytest.raises(K2Error, match="CUDA"):
        getattr(ops, op)(*args(torch.zeros(2, 4, 8, 8)))


def _bare_batcher(slots=2, emb_dim=16, max_steps=10):
    """A Batcher with its host state only (no pipeline, plan or graph): enough for submit's checks and the admission loop."""
    from kandinsky2.batching import Batcher, SlotSteps, _SlotBatcher
    b = Batcher.__new__(Batcher)
    b.pipe, b.max_steps, b._emb_dim = None, max_steps, emb_dim
    _SlotBatcher.__init__(b, slots)
    b.slots = SlotSteps(slots, (4, 1, 1), max_steps, "cpu")
    b.slots.state.fill_(7)
    return b


@pytest.mark.parametrize("pos,neg,what", [(torch.zeros(2, 16), torch.zeros(1, 16), "image_embeds"),
                                          (torch.zeros(1, 15), torch.zeros(1, 16), "image_embeds"),
                                          (torch.zeros(16), torch.zeros(1, 1, 16), "negative_image_embeds"),
                                          (torch.zeros(16, dtype=torch.int64), torch.zeros(16), "image_embeds"),
                                          (torch.zeros(16), [0.0] * 16, "negative_image_embeds")])
def test_submit_refuses_embeddings_of_another_shape(pos, neg, what):
    """image_embeds / negative_image_embeds must be one embedding of the UNet's width, [1, D] or [D]: anything else is refused
    at submit, naming the argument, before it can reach a slot."""
    b = _bare_batcher()
    with pytest.raises(ValueError, match=what):
        b.submit(image_embeds=pos, negative_image_embeds=neg, decoder_steps=5)
    assert not b.queue.waiting and not b._requests


def test_failed_admission_frees_its_slot_and_keeps_the_queue():
    """A request whose staging raises gives its slot back and leaves the device state of that slot idle; the requests behind it
    stay waiting, in order, and none of them holds a slot whose buffers were never written."""
    b = _bare_batcher(slots=3)
    for h in range(4):
        b._requests[h] = h
        b.queue.submit(h, 5)
    staged = []

    def stage(s, r):
        if r == 1:
            raise RuntimeError("bad embedding")
        staged.append((s, r))
    b._stage = stage
    with pytest.raises(RuntimeError, match="bad embedding"):
        b._admit()
    assert staged == [(0, 0)] and b.queue.holder == [0, None, None] and [h for h, _ in b.queue.waiting] == [2, 3]
    assert b.slots.state[:, 1].tolist() == [-1, 0] and 1 not in b._requests
    b._admit()
    assert staged == [(0, 0), (1, 2), (2, 3)] and b.queue.holder == [0, 2, 3]
