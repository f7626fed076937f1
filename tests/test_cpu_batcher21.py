"""CPU: the host side of the Kandinsky 2.1 batcher (batching.Batcher21) -- the per-request tables against the schedules the 2.1
sampling loops build, what Kandinsky2_1.batcher and submit refuse, and what the slot step ops refuse without a GPU."""
import numpy as np
import pytest
import torch

SAMPLERS_21 = ("p_sampler", "ddim_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")


def _bare_pipe(task_type="text2img"):
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.pipelines import Kandinsky2_1
    pipe = Kandinsky2_1.__new__(Kandinsky2_1)
    pipe.config, pipe.task_type = CONFIG_2_1, task_type
    return pipe


@pytest.mark.parametrize("sampler", SAMPLERS_21)
@pytest.mark.parametrize("steps", [2, 7, 25, 50, 100])
def test_request_tables_of_a_21_pipeline_are_its_sampling_loops(sampler, steps):
    """A request's staged tables, built from the pipeline (request_tables(pipe, ...)), are the rows _sampling_loop stages for
    Kandinsky2_1.generate_text2img(num_steps=steps): the schedule the pipeline builds for `sampler` over its _diffusion, last
    table row first."""
    from kandinsky2.batching import request_tables
    from kandinsky2.model.gaussian_diffusion import DDIMSampler
    from kandinsky2.pipelines import SCHEDULE_SAMPLERS
    pipe = _bare_pipe()
    ts, coef = request_tables(pipe, sampler, steps)
    diffusion = pipe._diffusion(sampler, steps)
    if sampler == "p_sampler":
        sched = diffusion
    elif sampler == "ddim_sampler":
        sched = DDIMSampler(None, diffusion)
        sched.make_schedule(steps)
    else:
        cls, kw = SCHEDULE_SAMPLERS[sampler]
        sched = cls(diffusion.base_alphas_cumprod, steps, **kw)
    want_coef = sched.coef_table()[::-1]
    want_ts = np.asarray(sched.model_timesteps(), dtype=np.float32)[::-1]
    n = sched.num_timesteps
    assert ts.dtype == coef.dtype == torch.float32 and coef.shape == (n, 8) and ts.shape == (n,)
    assert np.array_equal(coef.numpy(), want_coef) and np.array_equal(ts.numpy(), want_ts)
    if sampler == "p_sampler":
        # respaced to `steps`, the last step without noise, the UNet seeing the respaced timesteps
        assert n == steps and coef[-1, 6].item() == 0 and (coef[:-1, 6] == 1).all()
        assert ts.tolist() == [float(diffusion.model_timestep(i)) for i in range(steps)][::-1]
    elif sampler == "ddim_sampler":
        # raw DDIM timesteps 1, 1 + c, ... (c = 1000 // steps: more rows than steps when steps does not divide 1000), no noise
        c = 1000 // steps
        assert ts.tolist() == [float(t + 1) for t in range(0, 1000, c)][::-1]
        assert not coef[:, 4:7].any()
    else:
        assert n == steps


@pytest.mark.parametrize("kw,what", [(dict(sampler="plms_sampler"), "plms_sampler"),
                                     (dict(sampler="unipc_sampler"), "unipc_sampler"),
                                     (dict(sampler="dpmpp_2m_sde_sampler"), "dpmpp_2m_sde_sampler"),
                                     (dict(sampler="euler_sampler"), "euler_sampler"),
                                     (dict(sampler="heun_sampler"), "heun_sampler"),
                                     (dict(sampler="ddpm_sampler"), "ddpm_sampler"),
                                     (dict(max_loras=1), "max_loras"), (dict(max_loras=-1), "max_loras"),
                                     (dict(max_batch=0), "max_batch"), (dict(h=0), "h"), (dict(w=12.5), "w"),
                                     (dict(max_steps=0), "max_steps")])
def test_batcher21_refuses_by_name(kw, what):
    """Kandinsky2_1.batcher refuses a sampler it does not serve (PLMS among them), per-request LoRA and a geometry that is not
    positive, naming it, before any work (the bare object below has no model)."""
    from kandinsky2.pipelines import Kandinsky2_1
    args = dict(max_batch=4, h=512, w=512, max_steps=50)
    args.update(kw)
    pipe = Kandinsky2_1.__new__(Kandinsky2_1)
    with pytest.raises(ValueError, match=what):
        pipe.batcher(args.pop("max_batch"), args.pop("h"), args.pop("w"), **args)


@pytest.mark.parametrize("task", ["inpainting", "img2img"])
def test_batcher21_refuses_other_tasks(task):
    pipe = _bare_pipe(task)
    with pytest.raises(ValueError, match=task):
        pipe.batcher(2, 512, 512, sampler="p_sampler")


def _bare_batcher21(emb_dim=16, max_steps=10):
    from kandinsky2.batching import Batcher21, _SlotBatcher
    b = Batcher21.__new__(Batcher21)
    b.pipe, b.max_steps, b._emb_dim = None, max_steps, emb_dim
    _SlotBatcher.__init__(b, 2)
    return b


@pytest.mark.parametrize("prompt,kw,what", [
    (None, {}, "prompt"),
    ("a cat", dict(image_embeds=torch.zeros(2, 16)), "image_embeds"),
    ("a cat", dict(negative_image_embeds=torch.zeros(1, 15)), "negative_image_embeds"),
    ("a cat", dict(image_embeds=torch.zeros(16, dtype=torch.int64)), "image_embeds"),
    ("a cat", dict(num_steps=0), "num_steps"),
    ("a cat", dict(num_steps=11), "num_steps"),
    ("a cat", dict(num_steps=5.0), "num_steps")])
def test_submit21_refuses_bad_requests(prompt, kw, what):
    b = _bare_batcher21()
    with pytest.raises(ValueError, match=what):
        b.submit(prompt, **kw)
    assert not b.queue.waiting and not b._requests


@pytest.mark.parametrize("op,args", [
    ("slot_sampler_step", lambda t: ((t,) * 7, dict(cond_first=1, threshold_mode=1, sval=t))),
    ("slot_dpm_solver_step", lambda t: ((t,) * 6, dict(cond_first=1)))])
def test_slot_ops_with_row_order_and_threshold_refuse_host_tensors(op, args):
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    pos, kw = args(torch.zeros(2, 4, 8, 8))
    with pytest.raises(K2Error, match="CUDA"):
        getattr(ops, op)(*pos, **kw)
