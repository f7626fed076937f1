"""CPU: what every schedule sampler shares on the host -- the one name table (pipelines.SCHEDULE_SAMPLERS), the pipelines'
sampler-name check, the argument checks of the four solver step entry points and their ops wrappers without a GPU, and the
grids of the schedules that came before the sigma-space ones."""
import ctypes

import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests.sampler_cases import _ac22


def test_schedule_samplers_table():
    """Each name maps to its schedule class and keywords; SAMPLERS_21 / SAMPLERS_22 are each version's own samplers and
    these."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, EulerSchedule, HeunSchedule, UniPCSchedule
    from kandinsky2.pipelines import SAMPLERS_21, SAMPLERS_22, SCHEDULE_SAMPLERS
    assert SCHEDULE_SAMPLERS == {
        "dpmpp_2m_sampler": (DPMSolverSchedule, dict(spacing="linspace", sde=False)),
        "dpmpp_2m_karras_sampler": (DPMSolverSchedule, dict(spacing="karras", sde=False)),
        "dpmpp_2m_sde_sampler": (DPMSolverSchedule, dict(spacing="linspace", sde=True)),
        "dpmpp_2m_sde_karras_sampler": (DPMSolverSchedule, dict(spacing="karras", sde=True)),
        "unipc_sampler": (UniPCSchedule, dict(spacing="linspace")),
        "unipc_karras_sampler": (UniPCSchedule, dict(spacing="karras")),
        "euler_sampler": (EulerSchedule, dict(spacing="linspace")),
        "euler_karras_sampler": (EulerSchedule, dict(spacing="karras")),
        "euler_ancestral_sampler": (EulerSchedule, dict(spacing="linspace", ancestral=True)),
        "heun_sampler": (HeunSchedule, dict(spacing="linspace")),
        "heun_karras_sampler": (HeunSchedule, dict(spacing="karras"))}
    assert set(SAMPLERS_21) == {"p_sampler", "ddim_sampler", "plms_sampler"} | set(SCHEDULE_SAMPLERS)
    assert set(SAMPLERS_22) == {"ddpm_sampler"} | set(SCHEDULE_SAMPLERS)


# every pipeline method that takes a sampler: (version, method, its other arguments, its keywords)
SAMPLER_METHODS = [("2.1", "generate_text2img", ("x",), dict(num_steps=4)),
                   ("2.1", "mix_images", (["a"], [1.0]), dict(num_steps=4)),
                   ("2.1", "generate_img2img", ("x", None), dict(num_steps=4)),
                   ("2.1", "generate_inpainting", ("x", None, None), dict(num_steps=4)),
                   ("2.1", "generate_img", ("x", None), {}),
                   ("2.2", "generate_text2img", ("x",), {}),
                   ("2.2", "mix_images", (["a"], [1.0]), {}),
                   ("2.2", "generate_img2img", ("x", None), {}),
                   ("2.2", "generate_inpainting", ("x", None, None), {}),
                   ("2.2", "generate_controlnet", ("x", None), {}),
                   ("2.2", "generate_controlnet_img2img", ("x", None, None), {})]
UNKNOWN = ("euler", "heun", "dpmpp_2m", "unipc", "unipc_bh1_sampler", "uni_pc_sampler", "unipc_sde_sampler", "euler_a_sampler",
           "heun_ancestral_sampler", "euler_ancestral_karras_sampler", "dpm2_sampler")


@pytest.mark.parametrize("version,method,args,kw", SAMPLER_METHODS, ids=[f"{v}-{m}" for v, m, _, _ in SAMPLER_METHODS])
def test_pipelines_accept_every_sampler_and_reject_unknown_ones(version, method, args, kw):
    """The method gets past the sampler-name check with each of its version's names (the bare object below then fails for
    lack of an embedder, which is not a sampler-name error), and refuses unknown names, and the other version's own
    samplers, before doing any work."""
    from kandinsky2.pipelines import SAMPLERS_21, SAMPLERS_22, Kandinsky2_1, Kandinsky2_2
    cls, names, bad = ((Kandinsky2_1, SAMPLERS_21, UNKNOWN + ("ddpm_sampler",)) if version == "2.1" else
                       (Kandinsky2_2, SAMPLERS_22, UNKNOWN + ("p_sampler", "ddim_sampler", "plms_sampler")))
    call = getattr(cls.__new__(cls), method)
    for name in names:
        with pytest.raises(Exception) as ei:
            call(*args, sampler=name, **kw)
        assert "unknown sampler" not in str(ei.value), (name, ei.value)
    for name in bad:
        with pytest.raises(ValueError, match="unknown sampler"):
            call(*args, sampler=name, **kw)


P = ctypes.c_void_p(256)   # never dereferenced: every call below fails its checks first
# entry point -> (its arguments before the stream, all valid; [(the changed arguments, the message)])
STEP_ARGUMENTS = {
    "k2_dpm_solver_step": (
        [P, 8, P, P, P, 2, 4, 4, 4.0, 1, None, None, None],
        [({0: None}, "null pointer"), ({2: None}, "null pointer"), ({3: None}, "null pointer"), ({4: None}, "null pointer"),
         ({1: 3}, "C2 >= 4"), ({5: 0}, "must be >= 1"), ({6: 0}, "must be >= 1"), ({7: -1}, "must be >= 1"),
         ({10: P}, "init and mask go together"), ({11: P}, "init and mask go together"),
         ({12: P}, "inpaint_noise without init")]),
    "k2_dpm_solver_sde_step": (
        [P, 8, P, P, P, P, 2, 4, 4, 4.0, 1, None, None, None],
        [({4: None}, "null noise"), ({0: None}, "null pointer"), ({2: None}, "null pointer"), ({3: None}, "null pointer"),
         ({5: None}, "null pointer"), ({1: 3}, "C2 >= 4"), ({6: 0}, "must be >= 1"), ({7: 0}, "must be >= 1"),
         ({8: -1}, "must be >= 1"), ({11: P}, "init and mask go together"), ({12: P}, "init and mask go together"),
         ({13: P}, "inpaint_noise without init")]),
    "k2_unipc_step": (
        [P, 8, P, P, P, P, P, None, 2, 4, 4, 4.0, 1, None, None, None],
        [({0: None}, "null pointer"), ({2: None}, "null pointer"), ({3: None}, "null pointer"), ({4: None}, "null pointer"),
         ({5: None}, "null pointer"), ({6: None}, "null pointer"), ({1: 3}, "C2 >= 4"), ({8: 0}, "must be >= 1"),
         ({9: 0}, "must be >= 1"), ({10: -1}, "must be >= 1"), ({13: P}, "init and mask go together"),
         ({14: P}, "init and mask go together"), ({15: P}, "inpaint_noise without init")]),
    "k2_heun_step": (
        [P, 8, P, P, P, P, 2, 4, 4, 4.0, 1, None, None, None],
        [({0: None}, "null pointer"), ({2: None}, "null pointer"), ({3: None}, "null pointer"), ({4: None}, "null pointer"),
         ({5: None}, "null pointer"), ({1: 3}, "C2 >= 4"), ({6: 0}, "must be >= 1"), ({7: 0}, "must be >= 1"),
         ({8: -1}, "must be >= 1"), ({11: P}, "init and mask go together"), ({12: P}, "init and mask go together"),
         ({13: P}, "inpaint_noise without init")]),
}


@pytest.mark.parametrize("entry", list(STEP_ARGUMENTS))
def test_step_argument_errors_without_gpu(entry):
    """Each solver step entry point checks its arguments before any CUDA call: < 0 and a message naming the entry point, also
    on a machine without a GPU."""
    from kandinsky2 import _native
    lib = _native.load()
    ok, cases = STEP_ARGUMENTS[entry]
    for change, msg in cases:
        args = list(ok)
        for i, v in change.items():
            args[i] = v
        assert getattr(lib, entry)(*args, None) < 0, change
        err = lib.k2_last_error().decode()
        assert msg in err and entry[len("k2_"):] in err, (change, err)


# ops wrapper -> a call of it on CPU tensors (model output, a [1, 4, 8, 8] zero latent z)
STEP_CALLS = {
    "dpm_solver_step": lambda ops, mo, z: ops.dpm_solver_step(mo, z.clone(), z.clone(), torch.zeros(8), 4.0, True),
    "dpm_solver_sde_step": lambda ops, mo, z: ops.dpm_solver_step(mo, z.clone(), z.clone(), torch.zeros(8), 4.0, True,
                                                                  noise=z.clone()),
    "unipc_step": lambda ops, mo, z: ops.unipc_step(mo, z.clone(), z.clone(), z.clone(), z.clone(), torch.zeros(16), 4.0, True),
    "heun_step": lambda ops, mo, z: ops.heun_step(mo, z.clone(), z.clone(), z.clone(), torch.zeros(8), 4.0, True),
}


@pytest.mark.parametrize("step", list(STEP_CALLS))
def test_step_without_gpu_raises(step):
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only failure mode")
    with pytest.raises(K2Error):
        STEP_CALLS[step](ops, torch.zeros(2, 8, 8, 8), torch.zeros(1, 4, 8, 8))


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_existing_schedules_unchanged(spacing):
    """DPMSolverSchedule's grid is the restatement of its spacing (bit for bit: the oracle's linspace grid, or Karras sigmas
    through alpha = 1 / sqrt(1 + s^2)) and its rows are still 8 floats; the DPM++ and UniPC schedules keep a start noise
    scale of 1 and the solver grid; the DDPM table keeps its shape and step kind."""
    from kandinsky2.model.gaussian_diffusion import (DPMSolverSchedule, UniPCSchedule, _solver_grid, create_ddpm_v22,
                                                     karras_timesteps)
    ac = _ac22()
    for n in (1, 7, 20):
        if spacing == "linspace":
            sch = DPMSolverSchedule(ac, n)
            tau, alpha, sigma = do.grid(ac, n)
            assert np.array_equal(sch.timesteps, tau) and np.array_equal(sch.alphas, alpha) and np.array_equal(sch.sigmas, sigma)
            assert sch.step_kind == "dpmpp_2m"
        else:
            sch = DPMSolverSchedule(ac, n, spacing="karras", sde=True)
            t, s_hat = karras_timesteps(ac, n)
            a = 1.0 / np.sqrt(1.0 + s_hat ** 2)
            assert np.array_equal(sch.timesteps, t) and np.array_equal(sch.alphas[:-1], a)
            assert np.array_equal(sch.sigmas[:-1], s_hat * a)
            assert sch.step_kind == "dpmpp_2m_sde"
        assert sch.coef_table().shape == (n, 8)
    for cls in (DPMSolverSchedule, UniPCSchedule):
        sch = cls(ac, 10, spacing=spacing)
        tau, alpha, sigma = _solver_grid("x", ac, 10, spacing)
        assert sch.init_noise_scale == 1.0 and np.array_equal(sch.timesteps, tau) and np.array_equal(sch.alphas[:-1], alpha)
    d = create_ddpm_v22(50)
    assert d.coef_table().shape == (50, 8) and d.step_kind == "ddpm"
