"""Cost of the sigma-space samplers (Euler, Euler ancestral, Heun) against DPM-Solver++(2M) at the cfg-2 geometry (Kandinsky 2.2
decoder, 768x768, 4 images, guidance 4, the full-size UNet with random weights of the architecture).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * graph-replayed evaluations/s of each step kind -- k2_step_begin + UNet + the step kernel + k2_step_end, one graph launch
    per UNet evaluation: DPM++(2M) (k2_dpm_solver_step), Euler (the same kernel and graph with Euler's rows), Euler ancestral
    (k2_dpm_solver_sde_step) and Heun (k2_heun_step, its two stages alternating), the arms alternated --rounds times;
  * device time of one k2_dpm_solver_step, k2_dpm_solver_sde_step and k2_heun_step launch (stage 1 and stage 2) at this
    geometry: CUDA events over --kernel-reps back-to-back launches;
  * whole-call images/s through Kandinsky2_2.generate_text2img (latent init, the denoising loop, MoVQ decode, uint8 + PIL) for
    "dpmpp_2m_sampler" x 20, "euler_sampler" x 20, "euler_ancestral_sampler" x 20 and "heun_sampler" x 10 (19 evaluations):
    CUDA events, median of --calls steady-state calls after one warm-up call per arm.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/kdiff_steps.py [--out /tmp/kdiff_steps.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200"), os.path.join(ROOT, "profiles")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from sampler_steps import _card, _events_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=38, help="timed graph replays per evaluations/s measurement")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA sm_90 device")
    from bench import _init_pipe_with_model, build_unet
    from kandinsky2 import ops
    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.model.gaussian_diffusion import (DPMSolverSchedule, EulerSchedule, FusedStep, HeunSchedule,
                                                     create_ddpm_v22)
    from kandinsky2.pipelines import Kandinsky2_2
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.set_tuning(4, 1)  # programmatic dependent launch, as bench.py runs the step
    B, H, W = 4, 96, 96
    model = build_unet(dev)
    res = {"card": _card(), "torch": torch.__version__, "geometry": f"{B} images, {H}x{W} latents (768x768), guidance 4"}

    # ---- graph-replayed evaluations/s, the step kinds alternated
    g = torch.Generator(device=dev).manual_seed(1234)
    image_emb = torch.randn(2 * B, 1280, device=dev, generator=g)
    ac = create_ddpm_v22(50).base_alphas_cumprod
    scheds = {"dpmpp_2m_sampler x 20": DPMSolverSchedule(ac, 20), "euler_sampler x 20": EulerSchedule(ac, 20),
              "euler_ancestral_sampler x 20": EulerSchedule(ac, 20, ancestral=True), "heun_sampler x 10": HeunSchedule(ac, 10)}
    x_start = torch.randn(B, 4, H, W, device=dev, generator=g)
    noise = torch.randn(20, B, 4, H, W, device=dev, generator=g)
    arms = {}
    for name, sched in scheds.items():
        coef, ts = sched._tables(dev)
        order = torch.arange(sched.num_timesteps - 1, -1, -1, device=dev)
        step = FusedStep(model, B, H, W, dict(image_emb=image_emb), guidance_scale=4.0, cond_first=False, clip_range=2.0,
                         threshold_mode=0, step_kind=sched.step_kind)
        arms[name] = (step, ts[order], coef[order], noise[:sched.num_timesteps] if sched.draws_noise else None)
    eps_ = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, (step, ts_seq, coef_seq, nseq) in arms.items():
            step.set_schedule(ts_seq, coef_seq, nseq)
            x = step.latent()
            x.copy_(x_start)
            for _ in range(args.warmup):
                step.advance(x)
            ms = _events_ms(lambda: step.advance(x), args.steps)
            eps_[name].append(round(1e3 * args.steps / ms, 3))
    res["evaluations_per_s"] = eps_
    res["evaluations_per_s_note"] = (f"{args.steps} graph replays per run after {args.warmup} warm-up replays, arms alternated "
                                     f"{args.rounds} times; each schedule wraps around its rows (Heun: 19, both stages)")

    # ---- step-kernel device time
    mo = torch.randn(2 * B, 8, H, W, device=dev, generator=g)
    xk, hist, xs, ds, nz = (torch.randn(B, 4, H, W, device=dev, generator=g) for _ in range(5))
    coef_dpm = scheds["dpmpp_2m_sampler x 20"]._tables(dev)[0][10].clone()
    coef_anc = scheds["euler_ancestral_sampler x 20"]._tables(dev)[0][10].clone()
    heun_rows = scheds["heun_sampler x 10"]._tables(dev)[0]
    coef_h1, coef_h2 = heun_rows[10].clone(), heun_rows[9].clone()
    assert float(coef_dpm[4]) != 0.0 and float(coef_anc[7]) != 0.0 and float(coef_h1[7]) == 0.0 and float(coef_h2[7]) == 1.0
    kern = {"k2_dpm_solver_step": lambda: ops.dpm_solver_step(mo, xk, hist, coef_dpm, 4.0, False),
            "k2_dpm_solver_sde_step (Euler ancestral row)": lambda: ops.dpm_solver_step(mo, xk, hist, coef_anc, 4.0, False,
                                                                                         noise=nz),
            "k2_heun_step stage 1": lambda: ops.heun_step(mo, xk, xs, ds, coef_h1, 4.0, False),
            "k2_heun_step stage 2": lambda: ops.heun_step(mo, xk, xs, ds, coef_h2, 4.0, False)}
    for fn in kern.values():
        fn()
        _events_ms(fn, 50)
    kt = {name: {"us_per_launch": round(1e3 * _events_ms(fn, args.kernel_reps) / args.kernel_reps, 3)}
          for name, fn in kern.items()}
    n = B * 4 * H * W
    # fp32 words moved per latent element: DPM++ reads cond + uncond eps, x and hist and writes x and hist = 6; the Euler
    # ancestral row reads no history (c_P = 0) but the noise = 6; Heun stage 1 reads cond + uncond eps and x and writes x, the
    # pre-step latent and d = 6; stage 2 reads cond + uncond eps, the pre-step latent and d and writes x = 5
    words = {"k2_dpm_solver_step": 6, "k2_dpm_solver_sde_step (Euler ancestral row)": 6, "k2_heun_step stage 1": 6,
             "k2_heun_step stage 2": 5}
    for name, v in kt.items():
        v["bytes"] = 4 * n * words[name]
        v["achieved_GBps"] = round(v["bytes"] / (v["us_per_launch"] * 1e-6) / 1e9, 1)
    res["step_kernel"] = kt
    res["step_kernel_note"] = f"CUDA events over {args.kernel_reps} back-to-back launches of each kernel, cfg-2 geometry"

    # ---- whole-call images/s through the public pipeline
    arms.clear()
    model.del_cache()
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    _init_pipe_with_model(pipe, CONFIG_2_2, dev, model)
    calls = {}
    for sampler, steps in (("dpmpp_2m_sampler", 20), ("euler_sampler", 20), ("euler_ancestral_sampler", 20),
                           ("heun_sampler", 10)):
        ms_all = []
        for it in range(args.calls + 1):   # call 0 builds plans / graphs
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            pipe.generate_text2img("bench", batch_size=B, decoder_steps=steps, decoder_guidance_scale=4, h=768, w=768,
                                   sampler=sampler)
            e.record()
            torch.cuda.synchronize()
            if it > 0:
                ms_all.append(s.elapsed_time(e))
        med = sorted(ms_all)[len(ms_all) // 2]
        calls[f"{sampler} x {steps}"] = {"images_per_s": round(B / (med * 1e-3), 3), "ms_per_call": round(med, 1),
                                         "ms_per_call_all": [round(v, 1) for v in ms_all]}
    res["images_per_s"] = calls
    res["images_note"] = f"median of {args.calls} steady-state calls (CUDA events) after one warm-up call per arm"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
