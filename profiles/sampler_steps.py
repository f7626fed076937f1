"""Cost of the DPM-Solver++(2M) samplers (ODE and SDE, linspace and Karras spacing) and of UniPC against the default DDPM one at
the cfg-2 geometry (Kandinsky 2.2 decoder, 768x768, 4 images, guidance 4, the full-size UNet with random weights of the architecture).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * whole-call images/s through Kandinsky2_2.generate_text2img (latent init, the denoising steps, MoVQ decode, uint8 + PIL) for
    sampler="ddpm_sampler" x 50 steps, "dpmpp_2m_sampler" x 20 and x 25, "dpmpp_2m_sde_sampler" x 20 and
    "dpmpp_2m_karras_sampler" x 20, "unipc_sampler" x 10, 15 and 20: CUDA events, median of --calls steady-state calls after
    one warm-up call per arm;
  * graph-replayed steps/s of each step kind (k2_step_begin + UNet + k2_sampler_step, k2_dpm_solver_step,
    k2_dpm_solver_sde_step or k2_unipc_step + k2_step_end, one graph launch per step), the arms alternated --rounds times in
    this process;
  * device time of one k2_dpm_solver_step, k2_dpm_solver_sde_step, k2_unipc_step and k2_sampler_step launch (threshold mode 0,
    as the 2.2 step issues it) at this geometry: CUDA events over --kernel-reps back-to-back launches.
--arms unipc keeps only the UniPC arms and DPM++(2M), its baseline (dpmpp_2m_sampler x 20 for the whole call).
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/sampler_steps.py [--arms all|unipc] [--out /tmp/sampler_steps.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="timed graph replays per steps/s measurement")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=2000)
    ap.add_argument("--arms", default="all", choices=["all", "unipc"])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA sm_90 device")
    from bench import _init_pipe_with_model, build_unet
    from kandinsky2 import ops
    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, FusedStep, UniPCSchedule, create_ddpm_v22
    from kandinsky2.pipelines import Kandinsky2_2
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.set_tuning(4, 1)  # programmatic dependent launch, as bench.py runs the step
    B, H, W = 4, 96, 96
    model = build_unet(dev)
    res = {"card": _card(), "torch": torch.__version__, "geometry": f"{B} images, {H}x{W} latents (768x768), guidance 4"}

    # ---- graph-replayed steps/s, the two step kinds alternated
    g = torch.Generator(device=dev).manual_seed(1234)
    image_emb = torch.randn(2 * B, 1280, device=dev, generator=g)
    ddpm = create_ddpm_v22(50)
    dpm = DPMSolverSchedule(ddpm.base_alphas_cumprod, 20)
    sde = DPMSolverSchedule(ddpm.base_alphas_cumprod, 20, sde=True)
    unipc = UniPCSchedule(ddpm.base_alphas_cumprod, 20)
    only = None if args.arms == "all" else ("dpmpp_2m", "unipc")
    x_start = torch.randn(B, 4, H, W, device=dev, generator=g)
    noise = torch.randn(50, B, 4, H, W, device=dev, generator=g)
    arms = {}
    for name, sched, kind, nseq in (("ddpm_sampler", ddpm, "ddpm", noise), ("dpmpp_2m_sampler", dpm, "dpmpp_2m", None),
                                    ("dpmpp_2m_sde_sampler", sde, "dpmpp_2m_sde", noise[:20]), ("unipc_sampler", unipc, "unipc", None)):
        if only and kind not in only:
            continue
        coef, ts = sched._tables(dev)
        order = torch.arange(sched.num_timesteps - 1, -1, -1, device=dev)
        step = FusedStep(model, B, H, W, dict(image_emb=image_emb), guidance_scale=4.0, cond_first=False, clip_range=2.0,
                         threshold_mode=0, step_kind=kind)
        arms[name] = (step, ts[order], coef[order], nseq)
    sps = {name: [] for name in arms}
    for _ in range(args.rounds):
        for name, (step, ts_seq, coef_seq, nseq) in arms.items():
            step.set_schedule(ts_seq, coef_seq, nseq)
            x = step.latent()
            x.copy_(x_start)
            for _ in range(args.warmup):
                step.advance(x)
            ms = _events_ms(lambda: step.advance(x), args.steps)
            sps[name].append(round(1e3 * args.steps / ms, 3))
    res["steps_per_s"] = sps
    res["steps_per_s_note"] = (f"{args.steps} graph replays per run after {args.warmup} warm-up replays, arms alternated "
                               f"{args.rounds} times; the DPM++ and UniPC schedules wrap around their 20 rows")

    # ---- step-kernel device time
    mo = torch.randn(2 * B, 8, H, W, device=dev, generator=g)
    xk = torch.randn(B, 4, H, W, device=dev, generator=g)
    hist = torch.randn(B, 4, H, W, device=dev, generator=g)
    last, hist2 = torch.randn(B, 4, H, W, device=dev, generator=g), torch.randn(B, 4, H, W, device=dev, generator=g)
    nz = torch.randn(B, 4, H, W, device=dev, generator=g)
    work = torch.empty(B * 4 * H * W + 4096, device=dev)
    coef_ddpm = ddpm._tables(dev)[0][25].clone()
    coef_dpm = dpm._tables(dev)[0][10].clone()
    coef_sde = sde._tables(dev)[0][10].clone()
    coef_unipc = unipc._tables(dev)[0][10].clone()
    assert float(coef_dpm[4]) != 0.0 and float(coef_sde[4]) != 0.0 and float(coef_sde[7]) != 0.0  # history and noise are read
    assert all(float(coef_unipc[i]) != 0.0 for i in (3, 5, 6, 9))                                 # last, D_{k-1}, D_{k-2} too
    kern = {"k2_sampler_step": lambda: ops.sampler_step(mo, xk, nz, coef_ddpm, 4.0, False, 2.0, 0, work=work),
            "k2_dpm_solver_step": lambda: ops.dpm_solver_step(mo, xk, hist, coef_dpm, 4.0, False),
            "k2_dpm_solver_sde_step": lambda: ops.dpm_solver_step(mo, xk, hist, coef_sde, 4.0, False, noise=nz),
            "k2_unipc_step": lambda: ops.unipc_step(mo, xk, last, hist, hist2, coef_unipc, 4.0, False)}
    if only:
        kern = {k: v for k, v in kern.items() if k in ("k2_dpm_solver_step", "k2_unipc_step")}
    kt = {}
    for name, fn in kern.items():
        fn()
        _events_ms(fn, 50)
    for name, fn in kern.items():
        kt[name] = {"us_per_launch": round(1e3 * _events_ms(fn, args.kernel_reps) / args.kernel_reps, 3)}
    n = B * 4 * H * W
    # fp32 words moved per latent element: DDPM reads cond + uncond eps, the variance, x (twice: one per kernel), the noise,
    # writes and re-reads x0 through a scratch buffer and writes x = 9; DPM++ reads cond + uncond eps, x and hist and writes
    # x and hist = 6; the SDE step also reads the noise = 7; UniPC reads cond + uncond eps, x, last, D_{k-1} and D_{k-2} and writes
    # x, last and both history slots = 10
    words = {"k2_sampler_step": 9, "k2_dpm_solver_step": 6, "k2_dpm_solver_sde_step": 7, "k2_unipc_step": 10}
    for name in kt:
        kt[name]["bytes"] = 4 * n * words[name]
    for v in kt.values():
        v["achieved_GBps"] = round(v["bytes"] / (v["us_per_launch"] * 1e-6) / 1e9, 1)
    res["step_kernel"] = kt
    res["step_kernel_note"] = f"CUDA events over {args.kernel_reps} back-to-back launches of each kernel, cfg-2 geometry"

    # ---- whole-call images/s through the public pipeline
    arms.clear()
    model.del_cache()
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    _init_pipe_with_model(pipe, CONFIG_2_2, dev, model)
    calls = {}
    call_arms = (("ddpm_sampler", 50), ("dpmpp_2m_sampler", 20), ("dpmpp_2m_sampler", 25), ("dpmpp_2m_sde_sampler", 20),
                 ("dpmpp_2m_karras_sampler", 20), ("unipc_sampler", 10), ("unipc_sampler", 15), ("unipc_sampler", 20))
    if only:
        call_arms = (("dpmpp_2m_sampler", 20), ("unipc_sampler", 10), ("unipc_sampler", 15), ("unipc_sampler", 20))
    for sampler, steps in call_arms:
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
