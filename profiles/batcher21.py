"""Serving a staggered stream of Kandinsky 2.1 text2img requests at full size (synthetic weights of the architecture, the
synthetic embedder) with p_sampler (respaced DDPM, +-2 clamp and the dynamic threshold), three ways, in one process on cuda:0:
  * batcher:  Kandinsky2_1.batcher(max_batch=4, sampler="p_sampler"): every request is submitted when it arrives and joins the
              refilled batch at the next step; each slot clips with its own request's percentile;
  * single:   the requests one at a time, generate_text2img(batch_size=1), each starting when it has arrived and the previous
              one is done;
  * groups:   fixed groups of 4 in arrival order, generate_text2img(batch_size=4), each group starting when its last request
              has arrived and the previous group is done (one prompt per group call: the compute is that of 4 requests; the
              group clips with its sample 0's percentile, as the reference does, so only its timing is comparable).
The stream and the per-arm report are those of profiles/batcher.py (the Kandinsky 2.2 stream), so the two files compare.
Also reported: the batcher's step time with all 4 slots busy, and the kernel time of the per-slot percentile
(sampler_percentile_kernel<true>, one CTA per slot, 4 slots) against the batch percentile at B = 1
(sampler_percentile_kernel<false>) on the same 96 x 96 latents, from torch.profiler in a separate pass after the timed arms.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/batcher21.py [--requests 16] [--steps 50] [--gap-steps 3] [--out profiles/batcher21_h100.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from batcher import _card, _summary, _wait_until  # noqa: E402  (profiles/batcher.py)

SAMPLER = "p_sampler"


def run_batcher(b, prompts, arrive, steps):
    t0 = time.perf_counter()
    handles, finish = {}, {}
    nxt = 0
    while len(finish) < len(prompts):
        now = time.perf_counter() - t0
        while nxt < len(prompts) and arrive[nxt] <= now:
            handles[b.submit(prompts[nxt], num_steps=steps, seed=nxt)] = nxt
            nxt += 1
        if not b.pending():
            _wait_until(t0, arrive[nxt])
            continue
        for h in b.step():
            finish[handles[h]] = time.perf_counter() - t0
    return [finish[i] for i in range(len(prompts))]


def run_calls(pipe, prompts, arrive, steps, group, size):
    t0 = time.perf_counter()
    finish = []
    for g in range(0, len(prompts), group):
        members = range(g, min(g + group, len(prompts)))
        _wait_until(t0, max(arrive[i] for i in members))
        pipe.base_seed = g
        pipe.generate_text2img(prompts[g], batch_size=len(members), num_steps=steps, h=size, w=size, sampler=SAMPLER)
        finish += [time.perf_counter() - t0] * len(members)
    return finish


def percentile_kernels_us(S, H, W, reps=200):
    """-> {kernel: mean device time in us} of the slot percentile over S busy slots and the batch one at B = 1."""
    from torch.profiler import ProfilerActivity, profile
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    f = lambda *s: torch.randn(*s, device="cuda", generator=g)
    mo, x, noise = f(2 * S, 8, H, W), 3 * f(S, 4, H, W), f(S, 4, H, W)
    coef = torch.tensor([1.2, 0.6, 0.5, 0.5, -4.0, -3.0, 1.0, 0.9], device="cuda").repeat(S, 1).contiguous()
    guid = torch.full((S,), 7.0, device="cuda")
    state = torch.tensor([[0] * S, [10 ** 9] * S], dtype=torch.int32, device="cuda")   # every slot busy for every rep
    work, sval = torch.empty_like(x), torch.empty(S, device="cuda")
    bwork = torch.empty(4 * H * W + 4096, device="cuda")
    x1, m1 = x[:1].clone(), mo[::S].contiguous()

    def both():
        ops.slot_sampler_step(mo, x, noise, coef, guid, state, work, 2.0, cond_first=1, threshold_mode=1, sval=sval)
        ops.sampler_step(m1, x1, noise[:1], coef[0], 7.0, True, clip=2.0, threshold_mode=1, work=bwork)
    for _ in range(10):
        both()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            both()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for form in ("true", "false"):
            if f"sampler_percentile_kernel<{form}>" in e.key:
                out[f"sampler_percentile_kernel<{form}>"] = round(e.device_time_total / e.count, 2)
    if len(out) != 2:
        raise SystemExit(f"profiles/batcher21.py: the profiler did not report both percentile kernels: {sorted(out)}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--gap-steps", type=float, default=3.0)
    ap.add_argument("--size", type=int, default=768)
    ap.add_argument("--max-batch", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/batcher21.py needs a CUDA sm_90 device")
    from kandinsky2 import get_kandinsky2
    card = _card()
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.1", cache_dir="/nonexistent")
    S, size, steps = args.max_batch, args.size, args.steps
    b = pipe.batcher(S, size, size, sampler=SAMPLER, max_steps=steps)
    # warm-up of every arm: plan builds, tuning, graph captures; the batcher's step time with every slot occupied
    for i in range(S):
        b.submit(f"warm-up {i}", num_steps=steps, seed=100 + i)
    b.step()
    step_ms = []
    for _ in range(8):
        t = time.perf_counter()
        b.step()
        torch.cuda.synchronize()
        step_ms.append((time.perf_counter() - t) * 1e3)
    b.run()
    pipe.generate_text2img("warm-up", batch_size=1, num_steps=2, h=size, w=size, sampler=SAMPLER)
    pipe.generate_text2img("warm-up", batch_size=S, num_steps=2, h=size, w=size, sampler=SAMPLER)
    step_s = statistics.median(step_ms) / 1e3
    prompts = [f"request {i}" for i in range(args.requests)]
    arrive = [i * args.gap_steps * step_s for i in range(args.requests)]
    res = dict(card=card, sampler=SAMPLER, size=size, steps=steps, requests=args.requests, max_batch=S,
               gap_steps=args.gap_steps, batcher_step_ms_all_slots_busy=round(step_s * 1e3, 2),
               arrival_gap_s=round(args.gap_steps * step_s, 4))
    res["batcher"] = _summary(arrive, run_batcher(b, prompts, arrive, steps))
    res["single"] = _summary(arrive, run_calls(pipe, prompts, arrive, steps, 1, size))
    res["groups"] = _summary(arrive, run_calls(pipe, prompts, arrive, steps, S, size))
    H, W = b.slots.x.shape[2:]
    res["percentile_kernel_us"] = dict(slots=S, latent=[H, W], **percentile_kernels_us(S, H, W))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
