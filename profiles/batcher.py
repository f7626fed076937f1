"""Serving a staggered stream of Kandinsky 2.2 text2img requests at full size (synthetic weights of the architecture, the
synthetic embedder), three ways, in one process on cuda:0:
  * batcher:  Kandinsky2_2.batcher(max_batch=4): every request is submitted when it arrives and joins the refilled batch at
              the next step;
  * single:   the requests one at a time, generate_text2img(batch_size=1), each starting when it has arrived and the previous
              one is done;
  * groups:   fixed groups of 4 in arrival order, generate_text2img(batch_size=4), each group starting when its last request
              has arrived and the previous group is done (one prompt per group call: the compute is that of 4 requests).
The stream: --requests requests of --steps DDPM steps at --size x --size, request i arriving at i * --gap-steps batcher steps
(the batcher's step time with all 4 slots occupied, measured in the warm-up).  Arrivals and completions are read on one host
clock; every completion ends in the device-to-host copy of the image.  Reported per arm: images/s over the whole stream (first
arrival to last completion) and each request's latency (arrival to its image).  The card's name, power limit and maximum SM
clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/batcher.py [--requests 16] [--steps 50] [--gap-steps 3] [--out profiles/batcher_h100.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _wait_until(t0, t):
    while time.perf_counter() - t0 < t:
        time.sleep(0.0005)


def _summary(arrive, finish):
    lat = [f - a for a, f in zip(arrive, finish)]
    span = max(finish) - min(arrive)
    return dict(images_per_s=round(len(lat) / span, 3), span_s=round(span, 2), latency_mean_s=round(statistics.mean(lat), 2),
                latency_median_s=round(statistics.median(lat), 2), latency_max_s=round(max(lat), 2),
                latency_s=[round(x, 2) for x in lat])


def run_batcher(b, prompts, arrive, steps):
    t0 = time.perf_counter()
    handles, finish = {}, {}
    nxt = 0
    while len(finish) < len(prompts):
        now = time.perf_counter() - t0
        while nxt < len(prompts) and arrive[nxt] <= now:
            handles[b.submit(prompts[nxt], decoder_steps=steps, seed=nxt)] = nxt
            nxt += 1
        if not b.pending():
            _wait_until(t0, arrive[nxt])
            continue
        for h in b.step():
            finish[handles[h]] = time.perf_counter() - t0
    return [finish[i] for i in range(len(prompts))]


def run_calls(pipe, prompts, arrive, steps, group, size):
    t0 = time.perf_counter()
    finish, done = [], 0.0
    for g in range(0, len(prompts), group):
        members = range(g, min(g + group, len(prompts)))
        _wait_until(t0, max(arrive[i] for i in members))
        pipe.base_seed = g
        pipe.generate_text2img(prompts[g], batch_size=len(members), decoder_steps=steps, h=size, w=size)
        done = time.perf_counter() - t0
        finish += [done] * len(members)
    return finish


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
        raise SystemExit("profiles/batcher.py needs a CUDA sm_90 device")
    from kandinsky2 import get_kandinsky2
    card = _card()
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent")
    S, size, steps = args.max_batch, args.size, args.steps
    b = pipe.batcher(S, size, size, max_steps=steps)
    # warm-up of every arm: plan builds, tuning, graph captures; the batcher's step time with every slot occupied
    for i in range(S):
        b.submit(f"warm-up {i}", decoder_steps=steps, seed=100 + i)
    b.step()
    step_ms = []
    for _ in range(8):
        t = time.perf_counter()
        b.step()
        torch.cuda.synchronize()
        step_ms.append((time.perf_counter() - t) * 1e3)
    b.run()
    pipe.generate_text2img("warm-up", batch_size=1, decoder_steps=2, h=size, w=size)
    pipe.generate_text2img("warm-up", batch_size=S, decoder_steps=2, h=size, w=size)
    step_s = statistics.median(step_ms) / 1e3
    prompts = [f"request {i}" for i in range(args.requests)]
    arrive = [i * args.gap_steps * step_s for i in range(args.requests)]
    res = dict(card=card, size=size, steps=steps, requests=args.requests, max_batch=S, gap_steps=args.gap_steps,
               batcher_step_ms_all_slots_busy=round(step_s * 1e3, 2), arrival_gap_s=round(args.gap_steps * step_s, 4))
    res["batcher"] = _summary(arrive, run_batcher(b, prompts, arrive, steps))
    res["single"] = _summary(arrive, run_calls(pipe, prompts, arrive, steps, 1, size))
    res["groups"] = _summary(arrive, run_calls(pipe, prompts, arrive, steps, S, size))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
