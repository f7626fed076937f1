"""Serving the ControlNet notebook's stream -- Kandinsky 2.2 ControlNet-depth img2img requests, each with its own image, depth
hint and strength -- at full size (synthetic weights of the architecture, the synthetic embedder), three ways, in one process
on cuda:0:
  * batcher:  Kandinsky2_2(task_type="controlnet").batcher(max_batch=4): every request is submitted when it arrives (its image
              MoVQ-encoded then) and joins the refilled batch at the next step, running only the steps its strength keeps;
  * single:   the requests one at a time, generate_controlnet_img2img(batch_size=1), each starting when it has arrived and the
              previous one is done;
  * groups:   fixed groups of 4 in arrival order, generate_controlnet_img2img(batch_size=4) at the largest strength of the
              group (a fixed group runs as long as its longest member), each group starting when its last request has arrived
              and the previous group is done (one image and hint per group call: the compute is that of 4 requests).
The stream: --requests requests of --steps DDPM steps at --size x --size, strengths alternating 0.5 / 0.3 (25 and 15 of 50
steps kept), request i arriving at i * --gap-steps batcher steps (the batcher's step time with all 4 slots occupied, measured in
the warm-up).  Arrivals and completions are read on one host clock; every completion ends in the device-to-host copy of the
image.  Reported per arm: images/s over the whole stream (first arrival to last completion) and each request's latency
(arrival to its image).  Also reported: the admission cost of one request, split into the MoVQ encode of its image (at
submit), the hint stem at the plan's 2 S rows and the whole bind_slot it runs in (at admission), and the image embeddings
(at submit; here the synthetic embedder's).  The card's name, power limit and maximum SM clock are read in the same run
(nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/batcher_controlnet.py [--requests 16] [--steps 50] [--gap-steps 3] [--out profiles/batcher_controlnet.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from batcher import _card, _summary, _wait_until  # noqa: E402  (profiles/batcher.py)

STRENGTHS = (0.5, 0.3)


def _photo(size, seed):
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((size, size, 3)) * 255).astype("uint8"))


def run_batcher(b, reqs, arrive, steps):
    t0 = time.perf_counter()
    handles, finish = {}, {}
    nxt = 0
    while len(finish) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrive[nxt] <= now:
            prompt, image, hint, strength = reqs[nxt]
            handles[b.submit(prompt, image=image, hint=hint, strength=strength, decoder_steps=steps, seed=nxt)] = nxt
            nxt += 1
        if not b.pending():
            _wait_until(t0, arrive[nxt])
            continue
        for h in b.step():
            finish[handles[h]] = time.perf_counter() - t0
    return [finish[i] for i in range(len(reqs))]


def run_calls(pipe, reqs, arrive, steps, group, size):
    t0 = time.perf_counter()
    finish = []
    for g in range(0, len(reqs), group):
        members = range(g, min(g + group, len(reqs)))
        _wait_until(t0, max(arrive[i] for i in members))
        prompt, image, hint, _ = reqs[g]
        pipe.base_seed = g
        pipe.generate_controlnet_img2img(prompt, image, hint, strength=max(reqs[i][3] for i in members),
                                         batch_size=len(members), decoder_steps=steps, h=size, w=size)
        finish += [time.perf_counter() - t0] * len(members)
    return finish


def _ms(fn, reps=10):
    """Median wall time of fn() in ms, each call ending in a device synchronise."""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return round(statistics.median(out), 2)


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
        raise SystemExit("profiles/batcher_controlnet.py needs a CUDA sm_90 device")
    from kandinsky2 import get_kandinsky2
    card = _card()
    pipe = get_kandinsky2("cuda", task_type="controlnet", model_version="2.2", cache_dir="/nonexistent")
    S, size, steps = args.max_batch, args.size, args.steps
    reqs = [(f"request {i}", _photo(size, i), torch.rand(1, 3, size, size, generator=torch.Generator().manual_seed(1000 + i)),
             STRENGTHS[i % 2]) for i in range(args.requests)]
    b = pipe.batcher(S, size, size, max_steps=steps)
    # warm-up of every arm: plan builds, tuning, graph captures; the batcher's step time with every slot occupied
    for i in range(S):
        b.submit(f"warm-up {i}", image=reqs[i][1], hint=reqs[i][2], strength=1.0, decoder_steps=steps, seed=100 + i)
    b.step()
    step_ms = []
    for _ in range(8):
        t = time.perf_counter()
        b.step()
        torch.cuda.synchronize()
        step_ms.append((time.perf_counter() - t) * 1e3)
    b.run()
    for n in (1, S):
        pipe.generate_controlnet_img2img("warm-up", reqs[0][1], reqs[0][2], strength=0.3, batch_size=n, decoder_steps=2,
                                         h=size, w=size)
    step_s = statistics.median(step_ms) / 1e3
    # the admission cost of one request, split
    model, plan = pipe.model, b.plan
    hint_rows = torch.zeros(2 * S, 3, size, size, device=pipe.device)
    hint_rows[0] = hint_rows[S] = reqs[0][2][0].to(pipe.device)
    pos, neg = pipe._embeds("request 0", 1, "", None)
    admission = dict(
        movq_encode_ms=_ms(lambda: pipe._encode_image(reqs[0][1], size, size)),
        hint_stem_2S_rows_ms=_ms(lambda: model.hint_features(hint_rows)),
        bind_slot_ms=_ms(lambda: model.bind_slot(plan, 0, neg, pos, hint=reqs[0][2].to(pipe.device))),
        embeddings_ms=_ms(lambda: pipe._embeds("request 0", 1, "", None)))
    arrive = [i * args.gap_steps * step_s for i in range(args.requests)]
    res = dict(card=card, size=size, steps=steps, strengths=list(STRENGTHS),
               kept_steps=[int(steps * s) for s in STRENGTHS], requests=args.requests, max_batch=S,
               gap_steps=args.gap_steps, batcher_step_ms_all_slots_busy=round(step_s * 1e3, 2),
               arrival_gap_s=round(args.gap_steps * step_s, 4), admission=admission)
    res["batcher"] = _summary(arrive, run_batcher(b, reqs, arrive, steps))
    res["single"] = _summary(arrive, run_calls(pipe, reqs, arrive, steps, 1, size))
    res["groups"] = _summary(arrive, run_calls(pipe, reqs, arrive, steps, S, size))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
