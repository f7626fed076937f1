"""Serving Kandinsky 2.2 text2img with a real prior: the continuous batcher with the prior run at submit (prior_slots=0, one
batch-1 prior call per request, which blocks the host) against the batcher that samples the prior in 4 refilled slots
(prior_slots=4), in one process on cuda:0.  Everything is at full size with synthetic weights of the architecture: the UNet
and MoVQ of get_kandinsky2, the 2.2 prior (20 layers, width 2048, clip_dim 1280) and the ViT-bigG/14 CLIP text tower with a
synthetic BPE vocabulary.
The streams: --requests prompts at --size x --size, request i arriving at i * --gap-steps batcher steps (the decoder batcher's
step time with all 4 slots busy, measured in the warm-up); 50 DDPM steps, and then --dpm-steps dpmpp_2m_sampler steps; prior
defaults (25 steps, guidance 4).  The two arms run alternately, --rounds times each per stream.  Arrivals and completions are
read on one host clock; every completion ends in the device-to-host copy of the image.  Reported per arm and round:
images/s over the stream (first arrival to last completion) and each request's latency (arrival to its image).  Also
reported, with CUDA events over --reps replays after warm-up: one prior slot step at 8 rows (4 slots, all busy; its GEMMs
pinned to the batch-1 configurations), one step of the batch plan at B = 4 (8 rows, the GEMM configurations picked for 8
rows: what the pinning costs), one decoder step with 4 busy slots, and a prior and a decoder step replayed back to back.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90
device.

    python profiles/batcher_prior.py [--requests 16] [--gap-steps 3] [--rounds 2] [--out profiles/batcher_prior.json]
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

import torch  # noqa: E402

from batcher import _card, _summary, _wait_until  # noqa: E402  (profiles/batcher.py)


def _embedder():
    """PriorEmbedder22 at the released geometry: the synthetic full-size prior and bigG text tower."""
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower, CLIPTokenizer
    from kandinsky2.model.prior import PriorEmbedder22
    from tests import clip_text_oracle as cto
    from tests import prior22_oracle as p22
    from tests.test_gpu_zz_prior22 import _prior_from_diffusers
    prior, dsd = _prior_from_diffusers(p22.CONFIG_PRIOR22, seed=11, round_gemm=True)
    del dsd
    cfg = cto.CONFIG_BIGG
    fx = torch.load(cto.FIXTURE)
    tok = CLIPTokenizer(cto.synthetic_vocab(fx["merges"]), [tuple(m) for m in fx["merges"]], model_max_length=77)
    sd16 = {k: v.cuda().half() for k, v in cto.synth_weights(cfg, 1).items()}
    tower = CLIPTextTower(transformers_clip_text_to_k2(sd16), cfg, device="cuda", tokenizer=tok).finalize()
    del sd16
    torch.cuda.empty_cache()
    g = torch.Generator(device="cuda").manual_seed(3)
    D = prior.clip_dim
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    return PriorEmbedder22(prior, tower, mean, std, zero_image_emb=torch.randn(1, D, generator=torch.Generator().manual_seed(4)))


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


def _event_ms(fn, reps):
    """Median device time of fn() in ms over reps calls, CUDA events around each."""
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    fn()
    torch.cuda.synchronize()
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    return round(statistics.median(evs[i].elapsed_time(evs[i + 1]) for i in range(reps)), 3)


def _fill(b, steps):
    """Every decoder slot (and prior slot) of b busy for at least `steps` more replays."""
    for i in range(b.slots.S):
        b.submit(f"warm-up {i}", decoder_steps=steps, seed=100 + i)
    while b.queue.waiting or (b.prior is not None and b._held):
        b.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--dpm-steps", type=int, default=20)
    ap.add_argument("--gap-steps", type=float, default=3.0)
    ap.add_argument("--size", type=int, default=768)
    ap.add_argument("--max-batch", type=int, default=4)
    ap.add_argument("--prior-slots", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/batcher_prior.py needs a CUDA sm_90 device")
    from kandinsky2 import get_kandinsky2
    card = _card()
    emb = _embedder()
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent", embedder=emb)
    S, P, size = args.max_batch, args.prior_slots, args.size
    prompts = [f"a photograph of request {i}, highly detailed" for i in range(args.requests)]
    res = dict(card=card, size=size, requests=args.requests, max_batch=S, prior_slots=P, gap_steps=args.gap_steps,
               prior_steps=emb.prior_steps, prior_guidance_scale=emb.prior_guidance_scale, streams={})
    for sampler, steps in (("ddpm_sampler", args.steps), ("dpmpp_2m_sampler", args.dpm_steps)):
        arms = {"prior_slots=0": pipe.batcher(S, size, size, sampler=sampler, max_steps=steps),
                f"prior_slots={P}": pipe.batcher(S, size, size, sampler=sampler, max_steps=steps, prior_slots=P)}
        # warm-up of both arms (plan builds, tuning, graph captures, the batch-1 prior plan); step times with all slots busy
        for b in arms.values():
            _fill(b, steps)
        b0, bp = arms["prior_slots=0"], arms[f"prior_slots={P}"]
        # a prior batch of its own with every slot busy (its graph is the one bp.prior replays); the graphs are replayed
        # directly, so the host bookkeeping of the batchers is drained with run() afterwards
        pt = emb.batcher(P)
        for i in range(P):
            pt.submit(f"timing {i}", prior_steps=4 * args.reps)
        pt.step()
        times = dict(decoder_step_4_busy_ms=_event_ms(b0.graph.replay, args.reps),
                     prior_step_8_rows_ms=_event_ms(pt.graph.replay, args.reps),
                     decoder_plus_prior_step_ms=_event_ms(lambda: (pt.graph.replay(), bp.graph.replay()), args.reps))
        # what pinning the slot plan's GEMMs to the batch-1 configurations costs: the batch plan at B = 4 (8 rows, each GEMM
        # at the configuration the library and tuner pick for 8 rows) on the same step
        from kandinsky2.model.prior import UnCLIPSchedule
        D = emb.prior.clip_dim
        _, _, rows4, _ = emb._call_args("timing", 4, 25, 4.0, "")
        plan4 = emb.prior._step_plan(4)
        plan4.bind(*rows4)
        plan4.set_schedule(UnCLIPSchedule(4 * args.reps), torch.zeros(4, D, device="cuda"),
                           torch.zeros(4 * args.reps, 4, D, device="cuda"), 4.0)
        times["batch_plan_step_8_rows_ms"] = _event_ms(lambda: plan4.run(True), args.reps)
        torch.cuda.synchronize()
        t = time.perf_counter()
        emb.image_emb("one batch-1 prior call", 1)
        torch.cuda.synchronize()
        times["batch1_prior_call_ms"] = round((time.perf_counter() - t) * 1e3, 2)
        for b in arms.values():
            b.run()
        del pt
        gap_s = args.gap_steps * times["decoder_step_4_busy_ms"] / 1e3
        arrive = [i * gap_s for i in range(args.requests)]
        stream = dict(sampler=sampler, steps=steps, arrival_gap_s=round(gap_s, 4), **times,
                      rounds={name: [] for name in arms})
        for _ in range(args.rounds):
            for name, b in arms.items():
                stream["rounds"][name].append(_summary(arrive, run_batcher(b, prompts, arrive, steps)))
        res["streams"][sampler] = stream
        del arms, b0, bp, b
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
