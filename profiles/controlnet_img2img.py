"""Cost of the ControlNet notebook's image-guided workflow at full Kandinsky 2.2 size (synthetic weights of the architecture),
against the text-to-image calls it replaces.

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * the prior: PriorEmbedder22.emb2emb at strength 0.85 (the last 21 of 25 UnCLIP steps run, from the noised image embedding)
    against PriorEmbedder22.image_emb (all 25 steps from noise), guidance 4, B = 1 and 4 (full size: 20 layers, width 2048,
    CLIP-bigG 1280, 77 + 4 tokens);
  * the decoder: Kandinsky2_2(task_type="controlnet").generate_controlnet_img2img (strength 0.5: MoVQ encode of the image, then
    the last 25 of 50 DDPM steps) against generate_controlnet (50 steps), 768 x 768, B = 2 and 4, guidance 4, both with the
    depth hint and the synthetic embedder.
Each arm is a whole call timed with CUDA events (every call ends in a device-to-host copy); the arms alternate within each
repetition, after one warm-up call of each; median and min of --calls repetitions.  The card's name, power limit and maximum
SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/controlnet_img2img.py [--calls 3] [--out /tmp/controlnet_img2img.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def _alternate(arms, calls):
    for fn in arms.values():    # warm-up: plan builds, tuning, graph capture
        fn()
    times = {k: [] for k in arms}
    for _ in range(calls):
        for k, fn in arms.items():
            times[k].append(_timed(fn))
    return {k: dict(median_ms=round(statistics.median(v), 2), min_ms=round(min(v), 2), all_ms=[round(t, 2) for t in v])
            for k, v in times.items()}


def _prior_embedder():
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import prior22_oracle as p22
    dsd = {k: v.cuda() for k, v in synth.synth_state_dict(p22.diffusers_prior_spec(p22.CONFIG_PRIOR22), seed=1).items()}

    def clip_text(prompts):     # stand-in for the CLIP-bigG text tower: deterministic per prompt, CLIP-style masks
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(77, 1280, generator=g), torch.arange(77) < 2 + len(p)))
        return tuple(torch.stack(t) for t in zip(*outs))

    return PriorEmbedder22.from_diffusers(dsd, clip_text)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3, help="timed calls per arm")
    ap.add_argument("--prior-batches", default="1,4")
    ap.add_argument("--decoder-batches", default="2,4")
    ap.add_argument("--size", type=int, default=768)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("controlnet_img2img.py needs a CUDA sm_90 device")
    from PIL import Image
    from kandinsky2 import get_kandinsky2
    torch.backends.cuda.matmul.allow_tf32 = False
    res = dict(card=_card(), calls=args.calls, prior={}, decoder={})

    emb = _prior_embedder()
    image = torch.randn(1, 1280, generator=torch.Generator().manual_seed(2))
    prompt = "A capybara, 4k photo"
    for B in [int(b) for b in args.prior_batches.split(",")]:
        r = _alternate({"emb2emb_0.85": lambda: emb.emb2emb(prompt, image, B, strength=0.85, prior_steps=25),
                        "text_only": lambda: emb.image_emb(prompt, B, prior_steps=25)}, args.calls)
        r["ratio_median"] = round(r["emb2emb_0.85"]["median_ms"] / r["text_only"]["median_ms"], 3)
        r["steps_run"] = dict(emb2emb=21, text_only=25)
        res["prior"][str(B)] = r
    del emb
    torch.cuda.empty_cache()

    S = args.size
    pipe = get_kandinsky2("cuda", task_type="controlnet", model_version="2.2", cache_dir="/nonexistent")
    photo = Image.fromarray((np.random.default_rng(0).random((S, S, 3)) * 255).astype("uint8"))
    hint = torch.rand(1, 3, S, S, generator=torch.Generator().manual_seed(3))
    kw = dict(decoder_steps=50, h=S, w=S, decoder_guidance_scale=4)
    for B in [int(b) for b in args.decoder_batches.split(",")]:
        r = _alternate({"controlnet_img2img_0.5": lambda: pipe.generate_controlnet_img2img(prompt, photo, hint, strength=0.5,
                                                                                           batch_size=B, **kw),
                        "controlnet": lambda: pipe.generate_controlnet(prompt, hint, batch_size=B, **kw)}, args.calls)
        r["ratio_median"] = round(r["controlnet_img2img_0.5"]["median_ms"] / r["controlnet"]["median_ms"], 3)
        r["steps_run"] = dict(controlnet_img2img=25, controlnet=50)
        encode = _alternate({"movq_encode": lambda: pipe._encode_image(photo, S, S).cpu()}, args.calls)["movq_encode"]
        r["movq_encode_ms"] = encode["median_ms"]
        res["decoder"][str(B)] = r
    res["size"] = S
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
