"""Cost of the Kandinsky 2.1 CLIP ViT-L/14 towers (kandinsky2/model/clip_vitl14.py) at full size (synthetic weights of the
architecture: text 12 layers of width 768, 77 tokens; image 24 layers of width 1024, 16 heads of 64, 257 tokens; embeddings
of 768).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given): per B in --batches, the text
tower on 2B rows (generate_clip_emb encodes B prompts and B negative prompts) and the image tower on B images, each as one
CUDA graph replay of its launch plan; the two arms alternate within each repetition after a warm-up, median and min of --reps
repetitions of CUDA events around one call; plus the per-kernel-family device time of one eager pass (LaunchPlan.profile).
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90
device.

    python profiles/clip_vitl14.py [--reps 20] [--out profiles/clip_vitl14_h100.json]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from profiles.controlnet_img2img import _card, _timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batches", default="1,2,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_vitl14.py needs a CUDA sm_90 device")
    from kandinsky2.model.clip_vitl14 import load_openai_clip
    from tests import openai_clip_oracle as oo
    geo = oo.GEO_L14
    text, image = load_openai_clip({k: v.half() for k, v in oo.synth_weights(geo, 1).items()}, "cuda")
    res = dict(card=_card(), reps=args.reps, towers={})
    for B in [int(b) for b in args.batches.split(",")]:
        tp = text._plan(2 * B, geo["context"])
        tp.ids.copy_(oo.sample_tokens(geo, B, n=2 * B))
        ip = image._plan(B)
        ip.pix.copy_(torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B)))
        arms = {"text": lambda: tp.run(True), "image": lambda: ip.run(True)}
        for fn in arms.values():
            fn()
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(_timed(fn))
        r = {k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3)) for k, v in times.items()}
        r["text"]["rows"], r["image"]["images"] = 2 * B, B
        for k, plan in (("text", tp), ("image", ip)):
            r[k]["kernel_ms_eager"] = {n: round(v["ms"], 3) for n, v in plan.profile(reps=3).items()}
        res["towers"][str(B)] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
