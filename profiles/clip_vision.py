"""Cost of the Kandinsky 2.2 CLIP image tower (kandinsky2/model/clip_vision.py) at the full ViT-bigG/14 size (synthetic weights
of the architecture: 48 layers, hidden 1664, 16 heads of 104, MLP 8192, 257 tokens, projection 1280).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * the tower at B = 1, 4, 8: one CUDA graph replay of the launch plan, the same launch list issued eagerly, and the oracle's
    torch fp16 forward (tests/clip_vision_oracle.py, a side baseline on the same GPU, like bench.py --impl torch_gpu); the arms
    alternate within each repetition after a warm-up, median and min of --reps repetitions, CUDA events;
  * achieved TFLOP/s from the FLOPs computed from the shapes (flops_per_image), and at B = 1 the packed weights' bytes over the
    replay time;
  * the attention kernel's share of the tower's time (per-launch CUDA events around one eager pass, LaunchPlan.profile);
  * PriorEmbedder22.emb2emb at strength 0.85 from a PIL image (preprocess + tower + prior) against emb2emb from a precomputed
    embedding, B = 1, full-size 2.2 prior.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/clip_vision.py [--reps 10] [--out /tmp/clip_vision.json]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from profiles.controlnet_img2img import _card, _prior_embedder, _timed  # noqa: E402


def flops_per_image(cfg):
    """Multiply-adds x 2 of one 224^2 image: the patch-embedding GEMM (3 P^2 columns), per layer qkv / out_proj / fc1 / fc2 and
    the two attention products, the projection of the CLS row."""
    H, I, L, P = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"], cfg["patch_size"]
    T = (cfg["image_size"] // P) ** 2 + 1
    gemm = 2 * (T - 1) * 3 * P * P * H + L * 2 * T * (3 * H * H + H * H + 2 * H * I) + 2 * H * cfg["projection_dim"]
    attn = L * 4 * T * T * H
    return gemm + attn, attn


def _alternate(arms, reps):
    for fn in arms.values():
        fn()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(_timed(fn))
    return {k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3)) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--batches", default="1,4,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_vision.py needs a CUDA sm_90 device")
    from PIL import Image
    from kandinsky2.checkpoints import transformers_clip_vision_to_k2
    from kandinsky2.model.clip_vision import CLIPVisionTower
    from tests import clip_vision_oracle as cvo
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = cvo.CONFIG_BIGG
    total, attn = flops_per_image(cfg)
    sd16 = {k: v.cuda().half() for k, v in cvo.synth_weights(cfg, 1).items()}
    tower = CLIPVisionTower(transformers_clip_vision_to_k2(sd16), cfg, device="cuda").finalize()
    wbytes = sum(t.numel() * t.element_size() for L in tower._packed["layers"]
                 for t, _ in (L[n] for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")))
    wbytes += tower._packed["embed"].numel() * 2 + tower._packed["proj"].numel() * 4
    res = dict(card=_card(), reps=args.reps, flops_per_image=total, attention_flops_per_image=attn, weight_bytes=wbytes,
               tower={})
    for B in [int(b) for b in args.batches.split(",")]:
        pix = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B))
        plan = tower._plan(B)
        plan.pix.copy_(pix)
        with torch.no_grad():
            r = _alternate({"graph": lambda: plan.run(True), "eager": lambda: plan.run(False),
                            "torch_fp16": lambda: cvo.forward(sd16, cfg, pix, dtype=torch.float16)}, args.reps)
        g = r["graph"]["median_ms"]
        r["graph_tflops"] = round(B * total / (g * 1e-3) / 1e12, 1)
        r["speedup_vs_torch_fp16"] = round(r["torch_fp16"]["median_ms"] / g, 2)
        prof = plan.profile(reps=3)
        eager_sum = sum(v["ms"] for v in prof.values())
        r["attention_ms_eager"] = round(prof["attention"]["ms"], 3)
        r["attention_share"] = round(prof["attention"]["ms"] / eager_sum, 4)
        r["kernel_ms"] = {k: round(v["ms"], 3) for k, v in prof.items()}
        if B == 1:
            r["weight_tb_per_s"] = round(wbytes / (g * 1e-3) / 1e12, 2)
        res["tower"][str(B)] = r
    del sd16
    torch.cuda.empty_cache()

    from kandinsky2.model.prior import PriorEmbedder22
    base = _prior_embedder()
    emb = PriorEmbedder22(base.prior, base.clip_text, base.clip_mean, base.clip_std, clip_image=tower,
                          zero_image_emb=tower.zero_embed().cpu())
    photo = Image.fromarray((np.random.default_rng(0).random((512, 640, 3)) * 255).astype("uint8"))
    pre = tower(photo)
    prompt = "A capybara, 4k photo"
    r = _alternate({"from_pil": lambda: emb.emb2emb(prompt, photo, 1, strength=0.85, prior_steps=25),
                    "from_embedding": lambda: emb.emb2emb(prompt, pre, 1, strength=0.85, prior_steps=25),
                    "tower_call_pil": lambda: tower(photo)}, args.reps)
    res["emb2emb_b1"] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
