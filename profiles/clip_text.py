"""Cost of the Kandinsky 2.2 CLIP text tower (kandinsky2/model/clip_text.py) at the full ViT-bigG/14 text size (synthetic weights
of the architecture: 32 layers, hidden 1280, 20 heads of 64, MLP 5120, 77 tokens, projection 1280).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * the tower at n = 1, 2, 8 sequences of 77 tokens: one CUDA graph replay of the launch plan, the same launch list issued
    eagerly, and the oracle's torch fp16 forward (tests/clip_text_oracle.py, a side baseline on the same GPU); the arms
    alternate within each repetition after a warm-up, median and min of --reps repetitions, CUDA events;
  * achieved TFLOP/s from the FLOPs computed from the shapes (flops_per_sequence), and the packed layer weights' bytes over the
    replay time (the tower is weight-bound at small n);
  * the tokenizer's host time for a 2-prompt call (the synthetic tokenizer of tests/golden/clip_text_tiny.pt, perf_counter);
  * a full 2.2 prior call (PriorEmbedder22.image_emb, 25 steps, guidance 4) at B = 1 and 4 with the tower as clip_text against
    the same call with the tower's outputs precomputed.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/clip_text.py [--reps 10] [--out /tmp/clip_text.json]
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

from profiles.clip_vision import _alternate  # noqa: E402
from profiles.controlnet_img2img import _card, _prior_embedder  # noqa: E402


def flops_per_sequence(cfg, T=77):
    """Multiply-adds x 2 of one T-token sequence: per layer qkv / out_proj / fc1 / fc2 and the two (full, unmasked-count)
    attention products, the projection of the pooled row."""
    H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    gemm = L * 2 * T * (3 * H * H + H * H + 2 * H * I) + 2 * H * cfg["projection_dim"]
    attn = L * 4 * T * T * H
    return gemm + attn, attn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ns", default="1,2,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clip_text.py needs a CUDA sm_90 device")
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower, CLIPTokenizer
    from kandinsky2.model.prior import PriorEmbedder22
    from tests import clip_text_oracle as cto
    from tests.test_gpu_zz_clip_text import bigg_ids
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = cto.CONFIG_BIGG
    total, attn = flops_per_sequence(cfg)
    fx = torch.load(cto.FIXTURE)
    tok = CLIPTokenizer(cto.synthetic_vocab(fx["merges"]), [tuple(m) for m in fx["merges"]], model_max_length=77)
    sd16 = {k: v.cuda().half() for k, v in cto.synth_weights(cfg, 1).items()}
    tower = CLIPTextTower(transformers_clip_text_to_k2(sd16), cfg, device="cuda", tokenizer=tok).finalize()
    wbytes = sum(t.numel() * t.element_size() for L in tower._packed["layers"]
                 for t, _ in (L[n] for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")))
    res = dict(card=_card(), reps=args.reps, flops_per_sequence=total, attention_flops_per_sequence=attn,
               layer_weight_bytes=wbytes, tower={})
    for n in [int(x) for x in args.ns.split(",")]:
        ids = bigg_ids(n, seed=n, lengths=(77,))
        plan = tower._plan(n)
        plan.ids.copy_(ids)
        idc = ids.cuda()
        with torch.no_grad():
            r = _alternate({"graph": lambda: plan.run(True), "eager": lambda: plan.run(False),
                            "torch_fp16": lambda: cto.forward(sd16, cfg, idc, dtype=torch.float16)}, args.reps)
        g = r["graph"]["median_ms"]
        r["graph_tflops"] = round(n * total / (g * 1e-3) / 1e12, 1)
        r["weight_tb_per_s"] = round(wbytes / (g * 1e-3) / 1e12, 2)
        r["speedup_vs_torch_fp16"] = round(r["torch_fp16"]["median_ms"] / g, 2)
        prof = plan.profile(reps=3)
        r["kernel_ms"] = {k: round(v["ms"], 3) for k, v in prof.items()}
        r["launches"] = sum(v["launches"] for v in prof.values())
        res["tower"][str(n)] = r
    del sd16
    torch.cuda.empty_cache()

    prompts = ["A capybara, 4k photo", "lowres, text, error, cropped, worst quality, low quality, jpeg artifacts, ugly"]
    host = []
    for _ in range(args.reps):
        tok._cache.clear()
        t0 = time.perf_counter()
        tok(prompts)
        host.append((time.perf_counter() - t0) * 1e3)
    res["tokenizer_2_prompts_ms"] = dict(median_ms=round(statistics.median(host), 3), min_ms=round(min(host), 3))

    base = _prior_embedder()
    live = PriorEmbedder22(base.prior, tower, base.clip_mean, base.clip_std)
    cache = {}

    def precomputed(ps):
        key = tuple(ps)
        if key not in cache:
            cache[key] = tuple(t.clone() for t in tower(ps))
        return cache[key]

    pre = PriorEmbedder22(base.prior, precomputed, base.clip_mean, base.clip_std)
    prompt = prompts[0]
    res["prior_call"] = {}
    for B in (1, 4):
        res["prior_call"][str(B)] = _alternate({"with_tower": lambda: live.image_emb(prompt, B, prior_steps=25),
                                                 "precomputed_clip_text": lambda: pre.image_emb(prompt, B, prior_steps=25)},
                                                args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
