"""Cost of the hybrid DPT depth estimator (MiDaS v3 DPT-Hybrid, kandinsky2/model/depth.py) at the Intel/dpt-hybrid-midas
geometry (synthetic weights of the architecture: BiT ResNet-50 stem and stages [3, 4, 9], 12 ViT-B/16 layers of width 768,
neck 256 / 512 / 768 / 768, fusion 256) at 384 x 384 (B = 1, 4) and 512 x 512 (B = 1, the ControlNet annotator's size).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given): per size, three arms that
alternate within each repetition after a warm-up -- the launch plan as one CUDA graph replay, the same launch list issued
eagerly, and the oracle's torch fp16 forward (tests/dpt_hybrid_oracle.py, cuDNN / cuBLAS) -- median and min of --reps
repetitions of CUDA events around one call; the per-kernel-family device time of one eager pass (LaunchPlan.profile) with
the FLOPs of each family computed from shapes, and the share of that pass spent in the two stride-2 3x3 convolutions that run
at stride 1 (the first blocks of stages 2 and 3).  The card's name, power limit and maximum SM clock are read in the same run.

    python profiles/dpt_hybrid_depth.py [--reps 20] [--out profiles/dpt_hybrid_depth_h100_700w.json]
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
    ap.add_argument("--sizes", default="1x384x384,4x384x384,1x512x512")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpt_hybrid_depth.py needs a CUDA sm_90 device")
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_hybrid_oracle as ho
    cfg = ho.CFG_HYBRID
    sd = ho.synth_weights(cfg, 1, last_bias=ho.REAL_LAST_BIAS)
    est = DPTDepthEstimator.from_transformers(sd, cfg)
    sd16 = {k: v.to("cuda", torch.float16) for k, v in sd.items()}
    res = dict(card=_card(), reps=args.reps, sizes={})
    for key in args.sizes.split(","):
        B, h, w = (int(v) for v in key.split("x"))
        plan = est._plan(B, h, w)
        pix = ho.sample_pixels(h, w, seed=B, B=B).cuda()
        plan.pix.copy_(pix)
        arms = {"graph": lambda: plan.run(True), "eager": lambda: plan.run(False),
                "torch_fp16_oracle": lambda: ho.forward(sd16, cfg, pix, dtype=torch.float16)}
        for fn in arms.values():
            fn()
            fn()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():
                times[k].append(_timed(fn))
        r = {k: dict(median_ms=round(statistics.median(v), 3), min_ms=round(min(v), 3)) for k, v in times.items()}
        prof = plan.profile(reps=3)
        flops = sum(v["flops"] for v in prof.values())
        total_ms = sum(v["ms"] for v in prof.values())
        s2_conv_ms = prof["conv_stride2_at_1"]["ms"]   # the first blocks' 3x3 convolutions of stages 2 and 3
        r["gflop_from_shapes"] = round(flops / 1e9, 2)
        r["graph"]["tflops_achieved"] = round(flops / (r["graph"]["median_ms"] * 1e-3) / 1e12, 1)
        r["kernel_ms_eager"] = {n: dict(ms=round(v["ms"], 3), launches=v["launches"],
                                        **({"tflops": round(v["flops"] / (v["ms"] * 1e-3) / 1e12, 1)} if v["flops"] else {}))
                                for n, v in prof.items()}
        r["stride2_conv3x3_at_stride1"] = dict(ms=round(s2_conv_ms, 3), share_of_eager_pass=round(s2_conv_ms / total_ms, 4))
        res["sizes"][key] = r
        plan.graph = None
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
