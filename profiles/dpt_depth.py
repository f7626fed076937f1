"""Cost of the DPT depth estimator (kandinsky2/model/depth.py) at the Intel/dpt-large geometry (synthetic weights of the
architecture: 24 ViT-L/16 layers of width 1024 over 577 tokens, neck sizes 256 / 512 / 1024 / 1024, fusion 256) on 384 x 384
inputs.

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given): per B in --batches, three arms
that alternate within each repetition after a warm-up -- the launch plan as one CUDA graph replay, the same launch list
issued eagerly, and the oracle's torch fp16 forward (tests/dpt_oracle.py, cuDNN / cuBLAS) -- median and min of --reps
repetitions of CUDA events around one call; the per-kernel-family device time of one eager pass (LaunchPlan.profile, CUDA
events around every launch) with the FLOPs of each family computed from shapes, and the achieved rate from them.  The
card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/dpt_depth.py [--reps 20] [--out profiles/dpt_depth_h100.json]
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
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpt_depth.py needs a CUDA sm_90 device")
    from kandinsky2.model.depth import DPTDepthEstimator
    from tests import dpt_oracle as do
    cfg = do.CFG_LARGE
    sd = do.synth_weights(cfg, 1)
    est = DPTDepthEstimator.from_transformers(sd, cfg)
    sd16 = {k: v.to("cuda", torch.float16) for k, v in sd.items()}
    res = dict(card=_card(), reps=args.reps, size=est.size, batches={})
    for B in [int(b) for b in args.batches.split(",")]:
        plan = est._plan(B)
        pix = torch.rand(B, 3, 384, 384, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B)) * 2 - 1
        plan.pix.copy_(pix)
        arms = {"graph": lambda: plan.run(True), "eager": lambda: plan.run(False),
                "torch_fp16_oracle": lambda: do.forward(sd16, cfg, pix, dtype=torch.float16)}
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
        r["gflop_from_shapes"] = round(flops / 1e9, 2)
        r["graph"]["tflops_achieved"] = round(flops / (r["graph"]["median_ms"] * 1e-3) / 1e12, 1)
        r["kernel_ms_eager"] = {n: dict(ms=round(v["ms"], 3), launches=v["launches"],
                                        **({"tflops": round(v["flops"] / (v["ms"] * 1e-3) / 1e12, 1)} if v["flops"] else {}))
                                for n, v in prof.items()}
        res["batches"][str(B)] = r
        plan.graph = None
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
