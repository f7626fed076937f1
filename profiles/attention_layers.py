"""Per-launch throughput of the head-width-64 attention (k2_attention_d64) at the shapes the UNet step runs it at.

Shapes (UNet batch B, T spatial queries, Tc = 32 encoder keys prepended, heads of width 64, the reference's qkv layout):
  cfg-2 (4 images x CFG at 96 x 96 latents): level 1 48 x 48, level 2 24 x 24, level 3 12 x 12 (also the middle block);
  cfg-3 (2 images x CFG at 128 x 128 latents): level 1 64 x 64.
Each shape is timed with CUDA events around enough back-to-back launches to fill --min-ms after a warm-up, on fresh random
inputs.  FLOPs are the two products the kernel computes, 4 B heads T (T + Tc) 64.  The card's name, power limit and max SM
clock are read in the same run.  --lib times another build of libk2b200.so (e.g. the parent commit's), so that two builds can
be compared on one card.  Prints a table and writes one JSON file (--out).  Needs a CUDA sm_90 device.

    python profiles/attention_layers.py --out /tmp/attention.json [--lib /path/to/libk2b200.so]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

# (name, B, heads, T, Tc, launches per step)
SHAPES = [
    ("cfg-2 level 1 (48x48)", 8, 12, 2304, 32, 7),
    ("cfg-2 level 2 (24x24)", 8, 18, 576, 32, 7),
    ("cfg-2 level 3 + mid (12x12)", 8, 24, 144, 32, 8),
    ("cfg-3 level 1 (64x64)", 4, 12, 4096, 32, None),
]


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _time(run, min_ms):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(5):
        run()
    e.record()
    torch.cuda.synchronize()
    reps = max(10, int(min_ms / max(s.elapsed_time(e) / 5, 1e-3)) + 1)
    s.record()
    for _ in range(reps):
        run()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", default=None, help="libk2b200.so to time (default: the in-tree build)")
    ap.add_argument("--min-ms", type=float, default=100.0, help="timed window per shape")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA sm_90 device")
    from kandinsky2 import _native, ops
    if args.lib:
        _native.LIB_PATH = os.path.abspath(args.lib)
    _native.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.set_tuning(4, 1)  # programmatic dependent launch, as bench.py runs the step
    res = {"card": _card(), "torch": torch.__version__, "lib": _native.LIB_PATH, "min_ms": args.min_ms}
    g = torch.Generator(device=dev).manual_seed(11)
    rows = []
    for name, B, heads, T, Tc, per_step in SHAPES:
        qkv = torch.randn(B, T, heads * 192, device=dev, generator=g).half()
        enc = torch.randn(B, Tc, heads * 128, device=dev, generator=g).half()
        out = torch.empty(B, T, heads * 64, device=dev, dtype=torch.float16)
        ms, reps = _time(lambda: ops.attention_d64(qkv, heads, enc, out=out), args.min_ms)
        flops = 4.0 * B * heads * T * (T + Tc) * 64
        rows.append(dict(shape=name, B=B, heads=heads, T=T, Tc=Tc, launches_per_step=per_step, ms=round(ms, 5), reps=reps,
                         gflop=round(flops * 1e-9, 2), tflops=round(flops / (ms * 1e-3) / 1e12, 1),
                         ms_per_step=round(ms * per_step, 4) if per_step else None))
    res["shapes"] = rows
    print(f"# {res['card']}  {res['lib']}")
    print(f"{'shape':30s} {'ms':>9s} {'TFLOP/s':>8s} {'ms/step':>8s}")
    for r in rows:
        print(f"{r['shape']:30s} {r['ms']:9.4f} {r['tflops']:8.1f} " + (f"{r['ms_per_step']:8.3f}" if r["ms_per_step"] else ""))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
