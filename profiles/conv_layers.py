"""Per-layer throughput of the implicit-GEMM convolution (k2_conv_gemm) at the cfg-2 step geometry, for every N tile.

Builds the full-size cfg-2 step the way bench.py does (Kandinsky 2.2 decoder UNet with random weights, 4 images x CFG at 96x96
latents), takes the distinct conv / GEMM layer shapes from the keys the step's launch plan hands the autotuner (the keys of
launch_plan._tune_cache, counted as the plan is recorded, so also how often the step launches each one), then times every legal N tile of each shape, unsplit,
on fresh tensors of that shape: CUDA events around enough back-to-back launches to fill --min-ms after a warm-up.

Per shape and configuration it reports:
  * the FLOPs of the GEMM the kernel runs (2 M N K; an up2 conv -- 3x3 over a nearest-2x upsampling -- runs 4 taps per output
    pixel), the time and TFLOP/s;
  * shared-memory operand bytes per FLOP, modelled from the wgmma instruction shape: one m64nNk16 reads a 64 x 16 A slice
    (2 KB) and an N x 16 B slice (32 N bytes) for 2 * 64 * N * 16 FLOPs.  N is the N tile for a build that issues one
    instruction per tile (the default), or 64 for a build that splits the tile into m64n64k16 instructions (--mma-n 64);
  * L2 -> SM operand bytes per FLOP, modelled from the tile: 16 KB of A + BN * 128 B of B per 128 x BN x 64 chunk, and the rate
    that implies at the measured time (chunks the launch loads x bytes per chunk / time);
  * the configuration the autotuner picked for the step, and the shape's share of the step's conv time (launches per step x
    the time of the picked configuration, over the sum of that product across shapes).
The card's name, power limit and max SM clock are read in the same run.  Prints a table and writes one JSON file (--out).
Needs a CUDA sm_90 device.

    python profiles/conv_layers.py --out /tmp/conv_layers.json [--mma-n 64]
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

B, H, W = 4, 96, 96  # cfg-2: 768 x 768 images, batch 4, UNet batch 8 under classifier-free guidance


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _pad64(c):
    return (c + 63) // 64 * 64


def _layer(key, dev, g):
    """Launch closure run(cfg, info) on fresh random tensors of one autotuner key, plus its GEMM sizes."""
    from kandinsky2 import ops
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).half()
    kind, cout = key[0], key[1]
    if kind == "gemm":
        _, _, xshape, has_res = key
        x = rnd(*xshape)
        M, K = x.numel() // xshape[-1], xshape[-1]
        w = rnd(cout, K)
        bias = torch.randn(cout, device=dev, generator=g)
        res = rnd(*xshape[:-1], cout) if has_res else None
        out = torch.empty(*xshape[:-1], cout, device=dev, dtype=torch.float16)
        run = lambda cfg, info=None: ops.gemm_rows(x, w, cout, bias=bias, residual=res, out=out, cfg=cfg, info=info)
        return run, dict(M=M, N=cout, K=K, desc=f"gemm {M}x{K}->{cout}" + (" +res" if has_res else ""))
    _, _, oshape, geom, srcs_spec, has_res, has_part, out_mode, w_batched = key
    if w_batched:
        return None, None  # per-image weights: MoVQ attention, not part of the UNet step
    if geom is not None:
        NB, Ho, Wo = geom
    elif out_mode == 0:
        NB, Ho, Wo = oshape[:3]
    else:
        NB, Ho, Wo = oshape[0], oshape[2], oshape[3]
    up2 = srcs_spec[0][1] == 4
    Hs, Ws = (Ho // 2, Wo // 2) if up2 else (Ho, Wo)
    srcs = [(rnd(NB, Hs, Ws, c), taps) for c, taps in srcs_spec]
    K = sum(taps * _pad64(c) for c, taps in srcs_spec)  # per output pixel (up2: one 4-tap phase)
    w_rows = max(16, cout)
    w = rnd(w_rows, 4 * K if up2 else K)
    bias = torch.randn(cout, device=dev, generator=g)
    res = rnd(NB, Ho, Wo, cout) if has_res else None
    out = torch.empty(*oshape, device=dev, dtype=torch.float16 if out_mode == 0 else torch.float32)
    part = torch.zeros(ops.gn_part_floats(NB, Ho, Wo, cout), device=dev) if has_part else None
    run = lambda cfg, info=None: ops.conv_gemm(srcs, w, cout, bias=bias, residual=res, out=out, out_mode=out_mode, geom=geom,
                                               gn_part=part, cfg=cfg, info=info)
    desc = (f"{NB}x{Ho}x{Wo} " + "+".join(f"{c}{'x3x3' if t == 9 else ('up2' if t == 4 else 'x1x1')}" for c, t in srcs_spec)
            + f"->{cout}" + (" +res" if has_res else "") + (" fp32-nchw" if out_mode else ""))
    return run, dict(M=NB * Ho * Wo, N=cout, K=K, desc=desc)


def _time(run, cfg, min_ms):
    for _ in range(3):
        run(cfg)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(5):
        run(cfg)
    e.record()
    torch.cuda.synchronize()
    reps = max(10, int(min_ms / max(s.elapsed_time(e) / 5, 1e-3)) + 1)
    s.record()
    for _ in range(reps):
        run(cfg)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--min-ms", type=float, default=50.0, help="timed window per configuration")
    ap.add_argument("--mma-n", default="tile", choices=["tile", "64"],
                    help="wgmma N of the build: one instruction per N tile, or m64n64k16 per 64 columns")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA sm_90 device")
    import bench
    from kandinsky2 import launch_plan, ops
    from kandinsky2.model.gaussian_diffusion import FusedStep, create_ddpm_v22
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.set_tuning(4, 1)  # programmatic dependent launch, as bench.py runs the step
    res = {"card": _card(), "torch": torch.__version__, "geometry": f"cfg-2: UNet batch {2 * B}, {H}x{W} latents",
           "mma_n": args.mma_n, "min_ms": args.min_ms}

    # ---- the step, with a count of how often its plan launches each tuned shape
    counts = {}
    tune = launch_plan.tune

    def counting_tune(key, run, m_rows=0):
        counts[key] = counts.get(key, 0) + 1
        return tune(key, run, m_rows=m_rows)
    launch_plan.tune = counting_tune
    model = bench.build_unet(dev)
    image_emb = torch.randn(2 * B, 1280, generator=torch.Generator().manual_seed(1234)).to(dev)
    step = FusedStep(model, B, H, W, dict(image_emb=image_emb), guidance_scale=4.0, cond_first=False, clip_range=2.0,
                     threshold_mode=0)
    launch_plan.tune = tune
    diffusion = create_ddpm_v22(50)
    coef, ts = diffusion._tables(dev)
    order = torch.arange(diffusion.num_timesteps - 1, -1, -1, device=dev)
    step.set_schedule(ts[order], coef[order], torch.randn(len(order), B, 4, H, W, device=dev))
    x = step.latent()
    x.copy_(torch.randn(B, 4, H, W, device=dev))
    step.advance(x)
    torch.cuda.synchronize()
    res["plan_conv_launches"] = sum(1 for _, kind, _ in step.plan.steps if kind == "conv_gemm")
    res["counted_conv_launches"] = sum(counts.values())

    # ---- every shape x configuration
    g = torch.Generator(device=dev).manual_seed(7)
    layers = []
    for key, n in counts.items():  # (kind, Cout, ...)
        run, shp = _layer(key, dev, g)
        if run is None:
            continue
        info = [0] * 7
        picked = launch_plan._tune_cache.get((dev.index, launch_plan.TUNE_SMALL_M) + key)
        run(picked, info)
        picked_cfg = [info[0], 0, info[2], (picked[3] if picked and picked[3] else 1)]
        cout = shp["N"]
        cfgs = []
        if cout > 64:  # the tuner's candidates at splits 1
            cfgs = [(bn, 0, 1, 1) for bn in (128, 192, 256) if bn - 64 < cout or bn == info[0]]
        if tuple(picked_cfg) not in cfgs:
            cfgs.append(tuple(picked_cfg))
        rows = []
        for cfg in cfgs:
            info = [0] * 7
            run(cfg, info)
            bn, splits = info[0], info[2]
            ms, reps = _time(run, cfg, args.min_ms)
            flops = 2.0 * shp["M"] * cout * shp["K"]
            mma_n = bn if (args.mma_n == "tile" or bn < 64) else 64
            smem_bpf = (2048 + 32 * mma_n) / (2.0 * 64 * mma_n * 16)
            m_tiles = info[3] * (4 if "up2" in shp["desc"] else 1)
            chunks = m_tiles * ((cout + bn - 1) // bn) * (shp["K"] // 64)
            l2_bytes = chunks * (16384 + bn * 128)
            rows.append(dict(n_tile=bn, epilogue_sets=cfg[3], splits=splits, ms=round(ms, 5), reps=reps,
                             tflops=round(flops / (ms * 1e-3) / 1e12, 1),
                             smem_operand_bytes_per_flop=round(smem_bpf, 5),
                             l2_operand_bytes_per_flop=round(l2_bytes / flops, 5),
                             l2_operand_TBps=round(l2_bytes / (ms * 1e-3) / 1e12, 2)))
        pick = next((r for r in rows if [r["n_tile"], r["splits"], r["epilogue_sets"]] ==
                     [picked_cfg[0], picked_cfg[2], picked_cfg[3]]), rows[0])
        layers.append(dict(shape=shp["desc"], key=repr(key), launches_per_step=n, gemm_gflop=round(2e-9 * shp["M"] * cout * shp["K"], 3),
                           picked=dict(n_tile=picked_cfg[0], splits=picked_cfg[2], epilogue_sets=picked_cfg[3],
                                       tuned=picked is not None),
                           picked_ms=pick["ms"], configs=rows))
    total = sum(l["launches_per_step"] * l["picked_ms"] for l in layers)
    for l in layers:
        l["share_of_conv_time"] = round(l["launches_per_step"] * l["picked_ms"] / total, 4)
    layers.sort(key=lambda l: -l["share_of_conv_time"])
    res["conv_ms_per_step_at_picked"] = round(total, 3)
    res["layers"] = layers

    print(f"# {res['card']}  (mma_n={args.mma_n})  conv time per step at the picked configurations: {total:.2f} ms")
    print(f"{'shape':44s} {'n':>2s} {'share':>6s} {'pick':>9s}  " + "  ".join(f"{c:>9s}" for c in
          ("128", "192", "256")) + "   (TFLOP/s at N tile, splits 1)")
    for l in layers:
        by = {(r["n_tile"], r["epilogue_sets"]): r["tflops"] for r in l["configs"] if r["splits"] == 1}
        pk = l["picked"]
        print(f"{l['shape'][:44]:44s} {l['launches_per_step']:2d} {100 * l['share_of_conv_time']:5.1f}% "
              f"{pk['n_tile']:>3d}/{pk['epilogue_sets']}/{pk['splits']:<3d}  " +
              "  ".join(f"{by.get(c, float('nan')):9.1f}" for c in ((128, 1), (192, 1), (256, 1))))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
