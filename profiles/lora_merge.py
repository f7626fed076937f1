"""Cost of a LoRA adapter on the full-size Kandinsky 2.2 decoder UNet (random weights of the architecture).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * merge time of a rank-4 and a rank-64 notebook-format adapter: the 66 k2_lora_merge launches (qkv, encoder_kv and proj_out
    of the 22 attention blocks) with the factors already on the device, CUDA events over --merge-reps repeated merges; and
    Text2ImUNet.load_lora end to end (host parsing + factor upload + merges), host clock around a device synchronise;
  * achieved bandwidth of the merge launches: bytes they must move (fp16 base read + fp16 out write + the fp32 factors) over
    the event time, against the H100 SXM data sheet's 3.35 TB/s;
  * cfg-2 denoising steps/s (4 images x CFG at 96x96 latents, the 50-step schedule, one graph launch per step, as bench.py runs
    it) without and with a merged rank-4 adapter, alternated --rounds times.  The kernels are the same, so they should be equal.
The card's name and power limit are read in the same run.  Needs a CUDA sm_90 device.

    python profiles/lora_merge.py [--out /tmp/lora_merge.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

HBM_TBPS = 3.35


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _adapter(rank, seed):
    """Notebook-format adapter of the full-size decoder with both factors random (the same recipe as tests/lora_oracle.py)."""
    from kandinsky2.checkpoints import unet_block_map
    from kandinsky2.model.unet import _topology
    inp, mid, out = _topology(4, 384, (1, 2, 3, 4), 3, (2, 4, 8))
    chans = [layer[1] for blk in inp + [mid] + out for layer in blk if layer[0] == "attn"]
    prefixes = [dp for dp, _, kind in unet_block_map(4, 384, (1, 2, 3, 4), 3, (2, 4, 8)) if kind == "attn"]
    g = torch.Generator().manual_seed(seed)
    lora = {}
    for dp, C in zip(prefixes, chans):
        for proj in ("to_q", "to_k", "to_v", "to_out", "add_k_proj", "add_v_proj"):
            fan_in = 768 if proj.startswith("add_") else C
            lora[f"{dp}.processor.{proj}_lora.down.weight"] = torch.randn(rank, fan_in, generator=g) / fan_in ** 0.5
            lora[f"{dp}.processor.{proj}_lora.up.weight"] = torch.randn(C, rank, generator=g) * (0.3 / rank ** 0.5)
    return lora


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--merge-reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA sm_90 device")
    from kandinsky2 import ops
    from kandinsky2.checkpoints import lora_to_k2
    from kandinsky2.model.gaussian_diffusion import FusedStep, create_ddpm_v22
    from kandinsky2.model.unet import Text2ImUNet
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ops.set_tuning(4, 1)  # programmatic dependent launch, as bench.py runs the step
    m = Text2ImUNet(model_dim=768, image_encoder_in_dim=1280, num_image_embs=32, pooling_type="from_model", in_channels=4,
                    model_channels=384, out_channels=8, num_res_blocks=3, attention_resolutions=(2, 4, 8),
                    channel_mult=(1, 2, 3, 4), use_fp16=True, num_head_channels=64, use_scale_shift_norm=True,
                    resblock_updown=True, cond_version="2.2", device=dev, param_dtype=torch.float16)
    m.init_synthetic_(0).finalize(release_params=True)
    res = {"card": _card(), "torch": torch.__version__}

    # ---- merge time
    for rank in (4, 64):
        lora = _adapter(rank, seed=rank)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.load_lora(lora)
        torch.cuda.synchronize()
        load_ms = (time.perf_counter() - t0) * 1e3
        factors = lora_to_k2(lora)
        jobs, nbytes = [], 0
        for p, a in m._packed["attn"].items():
            for name, target in m._LORA_WEIGHTS:
                up, down = (t.to(dev) for t in factors[p + target + ".weight"])
                jobs.append((m._lora_base[p][name], up, down, a[name]))
                nbytes += 2 * 2 * up.shape[0] * down.shape[1] + 4 * (up.numel() + down.numel())
        run = lambda: [ops.lora_merge(b, u, d, 1.0, out=o) for b, u, d, o in jobs]
        run()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.merge_reps):
            run()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / args.merge_reps
        res[f"rank{rank}"] = {"merge_ms": round(ms, 4), "launches": len(jobs), "bytes": nbytes,
                              "achieved_GBps": round(nbytes / (ms * 1e-3) / 1e9, 1),
                              "frac_of_3.35TBps": round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3),
                              "load_lora_ms": round(load_ms, 2)}
    m.unload_lora()

    # ---- cfg-2 steps/s without / with a merged adapter, alternated
    B, H, W = 4, 96, 96
    lora = _adapter(4, seed=4)
    image_emb = torch.randn(2 * B, 1280, generator=torch.Generator().manual_seed(1234)).to(dev)
    diffusion = create_ddpm_v22(50)
    coef, ts = diffusion._tables(dev)
    order = torch.arange(diffusion.num_timesteps - 1, -1, -1, device=dev)
    g = torch.Generator(device=dev).manual_seed(1234)
    noise = torch.randn(len(order), B, 4, H, W, device=dev, generator=g)
    x0 = torch.randn(B, 4, H, W, device=dev, generator=g)
    sps = {"base": [], "lora_rank4": []}
    for _ in range(args.rounds):
        for arm in sps:
            if arm == "base":
                m.unload_lora()
            else:
                m.load_lora(lora)
            step = FusedStep(m, B, H, W, dict(image_emb=image_emb), guidance_scale=4.0, cond_first=False, clip_range=2.0,
                             threshold_mode=0)
            step.set_schedule(ts[order], coef[order], noise)
            x = step.latent()
            x.copy_(x0)
            for _ in range(args.warmup):
                step.advance(x)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.steps):
                step.advance(x)
            e.record()
            torch.cuda.synchronize()
            sps[arm].append(round(1e3 * args.steps / s.elapsed_time(e), 3))
    m.unload_lora()
    res["cfg2_steps_per_s"] = sps
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
