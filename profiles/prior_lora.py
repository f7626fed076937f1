"""Cost of a LoRA adapter on the full-size Kandinsky 2.2 diffusion prior (20 layers, width 2048, CLIP-bigG 1280, 77 + 4 tokens;
synthetic weights of the architecture).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * merge time of a rank-4 and a rank-64 notebook-format adapter: the 40 k2_lora_merge launches (attn.qkv and attn.proj of the
    20 layers) with the factors already on the device, CUDA events over --merge-reps repeated merges; and
    PriorTransformer.load_lora end to end (host parsing + factor upload + merges), host clock around a device synchronise;
  * achieved bandwidth of the merge launches: bytes they must move (fp16 base read + fp16 out write + the fp32 factors) over
    the event time, against the H100 SXM data sheet's 3.35 TB/s;
  * a prior call (sample_prior22: bind + 25 UnCLIP steps at guidance 4, one CUDA graph replay per step) at B = 1 and 4,
    without and with a merged rank-4 adapter, the arms alternated --rounds times.  The kernels are the same, so they should
    be equal within noise.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/prior_lora.py [--out /tmp/prior_lora.json]
"""
import argparse
import json
import os
import statistics
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


def _timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--merge-reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--rounds", type=int, default=5, help="alternated timed calls per arm and batch size")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prior_lora.py needs a CUDA sm_90 device")
    from kandinsky2 import ops
    from kandinsky2.checkpoints import prior_lora_to_k2
    from kandinsky2.model.prior import PriorTransformer, sample_prior22
    from oracle import prior_oracle as po, synth
    from tests import prior22_oracle as p22
    from tests import prior_lora_oracle as plo
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = p22.CONFIG_PRIOR22
    m = PriorTransformer(**cfg, device="cuda")
    m.load_state_dict({k: v.cuda() for k, v in synth.synth_state_dict(po.prior_param_spec(cfg), seed=1).items()}, strict=True)
    m.finalize()
    res = {"card": _card(), "torch": torch.__version__, "steps": args.steps, "guidance": 4.0}

    # ---- merge time
    for rank in (4, 64):
        lora = plo.synth_prior_lora(cfg, rank=rank, seed=rank, gain=0.1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.load_lora(lora)
        torch.cuda.synchronize()
        load_ms = (time.perf_counter() - t0) * 1e3
        factors = prior_lora_to_k2(lora, cfg["xf_width"], cfg["xf_layers"])
        jobs, nbytes = [], 0
        for i, (L, base) in enumerate(zip(m._packed["layers"], m._lora_base)):
            for name, target in m._LORA_WEIGHTS:
                up, down = (t.to(dev) for t in factors[f"transformer.resblocks.{i}.{target}.weight"])
                jobs.append((base[name], up, down, L[name][0]))
                nbytes += 2 * 2 * up.shape[0] * down.shape[1] + 4 * (up.numel() + down.numel())
        run = lambda: [ops.lora_merge(b, u, d, 1.0, out=o) for b, u, d, o in jobs]  # noqa: E731
        run()
        ms = _timed(lambda: [run() for _ in range(args.merge_reps)]) / args.merge_reps
        res[f"rank{rank}"] = {"merge_ms": round(ms, 4), "launches": len(jobs), "bytes": nbytes,
                              "achieved_GBps": round(nbytes / (ms * 1e-3) / 1e9, 1),
                              "frac_of_3.35TBps": round(nbytes / (ms * 1e-3) / (HBM_TBPS * 1e12), 3),
                              "load_lora_ms": round(load_ms, 2)}
    m.unload_lora()

    # ---- prior calls without / with a merged rank-4 adapter, alternated
    lora = plo.synth_prior_lora(cfg, rank=4, seed=4, gain=0.1)
    N, D, L = args.steps, cfg["clip_dim"], cfg["text_ctx"]
    res["batches"] = {}
    for B in [int(b) for b in args.batches.split(",")]:
        g = torch.Generator(device="cuda").manual_seed(B)
        te = torch.randn(2, D, device="cuda", generator=g).repeat_interleave(B, 0)
        tenc = torch.randn(2, L, D, device="cuda", generator=g).repeat_interleave(B, 0)
        mask = torch.arange(L, device="cuda")[None, :] < torch.tensor([2] * B + [12] * B, device="cuda")[:, None]
        x_T = torch.randn(B, D, device="cuda", generator=g)
        noise = torch.randn(N, B, D, device="cuda", generator=g)
        mean, std = torch.zeros(D, device="cuda"), torch.ones(D, device="cuda")
        call = lambda: sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise)  # noqa: E731

        def use(arm):
            if arm == "base":
                m.unload_lora()
            else:
                m.load_lora(lora)

        outs = {}
        for arm in ("base", "lora_rank4"):   # warm-up: plan build, tuning, graph capture
            use(arm)
            outs[arm] = call().clone()
        times = {"base": [], "lora_rank4": []}
        for _ in range(args.rounds):
            for arm in times:
                use(arm)
                call()
                times[arm].append(_timed(call))
        m.unload_lora()
        r = {k: dict(min_ms=round(min(v), 3), median_ms=round(statistics.median(v), 3), all_ms=[round(t, 3) for t in v])
             for k, v in times.items()}
        r["outputs_differ_max_abs"] = (outs["base"] - outs["lora_rank4"]).abs().max().item()
        res["batches"][str(B)] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
