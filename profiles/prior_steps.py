"""Cost of the Kandinsky 2.2 diffusion prior at full size (20 layers, width 2048, CLIP-bigG 1280, 77 + 4 tokens; synthetic
weights of the architecture), 25 UnCLIP steps with guidance 4, at B = 1 and 4 samples (2B CFG rows).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * the prior call (bind + 25 steps + the clip_std / clip_mean affine) with every step one CUDA graph replay (sample_prior22)
    against the eager loop: PriorTransformer.forward per step plus the same k2_sampler_step update.  CUDA events over
    --calls steady-state calls per arm, the arms alternated in this process; min and median;
  * the Kandinsky 2.1 prior's sample_prior (eager, cond-first CFG, its own 768-wide size) at the same B and steps, for reference;
  * per-kind device time of one step from the step plan's profile() (CUDA events around every launch, eager and serial);
  * the GEMM and linear weight bytes one step reads, over the graph-replayed step time, against the 3.35 TB/s of HBM3 in
    NVIDIA's H100 SXM data sheet (a share of the data-sheet figure, not of a measured peak).
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/prior_steps.py [--calls 5] [--out /tmp/prior_steps.json]
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

import torch  # noqa: E402

HBM_TBS = 3.35


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


def _prior(cfg, seed):
    from kandinsky2.model.prior import PriorTransformer
    from oracle import prior_oracle as po, synth
    m = PriorTransformer(**cfg, device="cuda")
    m.load_state_dict({k: v.cuda() for k, v in synth.synth_state_dict(po.prior_param_spec(cfg), seed=seed).items()}, strict=True)
    return m.finalize()


def _step_weight_bytes(m):
    """Bytes of weights one step reads: the fp16 packed GEMM matrices of the 20 blocks, and the fp32 time_embed, clip_img_proj
    and out_proj matrices (text_enc_proj and text_emb_proj run once per call)."""
    n = sum(L[k][0].numel() * L[k][0].element_size() for L in m._packed["layers"]
            for k in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2"))
    for mod in (getattr(m.time_embed, "0"), getattr(m.time_embed, "2"), m.clip_img_proj, m.out_proj):
        n += mod.weight.numel() * mod.weight.element_size()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--calls", type=int, default=5, help="timed calls per arm and batch size")
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prior_steps.py needs a CUDA sm_90 device")
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import space_timesteps
    from kandinsky2.model.prior import UnCLIPSchedule, sample_prior, sample_prior22
    from oracle import prior_oracle as po
    from tests import prior22_oracle as p22
    torch.backends.cuda.matmul.allow_tf32 = False
    N = args.steps
    res = dict(card=_card(), steps=N, guidance=4.0, calls=args.calls, batches={})
    m22 = _prior(p22.CONFIG_PRIOR22, seed=1)
    m21 = _prior(po.CONFIG_PRIOR, seed=2)
    wbytes = _step_weight_bytes(m22)
    res["weight_bytes_per_step"] = wbytes
    sched = UnCLIPSchedule(N)
    table = torch.from_numpy(sched.coef_table()).cuda()
    use21 = sorted(space_timesteps(1000, [N]))
    for B in [int(b) for b in args.batches.split(",")]:
        g = torch.Generator(device="cuda").manual_seed(B)

        def cond(D, X, L=77):
            te = torch.randn(2, D, device="cuda", generator=g).repeat_interleave(B, 0)
            tenc = torch.randn(2, L, X, device="cuda", generator=g).repeat_interleave(B, 0)
            mask = torch.arange(L, device="cuda")[None, :] < torch.tensor([2] * B + [12] * B, device="cuda")[:, None]
            return te, tenc, mask

        D = 1280
        te, tenc, mask = cond(D, D)
        x_T = torch.randn(B, D, device="cuda", generator=g)
        noise = torch.randn(N, B, D, device="cuda", generator=g)
        mean, std = torch.zeros(D, device="cuda"), torch.ones(D, device="cuda")
        mo = torch.zeros(2 * B, 2 * D, device="cuda")
        work = torch.empty(B * D + 4096, device="cuda")

        def graph_call():
            return sample_prior22(m22, te, tenc, mask, N, 4.0, mean, std, x_T, noise)

        def eager_call():
            x = x_T.clone()
            for k, t in enumerate(sched.timesteps):
                mo[:, :D] = m22(torch.cat([x, x]), torch.full((2 * B,), float(t), device="cuda"), text_emb=te, text_enc=tenc,
                                mask=mask)
                ops.sampler_step(mo.view(2 * B, 8, 1, D // 4), x.view(B, 4, 1, D // 4), noise[k].view(B, 4, 1, D // 4), table[k],
                                 4.0, 0, clip=10.0, work=work)
            return x * std + mean

        te21, tenc21, mask21 = cond(768, 768)
        mask21 = torch.cat([mask21[B:], mask21[:B]])       # 2.1 rows are [prompt | ""]
        x21, n21 = torch.randn(B, 768, device="cuda", generator=g), torch.randn(N, B, 768, device="cuda", generator=g)

        def call21():
            return sample_prior(m21, te21, tenc21, mask21, use21, 4.0, torch.zeros(768, device="cuda"),
                                torch.ones(768, device="cuda"), x21, n21)

        arms = {"graph": graph_call, "eager": eager_call, "prior21_eager": call21}
        for fn in arms.values():     # warm-up: plan build, tuning, graph capture
            fn()
        a, b = graph_call(), eager_call()
        times = {k: [] for k in arms}
        for _ in range(args.calls):
            for k, fn in arms.items():
                times[k].append(_timed(fn))
        plan = m22._step_plan(B)
        kinds = {k: dict(ms=round(v["ms"], 4), launches=v["launches"]) for k, v in plan.profile(reps=5).items()}
        step_ms = min(times["graph"]) / N
        r = {k: dict(min_ms=round(min(v), 3), median_ms=round(statistics.median(v), 3)) for k, v in times.items()}
        r["graph_vs_eager_speedup"] = round(min(times["eager"]) / min(times["graph"]), 3)
        r["graph_step_ms"] = round(step_ms, 4)
        r["weight_GBps_per_step"] = round(wbytes / (step_ms * 1e-3) / 1e9, 1)
        r["share_of_3p35TBps"] = round(wbytes / (step_ms * 1e-3) / (HBM_TBS * 1e12), 3)
        r["graph_vs_eager_max_abs"] = (a - b).abs().max().item()
        r["per_kind_ms_one_step"] = kinds
        res["batches"][str(B)] = r
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
