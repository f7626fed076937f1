"""Cost of the Kandinsky 2.1 text encoder (kandinsky2/model/text_encoders.py) at XLM-RoBERTa-large size (synthetic weights of the
architecture: 24 layers, hidden 1024, 16 heads of 64, MLP 4096, vocabulary 250002, 514 positions, 77 tokens, Linear 1024 ->
768).

Measures, in one process on cuda:0, and prints one JSON line (also written to --out if given):
  * the tower at n = 2 (encode_text's prompt + "") and n = 8 rows of 77 tokens: one CUDA graph replay of the launch plan, the
    same launch list issued eagerly, and the oracle's torch fp16 forward (tests/xlmr_oracle.py, the halved reference model's
    arithmetic, a side baseline on the same GPU); the arms alternate within each repetition after a warm-up, median and min of
    --reps repetitions, CUDA events;
  * per-kind kernel time of one eager pass (CUDA events around every launch);
  * the non-embedding weight stream (the packed GEMM weights, fp16) over the replay time, and its share of the 3.35 TB/s
    data-sheet bandwidth (the tower reads every weight once per call, so at small n that stream is its floor);
  * the tokenizer's host time for encode_text's two distinct prompts (the tiny tokenizer of tests/golden/xlmr_tiny.pt: the same
    code path, a smaller vocabulary than the released one), perf_counter.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/xlmr_text.py [--reps 10] [--out /tmp/xlmr_text.json]
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
from profiles.controlnet_img2img import _card  # noqa: E402

HBM_TB_PER_S = 3.35   # NVIDIA H100 SXM data sheet


def flops_per_row(cfg, out, T=77):
    """Multiply-adds x 2 of one T-token row: per layer qkv / out-proj / fc1 / fc2 and the two attention products, the Linear."""
    H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    gemm = L * 2 * T * (3 * H * H + H * H + 2 * H * I) + 2 * H * out
    attn = L * 4 * T * T * H
    return gemm + attn, attn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ns", default="2,8")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("xlmr_text.py needs a CUDA sm_90 device")
    from kandinsky2.checkpoints import mclip_to_k2
    from kandinsky2.model.text_encoders import MultilingualCLIP
    from tests import xlmr_oracle as xo
    from tests.test_gpu_zz_text_encoder import large_ids
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg, out = xo.CONFIG_LARGE, xo.OUT_LARGE
    total, attn = flops_per_row(cfg, out)
    sd16 = {k: v.cuda().half() for k, v in xo.synth_weights(cfg, out, 1).items()}
    tower = MultilingualCLIP(mclip_to_k2(sd16, cfg["num_hidden_layers"]), cfg, device="cuda").finalize()
    wbytes = sum(t.numel() * t.element_size() for L in tower._packed["layers"]
                 for t, _ in (L[n] for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")))
    res = dict(card=_card(), reps=args.reps, flops_per_row=total, attention_flops_per_row=attn, layer_weight_bytes=wbytes,
               weight_floor_ms=round(wbytes / (HBM_TB_PER_S * 1e12) * 1e3, 3), tower={})
    for n in [int(x) for x in args.ns.split(",")]:
        ids, mask = large_ids(n, seed=n, lengths=(20, 2))
        plan = tower._plan(n)
        plan.ids.copy_(ids)
        plan.mask.copy_(mask)
        idc, mc = ids.cuda(), mask.cuda()
        with torch.no_grad():
            r = _alternate({"graph": lambda: plan.run(True), "eager": lambda: plan.run(False),
                            "torch_fp16": lambda: xo.forward(sd16, cfg, idc, mc, dtype=torch.float16)}, args.reps)
        g = r["graph"]["median_ms"]
        r["graph_tflops"] = round(n * total / (g * 1e-3) / 1e12, 1)
        r["weight_tb_per_s"] = round(wbytes / (g * 1e-3) / 1e12, 2)
        r["weight_stream_share_of_datasheet"] = round(wbytes / (g * 1e-3) / 1e12 / HBM_TB_PER_S, 3)
        r["speedup_vs_torch_fp16"] = round(r["torch_fp16"]["median_ms"] / g, 2)
        prof = plan.profile(reps=3)
        r["kernel_ms"] = {k: round(v["ms"], 3) for k, v in prof.items()}
        r["launches"] = sum(v["launches"] for v in prof.values())
        res["tower"][str(n)] = r
    del sd16
    torch.cuda.empty_cache()

    tok = xo.k2_tokenizer(xo.fixture_json(torch.load(xo.FIXTURE)))
    prompts = ["A capybara, 4k photo, highly detailed, trending on artstation, красивый пейзаж, 富士山と桜の花", ""]
    host = []
    for _ in range(args.reps):
        tok.model._cache.clear()
        t0 = time.perf_counter()
        tok(prompts)
        host.append((time.perf_counter() - t0) * 1e3)
    res["tokenizer_2_prompts_ms"] = dict(median_ms=round(statistics.median(host), 3), min_ms=round(min(host), 3))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
