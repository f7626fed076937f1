"""What per-request LoRA adapters cost the Kandinsky 2.2 batcher at full size (synthetic weights of the architecture), in one
process on cuda:0:
  * step time: the mean time of one step() with all max_batch slots occupied, max_loras=0 (the plain batcher) against
    max_loras=4 with a different adapter in each slot (attention projections as mapped batched GEMMs, never split in K);
  * add_lora: the time to merge one adapter into a slab (every attention layer's qkv / proj_out / encoder_kv weights), rank 4
    and rank 64, ending in a device synchronise;
  * memory: the device bytes of one slab (qkv + proj_out of every attention layer) plus one adapter's merged encoder_kv
    weights, from the tensor sizes, and the allocator's growth per adapter slab between max_loras=0 and max_loras=4.
Step times are host clock over --timed steps, ending in a device synchronise, after --warmup steps with every slot busy.  The
card's name, power limit and maximum SM clock are read in the same run (nvidia-smi query only).  Needs a CUDA sm_90 device.

    python profiles/batcher_lora.py [--size 768] [--slots 4] [--steps 50] [--out profiles/batcher_lora_h100.json]
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


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def _adapter(model, rank, seed):
    from oracle import unet_oracle as uo
    from tests import lora_oracle as lo
    cfg = dict(uo.CONFIG_2_2, in_channels=model.in_channels, model_channels=model.model_channels,
               channel_mult=tuple(model.channel_mult), num_res_blocks=model.num_res_blocks,
               attention_ds=tuple(model.attention_resolutions), model_dim=model.model_dim, inpainting=False)
    return lo.synth_lora(cfg, rank=rank, seed=seed)


def step_time(b, req, loras, warmup, timed):
    """Mean seconds per step() with every slot occupied by a request of the batcher's max_steps steps."""
    for i, name in enumerate(loras):
        b.submit(**req, seed=i, lora=name)
    for _ in range(warmup):
        b.step()
    assert all(h is not None for h in b.queue.holder)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(timed):
        b.step()
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / timed
    assert all(h is not None for h in b.queue.holder)
    b.run()
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=768)
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--timed", type=int, default=40)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "batcher_lora_h100.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("batcher_lora.py needs a CUDA sm_90 device")
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent")
    pipe.model.finalize()
    pos = pipe.embedder.image_emb("a red cat", 1)
    neg = pipe.embedder.zero_image_emb(1)
    req = dict(image_embeds=pos, negative_image_embeds=neg, decoder_steps=a.steps, decoder_guidance_scale=4.0)
    S, L = a.slots, 4
    assert a.warmup + a.timed < a.steps

    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    b0 = pipe.batcher(S, a.size, a.size, max_steps=a.steps)
    torch.cuda.synchronize()
    mem_plain = torch.cuda.memory_allocated() - mem0
    t_plain = step_time(b0, req, [None] * S, a.warmup, a.timed)
    del b0
    torch.cuda.synchronize()

    mem0 = torch.cuda.memory_allocated()
    b4 = pipe.batcher(S, a.size, a.size, max_steps=a.steps, max_loras=L)
    torch.cuda.synchronize()
    mem_lora = torch.cuda.memory_allocated() - mem0
    layers = b4.plan.attn_slabs["layers"]
    slab_bytes = sum(t[0].numel() * t.element_size() for pair in layers.values() for t in pair)
    wenc_bytes = sum(w.numel() * w.element_size() for w in b4._wenc0.values())
    add = {}
    for rank in (4, 64):
        sd = _adapter(pipe.model, rank, seed=rank)
        b4.add_lora("warm", sd)   # first call: the per-adapter host work of lora_to_k2 is timed below as well
        b4.remove_lora("warm")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b4.add_lora("timed", sd)
        torch.cuda.synchronize()
        add[f"rank_{rank}_s"] = round(time.perf_counter() - t0, 4)
        b4.remove_lora("timed")
    names = [f"style_{i}" for i in range(S)]
    for i, n in enumerate(names):
        b4.add_lora(n, _adapter(pipe.model, 8, seed=100 + i))
    mem_after = torch.cuda.memory_allocated() - mem0
    t_lora = step_time(b4, req, [names[i % L] for i in range(S)], a.warmup, a.timed)

    out = dict(card=_card(), size=a.size, slots=S, request_steps=a.steps, sampler="ddpm_sampler", timed_steps=a.timed,
               step_ms=dict(max_loras_0=round(t_plain * 1e3, 2), max_loras_4_four_adapters=round(t_lora * 1e3, 2),
                            ratio=round(t_lora / t_plain, 4)),
               add_lora=add,
               memory=dict(attention_layers=len(layers), slab_bytes=slab_bytes, encoder_kv_bytes_per_adapter=wenc_bytes,
                           batcher_bytes_max_loras_0=mem_plain, batcher_bytes_max_loras_4=mem_lora,
                           growth_with_4_adapters_registered=mem_after - mem_lora))
    print(json.dumps(out))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
