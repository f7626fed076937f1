"""TEST INFRASTRUCTURE (oracle): LoRA adapters of the Kandinsky 2.2 diffusion prior in diffusers' attention-processor format,
and the prior's diffusers-form forward with the adapter run UNFUSED, as diffusers 0.19's `LoRAAttnProcessor` runs it.

  synth_prior_lora       <- the state dict `AttnProcsLayers` saves for `LoRAAttnProcessor(hidden_size=width)` on every
                            transformer_blocks.{i}.attn1 (notebooks/lora_decoder.ipynb cells 12-13, 18):
                            transformer_blocks.{i}.attn1.processor.{to_q,to_k,to_v,to_out}_lora.{down,up}.weight
  lora_prior_forward     <- tests/prior22_oracle.py's diffusers_prior_forward with LoRAAttnProcessor.__call__ in the attention:
                            to_q(h) + scale * up(down(h)), likewise to_k / to_v, and to_out[0](a) + scale * up(down(a))
                            (LoRALinearLayer without network_alpha)

Parity unpinned: diffusers is not installed and the notebook's adapter file is not available, so the key names and the
processor arithmetic are restated from diffusers 0.19's published classes.  It computes the adapter in the DIFFUSERS layout,
unfused, so it shares nothing with the product's packed path (checkpoints.prior_lora_to_k2 + k2_lora_merge).  With an empty
adapter it is diffusers_prior_forward (tests/test_cpu_prior_lora.py checks that)."""
import math

import torch
import torch.nn.functional as F

from tests import prior22_oracle as p22

PROJECTIONS = ("to_q", "to_k", "to_v", "to_out")


def synth_prior_lora(cfg, rank, seed=0, gain=0.3, projections=PROJECTIONS, dtype=torch.float32):
    """A notebook-format prior adapter with BOTH factors random (diffusers initialises `up` to zero, which would test nothing):
    down ~ N(0, 1/width), up ~ N(0, gain^2/rank), so each delta W = up @ down has entries of variance gain^2/width and
    ||delta W|| is about gain * ||W|| for a weight of oracle/synth.py (entries N(0, 1/width))."""
    g = torch.Generator().manual_seed(seed)
    W = cfg["xf_width"]
    out = {}
    for i in range(cfg["xf_layers"]):
        for proj in projections:
            p = f"transformer_blocks.{i}.attn1.processor.{proj}_lora."
            out[p + "down.weight"] = (torch.randn(rank, W, generator=g) / W ** 0.5).to(dtype)
            out[p + "up.weight"] = (torch.randn(W, rank, generator=g) * (gain / rank ** 0.5)).to(dtype)
    return out


def lora_prior_forward(sd, cfg, lora, scale, x, timesteps, text_emb, text_enc, mask, dtype=torch.float32):
    """diffusers_prior_forward (tests/prior22_oracle.py) with the adapter `lora` (synth_prior_lora's keys, any subset) applied
    unfused at `scale`.  sd: diffusers keys, in `dtype`; the factors are cast to `dtype` on sd's device, as LoRALinearLayer
    runs in its own dtype."""
    W, H = cfg["xf_width"], cfg["xf_heads"]
    N, d = x.shape[0], W // H
    dev = sd["positional_embedding"].device
    lin = lambda name, v: F.linear(v, sd[name + ".weight"], sd[name + ".bias"])  # noqa: E731
    ln = lambda v, name: F.layer_norm(v, (W,), sd[name + ".weight"], sd[name + ".bias"])  # noqa: E731

    def proj(i, name, weight, v):
        y = lin(f"transformer_blocks.{i}.attn1.{weight}", v)
        p = f"transformer_blocks.{i}.attn1.processor.{name}_lora."
        if p + "down.weight" in lora:
            down, up = (lora[p + s].to(dev, dtype) for s in ("down.weight", "up.weight"))
            y = y + scale * F.linear(F.linear(v, down), up)
        return y

    x, text_emb, text_enc = x.to(dtype), text_emb.to(dtype), text_enc.to(dtype)
    t_emb = lin("time_embedding.linear_2", F.silu(lin("time_embedding.linear_1", p22._time_proj(timesteps, W).to(dtype))))
    h = torch.cat([lin("encoder_hidden_states_proj", text_enc), lin("embedding_proj", text_emb)[:, None], t_emb[:, None],
                   lin("proj_in", x)[:, None], sd["prd_embedding"].expand(N, -1, -1)], dim=1)
    h = h + sd["positional_embedding"].to(dtype)
    n = h.shape[1]
    causal = torch.full((n, n), -10000.0, device=x.device).triu_(1)
    add = F.pad((1 - mask.to(dtype)) * -10000.0, (0, 4), value=0.0)
    add = (add[:, None, :] + causal).to(dtype)                                   # [N, n, n]
    for i in range(cfg["xf_layers"]):
        p = f"transformer_blocks.{i}."
        y = ln(h, p + "norm1")
        q, k, v = (proj(i, f"to_{c}", f"to_{c}", y).view(N, n, H, d).transpose(1, 2) for c in "qkv")
        w = (q @ k.transpose(-1, -2)) / math.sqrt(d) + add[:, None]
        a = (torch.softmax(w.float(), dim=-1).to(dtype) @ v).transpose(1, 2).reshape(N, n, W)
        h = h + proj(i, "to_out", "to_out.0", a)
        y = ln(h, p + "norm3")
        h = h + lin(p + "ff.net.2", F.gelu(lin(p + "ff.net.0.proj", y)))
    h = ln(h, "norm_out")
    return lin("proj_to_clip_embeddings", h[:, -1]).float()
