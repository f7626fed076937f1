"""Multi-GPU plumbing of the sampling path: one process per GPU, images sharded over ranks, ONE broadcast.

The reference is single-device (SURVEY.md 2.1); the path is embarrassingly parallel over images (8e): every
image's latent, CFG twin, noise stream and MoVQ decode are independent.  Rank r owns the contiguous block
[r*B/W, (r+1)*B/W) of the global batch; rank 0 holds the conditioning embeddings and broadcasts them once
(NCCL over NVLink on GPUs, gloo in the CPU tests); nothing else crosses ranks.  RNG is seeded per GLOBAL
sample index so results do not depend on the world size.  The 2.1 dynamic threshold uses GLOBAL sample 0's
percentile for the whole batch (gaussian_diffusion.py:290): rank 0 owns that sample and broadcasts the one float
per step (kandinsky2/model/gaussian_diffusion.py: FusedStep._update) -- the 2.1 p_sampler path's second,
4-byte collective; Kandinsky 2.2 has no threshold and keeps exactly one broadcast per generation.
"""
import torch


def world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(global_batch, rank, world_size):
    """Contiguous block of the global batch owned by `rank` (sizes differ by at most one)."""
    base, extra = divmod(global_batch, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def broadcast_conditioning(tensors, src=0):
    """In-place broadcast of a dict of equally-shaped-on-all-ranks tensors from `src`: the path's only collective.
    Packs everything into one flat buffer so exactly one collective is issued."""
    import torch.distributed as dist
    rank, ws = world()
    if ws == 1:
        return tensors
    keys = sorted(tensors)
    flat = torch.cat([tensors[k].reshape(-1).float() for k in keys])
    dist.broadcast(flat, src=src)
    off = 0
    for k in keys:
        n = tensors[k].numel()
        tensors[k].copy_(flat[off:off + n].reshape(tensors[k].shape).to(tensors[k].dtype))
        off += n
    return tensors


def sample_noise(global_indices, shape, base_seed=1234, device="cpu", steps=None):
    """N(0,1) draws keyed by GLOBAL sample index: [len(idx), *shape] (or [steps, len(idx), *shape])."""
    outs = []
    for gi in global_indices:
        g = torch.Generator(device="cpu").manual_seed(base_seed + int(gi))
        full = (steps,) + tuple(shape) if steps else tuple(shape)
        outs.append(torch.randn(full, generator=g))
    t = torch.stack(outs, 1 if steps else 0)
    return t.to(device)
