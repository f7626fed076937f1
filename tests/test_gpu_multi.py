"""2 GPUs (skipped on a 1-GPU box): the sharded pipelines reproduce the single-GPU images.

One process per GPU over NCCL; rank r denoises and decodes its contiguous block of the batch; the ONLY collective on the 2.2
path is the conditioning broadcast (plus, for Kandinsky 2.1's p_sampler, one 4-byte broadcast per step of the dynamic threshold,
which the reference takes from GLOBAL sample 0 for the whole batch, gaussian_diffusion.py:288-292).

Why not byte equality: a rank's UNet batch is half the single-GPU one, which changes the launch geometry (tile boxes at the small
levels may hold several images, split-K and the statistics kernels' chunking depend on the row count) and with it the fp32
summation ORDER of GroupNorm partial sums and split-K partial tiles -- nothing else.  A 1e-7 difference in a statistic flips the
fp16 rounding of a few activations (5e-4 each), and the random-weight test UNet (not a trained, well-conditioned denoiser)
amplifies that under classifier-free guidance 4 by roughly an order of magnitude per DDPM step, so after a few steps a sizeable share
of the uint8 pixels differ, mostly by 1.  So the assertion is a PSNR bound that
is far above what any sharding mistake (wrong noise stream, wrong conditioning row, wrong threshold) would leave: images of
DIFFERENT samples are < 20 dB apart, the sharded and single-GPU images of the SAME sample > 40 dB (2 steps) / > 30 dB (4)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tiny_overrides():
    return {"model_config": dict(num_channels=64, num_res_blocks=1, model_dim=128, channel_mult="1,2",
                                 attention_resolutions="32"),
            "image_enc_params": dict(params=dict(embed_dim=4, n_embed=64, ddconfig=dict(
                double_z=False, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=32, ch_mult=[1, 1, 2, 2],
                num_res_blocks=1, attn_resolutions=[32], dropout=0.0)))}


def _generate(version, batch):
    """-> {steps: uint8 [batch, 128, 128, 3]} for 2 and 4 denoising steps"""
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version=version, cache_dir="/nonexistent",
                          config_overrides=_tiny_overrides())
    out = {}
    for steps in (2, 4):
        if version == "2.2":
            imgs = pipe.generate_text2img("a red cat", batch_size=batch, decoder_steps=steps, h=128, w=128)
        else:  # p_sampler: DDPM with the per-step dynamic threshold of global sample 0
            imgs = pipe.generate_text2img("a red cat", num_steps=steps, batch_size=batch, guidance_scale=4, h=128, w=128,
                                          sampler="p_sampler")
        out[steps] = np.stack([np.asarray(im) for im in imgs])
    return out


def _worker(rank, world, port, version, batch, q):
    for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    imgs = _generate(version, batch)   # each rank returns ITS images (contiguous block of the global batch)
    q.put((rank, {k: v.copy() for k, v in imgs.items()}))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("version", ["2.2", "2.1"])
def test_two_gpus_reproduce_one_gpu(version):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    batch = 4
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, version, batch, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=150) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    single = _generate(version, batch)
    for steps in (2, 4):
        multi = np.concatenate([got[0][steps], got[1][steps]])
        assert multi.shape == single[steps].shape == (batch, 128, 128, 3)
        diff = np.abs(multi.astype(np.int16) - single[steps].astype(np.int16))
        frac = float((diff > 0).mean())
        psnr = [10 * np.log10(255.0 ** 2 / max(float((diff[i].astype(np.float64) ** 2).mean()), 1e-12)) for i in range(batch)]
        other = single[steps][[1, 0, 3, 2]].astype(np.int16)     # a DIFFERENT sample's image: what a sharding mistake looks like
        cross = 10 * np.log10(255.0 ** 2 / float(((multi.astype(np.int16) - other).astype(np.float64) ** 2).mean()))
        print(f"{version}, {steps} step(s): max uint8 difference {diff.max()}, differing pixels {frac:.2e}, PSNR per image "
              f"{[round(v, 1) for v in psnr]} dB (different samples: {cross:.1f} dB)")
        assert min(psnr) > (40.0 if steps == 2 else 30.0) and cross < 25.0, (psnr, cross)
