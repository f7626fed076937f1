"""CPU: the per-request LoRA adapters of the batcher without a GPU -- the argument checks of k2_conv_gemm_wmap (the mapped batched
GEMM the attention projections run as), ops.conv_gemm's refusal of a host map, and what the adapter registry refuses."""
import ctypes

import pytest
import torch

P = ctypes.c_void_p(256)   # never dereferenced: every call below fails its checks first


def _srcs():
    from kandinsky2._native import K2ConvSrc
    arr = (K2ConvSrc * 1)()
    arr[0].ptr, arr[0].C, arr[0].ld, arr[0].taps = 256, 128, 128, 1
    return arr


# arguments before the stream, all valid: 4 images of 12 x 12 tokens, 128 -> 384 channels, 3 slabs of 384 x 128
def _good():
    return [_srcs(), 1, 4, 12, 12, P, 384, 128, 128, 384, P, None, 0, P, 384, 0, None, 0, None, None, None, 384 * 128, 3, P]


WMAP_CASES = [({23: None}, "null w_map"), ({23: ctypes.c_void_p(258)}, "4-byte aligned"), ({22: 0}, "n_slabs"),
              ({22: -1}, "n_slabs"), ({21: 0}, "w_batch_stride must be > 0"), ({21: 12}, "multiple of 8"),
              ({5: None}, "null source, weight or output"), ({13: None}, "null source, weight or output"),
              ({0: None}, "null source, weight or output"), ({1: 4}, "1..3 sources"), ({15: 2}, "out_mode"),
              ({7: 100}, "Ktot"), ({14: 12}, "out alignment"), ({2: 0}, "bad geometry")]


@pytest.mark.parametrize("changes,msg", WMAP_CASES, ids=[m for _, m in WMAP_CASES])
def test_conv_gemm_wmap_refuses_bad_arguments_without_a_gpu(changes, msg):
    from kandinsky2 import _native
    lib = _native.load()
    args = _good()
    for i, v in changes.items():
        args[i] = v
    assert lib.k2_conv_gemm_wmap(*args, None) != 0
    assert msg in lib.k2_last_error().decode(), (changes, lib.k2_last_error())


def test_conv_gemm_refuses_a_host_map():
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    x = torch.zeros(2, 4, 4, 64, dtype=torch.float16)
    with pytest.raises(K2Error, match="CUDA"):
        ops.conv_gemm([(x, 1)], torch.zeros(64, 64, dtype=torch.float16), 64, w_batch_stride=64 * 64,
                      w_map=torch.zeros(2, dtype=torch.int32), n_slabs=1)


def test_batcher_refuses_a_negative_max_loras():
    from kandinsky2.pipelines import Kandinsky2_2
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="max_loras"):
            pipe.batcher(2, 64, 64, max_loras=bad)


def _bare_batcher(max_loras, slots=2, emb_dim=16, max_steps=10):
    """A Batcher with its host state only (a bare pipeline, no plan or graph): enough for the registry's refusals."""
    from kandinsky2.batching import Batcher, _SlotBatcher
    from kandinsky2.pipelines import Kandinsky2_2
    b = Batcher.__new__(Batcher)
    b.pipe, b.max_steps, b._emb_dim, b.max_loras = Kandinsky2_2.__new__(Kandinsky2_2), max_steps, emb_dim, max_loras
    b._loras, b.sampler = {}, "ddpm_sampler"
    _SlotBatcher.__init__(b, slots)
    return b


def _emb():
    return dict(image_embeds=torch.zeros(16), negative_image_embeds=torch.zeros(16), decoder_steps=5, seed=0)


def test_registry_refusals_on_a_bare_pipeline():
    """add_lora refuses a batcher made without slabs, a duplicate name and a full table before touching a weight; submit
    refuses an unknown adapter; remove_lora refuses an unknown name and an adapter a waiting request uses."""
    with pytest.raises(ValueError, match="max_loras=0"):
        _bare_batcher(0).add_lora("a", {})
    b = _bare_batcher(2)
    b._loras = {"a": (1, {}), "b": (2, {})}
    with pytest.raises(ValueError, match="already registered"):
        b.add_lora("a", {})
    with pytest.raises(ValueError, match="slabs are in use"):
        b.add_lora("c", {})
    with pytest.raises(ValueError, match="no adapter named 'c'"):
        b.submit(**_emb(), lora="c")
    with pytest.raises(ValueError, match="no adapter named 'a'"):
        _bare_batcher(0).submit(**_emb(), lora="a")
    assert not b.queue.waiting and not b._requests
    h = b.submit(**_emb(), lora="a")
    b.submit(**_emb())
    with pytest.raises(ValueError, match="used by a waiting or active request"):
        b.remove_lora("a")
    with pytest.raises(ValueError, match="no adapter named 'z'"):
        b.remove_lora("z")
    b.remove_lora("b")
    assert list(b._loras) == ["a"]
    del b._requests[h]
    b.remove_lora("a")
    assert not b._loras
