"""kandinsky2 (H100-native): drop-in for the ai-forever/Kandinsky-2 denoising hot path.

Same import name and entry points as the reference package (kandinsky2/__init__.py:164-192):
`get_kandinsky2(device, task_type, ..., model_version)` returning an object with
`generate_text2img / mix_images / generate_img2img / generate_inpainting`; the arithmetic of the
UNet + sampler + MoVQ decoder runs in libk2b200.so (hand-written sm_90a CUDA, see include/k2b200.h).
"""
__version__ = "0.1.0"


def get_kandinsky2(*args, **kwargs):
    from .factory import get_kandinsky2 as _g
    return _g(*args, **kwargs)
