"""CPU: the diffusion prior's entry points (csrc/k2_prior.cu) refuse bad sequence lengths, strides and pointers before any
CUDA call, and ops.attention_small refuses keep masks the kernel would misread.  Fabricated device addresses, one defect per
call, as in tests/test_cpu_vector_arg_checks.py: nothing is launched."""
import pytest
import torch

from tests.test_cpu_vector_arg_checks import A, P, _refused, _with

# k2_attention_small(qkv, ldq, keep_mask, causal, out, ldo, B, T, heads, scale, stream)
ATTN = dict(qkv=P(A), ldq=6144, keep=P(A), causal=1, out=P(A), ldo=2048, B=2, T=81, heads=32, scale=0.125, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(T=0), "sequence length"),
    (dict(T=129), "sequence length"),
    (dict(T=-1), "sequence length"),
    (dict(ldq=6145), "row strides"),              # odd: the q row is read as half2
    (dict(ldo=2049), "row strides"),              # odd: the output is written as half2
    (dict(ldq=6142), "row strides"),              # < heads * 192
    (dict(ldo=2046), "row strides"),              # < heads * 64
    (dict(qkv=P(A + 2)), "alignment"),
    (dict(out=P(A + 6)), "alignment"),
    (dict(qkv=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(heads=0), "bad arguments"),
])
def test_attention_small_refuses(change, msg):
    _refused("k2_attention_small", list(_with(ATTN, **change).values()), msg)


@pytest.mark.parametrize("change", [dict(M=0), dict(N=0), dict(ldx=2047), dict(ldy=100), dict(gamma=None), dict(y=None)])
def test_layernorm_f16_refuses(change):
    # k2_layernorm_f16(x, ldx, gamma, beta, y, ldy, M, N, eps, stream)
    base = dict(x=P(A), ldx=2048, gamma=P(A), beta=P(A), y=P(A), ldy=2048, M=81, N=2048, eps=1e-5, stream=None)
    _refused("k2_layernorm_f16", list(_with(base, **change).values()), "layernorm_f16")


@pytest.mark.parametrize("x,y,n,msg", [
    (A, A, 7, "even element count"),
    (A, A, 0, "even element count"),
    (A + 2, A, 8, "alignment"),
    (A, A + 2, 8, "alignment"),
])
def test_gelu_f16_refuses(x, y, n, msg):
    _refused("k2_gelu_f16", [P(x), P(y), n, None], msg)


def _cpu_attention_args(B=2, T=9, heads=2):
    return torch.zeros(B, T, heads * 192, dtype=torch.float16), heads


@pytest.mark.parametrize("keep", [
    torch.ones(2, 9, dtype=torch.int64),            # wrong dtype: 8 bytes per key
    torch.ones(2, 9, dtype=torch.float32),
    torch.ones(2, 8, dtype=torch.uint8),            # wrong shape
    torch.ones(2, 9, 1, dtype=torch.uint8),
    torch.ones(9, 2, dtype=torch.uint8).t(),        # [B, T] but not contiguous
    torch.ones(2, 18, dtype=torch.bool)[:, ::2],
])
def test_attention_small_refuses_bad_keep_mask(keep):
    """Checked in Python before the library is reached (the tensors here are on the CPU and must never get to a kernel)."""
    from kandinsky2 import ops
    qkv, heads = _cpu_attention_args()
    with pytest.raises(AssertionError):
        ops.attention_small(qkv, heads, keep_mask=keep)


def test_attention_small_refuses_bad_qkv():
    from kandinsky2 import ops
    qkv, heads = _cpu_attention_args()
    with pytest.raises(AssertionError):
        ops.attention_small(qkv.float(), heads)
    with pytest.raises(AssertionError):
        ops.attention_small(qkv, heads + 1)           # width is not heads * 192
