"""GPU: the CLIP text tower's two kernels (csrc/k2_clip_text.cu), bit for bit against the torch composition.

k2_clip_text_embed: fp16(float(tok[id]) + float(pos[t])) with one rounding, at the ids 0 and V - 1 and the tower's geometry, on
row-strided views: the ids rows have poison in their gap columns (ids that would read far out of the table), the output rows
sit in a guarded buffer whose gaps must stay untouched; an out-of-range id gives a NaN row.
k2_clip_text_pool: the pooled index (both rules: the first argmax, and the first eos or 0) and the widened row, with no eos, a
repeated eos and a literal eos early in the row, the hidden rows NaN-guarded and row-strided."""
import pytest
import torch

from tests.test_gpu_kernel_bounds import _Guarded, _bits

pytestmark = pytest.mark.gpu


def _strided_ids(ids, ldi, poison):
    """int32 [B, T] -> a [B, T] view with row stride ldi whose gap columns hold `poison`."""
    B, T = ids.shape
    buf = torch.full((B, ldi), poison, dtype=torch.int32, device="cuda")
    buf[:, :T] = ids
    return buf[:, :T]


@pytest.mark.parametrize("B,T,V,H", [(1, 77, 49408, 1280), (3, 77, 814, 128), (2, 5, 100, 8), (4, 128, 300, 64)])
def test_clip_text_embed_bit_exact(B, T, V, H):
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + T)
    tok = (torch.randn(V, H, device="cuda", generator=g) * 3).half()
    pos = (torch.randn(T + 3, H, device="cuda", generator=g) * 0.5).half()
    tok[0, :4] = torch.tensor([65504.0, -65504.0, 6e-8, 1.0], device="cuda").half()     # overflow and subnormal edges
    pos[0, :4] = torch.tensor([32.0, -32.0, 6e-8, 2 ** -11], device="cuda").half()
    ids = torch.randint(0, V, (B, T), device="cuda", generator=g, dtype=torch.int32)
    ids[0, 0], ids[-1, -1] = 0, V - 1
    iv = _strided_ids(ids, T + 5, V + 100000)
    go = _Guarded((B, T), H, ld=H + 16, out=True)
    ops.clip_text_embed(iv, tok, pos, out=go.view)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    ref = (tok.float()[ids.long()] + pos.float()[:T][None]).half()
    assert torch.equal(_bits(go.view), _bits(ref))
    assert torch.equal(_bits(ops.clip_text_embed(ids, tok, pos)), _bits(ref))       # the contiguous call


def test_clip_text_embed_out_of_range_id_is_a_nan_row():
    from kandinsky2 import ops
    tok = torch.randn(50, 64, device="cuda").half()
    pos = torch.randn(6, 64, device="cuda").half()
    ids = torch.tensor([[1, 50, 2, -1, 49, 3]], device="cuda", dtype=torch.int32)
    y = ops.clip_text_embed(ids, tok, pos)
    bad = torch.tensor([False, True, False, True, False, False], device="cuda")
    assert torch.isnan(y[0, bad]).all() and torch.isfinite(y[0, ~bad]).all()


def _pool_ref(ids, hidden, eos_id):
    if eos_id < 0:
        idx = ids.argmax(-1)
    else:
        idx = (ids == eos_id).int().argmax(-1)
    return idx, hidden[torch.arange(ids.shape[0], device=ids.device), idx].float()


@pytest.mark.parametrize("rule", ["argmax", "eos"])
def test_clip_text_pool_bit_exact(rule):
    from kandinsky2 import ops
    V, T, H = 49408, 77, 1280
    bos, eos, pad = V - 2, V - 1, 0
    g = torch.Generator(device="cuda").manual_seed(7 + (rule == "eos"))
    rows = []
    body = lambda n: torch.randint(1, bos, (n,), device="cuda", generator=g, dtype=torch.int32).tolist()  # noqa: E731
    for n in (0, 3, 20, 75):                                   # bos, n tokens, eos, pad
        rows.append([bos] + body(n) + [eos] + [pad] * (T - n - 2))
    rows.append([bos] + body(76))                              # no eos: the argmax is bos, the eos rule gives 0
    r = [bos] + body(10) + [eos] * 66                          # eos repeated as padding: the first one
    rows.append(r)
    r = [bos] + body(2) + [eos] + body(20) + [eos] + [pad] * 52   # a literal eos early in the row
    rows.append(r)
    rows.append([eos] * T)                                     # eos at position 0
    rows.append([7] * T)                                       # all equal: the first position
    ids = torch.tensor(rows, device="cuda", dtype=torch.int32)
    B = ids.shape[0]
    assert all(len(x) == T for x in rows)
    hidden = (torch.randn(B, T, H, device="cuda", generator=g) * 4).half()
    gh = _Guarded.of(hidden, ld=H + 8)
    go = _Guarded((B,), H, ld=H + 4, dtype=torch.float32, out=True)
    index = torch.full((B,), -5, device="cuda", dtype=torch.int32)
    eos_id = -1 if rule == "argmax" else eos
    iv = _strided_ids(ids, T + 3, V + 7 if rule == "argmax" else eos)     # the gaps would win if they were read
    ops.clip_text_pool(iv, gh.view, eos_id, out=go.view, index_out=index)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    idx, ref = _pool_ref(ids.long(), hidden, eos_id)
    assert index.long().tolist() == idx.tolist()
    assert torch.equal(_bits(go.view), _bits(ref))
    if rule == "argmax":
        assert idx.tolist()[4] == 0 and idx.tolist()[-1] == 0
    else:
        assert idx.tolist()[4:] == [0, 11, 3, 0, 0]
    assert torch.equal(ops.clip_text_pool(ids, hidden, eos_id), ref)      # contiguous, no index
