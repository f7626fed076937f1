"""GPU: the Kandinsky 2.1 text encoder's kernels against float64 evaluations of the same fp16 inputs, bounds in fp16 ulps.

k2_xlmr_embed: LayerNorm(word[id] + type_row + pos[p]) with the positions computed from the ids, at XLM-R-large's width;
padding at the end, in the middle and rows of padding only, T = 1..77, rows offset by large means, out-of-range ids and
positions (NaN rows), id rows whose gap columns hold ids that would move the positions if they were read, output rows in a
guarded buffer whose gaps must stay untouched.
k2_masked_mean_f16: holed masks, a row with no kept token (NaN), strided and guarded views.
k2_attention_small as the text encoder calls it: not causal, tokenizer-style key masks, 16 heads, T = 77."""
import pytest
import torch

from tests.test_gpu_kernel_bounds import _Guarded, _bits
from tests.test_gpu_prior_kernels import _check_attention, _qkv, _ulp16
from tests.xlmr_oracle import position_ids

pytestmark = pytest.mark.gpu

PAD = 1


def _tables(V, P, H, seed, offset=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    word = (torch.randn(V, H, device="cuda", generator=g) * 0.5 + offset).half()
    pos = (torch.randn(P, H, device="cuda", generator=g) * 0.3).half()
    typ = (torch.randn(H, device="cuda", generator=g) * 0.1).half()
    gamma = 1.0 + 0.1 * torch.randn(H, device="cuda", generator=g)
    beta = 0.1 * torch.randn(H, device="cuda", generator=g)
    return word, pos, typ, gamma, beta


def _embed_ref(ids, word, pos, typ, gamma, beta, eps):
    """float64 of transformers' embeddings (positions from the ids), and the kernel's allowance: one fp16 ulp plus the
    LayerNorm affine term of the prior's LayerNorm test, plus the two fp32 roundings of the table sum (2^-23 of the summands'
    magnitude each, carried through x_hat with a factor 2 for their effect on the statistics)."""
    p = position_ids(ids.long(), PAD)
    w, t, q = word.double()[ids.long()], typ.double(), pos.double()[p]
    x = w + t + q
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + eps)
    xhat = (x - mean) * rstd
    ref = xhat * gamma.double() + beta.double()
    mag = (w.abs() + t.abs() + q.abs()) * rstd * gamma.double().abs()
    allow = _ulp16(ref) + 2.0 ** -20 * ((gamma.double() * xhat).abs() + beta.double().abs()) + 2.0 ** -21 * mag
    return ref, allow


def _check_embed(y, ref, allow, what):
    err = (y.double() - ref).abs()
    bad = err > allow
    assert not bad.any(), (what, int(bad.sum()), err[bad][:4].tolist(), ref[bad][:4].tolist())
    return (err / _ulp16(ref)).max().item()


def _strided_ids(ids, ldi, poison):
    B, T = ids.shape
    buf = torch.full((B, ldi), poison, dtype=torch.int32, device="cuda")
    buf[:, :T] = ids
    return buf[:, :T]


def _rows(B, T, V, seed, lengths):
    """<s>, random ids, </s>, then padding, per row of the given real length."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ids = torch.full((B, T), PAD, dtype=torch.int32, device="cuda")
    for r in range(B):
        L = lengths[r % len(lengths)]
        if L:
            ids[r, :L] = torch.randint(3, V, (L,), device="cuda", generator=g, dtype=torch.int32)
            ids[r, 0] = 0
            ids[r, L - 1] = 2
    return ids


@pytest.mark.parametrize("offset", [0.0, 30.0, 1000.0])
@pytest.mark.parametrize("T", [1, 2, 5, 33, 64, 77])
def test_xlmr_embed_vs_float64(T, offset):
    from kandinsky2 import ops
    V, P, H, eps = 1000, T + PAD + 3, 1024, 1e-5
    word, pos, typ, gamma, beta = _tables(V, P, H, seed=T, offset=offset)
    ids = _rows(4, T, V, seed=T + 1, lengths=(T, max(T // 2, 1), 0, 1))
    if T >= 5:
        ids[1, 1] = PAD                               # padding in the middle: the later positions do not count it
        ids[0, 2:4] = PAD
    iv = _strided_ids(ids, T + 7, 5)                  # gap ids are real tokens: reading them would move the positions
    go = _Guarded((4, T), H, ld=H + 16, out=True)
    ops.xlmr_embed(iv, PAD, word, pos, typ, gamma, beta, eps, out=go.view)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    ref, allow = _embed_ref(ids, word, pos, typ, gamma, beta, eps)
    worst = _check_embed(go.view, ref, allow, (T, offset))
    assert torch.equal(_bits(ops.xlmr_embed(ids, PAD, word, pos, typ, gamma, beta, eps)), _bits(go.view))
    print(f"xlmr_embed T={T} offset={offset}: worst {worst:.3f} ulp")


def test_xlmr_embed_nan_rows():
    """An id outside [0, V) or a position beyond the table gives a NaN row; its neighbours are exact."""
    from kandinsky2 import ops
    V, H, T = 50, 64, 12
    P = PAD + 1 + 8                                    # positions up to 9: the 9th real token of a row is out of the table
    word, pos, typ, gamma, beta = _tables(V, P, H, seed=3)
    ids = torch.tensor([[0, 5, 6, 50, 7, -1, 2] + [PAD] * 5,
                        [0] + list(range(3, 13)) + [2]], dtype=torch.int32, device="cuda")
    y = ops.xlmr_embed(ids, PAD, word, pos, typ, gamma, beta, 1e-5)
    p = position_ids(ids.long(), PAD)
    bad = (ids < 0) | (ids >= V) | (p >= P)
    assert bad.sum().item() == 2 + 4
    assert torch.isnan(y[bad]).all() and torch.isfinite(y[~bad]).all()
    ok = ~bad
    ref, allow = _embed_ref(ids.clamp(0, V - 1), word, torch.cat([pos, pos[:8]]), typ, gamma, beta, 1e-5)
    _check_embed(y[ok], ref[ok], allow[ok], "neighbours")


@pytest.mark.parametrize("B,T,H", [(2, 77, 1024), (5, 77, 1024), (3, 9, 300)])
def test_masked_mean_vs_float64(B, T, H):
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(B * T)
    hidden = (torch.randn(B, T, H, device="cuda", generator=g) * 4).half()
    mask = (torch.rand(B, T, device="cuda", generator=g) < 0.6).to(torch.uint8)
    mask[:, 0] = 1
    mask[-1] = 0                                       # no kept token: NaN
    gh = _Guarded.of(hidden, ld=H + 8)
    mbuf = torch.full((B, T + 5), 1, dtype=torch.uint8, device="cuda")
    mbuf[:, :T] = mask
    go = _Guarded((B,), H, ld=H + 4, dtype=torch.float32, out=True)
    ops.masked_mean_f16(gh.view, mbuf[:, :T], out=go.view)
    torch.cuda.synchronize()
    ok, msg = go.untouched()
    assert ok, msg
    m = mask.double()[..., None]
    cnt = m.sum(1)
    ref = (hidden.double() * m).sum(1) / cnt
    # fp32 chain of at most T additions (gamma_T of the kept magnitudes) and the division's rounding
    allow = (T * 2.0 ** -24 * (hidden.double().abs() * m).sum(1) / cnt + 2.0 ** -24 * ref.abs())[:-1]
    got = go.view.double()
    assert torch.isnan(got[-1]).all()
    err = (got[:-1] - ref[:-1]).abs()
    assert (err <= allow).all(), (err.max().item(), allow.min().item())
    for m_ in (mask, mask.bool()):                                   # contiguous operands, uint8 or bool mask: the same bits
        assert torch.equal(_bits(ops.masked_mean_f16(hidden, m_)), _bits(go.view.contiguous()))


@pytest.mark.parametrize("B", [2, 8])
def test_attention_small_noncausal_key_masks(B):
    """The encoder's attention: 16 heads of 64, T = 77, not causal, the tokenizer's attention mask (a prefix that always keeps
    <s>) as the key keep-mask, within attention_small's existing float64 bound."""
    from kandinsky2 import ops
    T, heads = 77, 16
    lengths = [2, 3, 20, 77, 40, 2, 77, 11][:B]
    keep = (torch.arange(T, device="cuda")[None] < torch.tensor(lengths, device="cuda")[:, None]).to(torch.uint8)
    qkv = _qkv(B, T, heads, seed=B, std=1.5)
    out = ops.attention_small(qkv, heads, keep_mask=keep, causal=False, scale=0.125)
    ulps, share = _check_attention(out, qkv, heads, keep, False, 0.125, "text encoder")
    assert torch.isfinite(out).all()
    print(f"attention_small non-causal B={B}: worst {ulps:.2f} ulp, {share:.2f} of the bound")
