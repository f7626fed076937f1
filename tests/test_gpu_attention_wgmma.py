"""The head-width-64 attention kernel (k2_attention_d64: TMA-fed warp-specialised wgmma) against float64 within the fused
attention kernels' per-element bound (tests/attention_ref.py), at the UNet step's full shapes, at encoder / spatial lengths that leave ragged key and query blocks, with NaN in memory the kernel must
not read, and for run-to-run and graph-replay bit identity."""
import pytest
import torch

from tests.attention_ref import check_d64

pytestmark = pytest.mark.gpu


def _inputs(B, heads, T, Tc, seed, guard_rows=0):
    """Random fp16 qkv / enc; with guard_rows, each lives at the start of an allocation whose following rows are NaN."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, T, heads * 192, device="cuda", generator=g).half()
    enc = torch.randn(B, Tc, heads * 128, device="cuda", generator=g).half() if Tc else None
    if guard_rows:
        qb = torch.full((B * T + guard_rows, heads * 192), float("nan"), device="cuda", dtype=torch.float16)
        qb[:B * T] = qkv.reshape(B * T, -1)
        qkv = qb[:B * T].view(B, T, -1)
        if enc is not None:
            eb = torch.full((B * Tc + guard_rows, heads * 128), float("nan"), device="cuda", dtype=torch.float16)
            eb[:B * Tc] = enc.reshape(B * Tc, -1)
            enc = eb[:B * Tc].view(B, Tc, -1)
    return qkv, enc


def _check(out, qkv, enc, heads, what):
    ulps, share = check_d64(out, qkv, enc, heads, what)
    print(f"attention_d64 {what}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


def test_single_block():
    """One query tile against one key block: S = Q K^T from shared memory, P V with V read MN-major."""
    from kandinsky2 import ops
    qkv, _ = _inputs(1, 1, 128, 0, seed=1)
    out = ops.attention_d64(qkv, 1, None)
    torch.cuda.synchronize()
    _check(out, qkv, None, 1, "single block")


@pytest.mark.parametrize("B,heads,T", [
    (8, 12, 2304),   # cfg-2 level 1 (48 x 48)
    (8, 18, 576),    # cfg-2 level 2 (24 x 24)
    (8, 24, 144),    # cfg-2 level 3 and middle block (12 x 12)
    (4, 12, 4096),   # cfg-3 level 1 (64 x 64)
])
def test_step_shapes(B, heads, T):
    from kandinsky2 import ops
    qkv, enc = _inputs(B, heads, T, 32, seed=T)
    out = ops.attention_d64(qkv, heads, enc)
    torch.cuda.synchronize()
    _check(out, qkv, enc, heads, f"B={B} heads={heads} T={T}")


@pytest.mark.parametrize("Tc", [0, 1, 63, 64, 65, 200])
@pytest.mark.parametrize("T", [1, 100, 129, 300])
def test_ragged_blocks_nan_guards(T, Tc):
    """Encoder and spatial lengths that are not multiples of the 128-key block or the 128-row query tile; the rows after the
    last image's T qkv rows and Tc encoder rows are NaN, so a key box that reached them would poison the output."""
    from kandinsky2 import ops
    B, heads = 2, 3
    qkv, enc = _inputs(B, heads, T, Tc, seed=7 * T + Tc, guard_rows=256)
    out = ops.attention_d64(qkv, heads, enc)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    _check(out, qkv, enc, heads, f"T={T} Tc={Tc}")


@pytest.mark.parametrize("T,Tc", [(100, 65), (300, 32)])
def test_next_image_not_read(T, Tc):
    """Image 1 is all NaN: image 0's query, key and value boxes must stop at its own last row."""
    from kandinsky2 import ops
    heads = 2
    qkv, enc = _inputs(2, heads, T, Tc, seed=5)
    qkv[1] = float("nan")
    enc[1] = float("nan")
    out = ops.attention_d64(qkv, heads, enc)
    torch.cuda.synchronize()
    assert torch.isfinite(out[0]).all()
    _check(out[:1], qkv[:1], enc[:1], heads, f"next image NaN T={T} Tc={Tc}")


def test_bit_identical_repeats_and_graph_replay():
    from kandinsky2 import ops
    B, heads, T, Tc = 2, 4, 600, 32
    qkv, enc = _inputs(B, heads, T, Tc, seed=9)
    eager = [ops.attention_d64(qkv, heads, enc) for _ in range(3)]
    out = torch.empty_like(eager[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.attention_d64(qkv, heads, enc, out=out)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.attention_d64(qkv, heads, enc, out=out)
    replays = []
    for _ in range(3):
        out.zero_()
        graph.replay()
        replays.append(out.clone())
    torch.cuda.synchronize()
    for y in eager[1:] + replays:
        assert torch.equal(y, eager[0])
