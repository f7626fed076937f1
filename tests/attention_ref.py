"""float64 reference of softmax(q k^T * scale) v and the per-element error allowance of the fused attention kernels
(csrc/k2_attention.cu: flash_attention_kernel at head widths 104 and 512, attention_d64_kernel at 64).

Both kernels follow one recipe: fp32 scores from fp16 q / k, scale * log2(e) folded into ex2.approx, a running maximum m with
the rescale factor alpha = ex2(m_old - m_new) applied to the row sum l and to O, l summed from the unrounded fp32 weights, the
weights rounded to fp16 before P V, O / l rounded once to fp16.  The allowance below is first order in the fp32 unit roundoff
u = 2^-24.  A relative error eta_s of the unnormalised weight of key s moves the output by sum_s p_s eta_s (v_s - o), at most
sum_s p_s eta_s (|v_s| + |o|), where eta_s is bounded by
  D u scale sum_c |q_c k_c|     the D-term fp32 chain of the score (D = 64, 104 or 512; zero-filled padding columns add
                                exact zeros),
  2^-22 (|s| + |max|)           rounding of the scaled score and of its difference with the maximum, in natural units
                                (log2(e) u (|s| + |max|) per rounding, times ln 2 in the exponential; the error of the
                                maximum itself cancels between P and l).  The d64 kernel evaluates ex2(fmaf(s, c, -m)), one
                                rounding fewer than the flash template's ex2(s c - m): the same term bounds it,
  2^-21                         ex2.approx of the weight, and of alpha once the maximum has moved past the key's block.
Terms that do not depend on the key, relative to sum_s p_s |v_s|:
  2^-11                         P rounded to fp16 before P V (half an fp16 ulp),
  (Tkv + 16) u                  the fp32 P V chain and the chain of l: per block of BKV keys O takes one rescale and the
                                MMA's accumulation, l one rescale and BKV / 4 additions per thread, then 2 shuffles, 1 / l and
                                the product -- fewer than Tkv + 16 roundings in total for BKV = 16 and 128.
An absolute term: a weight in fp16's subnormal range is rounded to 2^-25 absolute, Tkv 2^-25 max|v| over all keys.
The caller adds one fp16 ulp of the float64 result (`_ulp16`) for the final rounding.

ref_attention_small / check_attention_small do the same for attention_small (csrc/k2_prior.cu), the masked and causal
attention of the prior and the text towers, with that kernel's own allowance derived where it is computed."""
import torch

U = 2.0 ** -24
INF = float("inf")
CHUNK_ELEMS = 2 ** 24    # float64 elements of one [heads, query chunk, keys] intermediate: 128 MB, five alive at once


def _ulp16(r):
    """fp16 ulp at float64 values r: 2^(e - 10) for |r| in [2^e, 2^(e+1)), 2^-24 below 2^-14."""
    a = r.abs()
    e = torch.floor(torch.log2(torch.where(a > 0, a, torch.full_like(a, 2.0 ** -30)))).clamp(min=-14)
    return torch.exp2(e - 10)


def ref_attention(q, k, v, scale, chain=None):
    """One image: q [T, H, D], k / v [Tkv, H, D] (fp16 or wider, on any device) -> (float64 out [T, H, D], float64
    allowance [T, H, D]).  chain = length of the score's fp32 chain (default D).  Evaluated in query chunks so that no
    float64 intermediate exceeds CHUNK_ELEMS elements."""
    q, k, v = q.double(), k.double(), v.double()
    T, H, D = q.shape
    Tkv = k.shape[0]
    chain = D if chain is None else chain
    ka, va = k.abs(), v.abs()
    vmax = va.amax(0)                                            # [H, D]
    rows = max(1, CHUNK_ELEMS // (H * Tkv))
    outs, allows = [], []
    for t0 in range(0, T, rows):
        qc = q[t0:t0 + rows]
        s = torch.einsum("thc,shc->hts", qc, k) * scale
        p = torch.softmax(s, -1)
        o = torch.einsum("hts,shc->thc", p, v)
        mx = s.amax(-1, keepdim=True).abs()
        eta = chain * U * scale * torch.einsum("thc,shc->hts", qc.abs(), ka)
        eta += 2.0 ** -22 * (s.abs() + mx) + 2.0 ** -21
        del s
        pe = p * eta
        del eta
        mag = torch.einsum("hts,shc->thc", p, va)
        del p
        allow = (torch.einsum("hts,shc->thc", pe, va) + pe.sum(-1).transpose(0, 1)[..., None] * o.abs()
                 + (2.0 ** -11 + (Tkv + 16) * U) * mag + Tkv * 2.0 ** -25 * vmax)
        del pe
        outs.append(o)
        allows.append(allow)
    return torch.cat(outs), torch.cat(allows)


def check(got, ref, allow, what):
    """got (any float dtype) against (ref, allow) of ref_attention: |got - ref| <= one fp16 ulp of ref + allow everywhere
    (NaN fails).  Returns (worst error in fp16 ulps, largest share of the bound)."""
    got = got.double()
    err = (got - ref).abs()
    ulp = _ulp16(ref)
    bound = ulp + allow
    bad = ~(err <= bound)
    assert not bad.any(), (what, int(bad.sum()), got[bad][:4].tolist(), ref[bad][:4].tolist(), bound[bad][:4].tolist())
    return (err / ulp).max().item(), (err / bound).max().item()


def check_d64(out, qkv, enc, heads, what, scale=0.125):
    """out [B, T, heads * 64] of k2_attention_d64 against float64, one image at a time: the encoder keys come first
    (unet.py:300-302).  Returns (worst ulps, worst share)."""
    ulps = share = 0.0
    B, T = qkv.shape[:2]
    for b in range(B):
        q, k, v = qkv[b].view(T, heads, 3, 64).unbind(2)
        if enc is not None and enc.shape[1]:
            ek, ev = enc[b].view(enc.shape[1], heads, 2, 64).unbind(2)
            k, v = torch.cat([ek, k]), torch.cat([ev, v])
        u, s = check(out[b].view(T, heads, 64), *ref_attention(q, k, v, scale), (what, b))
        ulps, share = max(ulps, u), max(share, s)
    return ulps, share


# ------------------------------------------------------------------------------------------------------------------------------
# attention_small (csrc/k2_prior.cu): heads of 64, at most 128 tokens, keep mask and causal mask
# ------------------------------------------------------------------------------------------------------------------------------
def ref_attention_small(qkv, heads, keep, causal, scale):
    """float64 QKVMultiheadAttention with the prior's additive mask (prior.py:92-103, 261-262): where(keep, 0, -inf) plus
    triu(-inf, 1), added to q.k * scale.  Returns (out [B, T, heads*64], per-element error allowance from the kernel's fp32
    arithmetic, see below)."""
    B, T = qkv.shape[:2]
    q, k, v = qkv.double().view(B, T, heads, 192).split(64, -1)
    add = torch.zeros(B, 1, T, T, dtype=torch.float64, device=qkv.device)
    if keep is not None:
        add = add + torch.where(keep.bool(), 0.0, -INF).double()[:, None, None, :]
    if causal:
        add = add + torch.full((T, T), -INF, dtype=torch.float64, device=qkv.device).triu(1)
    s = torch.einsum("bthc,bshc->bhts", q, k) * scale
    p = torch.softmax(s + add, -1)
    o = torch.einsum("bhts,bshc->bthc", p, v)
    # First-order error of the kernel's fp32 evaluation.  A relative error eta_s of the unnormalised weight of key s moves
    # the output by sum_s p_s eta_s (v_s - o), at most sum_s p_s eta_s (|v_s| + |o|), where eta_s is bounded by
    #   2^-18 * scale * sum_c |q_c k_c|   the 64-term fp32 fma chain of the score (gamma_64 = 64 * 2^-24),
    #   2^-22 * (|s| + |max|)             rounding of the scaled score, of s - max and of its product with log2(e),
    #   2^-21                             ex2.approx behind __expf.
    # The P.V chain over <= 128 keys, the sum of the weights and the final multiply by 1 / sum add 2^-16 of sum_s p_s |v_s|.
    reach = torch.isfinite(add).expand(B, heads, T, T)
    mx = torch.where(reach, s, -INF).amax(-1, keepdim=True)
    mx = torch.where(torch.isfinite(mx), mx.abs(), 0.0)
    eta = 2.0 ** -18 * scale * torch.einsum("bthc,bshc->bhts", q.abs(), k.abs()) + 2.0 ** -22 * (s.abs() + mx) + 2.0 ** -21
    pe = torch.where(reach, p * eta, 0.0)
    mag = torch.einsum("bhts,bshc->bthc", p, v.abs())
    allow = torch.einsum("bhts,bshc->bthc", pe, v.abs()) + pe.sum(-1).transpose(1, 2)[..., None] * o.abs() + 2.0 ** -16 * mag
    return o.reshape(B, T, heads * 64), allow.reshape(B, T, heads * 64)


def check_attention_small(got, qkv, heads, keep, causal, scale, what):
    ref, allow = ref_attention_small(qkv, heads, keep, causal, scale)
    got = got.double()
    dead = torch.isnan(ref)      # query rows that reach no key: NaN in torch, NaN in the kernel (the documented contract)
    assert torch.equal(torch.isnan(got), dead), (what, "NaN rows differ", int(torch.isnan(got).sum()), int(dead.sum()))
    r, g, a = ref[~dead], got[~dead], allow[~dead]
    err = (g - r).abs()
    bound = _ulp16(r) + a
    bad = err > bound
    assert not bad.any(), (what, int(bad.sum()), err[bad][:4].tolist(), r[bad][:4].tolist(), a[bad][:4].tolist())
    if not r.numel():
        return 0.0, 0.0
    # worst error in ulps (large only where the output cancels to near zero), and the largest share of the bound used
    return (err / _ulp16(r)).max().item(), (err / bound).max().item()
