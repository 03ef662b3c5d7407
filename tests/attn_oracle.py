"""float64 attention, an elementwise error bound for the 16-bit attention kernels, input builders for their tile, mask
and score edges, and a CPU emulation of the wgmma prefill kernel's arithmetic (TEST INFRASTRUCTURE ONLY).

The kernels (csrc/attn_fwd_sm100.cu, csrc/attn_generic_sm100.cu) compute softmax(q k^T * scale + mask) v with query i
of batch entry b seeing key j when ``key_mask[b, j]`` (or no mask) and, if causal, ``j <= past + i``.  A row that sees
no key gives output 0 and log-sum-exp +inf (DESIGN.md, "Attention masks").

Poison contracts:
* the generic kernel, both split-KV decode kernels and the shared-prefix decode never read a masked key or value
  (masked scores are never computed, and a zero weight skips its value row), so masked slots may hold NaN / +-Inf;
* the wgmma prefill kernel loads whole 64-key tiles and multiplies the masked slots' P = 0 into P V on the tensor
  cores, where 0 * NaN = NaN.  Its contract is that every slot below Tkv holds a finite number (``StaticKV.zero_from_``
  zeroes the unused tail of the cache), so its masked slots get the dtype's largest finite value instead.  Positions at
  or beyond Tkv are outside its tensor maps (TMA fills them with zeros) and may hold NaN.
"""
from __future__ import annotations

import math

import torch

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
U = {BF16: 2.0 ** -8, F16: 2.0 ** -11, F32: 2.0 ** -24}   # unit roundoff of one round-to-nearest
U32 = 2.0 ** -24
EX2 = 2.0 ** -22      # ex2.approx.ftz.f32 (fast_exp2, and __expf after its argument is multiplied by log2 e): 2 ulp
TILE = 64             # wgmma kernel: keys per tile (kBN)
CHUNK = 256           # generic kernel: keys per chunk (kAttnChunk); decode kernels: keys per split (kDecKeys)


# ---- visibility and the float64 reference ------------------------------------------------------------------------------
def visibility(B, Tq, Tkv, key_mask=None, causal=True, past=0, device="cpu"):
    """(B, Tq, Tkv) bool: query i of entry b sees key j."""
    vis = torch.ones((B, Tq, Tkv), dtype=torch.bool, device=device)
    if key_mask is not None:
        vis = vis & key_mask.to(device).bool()[:, None, :]
    if causal:
        j = torch.arange(Tkv, device=device)
        i = torch.arange(Tq, device=device)
        vis = vis & (j[None, :] <= past + i[:, None])[None]
    return vis


def reference(q, k, v, key_mask=None, causal=True, past=0, scale=None, vis=None):
    """float64 attention on the given (already 16-bit-rounded) inputs, one head at a time on their device.

    Returns a dict of float64 tensors: ``out`` (B, Tq, H, hd); ``mag`` = sum_j p_ij |v_jc| (B, Tq, H, hd); ``lse``
    (B, H, Tq), +inf where a row sees no key; ``smax`` = scale * max_j sum_d |q_id k_jd| over the visible keys
    (B, H, Tq), 0 where none; ``seen`` (B, Tq) bool; ``vmax`` = max |v_jc| over the keys any row of the entry sees
    (B, 1, H, hd).  Masked slots of k / v are never read (they may hold NaN)."""
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    scale = hd ** -0.5 if scale is None else scale
    if vis is None:
        vis = visibility(B, Tq, Tkv, key_mask, causal, past, q.device)
    vis = vis.to(q.device)
    seen = vis.any(-1)
    readable = vis.any(1)                                                   # (B, Tkv): keys some row sees
    out = torch.zeros((B, Tq, H, hd), dtype=torch.float64, device=q.device)
    mag = torch.zeros_like(out)
    lse = torch.full((B, H, Tq), math.inf, dtype=torch.float64, device=q.device)
    smax = torch.zeros((B, H, Tq), dtype=torch.float64, device=q.device)
    for h in range(H):
        qd = q[:, :, h].double()
        kd = torch.where(readable[..., None], k[:, :, h].double(), 0.0)
        vd = torch.where(readable[..., None], v[:, :, h].double(), 0.0)
        s = torch.where(vis, qd @ kd.transpose(1, 2) * scale, -math.inf)
        a = torch.where(vis, qd.abs() @ kd.abs().transpose(1, 2) * scale, 0.0)
        ls = torch.logsumexp(s, -1)
        p = torch.where(seen[..., None], torch.exp(s - torch.where(seen, ls, 0.0)[..., None]), 0.0)
        out[:, :, h] = p @ vd
        mag[:, :, h] = p @ vd.abs()
        lse[:, h] = torch.where(seen, ls, math.inf)
        smax[:, h] = a.amax(-1)
    vmax = torch.where(readable[..., None, None], v.double().abs(), 0.0).amax(1, keepdim=True)   # (B, 1, H, hd)
    return {"out": out, "mag": mag, "lse": lse, "smax": smax, "seen": seen, "vmax": vmax}


# ---- the elementwise bound ---------------------------------------------------------------------------------------------
# For output (i, c) with exact weights p_ij and m_ic = sum_j p_ij |v_jc|:
#
#   |out - ref| <= 1.01 * (u_P + 2 delta_i + 2 n_exp EX2 + n_i 2^-24) * m_ic + u_out |ref_ic| + sub_P + tiny
#
# * u_P: P is rounded to nearest in the 16-bit type before P V (wgmma kernel only, pack2<T>; its row sum l is summed
#   from the fp32 values, so only the numerator carries it): a relative error <= u of each weight, i.e. <= u * m_ic.
#   The generic and decode kernels keep P in fp32 (u_P = 0).
# * sub_P: below fp16's smallest normal (2^-14) the rounding of P is absolute, <= 2^-25; P is relative to the running
#   max (<= 1) and the final row sum is >= 1, so the K keys a row scans add <= K 2^-25 max_j |v_jc| (fp16 P only;
#   the max is taken over the entry's keys).
# * delta_i: every exponent argument (scaled score minus running max, natural-log units) is off by at most delta_i, so
#   each normalised weight p_ij = e^x_j / sum_k e^x_k is off by a factor within e^(+-2 delta_i).  With
#   S_i = scale * max_j sum_d |q_id k_jd| (so |scaled score| <= S_i and every max difference <= 2 S_i):
#     - the fp32 dot product over hd terms: <= hd u S_i for the serial fp32 fma chains of the generic and split
#       kernels (the hd-128 split kernel's chains are shorter); the tensor cores' fp32 accumulation (wgmma) is allowed
#       truncation, 2u per add: 2 hd u S_i;
#     - the scale: fl(q * scale) (generic, split) or fl(dot * scale) (split-128), or fl(scale * log2 e) (wgmma): u S_i;
#     - the argument: fl(-m * scale log2e) and the fmaf (wgmma), or s - m and __expf's x * log2 e (generic, split),
#       each <= u |x| with |x| <= 2 S_i: 4 u S_i;
#     - the rescales alpha / corr = exp(m_old - m_new): the rises sum to <= 2 S_i, and their subtraction and scaling
#       round to <= 4 u S_i in all;
#   delta_i = (n_dot + 9) u S_i with n_dot = hd or 2 hd, kept at (n_dot + 12) u S_i.  It matters only when scores
#   are large, or at fp32 output.
# * n_exp: ex2.approx.ftz.f32 has a relative error <= 2 ulp = EX2 (CUDA C Programming Guide, exp2f / __expf; the
#   |x|-dependent part of __expf's error is its argument rounding, counted in delta_i).  A weight is the product of
#   its own exponential and of every rescale factor applied to it after (n_exp factors), and appears in the numerator
#   and in the row sum: 2 n_exp EX2.
# * n_i: the longest chain of fp32 roundings in the numerator P V plus the row sum l plus the final 1 / l, x (or /),
#   each <= 2^-24 relative for sums of non-negative terms (gamma_n bound); per kernel below.
# * u_out: the output's rounding to its type (relative u; fp32: 2^-24).  tiny: fp16's subnormal output step.
# * 1.01 covers the second-order products of the terms above.
def arith_wgmma(Tkv, dtype, hd):
    """wgmma prefill (attn_fwd_sm100.cu).  Per 64-key tile of the <= ceil(Tkv / 64) a row scans: O += P V over 64 keys
    plus O *= alpha, 2u each for tensor-core accumulation (2 (64 + 1)); the row sum: 16 per-thread adds, 2 quad
    shuffles, l alpha + ls (<= 18).  Then 1 / l and the multiply (2) and one spare.  n_exp: own ex2 + one alpha per
    later tile."""
    nt = -(-Tkv // TILE)
    return dict(u_p=U[dtype], n_sum=148 * nt + 4, n_exp=nt, n_dot=2 * hd, out=dtype, p16=dtype, keys=nt * TILE)


def arith_generic(Tkv, dtype, hd):
    """warp-per-row generic kernel.  P V: one fma per key plus acc *= corr per 256-key chunk; the row sum: 8 per-lane
    adds, 5 shuffles, l corr + csum (15 per chunk); 1 / l and the multiply (2).  n_exp: own __expf + one corr per later
    chunk."""
    nc = -(-Tkv // CHUNK)
    return dict(u_p=0.0, n_sum=Tkv + 16 * nc + 2, n_exp=nc, n_dot=hd, out=dtype, p16=None, keys=Tkv)


def arith_split128(Tkv, dtype, hd=128):
    """hd-128 16-bit split-KV decode.  A warp's 64 keys: 32 fmas per lane and one shuffle add (P V), 2 + 5 for its sum;
    the CTA combine: 4 fmas each; the merge: one fma per 256-key split each; num / den (1).  n_exp: own __expf, the
    warp combine's and the merge's."""
    ns = -(-Tkv // CHUNK)
    return dict(u_p=0.0, n_sum=50 + 2 * ns, n_exp=3, n_dot=hd, out=dtype, p16=None, keys=Tkv)


def arith_split(Tkv, dtype, hd):
    """generic split-KV decode + merge kernel.  A warp's 64 keys in two passes of 32: 64 fmas + 2 corr multiplies (P V)
    and 2 x (5 shuffles + 2) for its sum; the CTA combine: 4 each; the merge: one fma per split each; num / den (1).
    n_exp: own __expf, the corr between the two passes, the CTA combine's and the merge's."""
    ns = -(-Tkv // CHUNK)
    return dict(u_p=0.0, n_sum=90 + 2 * ns, n_exp=4, n_dot=hd, out=dtype, p16=None, keys=Tkv)


def bound(ref, arith):
    """The elementwise bound above, (B, Tq, H, hd) float64."""
    delta = (arith["n_dot"] + 12) * U32 * ref["smax"].transpose(1, 2)[..., None]            # (B, Tq, H, 1)
    rel = arith["u_p"] + 2 * delta + 2 * arith["n_exp"] * EX2 + arith["n_sum"] * U32
    b = 1.01 * rel * ref["mag"] + U[arith["out"]] * ref["out"].abs()
    if arith["p16"] is F16:
        b = b + arith["keys"] * 2.0 ** -25 * ref["vmax"]
    tiny = U[F16] * torch.finfo(F16).smallest_normal if arith["out"] is F16 else 1e-300
    return b + tiny


def check(out, ref, arith, what=""):
    """Assert the kernel output (B, Tq, H*hd) or (B, Tq, H, hd) is within the bound, finite, and exactly 0 on rows that
    see no key."""
    o = out.reshape(ref["out"].shape).double()
    assert bool(torch.isfinite(o).all()), f"{what}: non-finite output"
    dead = ~ref["seen"]
    assert not bool(o[dead].any()), f"{what}: a row that sees no key must give exact zeros"
    err = (o - ref["out"]).abs()
    b = bound(ref, arith)
    bad = err > b
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound, "
                                 f"worst err / bound {float((err / b).max()):.3g}")


# ---- log-sum-exp bound -------------------------------------------------------------------------------------------------
# lse = (m scale log2e + lg2.approx(l)) ln 2 (attn_fwd_kernel, LSE).  Each score shifts by <= delta_i; l carries the
# relative error of its sum (n_sum 2^-24) and of its exponentials (n_exp EX2), i.e. an absolute error of lse; lg2.approx
# errs by <= 2^-22 absolute on [0.5, 2] and 2 ulp of log2 l elsewhere; the fmaf, the rounding of ln 2 and the final
# multiply add <= 3 u |lse / ln 2| ~ 4.4 u |lse|, kept at 6 u (|lse| + 1).
def lse_bound(ref, arith):
    d = (arith["n_dot"] + 12) * U32 * ref["smax"]
    return (d + arith["n_sum"] * U32 + arith["n_exp"] * EX2 + EX2 * (1 + math.log2(max(arith["keys"], 2)))
            + 6 * U32 * (ref["lse"].abs() + 1))


def check_lse(lse, ref, arith, what=""):
    l = lse.double()
    fin = torch.isfinite(ref["lse"])
    assert bool((l[~fin] == math.inf).all()), f"{what}: lse of a row that sees no key must be +inf"
    assert bool(torch.isfinite(l[fin]).all()), f"{what}: non-finite lse on a row that sees keys"
    err = (l - ref["lse"])[fin].abs()
    b = lse_bound(ref, arith)[fin]
    assert bool((err <= b).all()), f"{what}: lse outside the bound, worst err / bound {float((err / b).max()):.3g}"


# ---- inputs --------------------------------------------------------------------------------------------------------------
PATTERNS = ("gauss", "sink", "rising", "falling", "uniform", "large")
PADS = (0, 5, 63, 64, 65, 128, 200, 300)


def key_mask(B, Tkv, pad=0, hole=False, dead_row=False, device="cpu"):
    """(B, Tkv) uint8: left padding of ``pad`` keys on the last entry, a 40-key hole in the middle of entry 0, and all
    keys of entry 1 masked (a row that sees nothing).  None when nothing is masked."""
    if not (pad or hole or dead_row):
        return None
    km = torch.ones((B, Tkv), dtype=torch.uint8, device=device)
    km[-1, :min(pad, Tkv)] = 0
    if hole:
        km[0, Tkv // 2 - 20:Tkv // 2 + 20] = 0
    if dead_row:
        km[min(1, B - 1)] = 0
    return km


def make_qkv(B, Tq, Tkv, H, hd, pattern="gauss", dtype=BF16, key_mask=None, seed=0, device="cpu", scale=None):
    """q (B, Tq, H, hd), k / v (B, Tkv, H, hd) of ``dtype`` with scaled scores following ``pattern``:

    gauss    q, k ~ N(0, 1): scaled scores ~ N(0, 1);
    sink     the first key the mask leaves visible in each entry scores 35 +- a few above the rest, for every query;
    rising   the keys of 64-key tile t score 10 t (+- 0.3): each tile raises the running max by >= 8;
    falling  the reverse: tile t scores 10 (n_tiles - 1 - t);
    uniform  every key identical: the output is the mean of the visible value rows;
    large    q, k ~ N(0, 50): |scaled score| up to ~150, nearly one-hot.
    Channel 0 of q is 1 and channel 0 of k carries the pattern's offset for sink / rising / falling."""
    scale = hd ** -0.5 if scale is None else scale
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((B, Tq, H, hd), generator=g)
    k = torch.randn((B, Tkv, H, hd), generator=g)
    v = torch.randn((B, Tkv, H, hd), generator=g)
    if pattern == "large":
        q, k = q * 50 ** 0.5, k * 50 ** 0.5
    elif pattern == "uniform":
        k = k[:, :1].expand(B, Tkv, H, hd).clone()
    elif pattern in ("sink", "rising", "falling"):
        k = k * 0.3
        q[..., 0] = 1.0
        k[..., 0] = 0.0
        if pattern == "sink":
            first = torch.zeros(B, dtype=torch.long)
            if key_mask is not None:
                first = torch.argmax(key_mask.cpu().to(torch.uint8), dim=1)  # first visible key (0 for a dead row)
            for b in range(B):
                k[b, int(first[b]), :, 0] = 35.0 / scale
        else:
            t = torch.arange(Tkv) // TILE
            lvl = t if pattern == "rising" else (t.max() - t)
            k[..., 0] = (10.0 * lvl.float() / scale)[None, :, None]
    elif pattern != "gauss":
        raise ValueError(pattern)
    return tuple(x.to(dtype).to(device) for x in (q, k, v))


def hidden_slots(vis):
    """(B, Tkv) bool: keys no query row of the entry sees."""
    return ~vis.any(1)


def poison(k, v, hidden, finite=False):
    """Copies of k / v with every hidden slot poisoned: NaN in k and +-Inf in v, or (``finite``: the wgmma kernel's
    contract) the dtype's largest finite value."""
    k, v = k.clone(), v.clone()
    hid = hidden.to(k.device)
    if finite:
        big = torch.finfo(k.dtype).max
        k[hid] = big
        v[hid] = -big
    else:
        k[hid] = float("nan")
        vv = v[hid]
        vv[..., 0::2] = float("inf")
        vv[..., 1::2] = float("-inf")
        v[hid] = vv
    return k, v


def in_cache(x, extra=37):
    """``x`` (B, T, H, hd) as the view [:, :T] of a (B, T + extra, H, hd) cache that holds NaN past T (the chunked
    prefill's and the decoder's K / V are such views)."""
    B, T, H, hd = x.shape
    c = torch.full((B, T + extra, H, hd), float("nan"), dtype=x.dtype, device=x.device)
    c[:, :T] = x
    return c[:, :T]


# ---- CPU emulation of the wgmma prefill kernel ---------------------------------------------------------------------------
MUTANTS = ("causal_plus1", "causal_minus1", "drop_tile", "drop_last_partial", "no_rescale", "masked_in_sum",
           "mask_wrong_row", "dead_row_mean", "scale_twice")


def emulate_wgmma(q, k, v, key_mask=None, causal=True, past=0, scale=None, mutant=None, drop=1):
    """attn_fwd_kernel's arithmetic on the CPU: 64-key tiles in order, fp32 scores, fp32 running max / sum, alpha
    rescale, P = exp2(s scale log2e - m scale log2e) rounded to the 16-bit type before P V, O / l at the end and zeros
    for a row that sees no key.  ``mutant`` injects one of MUTANTS (``drop``: the tile ``drop_tile`` skips).  Returns
    (B, Tq, H, hd) of q's dtype."""
    B, Tq, H, hd = q.shape
    Tkv = k.shape[1]
    scale = hd ** -0.5 if scale is None else scale
    dt = q.dtype
    qf, kf, vf = (x.float().permute(0, 2, 1, 3) for x in (q, k, v))         # (B, H, T, hd)
    km = key_mask
    if mutant == "mask_wrong_row" and km is not None:
        km = km.roll(1, 0)
    shift = {"causal_plus1": 1, "causal_minus1": -1}.get(mutant, 0)
    vis = visibility(B, Tq, Tkv, km, causal, past + shift)[:, None]          # (B, 1, Tq, Tkv)
    c = torch.tensor(scale * math.log2(math.e), dtype=torch.float32)
    if mutant == "scale_twice":
        c = c * scale
    m = torch.full((B, H, Tq), -math.inf)
    l = torch.zeros((B, H, Tq))
    o = torch.zeros((B, H, Tq, hd))
    nt = -(-Tkv // TILE)
    for t in range(nt):
        if mutant == "drop_tile" and t == drop:
            continue
        if mutant == "drop_last_partial" and t == nt - 1 and Tkv % TILE:
            continue
        ks = slice(t * TILE, min((t + 1) * TILE, Tkv))
        raw = qf @ kf[:, :, ks].transpose(-1, -2)
        s = torch.where(vis[..., ks], raw, -math.inf)
        m_new = torch.maximum(m, s.amax(-1))
        alpha = torch.where(m_new == -math.inf, 1.0, torch.exp2((m - m_new) * c))
        if mutant == "no_rescale":
            alpha = torch.ones_like(alpha)
        neg_m = torch.where(m_new == -math.inf, 0.0, -m_new * c)
        e = torch.exp2(s * c + neg_m[..., None])
        if mutant == "masked_in_sum":                                       # key-masked slots also summed
            kvis = visibility(B, Tq, Tkv, None, causal, past)[:, None, :, ks]
            es = torch.exp2(torch.where(kvis, raw, -math.inf) * c + neg_m[..., None])
            es = torch.where(m_new[..., None] == -math.inf, 0.0, es)
            l = l * alpha + es.sum(-1)
        else:
            l = l * alpha + e.sum(-1)
        o = o * alpha[..., None] + e.to(dt).float() @ vf[:, :, ks]
        m = m_new
    out = torch.where(l[..., None] > 0, o / l[..., None], 0.0)
    if mutant == "dead_row_mean":                                          # the reference's finfo.min clamp
        out = torch.where(l[..., None] > 0, out, vf.mean(2, keepdim=True))
    return out.permute(0, 2, 1, 3).to(dt)
