"""CPU checks of tests/attn_oracle.py, the float64 reference and elementwise bound the attention edge tests hold the
16-bit kernels to: a tile-wise emulation of the wgmma kernel's arithmetic passes the bound at every score pattern and
mask edge, and each of a set of plausible kernel bugs, injected into the emulation, fails it."""
import math

import pytest
import torch

from tests import attn_oracle as ao

BF16, F16 = torch.bfloat16, torch.float16


def _run(B, H, Tq, Tkv, hd, pattern, dtype, km, causal, past, mutant=None, seed=0):
    q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, pattern, dtype, key_mask=km, seed=seed)
    ref = ao.reference(q, k, v, km, causal, past)
    out = ao.emulate_wgmma(q, k, v, km, causal, past, mutant=mutant)
    return out, ref


def test_reference_matches_a_plain_float64_statement():
    B, Tq, Tkv, H, hd = 2, 7, 19, 3, 16
    q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, "gauss", torch.float64, seed=3)
    km = ao.key_mask(B, Tkv, pad=15)                                      # rows 0..2 of entry 1 see no key
    ref = ao.reference(q, k, v, km, causal=True, past=12)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(hd)
    allow = km.bool()[:, None, None, :] & (torch.arange(Tkv)[None, :] <= 12 + torch.arange(Tq)[:, None])
    s = s.masked_fill(~allow, -math.inf)
    p = torch.softmax(s, -1).nan_to_num(0.0)
    want = torch.einsum("bhqk,bkhd->bqhd", p, v)
    torch.testing.assert_close(ref["out"], want, rtol=1e-12, atol=1e-12)
    seen = allow.any(-1).expand(B, H, Tq)
    assert int((~seen).sum()) == 3 * H
    assert torch.equal(torch.isinf(ref["lse"]), ~seen) and torch.equal(ref["seen"], seen[:, 0])
    torch.testing.assert_close(ref["lse"][seen], torch.logsumexp(s, -1)[seen])
    assert not bool(ref["out"][1, :3].any())                               # a row that sees nothing: output 0
    q0 = q[:, :1]
    r0 = ao.reference(q0, k, v, torch.zeros((B, Tkv), dtype=torch.uint8), causal=False)
    assert not bool(r0["out"].any()) and bool((r0["lse"] == math.inf).all())


def test_reference_ignores_poisoned_hidden_slots():
    B, Tq, Tkv, H, hd = 2, 5, 40, 2, 32
    q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, "gauss", BF16, seed=1)
    km = ao.key_mask(B, Tkv, pad=7, hole=True)
    vis = ao.visibility(B, Tq, Tkv, km, True, 20)
    kp, vp = ao.poison(k, v, ao.hidden_slots(vis))
    assert bool(kp.isnan().any()) and bool(vp.isinf().any())
    a = ao.reference(q, k, v, km, True, 20)
    b = ao.reference(q, kp, vp, km, True, 20)
    assert all(torch.equal(a[x], b[x]) for x in ("out", "mag", "lse", "smax"))


def test_patterns_have_the_scores_they_promise():
    B, Tq, Tkv, H, hd = 2, 8, 300, 1, 128
    km = ao.key_mask(B, Tkv, pad=65)
    for pattern in ao.PATTERNS:
        q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, pattern, BF16, key_mask=km, seed=2)
        s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double()) / math.sqrt(hd)
        s = s.masked_fill(~km.bool()[:, None, None, :], -math.inf)[:, 0]      # (B, Tq, Tkv)
        if pattern == "sink":
            for b, first in ((0, 0), (1, 65)):
                top2 = s[b].topk(2, -1).values
                assert bool((s[b].argmax(-1) == first).all())
                assert bool((top2[:, 0] - top2[:, 1] > 25).all()) and bool((top2[:, 0] - top2[:, 1] < 45).all())
        elif pattern in ("rising", "falling"):
            tmax = torch.stack([s[0, :, t * 64:(t + 1) * 64].amax(-1) for t in range(5)], -1)
            d = tmax.diff(dim=-1)
            assert bool((d >= 8).all()) if pattern == "rising" else bool((d <= -8).all())
        elif pattern == "uniform":
            assert bool((s[0] == s[0, :, :1]).all())
        elif pattern == "large":
            assert 100 < float(s[torch.isfinite(s)].abs().max()) < 250


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("pattern", ao.PATTERNS)
def test_emulator_passes_the_bound_at_every_mask_edge(pattern, dtype):
    B, H, hd, T = 2, 1, 64, 330
    for pad in ao.PADS:
        km = ao.key_mask(B, T, pad=pad)
        out, ref = _run(B, H, T, T, hd, pattern, dtype, km, True, 0, seed=pad)
        ao.check(out, ref, ao.arith_wgmma(T, dtype, hd), f"{pattern} pad {pad}")
    for hole, dead in ((True, False), (False, True), (True, True)):
        km = ao.key_mask(B, T, hole=hole, dead_row=dead)
        out, ref = _run(B, H, 90, T, hd, pattern, dtype, km, False, 0, seed=7)
        ao.check(out, ref, ao.arith_wgmma(T, dtype, hd), f"{pattern} hole {hole} dead row {dead}")
    # a chunk on a cache: Tq = 17 queries at past = 200, with left padding across three tiles
    km = ao.key_mask(B, 217, pad=130)
    out, ref = _run(B, H, 17, 217, hd, pattern, dtype, km, True, 200, seed=9)
    ao.check(out, ref, ao.arith_wgmma(217, dtype, hd), f"{pattern} chunk")


# Each mutant is a plausible bug of a tiled online softmax.  Shapes are chosen so that the mutated key, tile or row
# carries weight well above the bound; every one must be caught.
MUTANT_CASES = {
    # mutant: (B, H, Tq, Tkv, hd, pattern, pad, hole, dead_row, causal, past)
    "causal_plus1": (1, 2, 130, 130, 64, "gauss", 0, False, False, True, 0),
    "causal_minus1": (1, 2, 130, 130, 64, "gauss", 0, False, False, True, 0),
    "drop_tile": (2, 2, 32, 200, 64, "uniform", 0, False, False, False, 0),
    "drop_last_partial": (2, 2, 32, 200, 64, "uniform", 0, False, False, False, 0),
    "no_rescale": (2, 2, 32, 200, 64, "rising", 0, False, False, False, 0),
    "masked_in_sum": (2, 2, 32, 200, 64, "uniform", 65, True, False, False, 0),
    "mask_wrong_row": (2, 2, 32, 200, 64, "gauss", 128, False, False, False, 0),
    "dead_row_mean": (2, 2, 32, 200, 64, "gauss", 0, False, True, False, 0),
    "scale_twice": (2, 2, 32, 200, 64, "gauss", 0, False, False, False, 0),
}


def test_every_mutant_is_listed():
    assert set(MUTANT_CASES) == set(ao.MUTANTS)


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("mutant", ao.MUTANTS)
def test_mutants_fail_the_check(mutant, dtype):
    B, H, Tq, Tkv, hd, pattern, pad, hole, dead, causal, past = MUTANT_CASES[mutant]
    km = ao.key_mask(B, Tkv, pad=pad, hole=hole, dead_row=dead)
    arith = ao.arith_wgmma(Tkv, dtype, hd)
    out, ref = _run(B, H, Tq, Tkv, hd, pattern, dtype, km, causal, past)
    ao.check(out, ref, arith, "unmutated")                                 # the same case passes without the bug
    bad, _ = _run(B, H, Tq, Tkv, hd, pattern, dtype, km, causal, past, mutant=mutant)
    with pytest.raises(AssertionError):
        ao.check(bad, ref, arith, mutant)


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_one_wrong_key_in_a_long_row_is_visible(dtype):
    """The bound is tight enough that dropping one of 1000 equally weighted keys is caught when its value stands out
    (16 against N(0, 1) values: it moves the output by ~1.6e-2, the bound is ~4e-3 in bf16)."""
    B, H, T, hd = 1, 1, 1000, 128
    q, k, v = ao.make_qkv(B, 4, T, H, hd, "uniform", dtype, seed=5)
    v[:, 500] = 16.0
    ref = ao.reference(q, k, v, None, causal=False)
    km = torch.ones((B, T), dtype=torch.uint8)
    km[0, 500] = 0
    out = ao.emulate_wgmma(q, k, v, None, causal=False)
    ao.check(out, ref, ao.arith_wgmma(T, dtype, hd), "exact")
    bad = ao.emulate_wgmma(q, k, v, km, causal=False)
    with pytest.raises(AssertionError):
        ao.check(bad, ref, ao.arith_wgmma(T, dtype, hd), "one key dropped")


def test_lse_bound_holds_for_fp32_logsumexp_and_catches_a_missing_tile():
    B, H, T, hd = 2, 2, 300, 64
    km = ao.key_mask(B, T, pad=64)
    for pattern in ao.PATTERNS:
        q, k, v = ao.make_qkv(B, T, T, H, hd, pattern, BF16, key_mask=km, seed=4)
        ref = ao.reference(q, k, v, km, causal=False)
        s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * hd ** -0.5
        s = s.masked_fill(~km.bool()[:, None, None, :], -math.inf)
        lse = torch.logsumexp(s, -1)
        lse = torch.where(ref["seen"][:, None, :].expand_as(lse), lse, math.inf)
        arith = ao.arith_wgmma(T, BF16, hd)
        ao.check_lse(lse, ref, arith, pattern)
        if pattern == "uniform":
            with pytest.raises(AssertionError):
                ao.check_lse(torch.logsumexp(s[..., 64:], -1), ref, arith, "missing tile")


def test_generic_and_decode_bounds_are_tighter_than_the_wgmma_one():
    """P stays fp32 in the generic and decode kernels: at fp32 output their bound stays below 2e-4 m_ic, most of it
    the worst case of the fp32 dot product (2 delta_i)."""
    B, H, T, hd = 1, 1, 513, 128
    q, k, v = ao.make_qkv(B, 1, T, H, hd, "gauss", torch.float32, seed=6)
    ref = ao.reference(q, k, v, None, causal=False)
    for arith in (ao.arith_generic(T, torch.float32, hd), ao.arith_split128(T, torch.float32),
                  ao.arith_split(T, torch.float32, hd)):
        rel = (ao.bound(ref, arith) / ref["mag"]).max()
        assert float(rel) < 2e-4, arith
