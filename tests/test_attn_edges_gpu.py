"""The 16-bit attention kernels against float64 at their tile, mask and score edges, with the elementwise bound of
tests/attn_oracle.py: the wgmma prefill kernel (one item per CTA and persistent), the warp-per-row generic kernel, the
hd-128 and generic split-KV decode kernels, the shared-prefix decode, and the attention backward at the same masking
and score edges.  Every case also checks finiteness, exact zeros for rows that see no key, and bit-identical reruns;
slots a kernel must not read are poisoned (NaN / +-Inf, or the largest finite value where the wgmma kernel's contract
asks for finite numbers)."""
import math

import pytest
import torch

from tests import attn_oracle as ao

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
DEV = "cuda"


def _ops():
    from mm_interleaved_b200 import ops
    return ops


def _resident(hd):
    """Resident CTAs of the wgmma kernel (1 per SM at hd 128, 2 at hd 64): more items than this run persistent."""
    return (2 if hd == 64 else 1) * torch.cuda.get_device_properties(0).multi_processor_count


def _heads(B, Tq, hd, persistent, few=2):
    """Heads giving B * H * ceil(Tq / 128) work items above the resident CTA count (persistent) or few of them."""
    if not persistent:
        return few
    return _resident(hd) // (B * -(-Tq // 128)) + 1


def _run_twice(fn):
    a = fn()
    b = fn()
    assert torch.equal(a, b), "two runs differ"
    return a


# ---- wgmma prefill ----------------------------------------------------------------------------------------------------
def _wgmma_case(B, H, Tq, Tkv, hd, dtype, pattern, km, causal, past, what, lse=False, seed=0):
    ops = _ops()
    q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, pattern, dtype, key_mask=km, seed=seed, device=DEV)
    vis = ao.visibility(B, Tq, Tkv, km, causal, past, DEV)
    kp, vp = ao.poison(k, v, ao.hidden_slots(vis), finite=True)
    kc, vc = ao.in_cache(kp), ao.in_cache(vp)                              # NaN past Tkv
    qv = torch.cat([q, q], dim=2)[:, :, :H]                                 # q a strided view, like the model's
    out = _run_twice(lambda: ops.attention(qv, kc, vc, key_mask=km, causal=causal, past=past))
    ref = ao.reference(q, k, v, km, causal, past, vis=vis)
    arith = ao.arith_wgmma(Tkv, dtype, hd)
    ao.check(out, ref, arith, what)
    if lse:
        o2, l2 = ops.attention_forward_lse(qv, kc, vc, key_mask=km, causal=causal)
        assert torch.equal(o2.reshape(out.shape), out), f"{what}: the LSE instantiation changed O"
        ao.check_lse(l2, ref, arith, what)


@pytest.mark.parametrize("persistent", [False, True])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_wgmma_causal_left_padding_over_whole_tiles(dtype, hd, persistent):
    """Left padding of 63 / 64 / 65 / 128 / 200 keys: whole query tiles see no key, and the first visible key is
    several key tiles in."""
    B, T = 2, 330
    H = _heads(B, T, hd, persistent)
    for pad in (63, 64, 65, 128, 200):
        km = ao.key_mask(B, T, pad=pad, device=DEV)
        _wgmma_case(B, H, T, T, hd, dtype, "gauss", km, True, 0, f"pad {pad}", lse=True, seed=pad)


@pytest.mark.parametrize("persistent", [False, True])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_wgmma_chunk_on_a_cache(dtype, hd, persistent):
    """A chunk of Tq in {16, 17, 63, 200} queries after ``past`` cached positions, K / V views of a longer cache that
    holds NaN past Tkv; left padding of 65 makes the chunk's first query at past 64 see nothing."""
    B = 2
    for past in (64, 1000):
        for Tq in (16, 17, 63, 200):
            Tkv = past + Tq
            H = _heads(B, Tq, hd, persistent)
            km = ao.key_mask(B, Tkv, pad=65, device=DEV)
            _wgmma_case(B, H, Tq, Tkv, hd, dtype, "gauss", km, True, past, f"past {past} Tq {Tq}", seed=Tq)


@pytest.mark.parametrize("persistent", [False, True])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_wgmma_score_patterns(dtype, hd, persistent):
    """Every score pattern, causal with left padding and non-causal Tq != Tkv with a hole, left padding and a fully
    masked entry."""
    B, T = 3, 300
    for i, pattern in enumerate(ao.PATTERNS):
        H = _heads(B, T, hd, persistent)
        km = ao.key_mask(B, T, pad=64, device=DEV)
        _wgmma_case(B, H, T, T, hd, dtype, pattern, km, True, 0, f"{pattern} causal", lse=True, seed=i)
        H = _heads(B, 90, hd, persistent)
        km = ao.key_mask(B, T, pad=65, hole=True, dead_row=True, device=DEV)
        _wgmma_case(B, H, 90, T, hd, dtype, pattern, km, False, 0, f"{pattern} non-causal", lse=True, seed=10 + i)


# ---- generic kernel ---------------------------------------------------------------------------------------------------
def _generic_mask(B, Tkv):
    """Entry 0: keys 256..511 masked (a whole 256-key chunk when Tkv > 511), entry 1: no key, entry 2: left padding 5."""
    km = torch.ones((B, Tkv), dtype=torch.uint8, device=DEV)
    km[0, 256:512] = 0
    km[1] = 0
    km[2, :5] = 0
    return km


@pytest.mark.parametrize("hd", [32, 64, 80, 96, 128, 256])
@pytest.mark.parametrize("dtype", [F32, BF16, F16])
def test_generic_kernel(dtype, hd):
    ops = _ops()
    B, H = 3, 2
    n = 0
    for Tkv in (255, 256, 257, 513):
        for Tq in (1, 2, 15):
            for km in (None, _generic_mask(B, Tkv)):
                pattern = ao.PATTERNS[n % len(ao.PATTERNS)]
                n += 1
                past = Tkv - Tq - 3                                         # the last 3 keys are seen by no row
                q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, pattern, dtype, key_mask=km, seed=n, device=DEV)
                vis = ao.visibility(B, Tq, Tkv, km, True, past, DEV)
                kp, vp = ao.poison(k, v, ao.hidden_slots(vis))
                kc, vc = ao.in_cache(kp), ao.in_cache(vp)
                what = f"Tkv {Tkv} Tq {Tq} {pattern} mask {km is not None}"
                out = _run_twice(lambda: ops.attention(q, kc, vc, key_mask=km, causal=True, past=past, force_generic=True))
                ref = ao.reference(q, k, v, km, True, past, vis=vis)
                ao.check(out, ref, ao.arith_generic(Tkv, dtype, hd), what)
                if Tq > 1:                                                  # the natural route at Tq < 16
                    nat = ops.attention(q, kc, vc, key_mask=km, causal=True, past=past)
                    assert torch.equal(nat, out), what


# ---- split-KV decode --------------------------------------------------------------------------------------------------
def _decode_masks(B, Tkv):
    """None, and: entry 0 with keys 256..511 (a whole split) and 64..127 (a whole warp range) masked where they exist,
    entry 1 fully masked, entry 2 left-padded by 300 keys."""
    km = torch.ones((B, Tkv), dtype=torch.uint8, device=DEV)
    km[0, 256:512] = 0
    km[0, 64:128] = 0
    km[1] = 0
    km[2, :300] = 0
    return (None, km)


def _decode_case(q, k, v, km, past, arith, what):
    ops = _ops()
    B, _, H, hd = q.shape
    Tkv = k.shape[1]
    vis = ao.visibility(B, 1, Tkv, km, True, past, DEV)
    kp, vp = ao.poison(k, v, ao.hidden_slots(vis))
    kc, vc = ao.in_cache(kp), ao.in_cache(vp)
    out = _run_twice(lambda: ops.attention(q, kc, vc, key_mask=km, causal=True, past=past))
    ao.check(out, ao.reference(q, k, v, km, True, past, vis=vis), arith, what)


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_decode_split128(dtype):
    """hd 128, 16-bit: one split (direct write) up to 256 keys, the ticket merge above, across the 64-key warp ranges;
    past at the end, in the middle and at 0 with NaN past it."""
    B, H, hd = 3, 2, 128
    for i, Tkv in enumerate((1, 63, 64, 65, 255, 256, 257, 2049)):
        pattern = ao.PATTERNS[i % len(ao.PATTERNS)]
        q, k, v = ao.make_qkv(B, 1, Tkv, H, hd, pattern, dtype, seed=Tkv, device=DEV)
        for past in sorted({Tkv - 1, Tkv // 2, 0}):
            for km in _decode_masks(B, Tkv):
                _decode_case(q, k, v, km, past, ao.arith_split128(Tkv, dtype),
                             f"Tkv {Tkv} past {past} {pattern} mask {km is not None}")


@pytest.mark.parametrize("dtype,hd", [(BF16, 32), (F16, 96), (BF16, 160), (F16, 192), (BF16, 256), (F32, 128),
                                      (BF16, 128), (F16, 128)])
def test_decode_split_generic(dtype, hd):
    """The generic split kernel and its merge: hd other than 128, fp32 at 128, and (16-bit hd 128) a q whose batch
    stride is not a multiple of 8 elements."""
    B, H = 3, 2
    for i, Tkv in enumerate((65, 257, 700)):
        pattern = ao.PATTERNS[(i + hd) % len(ao.PATTERNS)]
        q, k, v = ao.make_qkv(B, 1, Tkv, H, hd, pattern, dtype, seed=Tkv + hd, device=DEV)
        if dtype != F32 and hd == 128:                                      # q_bs = H * hd + 4: off the hd-128 kernel
            buf = torch.zeros((B, H * hd + 4), dtype=dtype, device=DEV)
            buf[:, :H * hd] = q.reshape(B, H * hd)
            q = buf[:, :H * hd].view(B, 1, H, hd)
            assert q.stride(0) % 8 != 0
        for past in sorted({Tkv - 1, Tkv // 2, 0}):
            for km in _decode_masks(B, Tkv):
                _decode_case(q, k, v, km, past, ao.arith_split(Tkv, dtype, hd),
                             f"hd {hd} Tkv {Tkv} past {past} {pattern} mask {km is not None}")


@pytest.mark.parametrize("hd", [128, 96])
def test_decode_graph_replay_follows_the_mask_on_the_device(hd):
    ops = _ops()
    B, H, Tkv = 3, 4, 700
    q, k, v = ao.make_qkv(B, 1, Tkv, H, hd, "gauss", BF16, seed=hd, device=DEV)
    km = torch.ones((B, Tkv), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.attention(q, k, v, key_mask=km, causal=True, past=Tkv - 1)     # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.attention(q, k, v, key_mask=km, causal=True, past=Tkv - 1)
    for mask_edit in (lambda m: m[0, 256:512].zero_(), lambda m: m[1].zero_(), lambda m: m[2, :300].zero_()):
        mask_edit(km)
        graph.replay()
        want = ops.attention(q, k, v, key_mask=km, causal=True, past=Tkv - 1)
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        ao.check(out, ao.reference(q, k, v, km, True, Tkv - 1), ao.arith_split128(Tkv, BF16) if hd == 128
                 else ao.arith_split(Tkv, BF16, hd), "graph replay")


# ---- shared-prefix decode ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,hd", [(BF16, 128), (F16, 128), (BF16, 64)])
@pytest.mark.parametrize("G", [1, 5])
def test_shared_prefix_decode(G, dtype, hd):
    """P = 2 prompts of G rows, a 520-position prefix buffer, prefix_len in {1, 300, 520}, against float64 over the
    logical cache; NaN in the prefix slots at and past prefix_len and in the generated rows past the step."""
    ops = _ops()
    P, Tp, max_new, H = 2, 520, 6, 2
    R = P * G
    Tkv = Tp + max_new
    g = torch.Generator(device=DEV).manual_seed(G * hd)
    kp = torch.randn((P, Tp, H, hd), generator=g, device=DEV).to(dtype)
    vp = torch.randn((P, Tp, H, hd), generator=g, device=DEV).to(dtype)
    kg = torch.randn((R, max_new, H, hd), generator=g, device=DEV).to(dtype)
    vg = torch.randn((R, max_new, H, hd), generator=g, device=DEV).to(dtype)
    q = torch.randn((R, 1, H, hd), generator=g, device=DEV).to(dtype)
    arith = ao.arith_split128(Tkv, dtype) if hd == 128 else ao.arith_split(Tkv, dtype, hd)
    for plen in (1, 300, 520):
        for step in (0, max_new - 1):
            past = plen + step
            km = torch.ones((R, Tkv), dtype=torch.uint8, device=DEV)
            km[-1, :min(plen, 200)] = 0                                     # a left-padded prompt row
            klog = torch.zeros((R, Tkv, H, hd), dtype=dtype, device=DEV)    # the logical per-row cache
            vlog = torch.zeros_like(klog)
            klog[:, :plen] = kp.repeat_interleave(G, 0)[:, :plen]
            vlog[:, :plen] = vp.repeat_interleave(G, 0)[:, :plen]
            klog[:, plen:past + 1] = kg[:, :step + 1]
            vlog[:, plen:past + 1] = vg[:, :step + 1]
            kpp, vpp, kgp, vgp = kp.clone(), vp.clone(), kg.clone(), vg.clone()
            for t in (kpp, vpp):
                t[:, plen:] = float("nan")
            for t in (kgp, vgp):
                t[:, step + 1:] = float("nan")
            plen_t = torch.tensor([plen], dtype=torch.int64, device=DEV)
            out = _run_twice(lambda: ops.attention_decode_shared(q, kpp, vpp, kgp, vgp, plen_t, key_mask=km, past=past))
            ref = ao.reference(q, klog, vlog, km, True, past)
            ao.check(out, ref, arith, f"G {G} prefix_len {plen} step {step}")


# ---- which kernel runs ------------------------------------------------------------------------------------------------
ATTN_KERNELS = ("attn_fwd_kernel", "attn_generic_kernel", "attn_decode_split128_kernel", "attn_decode_split_kernel",
                "attn_decode_merge_kernel")


def _kernels_run(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    # demangled ("mmfs::attn_fwd_kernel<...>(...)") or mangled ("...attn_fwd_kernelI...") names
    return {k for k in ATTN_KERNELS if any(k + "<" in n or k + "I" in n or k + "(" in n for n in names)}


def test_each_case_runs_on_the_kernel_it_is_meant_for():
    ops = _ops()
    q, k, v = ao.make_qkv(2, 200, 200, 2, 128, "gauss", BF16, device=DEV)
    q1, k1, v1 = ao.make_qkv(2, 1, 200, 2, 128, "gauss", BF16, device=DEV)
    qa, ka, va = ao.make_qkv(2, 1, 700, 2, 96, "gauss", BF16, device=DEV)
    routes = {
        "wgmma prefill": (lambda: ops.attention(q, k, v), {"attn_fwd_kernel"}),
        "generic, forced": (lambda: ops.attention(q, k, v, force_generic=True), {"attn_generic_kernel"}),
        "generic, Tq < 16": (lambda: ops.attention(q[:, :15], k, v, past=185), {"attn_generic_kernel"}),
        "split-128, one split": (lambda: ops.attention(q1, k1, v1, past=199), {"attn_decode_split128_kernel"}),
        "split-128, ticket merge": (lambda: ops.attention(q1, ao.in_cache(k1.repeat(1, 3, 1, 1)),
                                                          ao.in_cache(v1.repeat(1, 3, 1, 1)), past=599),
                                    {"attn_decode_split128_kernel"}),
        "generic split": (lambda: ops.attention(qa, ka, va, past=699),
                          {"attn_decode_split_kernel", "attn_decode_merge_kernel"}),
        "shared prefix": (lambda: ops.attention_decode_shared(
            q1, k1, v1, k1[:, :4], v1[:, :4], torch.tensor([150], device=DEV), past=151),
            {"attn_decode_split128_kernel"}),
    }
    for name, (fn, want) in routes.items():
        fn()                                                                # module load outside the trace
        got = _kernels_run(fn)
        assert got == want, f"{name}: ran {sorted(got)}, expected {sorted(want)}"


# ---- backward at the masking and score edges ---------------------------------------------------------------------------
ATTN_TOL = {BF16: 1e-2, F16: 2e-3}     # per tensor, of max |ref| (as tests/test_train_kernels_gpu.py)
U16 = {BF16: 2.0 ** -8, F16: 2.0 ** -11}


def _bwd_case(B, H, Tq, Tkv, hd, dtype, pattern, km, causal, general, seed):
    ops = _ops()
    q, k, v = ao.make_qkv(B, Tq, Tkv, H, hd, pattern, dtype, key_mask=km, seed=seed, device=DEV)
    d_out = torch.randn((B, Tq, H, hd), generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV).to(dtype)
    out, lse = ops.attention_forward_lse(q, k, v, key_mask=km, causal=causal)

    def grads():
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        if general:
            ops.attention_backward_general(q, k, v, out, d_out, lse, dq, dk, dv, key_mask=km, causal=causal)
        else:
            ops.attention_backward(q, k, v, out, d_out, lse, dq, dk, dv, key_mask=km)
        return torch.cat([dq.flatten(), dk.flatten(), dv.flatten()])

    flat = _run_twice(grads)
    n_q, n_k = q.numel(), k.numel()
    got = (flat[:n_q].view_as(q), flat[n_q:n_q + n_k].view_as(k), flat[n_q + n_k:].view_as(v))
    vis = ao.visibility(B, Tq, Tkv, km, causal, 0, DEV)
    x = [t.double().requires_grad_(True) for t in (q, k, v)]
    s = torch.einsum("bqhd,bkhd->bhqk", x[0], x[1]) * hd ** -0.5
    seen = vis.any(-1)[:, None, :, None]
    s = torch.where(seen, torch.where(vis[:, None], s, -math.inf), 0.0)
    p = torch.softmax(s, -1) * seen
    o_ref = torch.einsum("bhqk,bkhd->bqhd", p, x[2])
    o_ref.backward(d_out.double())
    # dQ = scale dS K and dK = scale dS^T Q with dS_ij = P_ij (dP_ij - D_i), dP_ij = dO_i . v_j, D_i = dO_i . O_i.
    # Two effects make max |ref| no scale for dQ / dK at these edges, and each gets a per-tensor floor:
    # * dS is rounded to 16 bits before its MMAs (relative u per entry): <= u scale sum_j |dS_ij| |k_jc| for dQ.
    #   Where the keys a row attends share a large component (the rising pattern: channel 0 of k is 10 t / scale for
    #   every key of tile t) sum_j dS_ij = 0 cancels it exactly in dQ, but its rounding errors do not cancel;
    # * dP_ij and D_i are fp32 dot products over hd that cancel where one key takes all the weight (the sink): each errs
    #   by <= 2 hd 2^-24 of its sum of |terms| (2u per add allows the tensor cores' truncation).
    with torch.no_grad():
        do, pd, qd, kd, vd = d_out.double(), p.detach(), x[0].detach(), x[1].detach(), x[2].detach()
        dp = torch.einsum("bqhd,bkhd->bhqk", do, vd)
        dd = torch.einsum("bqhd,bqhd->bhq", do, o_ref.detach())[..., None]
        ds = (pd * (dp - dd)).abs() * U16[dtype] * hd ** -0.5
        a = torch.einsum("bqhd,bkhd->bhqk", do.abs(), vd.abs())
        a = a + torch.einsum("bqhd,bqhd->bhq", do.abs(), o_ref.detach().abs())[..., None]
        w = pd * a * hd ** -0.5 * 2 * hd * 2.0 ** -24 + ds
        floor = (torch.einsum("bhqk,bkhd->bqhd", w, kd.abs()).max().item(),
                 torch.einsum("bhqk,bqhd->bkhd", w, qd.abs()).max().item(), 0.0)
    for name, g, r, fl in zip(("dQ", "dK", "dV"), got, x, floor):
        assert bool(torch.isfinite(g).all()), f"{pattern}: {name} not finite"
        err = (g.double() - r.grad).abs().max().item()
        tol = ATTN_TOL[dtype] * r.grad.abs().max().item() + fl
        assert err <= tol, f"{pattern}: {name} max err {err:.3e} > {tol:.3e}"
    dead_q = ~vis.any(-1)                                                   # (B, Tq): rows that see no key
    dead_k = ~vis.any(1)                                                    # (B, Tkv): keys no row sees
    assert not bool(got[0][dead_q].any()), f"{pattern}: dQ of a row that sees no key must be 0"
    assert not bool(got[1][dead_k].any()) and not bool(got[2][dead_k].any()), f"{pattern}: dK / dV of unseen keys"


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_attention_backward_at_mask_and_score_edges(dtype):
    B, H, T, hd = 2, 2, 330, 128
    for pad in (64, 128, 200):
        for pattern in ("gauss", "sink", "rising"):
            km = ao.key_mask(B, T, pad=pad, device=DEV)
            _bwd_case(B, H, T, T, hd, dtype, pattern, km, True, False, seed=pad)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_attention_backward_general_at_mask_and_score_edges(dtype, causal):
    B, H, hd = 2, 2, 64
    Tq, Tkv = (330, 330) if causal else (90, 330)
    for pad in (64, 128, 200):
        for pattern in ("gauss", "sink", "rising"):
            km = ao.key_mask(B, Tkv, pad=pad, device=DEV)
            _bwd_case(B, H, Tq, Tkv, hd, dtype, pattern, km, causal, True, seed=pad)
