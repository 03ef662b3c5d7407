"""GPU parity of the specialised fused MMFS sampler (csrc/mmfs_sampler_v2_sm100.cu: 16-bit, D = 64, P = 8, 3 / 4 levels).

Oracle = the scalar C restatement of the reference kernel (oracle/msda_ref.c, cuh:36-87, 240-302) run on the sampling
locations / attention weights the EMIT kernel materialises from the same inputs (those are pinned to the reference
module's intermediates in tests/test_mmfs_gpu.py).  Bars:
  * fp32 tap weights (``exact_weights``): |out - oracle_fp32_accumulator| <= one storage ulp of it;
  * default (tap weights rounded to the element type, mixed-precision FMA): <= one storage ulp + eps_T * sum_k |w_k v_k| with
    eps_T = 2^-8 (bf16) / 2^-11 (f16), the unit roundoff -- the bound derived in the kernel's header, evaluated with the
    oracle on |value|;
  * specialised vs generic kernel on the full cfg-3 layer shape: <= 2 storage ulps (+ the weight-rounding term in the
    default mode), > 99 % bit-identical with fp32 weights.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

from oracle import level_start_index, msda_forward_ref  # noqa: E402

ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EPS_W = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}     # unit roundoff of the tap weight's storage type


def make_case(N, n_img, n_lvl, Lq, dtype, seed, mask_mode="3d", ref_mode="center", sizes=None, Lq_r=None):
    M, D, P = 16, 64, 8
    g = torch.Generator().manual_seed(seed)
    sizes = sizes or ([32, 16, 8] if n_lvl == 3 else [16, 8, 4, 2])
    shapes = torch.tensor([(s, s) for s in sizes] * n_img, dtype=torch.long)
    starts = level_start_index(shapes)
    S = int(shapes.prod(1).sum())
    C = M * P * 2 + M * n_lvl * (P + 1)
    value = (torch.randn((N, S, M, D), generator=g)).to(dtype)
    qproj = torch.randn((N, Lq, C), generator=g)
    qproj[..., :M * P * 2] = torch.rand((N, Lq, M * P * 2), generator=g) * 8 - 4          # a few points leave the map
    qproj = qproj.to(dtype)
    rtable = (0.3 * torch.randn((50, C), generator=g)).to(dtype)
    if mask_mode == "3d":
        mask = (torch.rand((N, Lq, n_img), generator=g) < 0.6).float()
        mask[:, :2] = 0                                                                 # rows without any visible image
    elif mask_mode == "2d":
        mask = (torch.rand((N, n_img), generator=g) < 0.7).float()
        mask[0] = 1
    else:
        mask = torch.ones((N, Lq, n_img))
    if ref_mode == "center":
        ref = torch.full((1, Lq, 1, 2), 0.5)
    else:                                                                               # SD flavour: pixel grid incl. the borders
        side = int(Lq ** 0.5)
        ys, xs = torch.meshgrid((torch.arange(side) + 0.5) / side, (torch.arange(side) + 0.5) / side, indexing="ij")
        ref = torch.stack((xs.reshape(-1), ys.reshape(-1)), -1)[None, :, None, :].contiguous()
    base = sizes[1] if n_lvl == 3 else sizes[-1]
    scale = torch.tensor([s / base for s in sizes], dtype=torch.float32)
    return dict(value=value, qproj=qproj, rtable=rtable, mask=mask, ref=ref.float(), scale=scale, shapes=shapes, starts=starts,
                n_lvl=n_lvl, P=P, M=M, Lq=Lq)


def run(case, **kw):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mmfs import _relative_image_index
    d = {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in case.items()}
    relpos = _relative_image_index(d["mask"], case["Lq"])
    out = m.mmfs_sampler_forward(d["value"], d["shapes"], d["starts"], d["qproj"], d["rtable"], relpos, d["ref"], d["scale"],
                                 case["n_lvl"], case["P"], **kw)
    return out, relpos, d


def oracle_of(case, relpos, d):
    import mm_interleaved_b200 as m
    loc, attn, _ = m.mmfs_sampler_locw(d["shapes"], d["starts"], d["qproj"], d["rtable"], relpos, d["ref"], d["scale"],
                                       case["M"], case["n_lvl"], case["P"])
    v = case["value"].float()
    ref = msda_forward_ref(v, case["shapes"], case["starts"], loc.float().cpu(), attn.float().cpu())
    mag = msda_forward_ref(v.abs(), case["shapes"], case["starts"], loc.float().cpu(), attn.float().cpu())
    return ref, mag


CASES = [
    ("llm_bf16", dict(N=2, n_img=4, n_lvl=3, Lq=96, dtype=torch.bfloat16, seed=1)),
    ("llm_f16", dict(N=1, n_img=3, n_lvl=3, Lq=64, dtype=torch.float16, seed=2)),
    ("sd_bf16_grid_2dmask", dict(N=3, n_img=2, n_lvl=4, Lq=64, dtype=torch.bfloat16, seed=3, mask_mode="2d", ref_mode="grid")),
    ("many_images_two_ballot_chunks", dict(N=1, n_img=40, n_lvl=3, Lq=24, dtype=torch.bfloat16, seed=4, sizes=[8, 4, 2])),
    ("non_pow2_maps_take_the_division_path", dict(N=1, n_img=2, n_lvl=3, Lq=48, dtype=torch.bfloat16, seed=5, sizes=[12, 6, 3])),
]


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_specialised_kernel_matches_oracle(name, kw):
    case = make_case(**kw)
    dtype = kw["dtype"]
    exact, relpos, d = run(case, exact_weights=True)
    fast, _, _ = run(case)
    generic, _, _ = run(case, generic=True)
    ref, mag = oracle_of(case, relpos, d)
    tiny = 1e-6
    e_exact = (exact.float().cpu() - ref).abs()
    assert bool((e_exact <= ULP[dtype] * ref.abs() + tiny).all()), float((e_exact - ULP[dtype] * ref.abs()).max())
    e_fast = (fast.float().cpu() - ref).abs()
    bound = ULP[dtype] * ref.abs() + EPS_W[dtype] * mag + tiny
    assert bool((e_fast <= bound).all()), float((e_fast - bound).max())
    if generic is not None:
        e_gen = (generic.float().cpu() - ref).abs()
        assert bool((e_gen <= ULP[dtype] * ref.abs() + tiny).all())
    # rows that see no image are exactly zero (mmfs.py:203-234: all weight on the null slots)
    vis_any = case["mask"].reshape(case["mask"].shape[0], -1, case["mask"].shape[-1]).sum(-1) > 0
    if vis_any.shape[1] == case["Lq"]:
        dead = ~vis_any
        assert float(exact.float().cpu()[dead].abs().max() if dead.any() else 0.0) == 0.0


def test_decode_row_mask_and_null_mass():
    """Lq = 1 with a (N, Tm, n) mask whose LAST row applies (mmfs.py:161-162), plus the null-mass output."""
    case = make_case(N=3, n_img=4, n_lvl=3, Lq=1, dtype=torch.bfloat16, seed=9)
    case["mask"] = (torch.rand((3, 7, 4), generator=torch.Generator().manual_seed(1)) < 0.5).float()
    case["mask"][0, -1] = 0
    a, relpos, d = run(case, want_null_mass=True)
    b, _, _ = run(case, want_null_mass=True, generic=True)
    assert relpos.shape == (3, 4, 1)
    assert torch.equal(a[1], b[1])                                     # null mass: same arithmetic in both kernels
    assert float(a[0][0].abs().max()) == 0.0
    ref, mag = oracle_of(case, relpos, d)
    err = (a[0].float().cpu() - ref).abs()
    assert bool((err <= ULP[torch.bfloat16] * ref.abs() + EPS_W[torch.bfloat16] * mag + 1e-6).all())


def test_full_cfg3_layer_specialised_vs_generic():
    """BASELINE cfg 3 layer shape (4 sequences x 2048 tokens x 4 images, bench token layout)."""
    from benchmarks.workloads import InterleavedCfg3
    from mm_interleaved_b200.mm_interleaved import cross_attention_mask_from_ids
    wl = InterleavedCfg3(0, 1, 4)
    wl.make_host_inputs(pin=False)
    case = make_case(N=4, n_img=4, n_lvl=3, Lq=2048, dtype=torch.bfloat16, seed=11, mask_mode="ones")
    case["mask"] = cross_attention_mask_from_ids(wl.host[0], 4, 1, wl.SOI_ID).cpu()
    exact, _, _ = run(case, exact_weights=True)
    fast, _, _ = run(case)
    generic, _, _ = run(case, generic=True)
    vmax = float(case["value"].float().abs().max())
    # sum_k w_k <= 1, so the weight-rounding term of the bound is at most eps * max|value|
    for got, frac, atol in ((exact, 0.99, 1e-5), (fast, 0.5, EPS_W[torch.bfloat16] * vmax)):
        diff = (got.float() - generic.float()).abs()
        assert bool((diff <= 2 * ULP[torch.bfloat16] * generic.float().abs() + atol).all()), float(diff.max())
        assert float((got == generic).float().mean()) > frac


def test_strict_flag_propagates_non_finite_values_like_the_reference():
    """MMFS_MSDA_STRICT: taps whose attention weight underflowed to exactly 0 are fetched too, so 0 * inf = NaN as in
    the reference (which multiplies every tap in); the default skips them."""
    case = make_case(N=1, n_img=2, n_lvl=3, Lq=16, dtype=torch.bfloat16, seed=12, mask_mode="ones")
    M, P, n_lvl = 16, 8, 3
    logits = case["qproj"][..., M * P * 2:].view(1, 16, M, n_lvl, P + 1)
    logits[:, :, :, 2, :] = -300.0                                      # level-2 items: exp(-300 - max) == 0 in fp32
    case["rtable"][:, M * P * 2:] = 0
    per_img = 32 * 32 + 16 * 16 + 8 * 8
    for i in range(2):
        case["value"][:, i * per_img + 32 * 32 + 16 * 16:(i + 1) * per_img] = float("inf")   # the 8x8 maps
    plain, _, _ = run(case)
    strict, _, _ = run(case, strict=True)
    assert bool(torch.isfinite(plain.float()).all())
    assert bool(torch.isnan(strict.float()).any())
