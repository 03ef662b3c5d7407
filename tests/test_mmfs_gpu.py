"""GPU parity of the H100 ``MMFS`` module (fused sampler kernel) against the committed outputs of
the reference module (tests/golden/mmfs_*.npz) and against the CPU oracle's intermediates.

Tolerances:
  * fp32 module output vs the reference's fp64 run: |err| <= 1e-3 * |ref| + 1e-6 (north-star 1e-3 rel, with
    an absolute floor for outputs that are themselves ~0), in practice max-abs ~2e-7 (TF32 is NOT used: the tests pin torch.backends.cuda.matmul.allow_tf32=False);
  * materialised sampling locations / attention weights (fp32) vs the oracle restatement:
    max-abs <= 2e-6;
  * bf16 module output vs the fp32 golden: max-abs <= 4e-2 * max|ref| -- bf16 storage of weights,
    activations, offsets and locations (what the reference's own bf16 run incurs).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import error_metrics  # noqa: E402
from oracle.mmfs import mmfs_forward_ref  # noqa: E402
from tests.test_oracle_mmfs import NAMES, load_mmfs_case  # noqa: E402

DEV = "cuda"


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def build_module(case, params, dtype=torch.float32):
    import mm_interleaved_b200 as m
    mod = m.MMFS(**case["ctor"])
    missing = mod.load_state_dict(params, strict=True)     # same state-dict keys as the reference
    assert not missing.missing_keys and not missing.unexpected_keys
    return mod.to(DEV, dtype).eval()


def run_module(mod, t, dtype=torch.float32):
    with torch.no_grad():
        return mod(t["query"].to(DEV, dtype), t["reference_points"].to(DEV), t["input_flatten"].to(DEV, dtype),
                   t["spatial_shapes"].to(DEV), t["level_start_index"].to(DEV), None, t["attention_mask"].to(DEV))


@pytest.mark.parametrize("name", NAMES)
def test_module_fp32_matches_reference_golden(name):
    params, t, kw, case = load_mmfs_case(name)
    out = run_module(build_module(case, params), t)
    ref = t["out_fp64"]
    err = (out.double().cpu() - ref).abs()
    assert (err <= 1e-3 * ref.abs() + 1e-6).all(), error_metrics(out, ref)
    assert error_metrics(out, ref)["max_abs"] <= 2e-5


@pytest.mark.parametrize("name", NAMES)
def test_module_bf16_close_to_reference(name):
    params, t, kw, case = load_mmfs_case(name)
    out = run_module(build_module(case, params, torch.bfloat16), t, torch.bfloat16)
    ref = t["out_fp32"]
    assert (out.float().cpu() - ref).abs().max() <= 4e-2 * ref.abs().max()


@pytest.mark.parametrize("name", NAMES)
def test_materialised_locations_and_weights_match_oracle(name):
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.mmfs import relative_image_index
    params, t, kw, case = load_mmfs_case(name)
    _, inter = mmfs_forward_ref(params, t["query"], t["reference_points"], t["input_flatten"], t["spatial_shapes"],
                                t["level_start_index"], t["attention_mask"], return_intermediates=True, **kw)
    mod = build_module(case, params)
    with torch.no_grad():
        w_cat, b_cat, rtable = mod._fused_weights()
        q1 = mod.dynamic_offset_mask(t["query"].to(DEV))
        qproj = torch.nn.functional.linear(q1, w_cat, b_cat).contiguous()
        relpos = relative_image_index(t["attention_mask"].to(DEV), t["query"].shape[1])
        loc, attn, null_mass = m.mmfs_sampler_locw(
            t["spatial_shapes"].to(DEV), t["level_start_index"].to(DEV), qproj, rtable, relpos,
            t["reference_points"].to(DEV).float().contiguous(), mod.scale_ratios.float().contiguous(),
            mod.n_heads, mod.n_levels, mod.n_points)
    assert torch.equal(relpos.cpu().long().squeeze(-1) if relpos.shape[-1] == 1 else relpos.cpu().long(),
                       inter["relpos"][..., :relpos.shape[-1]].squeeze(-1) if relpos.shape[-1] == 1 else inter["relpos"])
    # attention weights: masked images exactly zero, the rest within fp32 noise
    aw = inter["attention_weights"]
    assert (attn.cpu() - aw).abs().max() <= 2e-6
    assert torch.equal(attn.cpu() == 0, aw == 0)
    visible = (aw != 0)[..., None].expand_as(loc.cpu())
    assert ((loc.cpu() - inter["sampling_locations"]).abs()[visible]).max() <= 2e-6
    assert (null_mass.cpu() - inter["null_weights"].sum(3).squeeze(-1)).abs().max() <= 2e-6
    # fused gather == un-fused op on the materialised tensors (same taps, same weights)
    with torch.no_grad():                                  # the ctypes kernels are inference-only (ops.inference_only)
        value = mod.project_value(t["input_flatten"].to(DEV))
        unfused = m.ms_deform_attn_forward(value, t["spatial_shapes"].to(DEV), t["level_start_index"].to(DEV), loc, attn, 1)
        if value.shape[-1] in (32, 64, 128):
            fused = m.mmfs_sampler_forward(value, t["spatial_shapes"].to(DEV), t["level_start_index"].to(DEV), qproj, rtable,
                                           relpos, t["reference_points"].to(DEV).float().contiguous(),
                                           mod.scale_ratios.float().contiguous(), mod.n_levels, mod.n_points)
            assert (fused - unfused).abs().max() <= 1e-6
    # and the index stream of those locations is bit-exact against the oracle's
    from oracle import msda_forward_ref
    _, idx_ref = msda_forward_ref(value.cpu(), t["spatial_shapes"], t["level_start_index"], loc.cpu(), attn.cpu(),
                                  want_index_stream=True)
    idx = m.msda_index_stream(t["spatial_shapes"].to(DEV), t["level_start_index"].to(DEV), loc, mod.n_heads, value.shape[-1])
    assert torch.equal(idx.cpu(), idx_ref)


def test_value_projection_is_cached_across_calls():
    params, t, kw, case = load_mmfs_case("llm_tiny")
    mod = build_module(case, params)
    feat = t["input_flatten"].to(DEV)
    with torch.no_grad():
        v1 = mod.project_value(feat)
        v2 = mod.project_value(feat)
        assert v1 is v2
        feat.add_(1.0)                                  # in-place change invalidates the cache
        v3 = mod.project_value(feat)
        assert v3 is not v1


def test_cpu_tensors_fail_loudly():
    params, t, kw, case = load_mmfs_case("sd_tiny")
    import mm_interleaved_b200 as m
    mod = m.MMFS(**case["ctor"])
    mod.load_state_dict(params)
    with pytest.raises(RuntimeError, match="CUDA"):
        mod(t["query"], t["reference_points"], t["input_flatten"], t["spatial_shapes"], t["level_start_index"], None,
            t["attention_mask"])


def test_kernels_refuse_to_run_where_a_gradient_would_be_dropped():
    """None of the ctypes kernels is autograd-aware: with grad enabled and a trainable input they raise instead of
    silently cutting the graph (ADVICE r01)."""
    params, t, kw, case = load_mmfs_case("llm_tiny")
    mod = build_module(case, params)
    with pytest.raises(RuntimeError, match="inference-only"):
        mod(t["query"].to(DEV), t["reference_points"].to(DEV), t["input_flatten"].to(DEV), t["spatial_shapes"].to(DEV),
            t["level_start_index"].to(DEV), None, t["attention_mask"].to(DEV))
    from mm_interleaved_b200 import ops
    w = torch.nn.Parameter(torch.ones(64, device=DEV))
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.rmsnorm(torch.randn((2, 64), device=DEV), w, 1e-6)
    with torch.no_grad():
        ops.rmsnorm(torch.randn((2, 64), device=DEV), w, 1e-6)
