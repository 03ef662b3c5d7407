"""CPU tests of the switch between the inference path and the training path, which lives in the entry points of
``autograd_ops``: the call each entry point makes under ``no_grad``, with grad on and nothing requiring grad, with its
input requiring grad and with only a weight (or another argument) requiring grad; the dtype refusal of a recording call
before any work; and ``records`` being false exactly where ``inference_only`` lets a kernel run.  The ops.py kernels,
``Conv2d.fused`` and each Function's ``apply`` are replaced by stand-ins that log the call."""
import pytest
import torch
import torch.nn.functional as F

from mm_interleaved_b200 import autograd_ops, ops, unet_sd
from mm_interleaved_b200.msda import inference_only, records

BF16 = torch.bfloat16


def _t(*shape, dtype):
    return torch.randn(shape).to(dtype)


def _conv(dtype):
    return unet_sd.Conv2d(8, 8, 3, padding=1).to(dtype).requires_grad_(False)


# entry point -> (its call on the argument dict, the arguments for a dtype (the first one is the input), the other
# arguments that can require grad, the inference call: a stand-in's name or the torch expression's value, the Function)
SPECS = {
    "layernorm": (lambda a: autograd_ops.layernorm(a["x"], a["weight"], a["bias"], 1e-5),
                  lambda dt: dict(x=_t(2, 8, dtype=dt), weight=_t(8, dtype=dt), bias=_t(8, dtype=dt)),
                  ["weight", "bias"], "ops.layernorm", autograd_ops.LayerNormFunction),
    "rmsnorm": (lambda a: autograd_ops.rmsnorm(a["x"], a["weight"], 1e-6),
                lambda dt: dict(x=_t(2, 8, dtype=dt), weight=_t(8, dtype=dt)),
                ["weight"], "ops.rmsnorm", autograd_ops.RMSNormFunction),
    "swiglu": (lambda a: autograd_ops.swiglu(a["gate_up"]), lambda dt: dict(gate_up=_t(2, 16, dtype=dt)),
               [], "ops.swiglu", autograd_ops.SwiGLUFunction),
    "geglu": (lambda a: autograd_ops.geglu(a["value_gate"]), lambda dt: dict(value_gate=_t(2, 16, dtype=dt)),
              [], "ops.geglu", autograd_ops.GEGLUFunction),
    "quick_gelu": (lambda a: autograd_ops.quick_gelu(a["h"]), lambda dt: dict(h=_t(2, 8, dtype=dt)),
                   [], lambda a: a["h"] * torch.sigmoid(1.702 * a["h"]), autograd_ops.QuickGELUFunction),
    "resize_bilinear": (lambda a: autograd_ops.resize_bilinear(a["x"], 2), lambda dt: dict(x=_t(1, 2, 4, 4, dtype=dt)),
                        [], lambda a: F.interpolate(a["x"], scale_factor=2, mode="bilinear", align_corners=False),
                        autograd_ops.ResizeBilinearFunction),
    "attention": (lambda a: autograd_ops.attention(a["qkv"], a["key_mask"], causal=False),
                  lambda dt: dict(qkv=_t(1, 4, 3, 2, 8, dtype=dt), key_mask=torch.ones(1, 4, dtype=torch.uint8)),
                  [], "ops.attention", autograd_ops.AttentionFunction),
    "attention_general": (lambda a: autograd_ops.attention_general(a["q"], a["k"], a["v"]),
                          lambda dt: dict(q=_t(1, 4, 2, 8, dtype=dt), k=_t(1, 5, 2, 8, dtype=dt),
                                          v=_t(1, 5, 2, 8, dtype=dt)),
                          ["k", "v"], "ops.attention", autograd_ops.GeneralAttentionFunction),
    "group_norm_nhwc": (lambda a: autograd_ops.group_norm_nhwc(a["x"], 4, a["weight"], a["bias"], 1e-5, silu=True),
                        lambda dt: dict(x=_t(1, 8, 2, 2, dtype=dt), weight=_t(8, dtype=dt), bias=_t(8, dtype=dt)),
                        ["weight", "bias"], "ops.group_norm_nhwc", autograd_ops.GroupNormNHWCFunction),
    "conv": (lambda a: autograd_ops.conv(a["x"], a["conv"], a["add_bc"], a["residual"]),
             lambda dt: dict(x=_t(1, 8, 4, 4, dtype=dt), conv=_conv(dt), add_bc=_t(1, 8, dtype=dt),
                             residual=_t(1, 8, 4, 4, dtype=dt)),
             ["conv", "add_bc", "residual"], "Conv2d.fused", autograd_ops.ConvFunction),
}
KERNELS = ("layernorm", "rmsnorm", "swiglu", "geglu", "attention", "group_norm_nhwc")
TAKES_FP32 = {"group_norm_nhwc", "conv"}     # backward takes fp32 too (the convolution's data gradient on cuDNN)

CASES = [(e, c) for e, spec in SPECS.items() for c in ("no_grad", "nothing", "input", *spec[2])]


@pytest.fixture
def calls(monkeypatch):
    log = []
    for name in KERNELS:
        monkeypatch.setattr(ops, name, lambda *a, _n=f"ops.{name}", **k: log.append(_n))
    monkeypatch.setattr(unet_sd.Conv2d, "fused", lambda *a, **k: log.append("Conv2d.fused"))
    for spec in SPECS.values():
        fn = spec[4]
        monkeypatch.setattr(fn, "apply", staticmethod(lambda *a, _n=fn.__name__: log.append(_n)))
    return log


def _requires_grad(args, names):
    for n in names:
        args[n].requires_grad_(True)          # a module: all its parameters


@pytest.mark.parametrize("entry,case", CASES)
def test_entry_point_takes_the_function_exactly_when_autograd_records(calls, entry, case):
    call, build, others, inference, function = SPECS[entry]
    args = build(BF16)
    first = next(iter(args))
    _requires_grad(args, {"no_grad": [first, *others], "nothing": [], "input": [first]}.get(case, [case]))
    with torch.set_grad_enabled(case != "no_grad"):
        recording = records(*args.values())
        out = call(args)
        try:
            inference_only(entry, *args.values())
            refused = False
        except RuntimeError:
            refused = True
    assert recording == (case not in ("no_grad", "nothing"))
    assert refused == recording
    if recording:
        assert calls == [function.__name__]
    elif isinstance(inference, str):
        assert calls == [inference]
    else:
        assert calls == [] and torch.equal(out, inference(args))


@pytest.mark.parametrize("entry", list(SPECS))
def test_fp32_recording_call_is_refused_before_any_work(calls, entry):
    call, build, _, _, function = SPECS[entry]
    args = build(torch.float32)
    _requires_grad(args, [next(iter(args))])
    if entry in TAKES_FP32:
        call(args)
        assert calls == [function.__name__]
    else:
        with pytest.raises(RuntimeError, match="bf16 / fp16 only"):
            call(args)
        assert calls == []


def test_records_reads_tensors_and_module_parameters_only():
    conv = _conv(torch.float32)
    x = torch.zeros(2, requires_grad=True)
    assert not records(None, 1.0, object(), conv, torch.zeros(2))
    assert records(None, object(), x)
    conv.bias.requires_grad_(True)
    assert records(conv)
    with torch.no_grad():
        assert not records(conv, x)
