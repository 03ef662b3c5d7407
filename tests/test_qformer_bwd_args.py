"""CPU tests of the argument checks of the Q-Former head's backward kernels (``mmfs_attn_backward_general``,
``mmfs_layernorm_backward``) and of their Python wrappers: every malformed or unsupported call is rejected with
MMFS_EINVAL / MMFS_EUNSUPPORTED and a message before any CUDA call (these run without a GPU, so a check that reached
CUDA would report a CUDA error)."""
import pytest
import torch

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it
BF16, F32 = 2, 0

_PTRS = ["q", "k", "v", "out", "d_out", "lse", "dq", "dk", "dv", "delta"]


def _bwd(**over):
    from mm_interleaved_b200 import _lib
    a = dict({n: GOOD for n in _PTRS}, key_mask=None, B=2, H=12, Tq=64, Tkv=257, hd=64, causal=0, dtype=BF16)
    q_bs, q_ts, kv_bs, kv_ts = 64 * 768, 768, 257 * 768, 768
    strides = dict(q_bs=q_bs, q_ts=q_ts, k_bs=kv_bs, k_ts=kv_ts, v_bs=kv_bs, v_ts=kv_ts, o_bs=q_bs, o_ts=q_ts,
                   do_bs=q_bs, do_ts=q_ts, dq_bs=q_bs, dq_ts=q_ts, dk_bs=kv_bs, dk_ts=kv_ts, dv_bs=kv_bs, dv_ts=kv_ts)
    a.update(strides)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_attn_backward_general(*[a[n] for n in _PTRS], a["key_mask"], a["B"], a["H"], a["Tq"], a["Tkv"], a["hd"],
                                        *[a[n] for n in strides], 0.125, a["causal"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


def _ln(**over):
    from mm_interleaved_b200 import _lib
    a = dict(x=GOOD, w=GOOD, dy=GOOD, dx=GOOD, dw=GOOD, db=GOOD, partials=GOOD, rows=300, cols=768, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_layernorm_backward(a["x"], a["w"], a["dy"], a["dx"], a["dw"], a["db"], a["partials"], a["rows"],
                                     a["cols"], 1e-12, a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("name", _PTRS)
def test_attn_backward_general_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _bwd(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


@pytest.mark.parametrize("over,code,text", [
    (dict(B=-1), "EINVAL", "bad shape"), (dict(H=0), "EINVAL", "bad shape"), (dict(Tq=0), "EINVAL", "bad shape"),
    (dict(Tkv=0), "EINVAL", "bad shape"), (dict(hd=0), "EINVAL", "bad shape"),
    (dict(causal=1), "EINVAL", "Tq == Tkv"),
    (dict(hd=96), "EUNSUPPORTED", "hd in {64, 128}"), (dict(hd=256), "EUNSUPPORTED", "hd in {64, 128}"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(dtype=3), "EUNSUPPORTED", "bf16"),
    (dict(k_ts=768 + 4), "EUNSUPPORTED", "16-byte"), (dict(dk_bs=257 * 768 + 2), "EUNSUPPORTED", "16-byte"),
    (dict(q=GOOD + 2), "EUNSUPPORTED", "16-byte"), (dict(dv=GOOD + 8), "EUNSUPPORTED", "16-byte"),
    (dict(H=70000), "EUNSUPPORTED", "65535"), (dict(B=70000), "EUNSUPPORTED", "65535"),
])
def test_attn_backward_general_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _bwd(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_attn_backward_general_takes_the_supported_cases_up_to_the_launch():
    """Causal with Tq = Tkv and hd 128 pass every check (the empty batch returns before touching a pointer)."""
    from mm_interleaved_b200 import _lib
    assert _bwd(B=0, q=None)[0] == _lib.OK
    assert _bwd(B=0, causal=1, Tq=64, Tkv=64, hd=128)[0] == _lib.OK


@pytest.mark.parametrize("over,code,text", [
    (dict(x=None), "EINVAL", "null pointer"), (dict(w=None), "EINVAL", "null pointer"),
    (dict(dy=None), "EINVAL", "null pointer"), (dict(dx=None), "EINVAL", "null pointer"),
    (dict(partials=None), "EINVAL", "null pointer"), (dict(dw=None, partials=None), "EINVAL", "null pointer"),
    (dict(cols=0), "EINVAL", "bad shape"), (dict(rows=-1), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(cols=772), "EUNSUPPORTED", "cols"),
    (dict(cols=8200), "EUNSUPPORTED", "cols"), (dict(dy=GOOD + 8), "EUNSUPPORTED", "aligned"),
])
def test_layernorm_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _ln(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_layernorm_backward_partials_may_be_null_without_dweight_and_dbias():
    from mm_interleaved_b200 import _lib
    rc, msg = _ln(dw=None, db=None, partials=None, cols=772)     # passes the pointer check, stops at the width
    assert rc == _lib.EUNSUPPORTED and "cols" in msg, msg
    assert _ln(rows=0)[0] == _lib.OK


def test_wrappers_refuse_bad_tensors():
    """The Python wrappers check shapes and dtypes before the library sees the call (CPU tensors fail the first check)."""
    from mm_interleaved_b200 import ops
    q = torch.zeros(1, 8, 2, 64)
    with pytest.raises(RuntimeError, match="attention_backward_general"):
        ops.attention_backward_general(q, q, q, q, q, torch.zeros(1, 2, 8), q, q, q)
    with pytest.raises(RuntimeError, match="attention_forward_lse"):
        ops.attention_forward_lse(q, q, q, causal=False)
    with pytest.raises(RuntimeError, match="layernorm_backward"):
        ops.layernorm_backward(torch.zeros(4, 64), torch.ones(64), torch.zeros(4, 64), 1e-5)


def test_wrappers_refuse_to_run_under_autograd():
    from mm_interleaved_b200 import ops
    x = torch.zeros(4, 64, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference-only"):
        ops.layernorm_backward(x, torch.ones(64), torch.zeros(4, 64), 1e-5)
