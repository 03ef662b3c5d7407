"""CPU tests of the argument checks of the training-path kernels (``mmfs_attn_forward_lse``, ``mmfs_attn_backward``,
``mmfs_rmsnorm_backward``, ``mmfs_swiglu_backward``): every malformed or unsupported call is rejected with
MMFS_EINVAL / MMFS_EUNSUPPORTED and a message before any CUDA call (these run without a GPU, so a check that reached
CUDA would report a CUDA error)."""
import pytest

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it
BF16, F32 = 2, 0


def _fwd_lse(**over):
    from mm_interleaved_b200 import _lib
    a = dict(q=GOOD, k=GOOD, v=GOOD, out=GOOD, lse=GOOD, key_mask=None, B=2, H=4, Tq=256, Tkv=256, hd=128,
             q_bs=256 * 3 * 512, q_ts=3 * 512, k_bs=256 * 3 * 512, k_ts=3 * 512, v_bs=256 * 3 * 512, v_ts=3 * 512,
             o_bs=256 * 512, o_ts=512, dtype=BF16, counter=GOOD)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_attn_forward_lse(a["q"], a["k"], a["v"], a["out"], a["lse"], a["key_mask"], a["B"], a["H"], a["Tq"],
                                   a["Tkv"], a["hd"], a["q_bs"], a["q_ts"], a["k_bs"], a["k_ts"], a["v_bs"], a["v_ts"],
                                   a["o_bs"], a["o_ts"], 0.088, 1, 0, a["dtype"], a["counter"], None)
    return rc, lib.mmfs_last_error().decode()


_BWD_PTRS = ["q", "k", "v", "out", "d_out", "lse", "dq", "dk", "dv", "delta"]


def _bwd(**over):
    from mm_interleaved_b200 import _lib
    a = dict({n: GOOD for n in _BWD_PTRS}, key_mask=None, B=2, H=4, T=256, hd=128, dtype=BF16)
    qkv_bs, qkv_ts, o_bs, o_ts = 256 * 3 * 512, 3 * 512, 256 * 512, 512
    strides = dict(q_bs=qkv_bs, q_ts=qkv_ts, k_bs=qkv_bs, k_ts=qkv_ts, v_bs=qkv_bs, v_ts=qkv_ts, o_bs=o_bs, o_ts=o_ts,
                   do_bs=o_bs, do_ts=o_ts, dq_bs=qkv_bs, dq_ts=qkv_ts, dk_bs=qkv_bs, dk_ts=qkv_ts, dv_bs=qkv_bs, dv_ts=qkv_ts)
    a.update(strides)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_attn_backward(*[a[n] for n in _BWD_PTRS], a["key_mask"], a["B"], a["H"], a["T"], a["hd"],
                                *[a[n] for n in strides], 0.088, a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


def _rms(**over):
    from mm_interleaved_b200 import _lib
    a = dict(x=GOOD, w=GOOD, dy=GOOD, dx=GOOD, dw=GOOD, partials=GOOD, rows=300, cols=5120, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_rmsnorm_backward(a["x"], a["w"], a["dy"], a["dx"], a["dw"], a["partials"], a["rows"], a["cols"], 1e-6,
                                   a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


def _swiglu(**over):
    from mm_interleaved_b200 import _lib
    a = dict(gu=GOOD, d=GOOD, dgu=GOOD, rows=300, inter=13824, dtype=BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_swiglu_backward(a["gu"], a["d"], a["dgu"], a["rows"], a["inter"], a["dtype"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("over,code,text", [
    (dict(lse=None), "EINVAL", "null pointer"), (dict(q=None), "EINVAL", "null pointer"),
    (dict(B=-1), "EINVAL", "bad shape"), (dict(hd=96), "EUNSUPPORTED", "hd"), (dict(dtype=F32), "EUNSUPPORTED", "bf16"),
    (dict(q_ts=3 * 512 + 4), "EUNSUPPORTED", "16-byte"), (dict(out=GOOD + 8), "EUNSUPPORTED", "16-byte"),
])
def test_attn_forward_lse_rejects(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _fwd_lse(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


@pytest.mark.parametrize("name", _BWD_PTRS)
def test_attn_backward_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _bwd(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


@pytest.mark.parametrize("over,code,text", [
    (dict(B=-1), "EINVAL", "bad shape"), (dict(H=0), "EINVAL", "bad shape"), (dict(hd=0), "EINVAL", "bad shape"),
    (dict(hd=64), "EUNSUPPORTED", "hd = 128"), (dict(hd=256), "EUNSUPPORTED", "hd = 128"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(dtype=3), "EUNSUPPORTED", "bf16"),
    (dict(dq_ts=3 * 512 + 2), "EUNSUPPORTED", "16-byte"), (dict(k=GOOD + 2), "EUNSUPPORTED", "16-byte"),
    (dict(dv=GOOD + 8), "EUNSUPPORTED", "16-byte"), (dict(H=70000), "EUNSUPPORTED", "65535"),
])
def test_attn_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _bwd(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_empty_problems_are_no_ops():
    from mm_interleaved_b200 import _lib
    assert _bwd(B=0, q=None)[0] == _lib.OK and _bwd(T=0)[0] == _lib.OK
    assert _rms(rows=0)[0] == _lib.OK and _swiglu(rows=0)[0] == _lib.OK


@pytest.mark.parametrize("over,code,text", [
    (dict(x=None), "EINVAL", "null pointer"), (dict(dy=None), "EINVAL", "null pointer"),
    (dict(dx=None), "EINVAL", "null pointer"), (dict(partials=None), "EINVAL", "null pointer"),
    (dict(cols=0), "EINVAL", "bad shape"), (dict(rows=-1), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(cols=5124), "EUNSUPPORTED", "cols"),
    (dict(cols=8200), "EUNSUPPORTED", "cols"), (dict(x=GOOD + 8), "EUNSUPPORTED", "aligned"),
])
def test_rmsnorm_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _rms(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)


def test_rmsnorm_backward_partials_may_be_null_without_dweight():
    from mm_interleaved_b200 import _lib
    rc, msg = _rms(dw=None, partials=None, cols=5124)     # passes the pointer check, stops at the width
    assert rc == _lib.EUNSUPPORTED and "cols" in msg, msg


@pytest.mark.parametrize("over,code,text", [
    (dict(gu=None), "EINVAL", "null pointer"), (dict(d=None), "EINVAL", "null pointer"),
    (dict(dgu=None), "EINVAL", "null pointer"), (dict(inter=0), "EINVAL", "bad shape"),
    (dict(dtype=F32), "EUNSUPPORTED", "bf16"), (dict(inter=13826), "EUNSUPPORTED", "inter"),
    (dict(d=GOOD + 4), "EUNSUPPORTED", "aligned"),
])
def test_swiglu_backward_bad_arguments_are_rejected(over, code, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _swiglu(**over)
    assert rc == getattr(_lib, code) and text in msg, (over, rc, msg)
