"""CPU tests of ``mmfs_attn_decode_shared`` (decode attention over a prompt stored once per group of rows): every
refusal returns the documented code with a message before any CUDA call, and a ``SharedPrefixKV`` refuses to be used
for anything but a one-token graph step."""
import pytest
import torch

# fake, never dereferenced device addresses: every call below is refused before a launch
A, B_, C, D, E, O, M, P, S = (0x10000 * (i + 1) for i in range(9))


def _call(**over):
    from mm_interleaved_b200 import _lib
    R, G, H, Tp, max_new, hd = 10, 5, 2, 64, 4, 128
    a = dict(q=A, kp=B_, vp=C, kg=D, vg=E, out=O, mask=M, plen=P, scratch=S, R=R, G=G, H=H, Tkv=Tp + max_new, Tp=Tp,
             max_new=max_new, hd=hd, q_bs=3 * H * hd, kp_bs=Tp * H * hd, kp_ts=H * hd, vp_bs=Tp * H * hd, vp_ts=H * hd,
             kg_bs=max_new * H * hd, kg_ts=H * hd, vg_bs=max_new * H * hd, vg_ts=H * hd, o_bs=H * hd, scale=0.125,
             causal=1, past=Tp + max_new - 1, dtype=_lib.BF16)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_attn_decode_shared(*a.values(), None)
    return rc, lib.mmfs_last_error().decode()


def test_declared_with_a_ctypes_signature():
    from mm_interleaved_b200 import _lib
    assert "mmfs_attn_decode_shared" in _lib.SIGNATURES
    assert len(_lib.SIGNATURES["mmfs_attn_decode_shared"][1]) == 31


@pytest.mark.parametrize("name", ["q", "kp", "vp", "kg", "vg", "out", "plen", "scratch"])
def test_null_pointers_are_invalid(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg


def test_key_mask_may_be_null_and_empty_batches_are_a_no_op():
    from mm_interleaved_b200 import _lib
    rc, _ = _call(R=0, q=None, kp=None, vp=None, kg=None, vg=None, out=None, plen=None, scratch=None)
    assert rc == _lib.OK
    rc, msg = _call(mask=None, kg=8)                     # gets past the pointer checks to the alignment check
    assert rc == _lib.EUNSUPPORTED and "aligned" in msg


@pytest.mark.parametrize("R, G", [(10, 3), (7, 2), (5, 10)])
def test_rows_must_be_whole_groups(R, G):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(R=R, G=G)
    assert rc == _lib.EINVAL and "whole groups" in msg


@pytest.mark.parametrize("over", [dict(G=0), dict(G=-1), dict(H=0), dict(Tkv=0), dict(Tp=0), dict(hd=0), dict(R=-5)])
def test_bad_shapes_are_invalid(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EINVAL and "bad shape" in msg


@pytest.mark.parametrize("max_new", [0, -3])
def test_max_new_below_one_is_invalid(max_new):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(max_new=max_new)
    assert rc == _lib.EINVAL and "max_new" in msg


@pytest.mark.parametrize("over", [dict(kp=B_ + 8), dict(vp=C + 2), dict(kg=D + 4), dict(vg=E + 8),
                                  dict(kp_bs=64 * 256 + 1), dict(kp_ts=257), dict(vp_ts=260), dict(vp_bs=3),
                                  dict(kg_bs=4), dict(kg_ts=255), dict(vg_bs=1), dict(vg_ts=6)])
def test_misaligned_rows_and_strides_are_unsupported(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EUNSUPPORTED and "16-byte aligned" in msg


@pytest.mark.parametrize("over", [dict(hd=96 + 16), dict(hd=288), dict(hd=48), dict(dtype=3), dict(dtype=99)])
def test_head_dims_and_dtypes_outside_attn_decode_are_unsupported(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EUNSUPPORTED and "f32/f16/bf16" in msg


def test_negative_past_is_invalid():
    from mm_interleaved_b200 import _lib
    rc, msg = _call(past=-1)
    assert rc == _lib.EINVAL and "negative past" in msg


def test_too_many_prompts_for_the_grid_are_unsupported():
    from mm_interleaved_b200 import _lib
    rc, msg = _call(R=65536 * 2, G=2)
    assert rc == _lib.EUNSUPPORTED and "65535" in msg


def test_shared_prefix_kv_refuses_anything_but_a_one_token_step():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.llama_mmfs import LlamaAttention, SharedPrefixKV
    cfg = m.LlamaMMFSConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=1)
    attn = LlamaAttention(cfg)
    P, G, Tp, max_new = 2, 3, 8, 4
    pre = torch.zeros((P, Tp, 2, 32))
    gen = torch.zeros((P * G, max_new, 2, 32))
    c = SharedPrefixKV(pre, pre.clone(), gen, gen.clone(), torch.zeros(1, dtype=torch.long), torch.zeros(1, dtype=torch.long))
    assert c.G == G and c.length == Tp + max_new - 1
    with torch.no_grad(), pytest.raises(RuntimeError, match="graph-decode cache"):
        attn(torch.zeros((P * G, 2, 64)), past_key_value=c)
