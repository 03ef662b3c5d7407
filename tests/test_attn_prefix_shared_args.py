"""CPU tests of ``mmfs_attn_prefix_shared`` (answer options scored against one stored context): every refusal returns
the documented code with a message before any CUDA call; ``PrefixKV`` refuses a cache-writing or position-less use;
and the shared-context ``generate_scores`` refuses options that hold the bos, soi or image-token id."""
import pytest
import torch

# fake, never dereferenced device addresses: every call below is refused before a launch
A, B_, C, D, E, O, PM, KM, W = (0x10000 * (i + 1) for i in range(9))


def _call(**over):
    from mm_interleaved_b200 import _lib
    P, H, G, L, Tp, hd = 2, 2, 5, 4, 64, 128
    Tq = G * L
    a = dict(q=A, k=B_, v=C, kp=D, vp=E, out=O, pmask=PM, kmask=KM, P=P, H=H, Tq=Tq, Tp=Tp, seg_len=L, hd=hd,
             q_bs=Tq * H * hd, q_ts=H * hd, k_bs=Tq * H * hd, k_ts=H * hd, v_bs=Tq * H * hd, v_ts=H * hd,
             kp_bs=Tp * H * hd, kp_ts=H * hd, vp_bs=Tp * H * hd, vp_ts=H * hd, o_bs=Tq * H * hd, o_ts=H * hd,
             scale=0.125, dtype=_lib.BF16, counter=W)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_attn_prefix_shared(*a.values(), None)
    return rc, lib.mmfs_last_error().decode()


def test_declared_with_a_ctypes_signature():
    from mm_interleaved_b200 import _lib
    assert "mmfs_attn_prefix_shared" in _lib.SIGNATURES
    res, args = _lib.SIGNATURES["mmfs_attn_prefix_shared"]
    assert len(args) == 30 and res is not None


def test_declared_in_the_header():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert "int mmfs_attn_prefix_shared(" in open(os.path.join(root, "include", "mmfs_b200.h")).read()


@pytest.mark.parametrize("name", ["q", "k", "v", "kp", "vp", "out", "counter"])
def test_null_pointers_are_invalid(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg


def test_masks_may_be_null_and_empty_batches_are_a_no_op():
    from mm_interleaved_b200 import _lib
    rc, _ = _call(P=0, q=None, k=None, v=None, kp=None, vp=None, out=None, counter=None)
    assert rc == _lib.OK
    rc, _ = _call(Tq=0, q=None, k=None, v=None, kp=None, vp=None, out=None, counter=None)
    assert rc == _lib.OK
    rc, msg = _call(pmask=None, kmask=None, dtype=3)     # past the pointer checks to the dtype check
    assert rc == _lib.EUNSUPPORTED and "f32/f16/bf16" in msg


@pytest.mark.parametrize("over", [dict(P=-1), dict(H=0), dict(Tq=-4), dict(Tp=0), dict(hd=0), dict(hd=288)])
def test_bad_shapes_are_invalid(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EINVAL and "bad shape" in msg


@pytest.mark.parametrize("seg_len", [0, -2])
def test_seg_len_below_one_is_invalid(seg_len):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(seg_len=seg_len)
    assert rc == _lib.EINVAL and "seg_len" in msg


@pytest.mark.parametrize("Tq, seg_len", [(20, 3), (21, 4), (5, 10)])
def test_queries_must_be_whole_segments(Tq, seg_len):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(Tq=Tq, seg_len=seg_len)
    assert rc == _lib.EINVAL and "whole segments" in msg


def test_misaligned_work_counter_is_invalid():
    from mm_interleaved_b200 import _lib
    rc, msg = _call(counter=W + 2)
    assert rc == _lib.EINVAL and "4-byte aligned" in msg


@pytest.mark.parametrize("over", [dict(dtype=3), dict(dtype=99), dict(dtype=-1)])
def test_dtypes_outside_f32_f16_bf16_are_unsupported(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EUNSUPPORTED and "f32/f16/bf16" in msg


@pytest.mark.parametrize("over", [dict(q=A + 1), dict(k=B_ + 1), dict(vp=E + 3), dict(out=O + 1),
                                  dict(kp=D + 2, dtype=0)])
def test_pointers_off_their_element_size_are_unsupported(over):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EUNSUPPORTED and "element size" in msg


def _tiny_attention():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.llama_mmfs import LlamaAttention
    cfg = m.LlamaMMFSConfig(hidden_size=64, num_attention_heads=2, intermediate_size=128, num_hidden_layers=1)
    return cfg, LlamaAttention(cfg)


def test_prefix_kv_refuses_use_cache():
    from mm_interleaved_b200.llama_mmfs import PrefixKV
    _, attn = _tiny_attention()
    pre = torch.zeros((1, 8, 2, 32))
    c = PrefixKV(pre, pre.clone(), None, 3)
    with torch.no_grad(), pytest.raises(RuntimeError, match="read-only"):
        attn(torch.zeros((1, 6, 64)), position_ids=torch.arange(6)[None], past_key_value=c, use_cache=True)


def test_prefix_kv_needs_explicit_position_ids():
    from mm_interleaved_b200.llama_mmfs import PrefixKV
    _, attn = _tiny_attention()
    pre = torch.zeros((1, 8, 2, 32))
    c = PrefixKV(pre, pre.clone(), None, 3)
    with torch.no_grad(), pytest.raises(RuntimeError, match="position_ids"):
        attn(torch.zeros((1, 6, 64)), past_key_value=c)


def test_decoder_with_prefix_kv_refuses_use_cache_and_missing_positions():
    import mm_interleaved_b200 as m
    from mm_interleaved_b200.llama_mmfs import LlamaModel, PrefixKV
    cfg = m.LlamaMMFSConfig(vocab_size=32, hidden_size=64, num_attention_heads=2, intermediate_size=128,
                            num_hidden_layers=1, cross_attention_frequency=4)
    model = LlamaModel(cfg).eval()
    pre = [PrefixKV(torch.zeros((1, 8, 2, 32)), torch.zeros((1, 8, 2, 32)), None, 3)]
    ids = torch.ones((1, 6), dtype=torch.long)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="read-only"):
            model(input_ids=ids, past_key_values=pre, position_ids=torch.arange(6)[None], use_cache=True)
        with pytest.raises(ValueError, match="position_ids"):
            model(input_ids=ids, past_key_values=pre, use_cache=False)
        with pytest.raises(ValueError, match="positions"):
            model(input_ids=ids, past_key_values=pre, position_ids=torch.arange(6)[None] + 8, use_cache=False)


class _StubScorer:
    """Just enough of MMInterleaved for the option check, which runs before any model work."""
    special_token_dict = dict(bos_token_id=1, eos_token_id=2, pad_token_id=0, soi_token_id=62, image_token_id=63)
    _shared_context_scores = True


@pytest.mark.parametrize("special", [1, 62, 63])
def test_shared_context_scores_refuse_options_with_special_ids(special):
    from mm_interleaved_b200.mm_interleaved import MMInterleaved
    _StubScorer._shared_context_scores_of = MMInterleaved._shared_context_scores_of
    opts = torch.randint(3, 60, (4, 3))
    opts[2, 1] = special
    with pytest.raises(ValueError, match="bos, soi or image-token"):
        MMInterleaved.generate_scores(_StubScorer(), text_ids=[torch.ones(5, dtype=torch.long)], image_tensors=None,
                                      num_image_per_seq=torch.ones(1), attention_mask=[torch.ones(5)],
                                      options_ids=[opts], options_attn_masks=[torch.ones((4, 3))])


def test_switch_is_off_by_default_and_toggles():
    from mm_interleaved_b200.mm_interleaved import MMInterleaved
    assert MMInterleaved.enable_shared_context_scores.__doc__
    stub = _StubScorer()
    stub._shared_context_scores = False
    assert MMInterleaved.enable_shared_context_scores(stub, True) is stub and stub._shared_context_scores
    MMInterleaved.enable_shared_context_scores(stub, False)
    assert not stub._shared_context_scores
