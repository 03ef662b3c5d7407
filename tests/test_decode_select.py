"""CPU tests of ``mmfs_decode_select``'s argument checks: every malformed call is rejected with MMFS_EINVAL and a
message before any CUDA call (these run without a GPU, so a check that reached CUDA would report a CUDA error)."""
import pytest

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it


def _call(**over):
    from mm_interleaved_b200 import _lib
    a = dict(logits=GOOD, ld=32002, out_ids=GOOD, step=GOOD, finished=GOOD, next_ids=GOOD, eos=GOOD, n_eos=2, pad_id=0,
             min_length=8, params=GOOD, seed=GOOD, uniforms=None, B=4, V=32002, max_new=90, mode=_lib.SELECT_SAMPLE)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_decode_select(a["logits"], a["ld"], a["out_ids"], a["step"], a["finished"], a["next_ids"], a["eos"],
                                a["n_eos"], a["pad_id"], a["min_length"], a["params"], a["seed"], a["uniforms"], a["B"],
                                a["V"], a["max_new"], a["mode"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("name", ["logits", "out_ids", "step", "finished", "next_ids", "params", "eos", "seed"])
def test_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


def test_optional_pointers_follow_the_mode():
    from mm_interleaved_b200 import _lib
    # eos may be NULL only with n_eos == 0, the seed only in greedy mode or with uniforms: these calls get past the
    # pointer check and stop at the next bad argument (ld < V)
    for over in (dict(eos=None, n_eos=0), dict(seed=None, mode=_lib.SELECT_GREEDY), dict(seed=None, uniforms=GOOD)):
        rc, msg = _call(ld=5, **over)
        assert rc == _lib.EINVAL and "ld" in msg, (over, msg)


@pytest.mark.parametrize("over,text", [
    (dict(V=0), "positive"), (dict(V=-3), "positive"), (dict(B=0), "positive"), (dict(B=-1), "positive"),
    (dict(max_new=0), "positive"), (dict(max_new=-2), "positive"), (dict(ld=32001), "ld"),
    (dict(mode=2), "mode"), (dict(mode=-1), "mode"), (dict(n_eos=-1), "eos"), (dict(V=1 << 20, ld=1 << 20), "exceeds"),
])
def test_bad_sizes_and_mode_are_rejected(over, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _call(**over)
    assert rc == _lib.EINVAL and text in msg, (over, rc, msg)
