"""CPU tests of the argument checks of ``mmfs_beam_sample``: every malformed call is rejected with MMFS_EINVAL and a
message before any CUDA call (these run without a GPU, so a check that reached CUDA would report a CUDA error)."""
import pytest

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it


def _sample(**over):
    from mm_interleaved_b200 import _lib
    a = dict(logits=GOOD, ld=32002, step=GOOD, params=GOOD, seed=GOOD, uniforms=None, beam_scores=GOOD, history=GOOD,
             next_ids=GOOD, parent=GOOD, done=GOOD, hyp_scores=GOOD, hyp_ids=GOOD, hyp_meta=GOOD, error=GOOD, eos=GOOD,
             n_eos=2, pad_id=0, min_length=8, top_k=50, scratch=GOOD, B=4, num_beams=5, V=32002, max_new=20)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_beam_sample(a["logits"], a["ld"], a["step"], a["params"], a["seed"], a["uniforms"], a["beam_scores"],
                              a["history"], a["next_ids"], a["parent"], a["done"], a["hyp_scores"], a["hyp_ids"],
                              a["hyp_meta"], a["error"], a["eos"], a["n_eos"], a["pad_id"], a["min_length"], a["top_k"],
                              a["scratch"], a["B"], a["num_beams"], a["V"], a["max_new"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("name", ["logits", "step", "params", "beam_scores", "history", "next_ids", "parent", "done",
                                  "hyp_scores", "hyp_ids", "hyp_meta", "error", "eos", "scratch", "seed"])
def test_beam_sample_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _sample(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


def test_beam_sample_optional_pointers():
    """eos may be NULL without eos ids; the seed may be NULL when uniforms replace the draw."""
    from mm_interleaved_b200 import _lib
    rc, msg = _sample(eos=None, n_eos=0, ld=5)          # passes the pointer check, stops at ld < V
    assert rc == _lib.EINVAL and "ld" in msg, msg
    rc, msg = _sample(seed=None, uniforms=GOOD, ld=5)
    assert rc == _lib.EINVAL and "ld" in msg, msg


@pytest.mark.parametrize("over,text", [
    (dict(V=0), "positive"), (dict(V=-3), "positive"), (dict(B=0), "positive"), (dict(B=-1), "positive"),
    (dict(max_new=0), "positive"), (dict(max_new=-2), "positive"), (dict(num_beams=0), "positive"),
    (dict(num_beams=9), "num_beams"), (dict(n_eos=5), "eos"), (dict(n_eos=-1), "eos"), (dict(ld=32001), "ld"),
    (dict(top_k=-1), "top_k"), (dict(V=1 << 20, ld=1 << 20), "exceeds"), (dict(V=(1 << 17) + 1, ld=1 << 18), "exceeds"),
    (dict(V=9, ld=9, num_beams=5), "candidate count"),                # 2 * 5 = 10 > V
    (dict(V=15, ld=15, num_beams=8, n_eos=4), "candidate count"),     # 2 * 8 = 16 > V
])
def test_beam_sample_bad_sizes_are_rejected(over, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _sample(**over)
    assert rc == _lib.EINVAL and text in msg, (over, rc, msg)


def test_beam_sample_supported_agrees_with_the_library():
    """Every (num_beams, n_eos, V) that ``beam_sample_supported`` accepts passes the library's size checks (the call
    then stops at the deliberately short row stride), and every one it refuses is rejected on its size."""
    from mm_interleaved_b200 import _lib, ops
    for nb in (0, 1, 3, 5, 8, 9):
        for n_eos in (-1, 0, 2, 4, 5):
            for V in (2 * max(nb, 1) - 1, 2 * max(nb, 1), 64, 32002, 1 << 17, (1 << 17) + 1):
                rc, msg = _sample(num_beams=nb, n_eos=n_eos, V=V, ld=V - 1, eos=GOOD if n_eos else None)
                assert rc == _lib.EINVAL, (nb, n_eos, V)
                assert ("ld" in msg) == ops.beam_sample_supported(nb, n_eos, V), (nb, n_eos, V, msg)
    assert ops.beam_sample_supported(5, 2, 32002) and ops.beam_sample_supported(8, 4, 16)
    assert not ops.beam_sample_supported(8, 4, 15) and not ops.beam_sample_supported(9, 2, 32002)
