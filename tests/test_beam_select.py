"""CPU tests of the argument checks of ``mmfs_beam_select`` and ``mmfs_kv_beam_reorder``: every malformed call is
rejected with MMFS_EINVAL and a message before any CUDA call (these run without a GPU, so a check that reached CUDA
would report a CUDA error)."""
import pytest

GOOD = 0x1000            # stands for a valid device pointer; no call below gets far enough to dereference it


def _select(**over):
    from mm_interleaved_b200 import _lib
    a = dict(logits=GOOD, ld=32002, step=GOOD, params=GOOD, beam_scores=GOOD, history=GOOD, next_ids=GOOD, parent=GOOD,
             done=GOOD, hyp_scores=GOOD, hyp_ids=GOOD, hyp_meta=GOOD, eos=GOOD, n_eos=2, pad_id=0, min_length=8,
             scratch=GOOD, B=4, num_beams=5, V=32002, max_new=20)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_beam_select(a["logits"], a["ld"], a["step"], a["params"], a["beam_scores"], a["history"], a["next_ids"],
                              a["parent"], a["done"], a["hyp_scores"], a["hyp_ids"], a["hyp_meta"], a["eos"], a["n_eos"],
                              a["pad_id"], a["min_length"], a["scratch"], a["B"], a["num_beams"], a["V"], a["max_new"], None)
    return rc, lib.mmfs_last_error().decode()


def _reorder(**over):
    from mm_interleaved_b200 import _lib
    a = dict(cache=GOOD, n_caches=80, cache_stride=1 << 20, rows=20, row_stride=1 << 14, pos_stride=10240,
             row_bytes=10240, num_beams=5, parent=GOOD, cur=GOOD, step=GOOD, done=GOOD, max_positions=20)
    a.update(over)
    lib = _lib.lib()
    rc = lib.mmfs_kv_beam_reorder(a["cache"], a["n_caches"], a["cache_stride"], a["rows"], a["row_stride"],
                                  a["pos_stride"], a["row_bytes"], a["num_beams"], a["parent"], a["cur"], a["step"],
                                  a["done"], a["max_positions"], None)
    return rc, lib.mmfs_last_error().decode()


@pytest.mark.parametrize("name", ["logits", "step", "params", "beam_scores", "history", "next_ids", "parent", "done",
                                  "hyp_scores", "hyp_ids", "hyp_meta", "eos", "scratch"])
def test_beam_select_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _select(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


def test_beam_select_eos_may_be_null_only_without_eos_ids():
    from mm_interleaved_b200 import _lib
    rc, msg = _select(eos=None, n_eos=0, ld=5)          # passes the pointer check, stops at ld < V
    assert rc == _lib.EINVAL and "ld" in msg, msg


@pytest.mark.parametrize("over,text", [
    (dict(V=0), "positive"), (dict(V=-3), "positive"), (dict(B=0), "positive"), (dict(B=-1), "positive"),
    (dict(max_new=0), "positive"), (dict(max_new=-2), "positive"), (dict(num_beams=0), "positive"),
    (dict(num_beams=9), "num_beams"), (dict(n_eos=5), "eos"), (dict(n_eos=-1), "eos"), (dict(ld=32001), "ld"),
    (dict(V=1 << 20, ld=1 << 20), "exceeds"),
    (dict(V=14, ld=14, num_beams=5, n_eos=2), "candidate count"),     # K = 3 * 5 = 15 > V
    (dict(V=39, ld=39, num_beams=8, n_eos=4), "candidate count"),     # K = 5 * 8 = 40 > V
])
def test_beam_select_bad_sizes_are_rejected(over, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _select(**over)
    assert rc == _lib.EINVAL and text in msg, (over, rc, msg)


@pytest.mark.parametrize("name", ["cache", "parent", "cur", "step"])
def test_kv_beam_reorder_null_pointers_are_rejected(name):
    from mm_interleaved_b200 import _lib
    rc, msg = _reorder(**{name: None})
    assert rc == _lib.EINVAL and "null pointer" in msg, (rc, msg)


@pytest.mark.parametrize("over,text", [
    (dict(n_caches=0), "positive"), (dict(rows=0), "positive"), (dict(rows=-5), "positive"),
    (dict(num_beams=0), "positive"), (dict(row_bytes=0), "positive"), (dict(max_positions=0), "positive"),
    (dict(num_beams=9, rows=18), "num_beams"), (dict(rows=21), "multiple"), (dict(row_bytes=10248), "16 bytes"),
    (dict(row_stride=(1 << 14) + 8), "16 bytes"), (dict(cache=GOOD + 4), "16 bytes"),
])
def test_kv_beam_reorder_bad_arguments_are_rejected(over, text):
    from mm_interleaved_b200 import _lib
    rc, msg = _reorder(**over)
    assert rc == _lib.EINVAL and text in msg, (over, rc, msg)


def test_supported_limits_match_the_library():
    from mm_interleaved_b200 import ops
    assert ops.beam_candidates(5, 2) == 15 and ops.beam_candidates(3, 0) == 6 and ops.beam_candidates(3, 1) == 6
    assert ops.beam_select_supported(5, 2, 32002) and ops.beam_select_supported(8, 4, 40)
    assert not ops.beam_select_supported(9, 2, 32002) and not ops.beam_select_supported(5, 5, 32002)
    assert not ops.beam_select_supported(5, 2, 14) and not ops.beam_select_supported(5, 2, (1 << 17) + 1)
