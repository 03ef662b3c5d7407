"""Caches of values derived from tensors, under one rule (DESIGN.md section 5).

A cached value matches its sources only while every source is the SAME Python tensor object (checked through a weak
reference, so a freed-and-reallocated tensor at the same address can never match) with the same in-place version
counter, ``data_ptr``, dtype, device and shape.  ``data_ptr`` alone is NOT an identity: the caching allocator hands the
next forward's feature tensor the address of the previous one.  Identity plus version is not one either:
``module.to()`` / ``.half()`` / ``p.data = t`` keep the Parameter object and its version and swap only its data.

``SourceCache`` holds one value derived from an ACTIVATION tensor (and the weights applied to it).  Writes that bypass
autograd's version counter (a CUDA-graph replay into a static input buffer) are invisible to the check: callers that
refill a tensor that way must call ``clear()`` (or ``clear_activation_caches(module)``) first.  ``WeightCache`` holds
values derived from WEIGHTS only; ``clear_activation_caches`` leaves them alone, as captured CUDA graphs read them.
"""
from __future__ import annotations

import weakref

import torch


def _as_seq(srcs):
    return srcs if isinstance(srcs, (list, tuple)) else (srcs,)


def _fingerprint(s):
    return s._version, s.data_ptr(), s.dtype, s.device, s.shape


def _make_entry(srcs, val):
    return val, tuple((weakref.ref(s), _fingerprint(s)) for s in srcs)


def _lookup(entry, srcs):
    """The value of ``entry`` if it was derived from exactly ``srcs``, else None."""
    if entry is None or len(entry[1]) != len(srcs):
        return None
    for (r, fp), s in zip(entry[1], srcs):   # _fingerprint(s) written out: ~80 hits per eager decode token
        if r() is not s or fp != (s._version, s.data_ptr(), s.dtype, s.device, s.shape):
            return None
    return entry[0]


class SourceCache:
    __slots__ = ("_extra", "_entry")

    def __init__(self):
        self.clear()

    def get(self, srcs, extra=()):
        """``srcs``: one tensor or a sequence of tensors the cached value was derived from; ``extra``: a further key."""
        return _lookup(self._entry, _as_seq(srcs)) if self._extra == extra else None

    def put(self, srcs, val, extra=()):
        self._extra, self._entry = extra, _make_entry(_as_seq(srcs), val)
        return val

    def get_or_build(self, srcs, build, extra=(), cache=True):
        """The value cached for ``srcs`` / ``extra``, else ``build()``, kept for the next call; ``cache=False``:
        ``build()`` and nothing else (the callers pass it while autograd records)."""
        if not cache:
            return build()
        val = self.get(srcs, extra)
        return self.put(srcs, build(), extra) if val is None else val

    def clear(self):
        self._extra, self._entry = None, None


class WeightCache:
    """One entry per ``key`` (e.g. a target shape), replaced when its sources change and never evicted otherwise: a
    CUDA graph captured while an entry was live keeps reading its tensors."""

    __slots__ = ("_entries",)

    def __init__(self):
        self._entries = {}

    def get(self, srcs, build, key=()):
        """The value ``build()`` returned for ``key``; rebuilt under ``no_grad`` unless ``srcs`` (one tensor or a
        sequence of tensors) are the ones it was built from."""
        if not isinstance(srcs, (list, tuple)):                       # _as_seq, inlined: this is the hot path
            srcs = (srcs,)
        val = _lookup(self._entries.get(key), srcs)
        if val is None:
            with torch.no_grad():
                val = build()
            self._entries[key] = _make_entry(srcs, val)
        return val


def clear_activation_caches(module) -> None:
    """Drop every ``SourceCache`` below ``module``.  Needed only when an input tensor is refilled behind autograd's back
    (CUDA-graph static buffers)."""
    for m in module.modules():
        for v in vars(m).values():
            if isinstance(v, SourceCache):
                v.clear()
