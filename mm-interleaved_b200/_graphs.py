"""CUDA-graph replay of launch-bound sub-graphs (SURVEY.md 8 f3): the visual tokenizer is ~2400 small kernels per 16
images and one decode step is ~1000 small kernels -- issued eagerly, the host cannot keep the GPU busy.

``GraphedCallable`` captures ``fn(*tensors)`` once per input signature (shapes, dtypes, device) over private static
input buffers and replays it on later calls after copying the new inputs in.  The returned tensors live in the
graph's memory pool and are OVERWRITTEN by the next replay of the same signature: consume (or clone) them first.
Activation-derived caches inside ``fn`` never see a replay (it bypasses Python), so ``fn`` must not depend on a
cache that is filled from a tensor the caller refills in place (see _cache.py).
"""
from __future__ import annotations

from typing import Any, Callable, Dict, Tuple

import torch

from . import ops


def _tree_map(f, x):
    if torch.is_tensor(x):
        return f(x)
    if isinstance(x, dict):
        return {k: _tree_map(f, v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_tree_map(f, v) for v in x)
    return x


class GraphedCallable:
    def __init__(self, fn: Callable, warmup: int = 2, max_entries: int = 8):
        self.fn, self.warmup, self.max_entries = fn, warmup, max_entries
        self._entries: Dict[Tuple, Any] = {}

    @staticmethod
    def _key(args):
        return tuple((tuple(a.shape), a.dtype, a.device) for a in args)

    def _capture(self, args):
        static_in = [a.clone() for a in args]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(self.warmup):                      # lazy handles, autotuning, weight-derived caches
                self.fn(*static_in)
        torch.cuda.current_stream().wait_stream(side)
        before = ops.launch_counter[0]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph), torch.no_grad():
            out = self.fn(*static_in)
        return dict(graph=graph, static_in=static_in, out=out, launches=ops.launch_counter[0] - before)

    def __call__(self, *args):
        key = self._key(args)
        e = self._entries.get(key)
        if e is None:
            if len(self._entries) >= self.max_entries:
                self._entries.pop(next(iter(self._entries)))
            e = self._entries[key] = self._capture(args)
        for dst, src in zip(e["static_in"], args):
            dst.copy_(src, non_blocking=True)
        e["graph"].replay()
        ops.launch_counter[0] += e["launches"]               # this repo's kernels inside one replay
        return e["out"]

    def launches(self, *args) -> int:
        e = self._entries.get(self._key(args))
        return 0 if e is None else e["launches"]

    def clear(self):
        self._entries.clear()
