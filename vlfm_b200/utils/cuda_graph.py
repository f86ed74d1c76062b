"""The CUDA-graph policy of every engine that replays its per-step launch sequence, keyed by what the engine's graph depends on
(shapes, caption ids, buffer pointers and parameters).  The first call of a key runs eagerly: it warms up function attributes,
tables and lazy allocations.  The second captures the step and replays it once, so it runs the work exactly once; later calls
copy their inputs into the key's static copies and replay.  Every call counts, whether graphs are enabled for it or not."""
from __future__ import annotations

import os
import warnings
from typing import Any, Callable, Dict, Hashable, NamedTuple, Optional, Tuple

import torch


def default_use_graph() -> bool:
    """The default of every engine's ``use_graph``: ``VLFM_NO_GRAPH=1`` makes every kernel an individual launch."""
    return os.environ.get("VLFM_NO_GRAPH") != "1"


class Captured(NamedTuple):
    graph: torch.cuda.CUDAGraph
    static: Tuple[torch.Tensor, ...]    # the inputs the graph reads
    result: Any                         # what the captured call returned: its tensors live in the graph's pool


class GraphCache:
    def __init__(self, max_keys: Optional[int] = None) -> None:
        """``max_keys`` bounds the keys kept, counted or captured; a new key beyond it drops the oldest with its graph."""
        self.max_keys = max_keys
        self.calls: Dict[Hashable, int] = {}
        self.captured: Dict[Hashable, Captured] = {}
        self.error: Optional[str] = None    # why a capture failed; the cache runs eagerly from then on

    def will_replay(self, key: Hashable, enabled: bool) -> bool:
        """Whether the next call with ``key`` captures or replays a graph rather than running eagerly."""
        return enabled and self.error is None and self.calls.get(key, 0) >= 1

    def __call__(self, key: Hashable, enabled: bool, fn: Callable[..., Any], *inputs: torch.Tensor) -> Any:
        """``fn(*inputs)``, run eagerly or by replaying the graph of ``key``.  A replay returns the captured call's result,
        rewritten in place."""
        replay = self.will_replay(key, enabled)
        if key not in self.calls and len(self.calls) == self.max_keys:
            oldest = next(iter(self.calls))
            del self.calls[oldest]
            self.captured.pop(oldest, None)
        self.calls[key] = self.calls.get(key, 0) + 1
        c = self.captured.get(key)
        if replay and c is None:
            static = tuple(t.clone() for t in inputs)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(graph):
                    result = fn(*static)
                c = self.captured[key] = Captured(graph, static, result)
            except Exception as e:  # e.g. a host synchronisation inside fn: stay eager (loudly, once)
                self.error = repr(e)
                warnings.warn(f"CUDA-graph capture failed, running eagerly from now on: {e}", RuntimeWarning)
                torch.cuda.synchronize()
                replay = False
        elif replay:
            for s, t in zip(c.static, inputs):
                s.copy_(t, non_blocking=True)
        if not replay:
            return fn(*inputs)
        c.graph.replay()
        return c.result

    def clear(self) -> None:
        """Forget every key: for when the buffers the graphs read are reallocated."""
        self.calls.clear()
        self.captured.clear()
