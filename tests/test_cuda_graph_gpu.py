"""The CUDA-graph policy every engine shares (vlfm_b200/utils/cuda_graph.py), on a toy step of a few torch ops."""
import pytest
import torch

from vlfm_b200.utils.cuda_graph import GraphCache

pytestmark = pytest.mark.gpu


def _ref(x):
    return (torch.sin(x) * 3.0 + x * x).cumsum(0)


class Toy:
    """_ref as a step that also counts its executions on the device (an in-place update, like an engine's recurrent state) and
    its Python calls."""

    def __init__(self):
        self.runs = torch.zeros((), dtype=torch.int64, device="cuda")
        self.calls = 0

    def __call__(self, x):
        self.calls += 1
        self.runs.add_(1)
        return _ref(x)


def _x(seed):
    return torch.randn(4096, generator=torch.Generator().manual_seed(seed)).cuda()


def test_first_call_eager_second_captures_then_replays():
    cache, toy, x = GraphCache(), Toy(), _x(0)
    assert not cache.will_replay("k", True)
    out = cache("k", True, toy, x)
    assert not cache.captured and cache.calls["k"] == 1 and toy.calls == 1
    assert torch.equal(out, _ref(x))
    assert cache.will_replay("k", True) and not cache.will_replay("k", False)
    got = cache("k", True, toy, x)
    assert "k" in cache.captured and cache.calls["k"] == 2 and cache.error is None
    assert int(toy.runs) == 2, "the capturing call must run the step exactly once"
    assert torch.equal(got, out)
    for seed in (1, 2):                          # new inputs: copied into the static copy, replayed, the same result tensor
        y = _x(seed)
        again = cache("k", True, toy, y)
        assert again is got and torch.equal(again, _ref(y))
    assert toy.calls == 2 and int(toy.runs) == 4 and len(cache.captured) == 1


def test_bound_drops_the_oldest_key():
    cache, toy = GraphCache(max_keys=2), Toy()
    for k in ("a", "a", "b", "b"):
        cache(k, True, toy, _x(3))
    assert set(cache.captured) == {"a", "b"}
    out = cache("c", True, toy, _x(4))
    assert set(cache.calls) == {"b", "c"} and set(cache.captured) == {"b"}
    assert torch.equal(out, _ref(_x(4)))
    assert not cache.will_replay("a", True)     # dropped with its count: its next call is eager again
    cache("a", True, toy, _x(5))
    assert "a" not in cache.captured and set(cache.calls) == {"c", "a"}


def test_disabled_counts_and_captures_nothing():
    cache, toy, x = GraphCache(), Toy(), _x(6)
    for n in (1, 2, 3):
        assert torch.equal(cache("k", False, toy, x), _ref(x))
        assert cache.calls["k"] == n and not cache.captured
    assert toy.calls == 3 and int(toy.runs) == 3
    got = cache("k", True, toy, x)               # the key has run before: the first enabled call captures
    assert "k" in cache.captured and int(toy.runs) == 4 and torch.equal(got, _ref(x))
    cache.clear()
    assert not cache.calls and not cache.captured
