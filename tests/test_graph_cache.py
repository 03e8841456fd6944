"""The CUDA-graph cache shared by the fused training step and the no-grad forward (mmdit_base.GraphCache), on the CPU: torch.cuda's
graph API is replaced by stand-ins, so the warm-up / capture / replay / eviction / re-recording / failure bookkeeping runs without a GPU."""
import contextlib
import warnings

import pytest
import torch

from qflux_b200 import lib
from qflux_b200.mmdit_base import GraphCache


class FakeGraph:
    """torch.cuda.CUDAGraph stand-in: counts replays."""

    def __init__(self):
        self.replays = 0

    def replay(self):
        self.replays += 1


class FakeModel:
    """What the cache reads of a fused model: its device, whether its weights are sharded, its current workspace, and whether it
    still holds a workspace a graph was recorded on."""

    def __init__(self):
        self.dev, self._sharded, self._fwd_gen, self.held = torch.device("cuda"), None, 0, []
        self.switch_ws("ws0")

    def switch_ws(self, key):  # a forward of another shape: the model builds and activates another workspace
        self._ws, self._ws_key = dict(rope=torch.zeros(1), kv_len=None), key
        self.held.append(self._ws)

    def _activate_ws(self, ws, key):
        if any(w is ws for w in self.held):
            self._ws, self._ws_key = ws, key
            return True
        return False


class LaunchSequence:
    """The function under the cache: three launches that scale the input; `fail_capture` makes it fail inside a capture."""

    def __init__(self, cuda):
        self.cuda, self.calls, self.fail_capture = cuda, [], False

    def __call__(self, x, k):
        lib.LAUNCHES += 3
        if self.cuda["capturing"] and self.fail_capture:
            raise RuntimeError("operation not permitted when stream is capturing")
        self.calls.append("capture" if self.cuda["capturing"] else "eager")
        return x * k


@pytest.fixture
def cuda(monkeypatch):
    state = dict(capturing=False, captures=0)

    @contextlib.contextmanager
    def graph(g):
        state["capturing"], state["captures"] = True, state["captures"] + 1
        try:
            yield
        finally:
            state["capturing"] = False

    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", graph)
    monkeypatch.setattr(lib, "LAUNCHES", 0)
    return state


def test_first_sighting_runs_eagerly_and_the_second_captures(cuda):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    x = torch.ones(2)
    assert torch.equal(cache.run(m, fn, (x, 2.0)), x * 2)
    assert fn.calls == ["eager"] and cache.captured() == 0
    out = cache.run(m, fn, (x * 3, 2.0))
    assert fn.calls == ["eager", "capture"] and cache.captured() == 1
    ent = next(iter(cache.entries.values()))
    assert ent["graph"].replays == 1 and ent["static"][0] is not x and out is ent["out"]
    assert ent["ws"] is m._ws and ent["keep"][0] is m._ws["rope"]  # the per-shape tables stay alive with the graph
    cache.run(m, fn, (x, 2.0), tag=True)  # another key (an accumulating micro-step): warmed up on its own
    assert fn.calls == ["eager", "capture", "eager"] and len(cache.entries) == 2


def test_replay_copies_new_inputs_into_the_static_buffers(cuda):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    for _ in range(2):
        cache.run(m, fn, (torch.ones(2), 2.0))
    ent = next(iter(cache.entries.values()))
    y = torch.tensor([5.0, 7.0])
    gen = m._fwd_gen
    assert cache.run(m, fn, (y, 2.0)) is ent["out"]
    assert torch.equal(ent["static"][0], y) and ent["graph"].replays == 2
    assert fn.calls == ["eager", "capture"]  # nothing re-issued
    assert m._fwd_gen == gen + 1             # a replay is a forward: autograd nodes of older forwards must refuse to run


def test_least_recently_used_graph_is_evicted_at_capacity(cuda):
    cache, m, fn = GraphCache(2, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    a, b, c = (torch.ones(n) for n in (1, 2, 3))  # three input signatures
    cache.run(m, fn, (a, 1.0))
    cache.run(m, fn, (b, 1.0))
    cache.run(m, fn, (a, 1.0))  # captures a: a is now the most recently used
    cache.run(m, fn, (c, 1.0))  # full: b goes
    assert len(cache.entries) == 2 and cache.captured() == 1
    cache.run(m, fn, (a, 1.0))  # still captured: replays
    cache.run(m, fn, (b, 1.0))  # evicted: a first sighting again (c goes)
    assert fn.calls == ["eager", "eager", "capture", "eager", "eager"]
    cache.run(m, fn, (a, 1.0))
    assert len(fn.calls) == 5 and cache.captured() == 1 and len(cache.entries) == 2


def test_graph_is_recorded_again_after_its_workspace_was_dropped(cuda):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    x = torch.ones(2)
    for _ in range(2):
        cache.run(m, fn, (x, 2.0))
    ws0 = m._ws
    m.switch_ws("ws1")  # the model still holds ws0: replay re-activates it
    cache.run(m, fn, (x, 2.0))
    assert fn.calls == ["eager", "capture"] and m._ws is ws0
    m.held.clear()
    m.switch_ws("ws2")  # ws0 is gone: record again, on the current workspace
    cache.run(m, fn, (x, 2.0))
    ent = next(iter(cache.entries.values()))
    assert fn.calls == ["eager", "capture", "capture"] and ent["ws"] is m._ws and ent["ws_key"] == "ws2"
    assert ent["graph"].replays == 1


def test_failed_capture_warns_once_and_stays_eager(cuda):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    fn.fail_capture = True
    x = torch.ones(2)
    cache.run(m, fn, (x, 2.0))
    with pytest.warns(UserWarning, match="CUDA-graph capture of the test sequence failed"):
        out = cache.run(m, fn, (x, 2.0))
    assert torch.equal(out, x * 2) and fn.calls == ["eager", "eager"] and cache.failed
    assert lib.LAUNCHES == 6  # the launches of the failed capture are not counted
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        for k in (2.0, 2.0, 4.0, 4.0):
            cache.run(m, fn, (x, k))
    assert fn.calls == ["eager"] * 6 and cuda["captures"] == 1 and cache.captured() == 0


def test_launch_counter_advances_by_the_captured_count_per_replay(cuda):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    x = torch.ones(2)
    cache.run(m, fn, (x, 2.0))
    assert lib.LAUNCHES == 3
    cache.run(m, fn, (x, 2.0))  # the capture launches nothing, its replay counts the recorded launches
    assert lib.LAUNCHES == 6 and next(iter(cache.entries.values()))["launches"] == 3
    for _ in range(3):
        cache.run(m, fn, (x, 2.0))
    assert lib.LAUNCHES == 15


@pytest.mark.parametrize("why", ["disabled", "sharded", "cpu"])
def test_eager_when_disabled_sharded_or_not_on_cuda(cuda, why):
    cache, m, fn = GraphCache(4, "the test sequence"), FakeModel(), LaunchSequence(cuda)
    if why == "sharded":
        m._sharded = object()
    if why == "cpu":
        m.dev = torch.device("cpu")
    for _ in range(3):
        cache.run(m, fn, (torch.ones(2), 2.0), enabled=why != "disabled")
    assert fn.calls == ["eager"] * 3 and cuda["captures"] == 0 and not cache.entries
