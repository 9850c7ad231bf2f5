"""The wave loop every search runs (engine.run_waves), on the CPU: a recording stand-in engine logs each call, counts launches the way
Engine does and finishes its search after a scripted number of waves.  For every search path the exact call sequence, the wave count
and the launch count are pinned, and a search that never finishes raises EngineError on the first iteration past 4 * playouts + 64
waves.

Log tokens: R refresh_if_stale, B<p>:<mask> begin_search, W wave, C wave_compact, L live_rows, U unfinished, E<rows> an evaluation,
G a graph replay, X raise_on_error."""
import numpy as np
import pytest
import torch

from cchess_zero_b200._lib import EngineError
from cchess_zero_b200.engine import Engine


class _RecEngine:
    """Engine-interface stand-in: logs every call, counts launches like Engine, and reports its search finished once `finish` waves
    have run (never when finish is None).  live_rows returns live[wave - 1] (0 past the end of the script)."""
    torch_device = "cpu"
    search = Engine.search

    def __init__(self, B, finish=None, leaves=1, live=()):
        self.B, self.leaves, self.finish, self.live = B, leaves, finish, list(live)
        self.device, self.launches, self.waves, self.replaying, self.log = 0, 0, 0, False, []

    def begin_search(self, playouts, mask=None):
        self.launches += 1
        self.log.append("B%d:%s" % (playouts, "*" if mask is None else "".join(str(int(x)) for x in mask)))

    def wave(self, nn_in, logits, value):
        self.launches += not self.replaying          # a replayed launch is no Python call: the caller counts it
        self.waves += 1
        self.log.append("W")

    def wave_compact(self, nn_stage, nn_dense, logits, value):
        self.launches += 3
        self.waves += 1
        self.log.append("C")

    def live_rows(self):
        self.log.append("L")
        return self.live[self.waves - 1] if self.waves <= len(self.live) else 0

    def unfinished(self):
        self.launches += 1
        self.log.append("U")
        return 0 if self.finish is not None and self.waves >= self.finish else 1

    def raise_on_error(self):
        self.log.append("X")
        return dict(error=0)


class _RecPlan:
    def __init__(self, log):
        self.log = log

    def make_input(self, rows):
        return torch.zeros((rows, 9, 10, 14))

    def refresh_if_stale(self):
        self.log.append("R")

    def __call__(self, x, logits, value):
        self.log.append("E%d" % len(x))


class _RecGraph:
    """A captured graph of `waves` stand-in waves."""

    def __init__(self, engine, waves=1):
        self.engine, self.waves = engine, waves

    def replay(self):
        e = self.engine
        e.log.append("G")
        e.replaying = True
        for _ in range(self.waves):
            e.wave(None, None, None)
        e.replaying = False


def _engine_search(finish):
    e = _RecEngine(3, finish, leaves=2)
    nn = torch.zeros((6, 9, 10, 14))
    return e, lambda: e.search(lambda x: e.log.append("E%d" % len(x)), 6, nn, None, None, mask=[1, 0, 1])


def _selfplay(finish, K=1, graph=False, compact=False, live=()):
    from cchess_zero_b200.selfplay import SelfPlay
    e = _RecEngine(4, finish, live=live)
    sp = SelfPlay(4, None, [6, 3, 6, 3], engine=e, plan=_RecPlan(e.log), search_threads=K, compact=compact)
    if graph:
        sp.graph = _RecGraph(e)
    return e, lambda: sp.search([1, 1, 1, 0])


def _mcts_graph(finish):
    from cchess_zero_b200.mcts import MCTS_tree
    e = _RecEngine(1, finish)
    t = MCTS_tree.__new__(MCTS_tree)          # the device buffers and the capture are replaced by the stand-ins
    t.engine, t.K, t._reps, t._plan, t._graph = e, 1, 8, _RecPlan(e.log), _RecGraph(e, 8)
    t._nn_in = t._logits = t._value = None
    t._side, t._rr = 0, 0
    return e, lambda: t.main("RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr", "w", 0, 12)


PATHS = {
    "engine_search": _engine_search,
    "selfplay_eager": _selfplay,
    "selfplay_eager_k2": lambda f: _selfplay(f, K=2),
    "selfplay_graph": lambda f: _selfplay(f, graph=True),
    "mcts_graph": _mcts_graph,
    "compact": lambda f: _selfplay(f, K=2, compact=True, live=[5, 3, 0, 2, 0] if f else [2] * 1000),
}

FINISH = dict(engine_search=5, selfplay_eager=8, selfplay_eager_k2=5, selfplay_graph=8, mcts_graph=24, compact=5)

# (call sequence, waves returned, launches) of each path, recorded from the loops as they were before they were merged
EXPECTED = {
    "compact": ("R B3:0100 B6:1010 C L E8 C L E4 C L U C L E4 C L U", 5, 19),
    "engine_search": ("B6:101 W E6 W E6 W E6 W U E6 W U", 5, 8),
    "mcts_graph": ("R B12:* G W W W W W W W W G W W W W W W W W U G W W W W W W W W U X", None, 27),
    "selfplay_eager": ("R B3:0100 B6:1010 W E4 W E4 W E4 W E4 W E4 W E4 W U E4 W U", 8, 12),
    "selfplay_eager_k2": ("R B3:0100 B6:1010 W E8 W E8 W E8 W U E8 W U", 5, 9),
    "selfplay_graph": ("R B3:0100 B6:1010 G W G W G W G W G W G W G W U G W U", 8, 12),
}

# a search that never finishes: (waves run when EngineError is raised, the last log entries)
PMAX = dict(engine_search=6, selfplay_eager=6, selfplay_eager_k2=6, selfplay_graph=6, mcts_graph=12, compact=6)
EXPECTED_GUARD = {
    "compact": (89, "C L E4 X"),
    "engine_search": (89, "W U E6 X"),
    "mcts_graph": (120, "W W U X"),
    "selfplay_eager": (89, "W U E4 X"),
    "selfplay_eager_k2": (89, "W U E8 X"),
    "selfplay_graph": (89, "G W U X"),
}


@pytest.mark.parametrize("path", sorted(PATHS))
def test_search_call_sequence(path):
    e, run = PATHS[path](FINISH[path])
    waves = run()
    assert (" ".join(e.log), waves, e.launches) == EXPECTED[path]
    assert e.waves == FINISH[path]


@pytest.mark.parametrize("path", sorted(PATHS))
def test_search_that_never_finishes_raises(path):
    e, run = PATHS[path](None)
    with pytest.raises(EngineError, match="did not converge"):
        run()
    assert (e.waves, " ".join(e.log[-4:])) == EXPECTED_GUARD[path]
    bound = 4 * PMAX[path] + 64
    assert e.waves > bound and e.waves - (8 if path == "mcts_graph" else 1) <= bound


def test_two_lane_selfplay_is_refused():
    from cchess_zero_b200.selfplay import SelfPlay
    e = _RecEngine(4)
    with pytest.raises(ValueError):
        SelfPlay(4, None, 8, engine=e, plan=_RecPlan(e.log), lanes=2)
