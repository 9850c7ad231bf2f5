"""CPU tier of the arena: match statistics (score, Elo, interval, gate), argument checks and the match oracle itself."""
import math

import numpy as np
import pytest

from cchess_zero_b200.arena import Match, MatchResult


def _result(w, d, l):
    games = []
    for i, r in enumerate(["win"] * w + ["draw"] * d + ["loss"] * l):
        games.append(dict(game=i, candidate_colour="wb"[i % 2], result=r))
    return MatchResult(games)


def test_elo_of_55_percent():
    r = _result(55, 0, 45)
    assert r.score == 0.55
    assert r.elo == pytest.approx(34.86, abs=0.01)            # -400 log10(1/0.55 - 1)
    lo, hi = r.elo_interval()
    # trinomial variance of the per-game score: 0.55 * 0.45 = 0.2475; standard error sqrt(0.2475 / 100) = 0.04975
    half = 1.959964 * math.sqrt(0.2475 / 100)
    assert lo == pytest.approx(-400 * math.log10(1 / (0.55 - half) - 1), rel=1e-12)
    assert hi == pytest.approx(-400 * math.log10(1 / (0.55 + half) - 1), rel=1e-12)
    assert lo < r.elo < hi
    assert r.promote() is False                               # 0.55 does not clear a gate of "more than 55 %"
    assert _result(56, 0, 44).promote() is True
    assert r.promote(0.5) is True


def test_all_draws_is_zero_elo_with_zero_width():
    r = _result(0, 40, 0)
    assert r.score == 0.5 and r.elo == 0.0
    assert r.elo_interval() == (0.0, 0.0)
    assert not r.promote()


def test_sweeps_are_infinite():
    assert _result(0, 0, 10).elo == -math.inf and _result(0, 0, 10).elo_interval() == (-math.inf, -math.inf)
    assert _result(10, 0, 0).elo == math.inf and _result(10, 0, 0).elo_interval() == (math.inf, math.inf)
    js = _result(10, 0, 0).to_json(games=False)
    assert '"elo": "inf"' in js and "Infinity" not in js


def test_totals_by_colour():
    r = _result(3, 2, 1)        # games alternate colours: w w b ... see _result
    assert (r.wins, r.draws, r.losses, r.n) == (3, 2, 1, 6)
    bc = r.by_colour
    assert sum(v["wins"] + v["draws"] + v["losses"] for v in bc.values()) == 6
    assert bc["w"]["wins"] + bc["b"]["wins"] == 3


@pytest.mark.parametrize("n", [0, 7, -2])
def test_match_rejects_odd_or_empty_game_counts(n):
    with pytest.raises(ValueError):
        Match(None, None, n, 10)


def test_match_oracle_is_deterministic_and_legal():
    from arena_oracle import match_game
    from oracle import oracle as O
    a = match_game("hash_signed", "mod17", 12, np.random.RandomState(3), 6, 1.0, 1e-3, max_plies=24, signatures=True)
    b = match_game("hash_signed", "mod17", 12, np.random.RandomState(3), 6, 1.0, 1e-3, max_plies=24, signatures=True)
    assert a["moves"] == b["moves"] and a["winner"] == b["winner"]
    assert all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a["sigs"], b["sigs"]))
    assert a["plies"] == len(a["moves"]) <= 24
    board, side = O.from_state(O.START), 0
    for mv in a["moves"]:
        assert mv in set(int(m) for m in O.legal_moves(board, side))
        board, _ = O.apply_move(board, mv)
        side ^= 1
