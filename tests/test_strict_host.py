"""CPU tier of strict legality: the product's per-lane attack test (csrc/cz_rules.cuh: attacked / in_check / move_is_strict),
compiled for the host, against the brute-force definition over the oracle's move generator (tests/strict_oracle.c); the host
side of cchess_main(strict=True) and the UCCI front-end's use of it over stand-in trees."""
import contextlib
import io
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import strict_support as S  # noqa: E402
from conftest import load_golden  # noqa: E402
from oracle import oracle as O  # noqa: E402

NAMES = ("moves", "counts", "legal mask", "flags")


def _agree(boards, sides):
    if S.host_lib() is None:
        pytest.skip("nvcc not available")
    want, got = S.oracle_strict(boards, sides), S.host_strict(boards, sides)
    for name, w, g in zip(NAMES, want, got):
        bad = np.nonzero((w != g).reshape(len(boards), -1).any(1))[0]
        assert len(bad) == 0, "%s differ on %d positions, first: %s side %d" % (name, len(bad), O.to_state(boards[bad[0]]), sides[bad[0]])
    return want


@pytest.fixture(scope="module")
def random_play():
    boards, sides = S.random_play(7, 200000)
    return boards, sides, _agree(boards, sides)


def test_golden_movegen_positions_for_both_sides():
    recs = load_golden("movegen.json.gz")["records"]
    boards = np.stack([O.from_state(r["state"]) for r in recs])
    _agree(np.concatenate([boards, boards]), np.concatenate([np.zeros(len(recs), np.uint8), np.ones(len(recs), np.uint8)]))


def test_random_play_positions(random_play):
    boards, sides, (mv, cnt, legal, flags) = random_play
    kingless = int(((boards == 1).sum(1) == 0).sum() + ((boards == 8).sum(1) == 0).sum())
    check, mated = int((flags & 1).sum()), int((flags & 2).sum())
    filtered = int((cnt - S.mask_bits(legal).sum(1)).astype(bool).sum())
    print("\n%d positions: %d in check, %d mated, %d with a king missing, %d with at least one move that is not strictly legal"
          % (len(boards), check, mated, kingless, filtered))
    assert check > 0 and mated > 0 and kingless > 0 and filtered > check


def test_set_up_boards():
    boards, sides = S.setup_boards()
    mv, cnt, legal, flags = _agree(boards, sides)
    assert (flags & 1).sum() > 0 and ((flags & 3) == 3).sum() > 0 and ((flags & 3) == 2).sum() > 0


def test_hand_made_positions():
    boards, sides = S.hand_made_boards()
    S.check_hand_made(*S.oracle_strict(boards, sides))
    if S.host_lib() is not None:
        S.check_hand_made(*S.host_strict(boards, sides))


def test_output_properties(random_play):
    boards, sides, (mv, cnt, legal, flags) = random_play
    ok = S.mask_bits(legal)
    assert not (ok & (np.arange(128)[None, :] >= cnt[:, None])).any()                 # no bit at or above the count
    assert np.array_equal((flags & 2) != 0, ~ok.any(1))                               # mated <=> empty mask
    assert not (mv * (np.arange(128)[None, :] >= cnt[:, None])).any()
    for g in range(0, len(boards), 997):                                              # the list is the pseudo-legal list
        assert np.array_equal(mv[g, :cnt[g]], O.legal_moves(boards[g], int(sides[g])))


# ---- cchess_main(strict=True) and UCCI over stand-in trees ----------------------------------------------------------------

class _Node:
    def __init__(self, N, P, Q=0.0):
        self.N, self.P, self.Q = N, P, Q


class _FixedTree:
    """MCTS_tree's surface with a root that holds given visit counts and priors for the position's pseudo-legal moves."""

    def __init__(self, state, player, visits=None, priors=None):
        moves = [O.move_str(m) for m in O.legal_moves(O.from_state(state), 0 if player == "w" else 1)]
        visits, priors = visits or {}, priors or {}
        self.root = type("R", (), {})()
        self.root.child = OrderedDict((m, _Node(visits.get(m, 0), priors.get(m, 0.0))) for m in moves)
        self.played = []

    def main(self, state, player, rr, playouts):
        pass

    def Q(self, move):
        return self.root.child[move].Q

    def update_tree(self, act):
        self.played.append(act)

    def _set_position(self, state, player, rr):
        pass


def _strict_main():
    from cchess_zero_b200.selfplay import cchess_main

    class StrictOnOracle(cchess_main):
        """cchess_main's own get_action / check_end / human_move text; only the device query is answered by the oracle."""
        strict = True

        def _strict_position(self):
            gb = self.game_borad
            mv, cnt, legal, fl = S.oracle_strict(O.from_state(gb.state)[None], [0 if gb.current_player == "w" else 1])
            return [O.move_str(m) for m in mv[0, :cnt[0]]], S.mask_bits(legal)[0, :cnt[0]], bool(fl[0] & 1), bool(fl[0] & 2)
    return StrictOnOracle


def _main_on(state, player, visits=None, priors=None, exploration=False):
    class GB:
        pass
    d = _strict_main().__new__(_strict_main())
    d.game_borad = GB()
    d.game_borad.state, d.game_borad.current_player, d.game_borad.restrict_round, d.game_borad.round = state, player, 0, 1
    d.mcts = _FixedTree(state, player, visits, priors)
    d.playout_counts, d.exploration, d.temperature, d.human_color = 10, exploration, 1, "b"
    return d


PIN = "4K4/9/9/9/4R4/9/9/9/9/4k4"          # the rook on e4 is pinned to the file by the facing kings


def test_get_action_never_plays_a_move_that_is_not_strictly_legal():
    np.random.seed(0)
    d = _main_on(PIN, "w", visits={"e4d4": 50, "e4a4": 9, "e4e6": 3, "e0d0": 1})
    act, move_probs, _ = d.get_action(PIN, 1)
    actions, probs = move_probs[0]
    p = dict(zip(actions, probs))
    assert act in ("e4e6", "e0d0") and p["e4d4"] == 0 and p["e4a4"] == 0
    assert abs(p["e4e6"] - 0.75) < 1e-12 and abs(p["e0d0"] - 0.25) < 1e-12 and abs(sum(probs) - 1) < 1e-12
    assert d.mcts.played == [act]
    # a banned move is filtered the same way
    d = _main_on(PIN, "w", visits={"e4d4": 50, "e4e6": 30, "e0d0": 1})
    d.banned_moves = ("e4e6",)
    assert d.get_action(PIN, 1e-3)[0] == "e0d0"
    # Dirichlet noise does not revive a filtered move
    d = _main_on(PIN, "w", visits={"e4d4": 50, "e4e6": 3}, exploration=True)
    assert {d.get_action(PIN, 1)[0] for _ in range(200)} == {"e4e6"}


def test_get_action_falls_back_to_the_largest_prior_among_playable_moves():
    d = _main_on(PIN, "w", visits={"e4d4": 50, "e4a4": 9}, priors={"e4d4": 0.9, "e0f0": 0.04, "e4e7": 0.04, "e4e1": 0.01})
    act, move_probs, _ = d.get_action(PIN, 1e-3)
    assert act == "e0f0"                                  # first maximum in move order among the strictly legal moves
    assert dict(zip(*move_probs[0]))["e0f0"] == 1.0 and sum(move_probs[0][1]) == 1.0
    d = _main_on(PIN, "w", visits={"e4d4": 5}, priors={"e0f0": 0.04})
    d.banned_moves = [m for m in d.mcts.root.child if m != "e4d4"]
    with pytest.raises(ValueError):
        d.get_action(PIN, 1e-3)


def test_check_end_reports_mate_and_human_move_refuses_self_check():
    by_name = {h[0]: h for h in S.HAND_MADE}
    with contextlib.redirect_stdout(io.StringIO()):
        assert _main_on(by_name["checkmate"][1], "w").check_end() == (True, "b")
        assert _main_on(by_name["stalemate"][1], "w").check_end() == (True, "b")
        assert _main_on(by_name["king_step_check_inside_the_attackers_palace"][1], "w").check_end() == (True, "b")
        assert _main_on(PIN, "w").check_end() == (False, "")
    d = _main_on(PIN, "w")
    with pytest.raises(ValueError):
        d.human_move((4, 4, 3, 4), "net")                 # e4d4 uncovers the king
    assert d.game_borad.state == PIN and d.game_borad.round == 1 and d.mcts.played == []


def _say(eng, *lines):
    eng.out = io.StringIO()
    with contextlib.redirect_stdout(io.StringIO()):
        for ln in lines:
            assert eng.handle(ln)
    return eng.out.getvalue().splitlines()


def _ucci_engine(visits=None):
    from cchess_zero_b200 import ucci
    made = []

    def make(options):
        d = _main_on(O.START, "w")
        tree = d.mcts

        def set_position(state, player, rr):              # a fresh root for the commanded position
            t = _FixedTree(state, player, visits)
            tree.root, tree.played = t.root, []
        tree._set_position = set_position
        made.append(d)
        return d
    return ucci.UcciEngine(make, playouts=10, legal_moves=S.strict_labels), made


def test_ucci_refuses_an_illegal_move_list_and_keeps_the_position():
    from cchess_zero_b200 import ucci
    eng, _ = _ucci_engine()
    fen = ucci.state_to_fen(PIN, "w")
    _say(eng, "position fen " + fen + " moves e4e5")
    before = _say(eng, "probe")
    assert _say(eng, "position fen " + fen + " moves e4d4") == ["info string error illegal move e4d4 (move 1)"]        # uncovers the king
    assert _say(eng, "position fen " + fen + " moves e0d0 e9d9") == ["info string error illegal move e9d9 (move 2)"]   # faces the king
    assert _say(eng, "position startpos moves h2e2 a5a6") == ["info string error illegal move a5a6 (move 2)"]               # empty square
    assert _say(eng, "position startpos moves b0b2") == ["info string error illegal move b0b2 (move 1)"]                    # not a knight move
    assert _say(eng, "probe") == before
    assert _say(eng, "position startpos moves h2e2 h9g7") == []


def test_ucci_banmoves_reach_the_driver_and_position_clears_them():
    from cchess_zero_b200 import ucci
    eng, made = _ucci_engine(visits={"e4e6": 30, "e0d0": 2})
    fen = ucci.state_to_fen(PIN, "w")
    out = _say(eng, "position fen " + fen, "banmoves e4e6 e4e7", "go")
    assert out[-1] == "bestmove e0d0" and made[0].banned_moves == ("e4e6", "e4e7")
    out = _say(eng, "position fen " + fen, "go")
    assert out[-1] == "bestmove e4e6" and made[0].banned_moves == ()
    assert "error" in _say(eng, "banmoves e4")[0]


def test_ucci_answers_nobestmove_when_mated():
    from cchess_zero_b200 import ucci
    eng, _ = _ucci_engine()
    mate = {h[0]: h for h in S.HAND_MADE}["checkmate"][1]
    out = _say(eng, "position fen " + ucci.state_to_fen(mate, "w"), "go")
    assert out == ["info string game over (b)", "nobestmove"]
