"""GPU tier of strict legality: k_strict_moves through the C ABI against the brute-force oracle, cchess_main(strict=True) on the
device engine with a network that wants a self-check move, and a UCCI session that starts in check."""
import contextlib
import ctypes as C
import io
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import strict_support as S  # noqa: E402
from oracle import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

PIN = "4K4/9/9/9/4R4/9/9/9/9/4k4"          # the rook on e4 is pinned to the file by the facing kings


def _device_strict(boards, sides):
    """cz_strict_moves_batch through rules.strict_moves_batch, back in the C layout's terms: (moves, counts, bool mask, flags)."""
    from cchess_zero_b200 import rules
    mv, cnt, legal, chk, mated = rules.strict_moves_batch(boards, sides)
    return mv, cnt, legal, chk.astype(np.uint8) | (mated.astype(np.uint8) << 1)


def test_kernel_matches_the_definition_and_the_pseudo_legal_kernel():
    from cchess_zero_b200 import rules
    rb, rs = S.random_play(11, 60000)
    sb, ss = S.setup_boards()
    hb, hs = S.hand_made_boards()
    boards, sides = np.concatenate([rb, sb, hb]), np.concatenate([rs, ss, hs])
    mv, cnt, legal, flags = _device_strict(boards, sides)
    omv, ocnt, olegal, oflags = S.oracle_strict(boards, sides)
    assert np.array_equal(mv, omv) and np.array_equal(cnt, ocnt)
    assert np.array_equal(legal, S.mask_bits(olegal)) and np.array_equal(flags, oflags)
    assert (oflags[:60000] & 1).sum() > 0 and (oflags[:60000] & 2).sum() > 0
    lmv, lcnt = rules.legal_moves_batch(boards, sides)
    assert np.array_equal(mv, lmv) and np.array_equal(cnt, lcnt)
    n = len(hb)
    packed = np.packbits(legal[-n:], axis=1, bitorder="little").view(np.uint32)
    S.check_hand_made(mv[-n:], cnt[-n:], packed, flags[-n:])


def test_argument_validation_and_boards_outside_the_input_domain():
    from cchess_zero_b200 import rules
    from cchess_zero_b200._lib import lib
    mv, cnt, legal, chk, mated = rules.strict_moves_batch(np.zeros((0, 90), np.uint8), np.zeros(0, np.uint8))
    assert mv.shape == (0, 128) and cnt.shape == (0,) and legal.shape == (0, 128) and chk.shape == (0,) and mated.shape == (0,)
    L = lib()
    assert L.cz_strict_moves_batch(0, None, None, 0, None, None, None, None) == 0
    assert L.cz_strict_moves_batch(0, None, None, 3, None, None, None, None) < 0 and b"null" in L.cz_last_error()
    b = np.zeros(90, np.uint8)
    assert L.cz_strict_moves_batch(0, b.ctypes.data_as(C.c_void_p), None, -1, None, None, None, None) < 0
    assert L.cz_version() == 2
    # piece codes above 14 are outside the input domain: whatever comes back, the call completes and the device is usable after it
    bad = np.random.RandomState(5).randint(0, 256, size=(64, 90)).astype(np.uint8)
    rules.strict_moves_batch(bad, np.zeros(64, np.uint8))
    hb, hs = S.hand_made_boards()
    S.check_hand_made(*S.oracle_strict(hb, hs))
    mv, cnt, legal, flags = _device_strict(hb, hs)
    S.check_hand_made(mv, cnt, np.packbits(legal, axis=1, bitorder="little").view(np.uint32), flags)


def test_gameboard_methods():
    from cchess_zero_b200.rules import GameBoard
    assert GameBoard.get_strict_moves(PIN, "w") == S.strict_labels(PIN, "w")
    assert GameBoard.get_strict_moves(O.START, "w") == GameBoard.get_legal_moves(O.START, "w")
    assert GameBoard.in_check(PIN, "b") and not GameBoard.in_check(PIN, "w")


# e0d0 walks into the rook on d7 and any sideways rook move uncovers the king; e0d0 is also the first move in generation order,
# which the reference's search visits first (its root has N = 0, so priors do not steer the first visits)
PLAY = "4K4/9/9/9/4R4/9/9/3r5/9/4k4"


class _Net:
    """policy_value_network stand-in: the given weight on each move label (Red to move, so no flip) and a constant value."""

    def __init__(self, weights, value):
        from cchess_zero_b200 import rules
        rules._init_tables()
        self.value = value
        self.row = np.full(2086, 1e-6, np.float32)
        for m, w in weights.items():
            self.row[rules.label2i[m]] = w

    def forward(self, x):
        n = np.asarray(x).shape[0]
        return np.tile(self.row, (n, 1)), np.full((n, 1), self.value, np.float32)


def _main(weights, value=0.0, strict=True, state=PLAY, playouts=40):
    from cchess_zero_b200.selfplay import cchess_main
    m = cchess_main(playout=playouts, in_search_threads=1, network=_Net(weights, value), exploration=False, log_file=False, strict=strict)
    m.game_borad.state = state
    m.mcts._set_position(state, "w", 0)
    return m


def test_strict_play_on_the_device_engine(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    legal = set(S.strict_labels(PLAY, "w"))
    assert "e0d0" not in legal and "e4d4" not in legal and "e4e9" in legal
    seen = []

    def spy(m):                                          # records the visit counts before and after the filter
        inner = m._strict_visits
        monkeypatch.setattr(m, "_strict_visits", lambda a, v: seen.append((dict(zip(a, v)), inner(a, v))) or seen[-1][1])
        return m
    with contextlib.redirect_stdout(io.StringIO()):
        np.random.seed(0)
        # all the network's weight on the self-check; a constant value spreads the visits over every move
        m = spy(_main({"e0d0": 1.0}, 0.5))
        act, move_probs, _ = m.get_action(PLAY, 1e-3)
        p = dict(zip(*move_probs[0]))
        assert seen[-1][0]["e0d0"] > 0 and seen[-1][0]["e4d4"] > 0          # the search did visit them
        assert act in legal and p["e0d0"] == 0.0 and p["e4d4"] == 0.0 and abs(sum(p.values()) - 1) < 1e-9
        # one playout: the only visit goes to e0d0, no legal child has one, so the largest prior among the legal moves decides
        m = spy(_main({"e0d0": 1.0, "e4e7": 0.05}, playouts=1))
        act, move_probs, _ = m.get_action(PLAY, 1e-3)
        assert seen[-1][0]["e0d0"] > 0 and not any(v for a, v in seen[-1][0].items() if a in legal) and sum(seen[-1][1]) == 1
        assert act == "e4e7" and dict(zip(*move_probs[0]))["e4e7"] == 1.0
        # a banned move is never played
        first = _main({"e0d0": 1.0}, 0.5).get_action(PLAY, 1e-3)[0]
        m = _main({"e0d0": 1.0}, 0.5)
        m.banned_moves = (first,)
        assert m.get_action(PLAY, 1e-3)[0] in legal - {first}
        # 'net' move choice takes its maximum over the playable moves
        m = _main({"e0d0": 1.0, "e4e7": 0.05, "e4e6": 0.04})
        m.banned_moves = ("e4e7",)
        m.select_move("net")
        assert m.game_borad.state == O.to_state(O.apply_move(O.from_state(PLAY), O.move_from_str("e4e6"))[0])
        # mate ends the game before any search; the reference's rules see no end
        mate = {h[0]: h for h in S.HAND_MADE}["checkmate"][1]
        assert _main({}, state=mate).check_end() == (True, "b")
        assert _main({}, strict=False, state=mate).check_end() == (False, "")
        # human_move refuses a self-check and leaves the board alone
        m = _main({})
        with pytest.raises(ValueError):
            m.human_move((4, 0, 3, 0), "mcts")
        assert m.game_borad.state == PLAY and m.game_borad.round == 1 and m.game_borad.current_player == "w"
        assert m.human_move((4, 4, 4, 5), "mcts") is not None and m.game_borad.current_player == "b"


def test_ucci_session_answers_a_check(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200 import ucci
    from cchess_zero_b200.rules import GameBoard
    from cchess_zero_b200.selfplay import cchess_main
    from oracle.fakenets_np import FAKE_NETS

    class Net:
        forward = staticmethod(FAKE_NETS["hash_signed"])

    def make(options):
        return cchess_main(playout=options["playouts"], in_search_threads=1, network=Net(), exploration=False, log_file=False, strict=True)

    def say(eng, *lines):
        eng.out = io.StringIO()
        with contextlib.redirect_stdout(io.StringIO()):
            for ln in lines:
                assert eng.handle(ln)
        return eng.out.getvalue().splitlines()

    np.random.seed(0)
    eng = ucci.UcciEngine(make, playouts=60, legal_moves=GameBoard.get_strict_moves)
    by_name = {h[0]: h for h in S.HAND_MADE}
    for name in ("cannon_check_answered_by_adding_a_screen", "double_check_only_a_king_move", "cannon_check_answered_by_removing_the_screen"):
        _, state, player, chk, _, good, _ = by_name[name]
        assert chk and GameBoard.in_check(state, player)
        out = say(eng, "position fen " + ucci.state_to_fen(state, player), "go")
        assert out[-1].startswith("bestmove ") and out[-1].split()[1] in good.split(), (name, out)
    fen = ucci.state_to_fen(PIN, "w")
    assert say(eng, "position fen " + fen + " moves e4d4") == ["info string error illegal move e4d4 (move 1)"]
    out = say(eng, "position fen " + fen, "banmoves " + " ".join(m for m in S.strict_labels(PIN, "w") if m != "e0e1"), "go nodes 30")
    assert out[-1] == "bestmove e0e1"
    out = say(eng, "position fen " + ucci.state_to_fen(by_name["checkmate"][1], "w"), "go")
    assert out[-1] == "nobestmove"
