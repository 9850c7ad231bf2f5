"""The strict-rules search on the CPU: the specification (tests/strict_search_oracle.c) against the brute-force strict legality,
hand-made mates in one, the format 2 snapshot checks of cz_snapshot_check, and the host side of SelfPlay / Match / Trainer under
strict rules on stand-in engines built over the specification trees."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import strict_search_support as S  # noqa: E402
from strict_support import mask_bits, oracle_strict, random_play, setup_boards  # noqa: E402
from test_snapshot_host import F_CUR, NONE, blob, block, check, game, mv, tree  # noqa: E402


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _children(board, side):
    """The spec's children of a position: its root expansion (a search of 0 playouts).  Set-up boards may hold moves without a label
    (error 2) or more than 128 pseudo-legal moves (error 16), as on the device."""
    t = S.StrictTree(board)
    assert t.search(side, 0, 0, "hash_pos") & ~(2 | 16) == 0
    return t.root_children()[0], t


@pytest.mark.parametrize("source", ["random_play", "setup"])
def test_children_are_the_strictly_legal_subset_of_the_pseudo_legal_list(source):
    if source == "random_play":
        boards, sides = random_play(31, 20000)
        boards, sides = boards[::10], sides[::10]
    else:
        boards, sides = setup_boards()
        boards, sides = boards[::15], sides[::15]
    mvs, cnt, legal, flags = oracle_strict(boards, sides)
    ok = mask_bits(legal)
    mated = 0
    for i in range(len(boards)):
        kids, t = _children(boards[i], int(sides[i]))
        n = min(int(cnt[i]), 128)
        want = mvs[i, :n][ok[i, :n]]
        assert np.array_equal(kids, want), i
        assert t.root_mated() == (len(want) == 0) == bool(flags[i] & 2), i
        mated += len(want) == 0
        if len(want):                       # priors: serial f32 sum seeded with 1e-8 over the strict children only
            p = t.root_children()[3]
            assert p.dtype == np.float32 and len(p) == len(want)
    assert mated > 0


def test_hand_made_mates_in_one(O):
    for name, state, side, mate, stalemate in S.MATE_IN_ONE:
        b, s = O.from_state(state), 0 if side == "w" else 1
        nb, _ = O.apply_move(b, O.move_from_str(mate))
        assert len(S.strict_moves(nb, s ^ 1)) == 0 and S.in_check(nb, s ^ 1) == (not stalemate), name
        assert mate in [O.move_str(x) for x in S.strict_moves(b, s)], name
        for net in S.NETS:
            t = S.StrictTree(b)
            assert t.search(s, 0, 200, net) == 0
            m, N, W, P, Q = t.root_children()
            sig = t.signature()
            labels = [O.move_str(x) for x in m]
            rec = _root_records(sig)
            found = 0
            for i in range(len(m)):
                child, _ = O.apply_move(b, int(m[i]))
                if N[i] and len(S.strict_moves(child, s ^ 1)) == 0:
                    # every playout through a mating move ends there worth exactly +1 (checkmate and stalemate alike)
                    assert Q[i] == np.float32(1.0) and W[i] == np.float32(N[i]), (name, net, labels[i])
                    r = sig[rec[i]]
                    assert r[5] == -1 and r[4] == np.float32(1.0).view(np.uint32) and r[1] == N[i], (name, net, labels[i])
                    assert S.game_end(child, s ^ 1, 0) == (3, s), name
                    found += 1
            # hash_pos priors are all positive, so every root child is tried; the signed nets may leave a mate unvisited
            assert found or net != "hash_pos", (name, net)


def _root_records(sig):
    """indices of the root's children in a depth-first signature (each record is followed by its subtree)"""
    def skip(k, n):
        for _ in range(n):
            c = int(sig[k, 5])
            k = skip(k + 1, c) if c > 0 else k + 1
        return k
    out, k = [], 0
    while k < len(sig):
        out.append(k)
        c = int(sig[k, 5])
        k = skip(k + 1, c) if c > 0 else k + 1
    return out


def test_mated_root_has_no_search(O):
    for name, state, side, mate, _ in S.MATE_IN_ONE:
        b, s = O.from_state(state), 0 if side == "w" else 1
        nb, _ = O.apply_move(b, O.move_from_str(mate))
        t = S.StrictTree(nb)
        assert t.search(s ^ 1, 0, 100, "hash_pos") == 0
        st = t.stats()
        assert t.root_mated() and st["n_expand"] == 1 and st["n_playout"] == 0 and st["sum_C"] == 0, name
        assert len(t.signature()) == 0 and len(t.root_children()[0]) == 0
        assert S.game_end(nb, s ^ 1, 0) == (3, s), name


def test_stalemate_loses():
    name, state, side, mate, stalemate = S.MATE_IN_ONE[1]
    from oracle import oracle as O
    b = O.from_state(state)
    nb, _ = O.apply_move(b, O.move_from_str(mate))
    assert stalemate and not S.in_check(nb, 0)
    end, winner = S.game_end(nb, 0, 0)
    assert (end, winner) == (3, 1)                                   # red has no move: black, who just moved, wins


# ---- snapshots: format 2 --------------------------------------------------------------------------------------------------------
def _strict(b):
    """a blob built by tests/test_snapshot_host.blob, marked format 2 (strict rules)"""
    b.view(np.uint64)[1] = 2 | (2 << 32)
    return b


def check_strict(b, B=1, K=1, narr=5, arena_words=1 << 16):
    """cz_snapshot_check_rules for a strict-rules engine -> (rc, message)"""
    import ctypes as C
    from cchess_zero_b200._lib import lib
    L = lib()
    rc = L.cz_snapshot_check_rules(b.ctypes.data_as(C.c_void_p), b.nbytes, B, K, narr, arena_words, 1)
    return rc, L.cz_last_error().decode() if rc else ""


def _mated_tree():
    """root (3 children) at 0: child 0 -> block A (2) at 48, child 1 -> a mated node (8-word block M at 96); alloc 104"""
    k = 48
    root = block([mv(1, 20), mv(7, 24), mv(64, 67)], [0, 0, NONE], [2, 0, 0])
    a = block([mv(81, 63), mv(83, 75)])
    m = np.zeros(8, np.uint32)
    root[8 + 4 * 8 + 0], root[8 + 4 * 8 + 1] = k, 2 * k
    return np.concatenate([root, a, m]), dict(root=0, A=k, M=2 * k)


def test_format_2_blob_with_mated_nodes_and_terminal_3_passes():
    ar, _ = _mated_tree()
    assert check_strict(_strict(blob([game(ar)]))) == (0, "")
    g = game(np.zeros(8, np.uint32), rootcnt=0, flags=F_CUR | (3 << 8) | (2 << 10))      # a mated root, won by black
    assert check_strict(_strict(blob([g]))) == (0, "")
    plain, _ = tree()
    assert check_strict(_strict(blob([game(plain)]))) == (0, "")                          # a strict engine's tree without mates


def test_format_2_refusals_each_with_its_own_message():
    msgs = {}
    ar, base = _mated_tree()
    # a format 1 blob (reference rules) with a mated node: what a strict engine wrote, relabelled
    rc, msgs["count-0 block in format 1"] = check(blob([game(ar)]))
    assert rc == -1
    longer = np.concatenate([ar, np.zeros(8, np.uint32)])             # 8 words after the mated block that no block covers
    rc, msgs["count-0 block longer than 8 words"] = check_strict(_strict(blob([game(longer)])))
    assert rc == -1
    plain, _ = tree()
    rc, msgs["terminal 3 in format 1"] = check(blob([game(plain, flags=F_CUR | (3 << 8) | (1 << 10))]))
    assert rc == -1
    rc, msgs["rules mismatch (strict blob, reference engine)"] = check(_strict(blob([game(ar)])))
    assert rc == -1
    rc, msgs["rules mismatch (reference blob, strict engine)"] = check_strict(blob([game(plain)]))
    assert rc == -1
    c = _strict(blob([game(plain)]))
    c.view(np.uint64)[1] += 1
    rc, msgs["format 3"] = check_strict(c)
    assert rc == -1
    want = {"count-0 block in format 1": "n_grandchildren 0", "count-0 block longer than 8 words": "count-0 block longer",
            "terminal 3 in format 1": "terminal code 3", "rules mismatch (strict blob, reference engine)": "rules differ",
            "rules mismatch (reference blob, strict engine)": "rules differ", "format 3": "unsupported format version"}
    for k, w in want.items():
        assert w in msgs[k], (k, msgs[k])
    texts = list(msgs.values())
    assert len(set(texts)) == len(texts), "two checks share a message"
    # format 1 validation is unchanged: the existing valid blob still passes, and a mated root count 0 is not looked at there
    assert check(blob([game(plain)]))[0] == 0
    assert check(blob([game(np.zeros(0, np.uint32), rootcnt=0, flags=F_CUR)]))[0] == 0


# ---- the host side of SelfPlay, Match and Trainer under strict rules ------------------------------------------------------------
class StrictStandIn:
    """Engine-interface stand-in over the specification trees, with strict rules: a new root without a strictly legal move ends the
    game with terminal code 3 (the winner is the side that just moved).  Test infrastructure only."""
    torch_device = "cpu"
    rules = "strict"

    def __init__(self, n, net):
        from oracle import oracle as O
        self.O, self.B, self.net, self.device, self.launches = O, n, net, 0, 0
        self.boards = np.tile(O.from_state(O.START), (n, 1))
        self.trees = [S.StrictTree(self.boards[g]) for g in range(n)]
        self.side = np.zeros(n, np.uint8); self.rr = np.zeros(n, np.int32); self.ply = np.zeros(n, np.int32)
        self.terminal = np.zeros(n, np.uint8); self.winner = -np.ones(n, np.int8)
        self.target = np.zeros(n, np.int64); self.pending = np.zeros(n, bool)

    def reset(self, mask=None, boards=None, sides=None, rr=None):
        for g in range(self.B):
            if mask is None or mask[g]:
                self.boards[g] = self.O.from_state(self.O.START) if boards is None else boards[g]
                self.side[g] = 0 if sides is None else sides[g]
                self.rr[g] = 0 if rr is None else rr[g]
                self.trees[g] = S.StrictTree(self.boards[g])
                self.ply[g] = 0; self.terminal[g] = 0; self.winner[g] = -1
                self._mate(g)

    def _mate(self, g):
        if self.terminal[g] == 0 and len(S.strict_moves(self.boards[g], int(self.side[g]))) == 0:
            self.terminal[g], self.winner[g] = 3, self.side[g] ^ 1

    def begin_search(self, playouts, mask=None):
        for g in range(self.B):
            if (mask[g] if mask is not None else not self.terminal[g]):
                self.target[g] = playouts; self.pending[g] = True

    def wave(self, nn_in, logits, value):
        for g in np.nonzero(self.pending)[0]:
            assert self.trees[g].search(int(self.side[g]), int(self.rr[g]), int(self.target[g]), self.net) == 0
        self.pending[:] = False

    def unfinished(self):
        return int(self.pending.sum())

    def root_children(self, want_wpq=True):
        n = np.zeros(self.B, np.int32); m = np.zeros((self.B, 128), np.uint16); v = np.zeros((self.B, 128), np.int32)
        for g, t in enumerate(self.trees):
            a, N = t.root_children()[:2]
            n[g] = len(a); m[g, :len(a)] = a; v[g, :len(a)] = N
        return dict(n=n, moves=m, visits=v, w=None, p=None, q=None)

    def _advance(self, g, move):
        self.boards[g], cap = self.O.apply_move(self.boards[g], int(move))
        self.side[g] ^= 1; self.rr[g] = self.rr[g] + 1 if cap == 0 else 0; self.ply[g] += 1
        if cap == 1: self.terminal[g], self.winner[g] = 1, 1
        elif cap == 8: self.terminal[g], self.winner[g] = 1, 0
        elif self.rr[g] >= 60: self.terminal[g] = 2
        self._mate(g)

    def play(self, choice, want_status=True):
        for g, c in enumerate(choice):
            if c >= 0:
                move = self.trees[g].root_children()[0][c]
                self.trees[g].update(int(c))
                self._advance(g, move)
        return self.status()

    def play_moves(self, moves, want_status=True):
        for g, m in enumerate(moves):
            if m == 0xFFFF:
                continue
            kids = list(self.trees[g].root_children()[0])
            assert self.terminal[g] == 0 and int(m) in [int(x) for x in S.strict_moves(self.boards[g], int(self.side[g]))]
            if kids:
                self.trees[g].update(kids.index(m))
                self._advance(g, m)
            else:
                self._advance(g, m)
                self.trees[g] = S.StrictTree(self.boards[g])
        return self.status()

    def status(self, boards=True):
        return dict(terminal=self.terminal.copy(), winner=self.winner.copy(), ply=self.ply.copy(), rr=self.rr.copy(),
                    side=self.side.copy(), boards=self.boards.copy(), q=np.zeros(self.B, np.float32))

    def counters(self):
        return dict(error=0)

    def raise_on_error(self):
        return self.counters()

    def tree_signature(self, g):
        return self.trees[g].signature()


def test_selfplay_host_loop_ends_mated_games_with_the_winners_z():
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net = 4, 24, "hash_pos"
    sp = SelfPlay(B, lambda x: None, P, seeds=[500 + g for g in range(B)], auto_reset=False, engine=StrictStandIn(B, net), rules="strict")
    with np.errstate(all="ignore"):
        out = sp.play_games()
    ends = []
    for slot, rec in out:
        with np.errstate(all="ignore"):
            r = S.selfplay_game(net, P, np.random.RandomState(500 + slot))
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot
        ends.append(r["end"])
        if r["end"] == 3:
            assert rec.winner == "wb"[r["players"][-1]] and rec.z[-1] == 1.0
    assert 3 in ends, ends


def test_match_host_loop_counts_a_mate_as_a_win(monkeypatch):
    import cchess_zero_b200.arena as A
    from cchess_zero_b200.selfplay import SelfPlay
    nets = {"a": "hash_signed", "b": "mod17"}

    class SP(SelfPlay):
        def __init__(self, n, evaluator, playouts, **kw):
            super().__init__(n, lambda x: None, playouts, engine=StrictStandIn(n, nets[evaluator]), **kw)

        def capture_graph(self, warmup=3):
            pass
    monkeypatch.setattr(A, "SelfPlay", SP)
    n, P, T0, plies0 = 4, 16, 1.0, 6
    m = A.Match("a", "b", n, P, seeds=range(n), opening_temperature=T0, opening_plies=plies0, max_plies=400, rules="strict")
    with np.errstate(all="ignore"):
        r = m.run()
    ends = []
    for g in range(n):
        red, black = ("hash_signed", "mod17") if g < n // 2 else ("mod17", "hash_signed")
        with np.errstate(all="ignore"):
            o = S.match_game(red, black, P, np.random.RandomState(g), plies0, T0, 1e-3, max_plies=400)
        rec = r.games[g]
        assert rec["moves"] == o["moves"] and rec["winner"] == "wbt"[o["winner"]] and rec["plies"] == o["plies"], g
        ends.append(o["end"])
        if o["end"] == 3:
            cc = 0 if g < n // 2 else 1
            assert rec["result"] == ("win" if o["winner"] == cc else "loss")
    assert 3 in ends, ends


def test_strict_match_ends_a_mated_opening_before_its_first_ply(monkeypatch):
    import cchess_zero_b200.arena as A
    from cchess_zero_b200.selfplay import SelfPlay
    from oracle import oracle as O

    class SP(SelfPlay):
        def __init__(self, n, evaluator, playouts, **kw):
            super().__init__(n, lambda x: None, playouts, engine=StrictStandIn(n, evaluator), **kw)

        def capture_graph(self, warmup=3):
            pass
    monkeypatch.setattr(A, "SelfPlay", SP)
    name, state, side, mate, _ = S.MATE_IN_ONE[0]
    mated, _ = O.apply_move(O.from_state(state), O.move_from_str(mate))            # red to move, checkmated
    openings = (np.stack([mated, O.from_state(O.START)]), np.array([0, 0], np.uint8), np.array([0, 0], np.int32))
    m = A.Match("hash_pos", "mod17", 4, 8, seeds=range(4), openings=openings, max_plies=4, rules="strict")
    assert list(m.live) == [False, True, False, True]
    with np.errstate(all="ignore"):
        r = m.run()
    for g, result in ((0, "loss"), (2, "win")):                     # the candidate is red in game 0, black in game 2
        assert r.games[g]["plies"] == 0 and r.games[g]["winner"] == "b" and r.games[g]["result"] == result, g
    assert r.games[1]["plies"] == r.games[3]["plies"] == 4


def test_rules_argument_is_validated():
    from cchess_zero_b200.arena import Match, random_openings
    from cchess_zero_b200.engine import Engine, check_rules
    from cchess_zero_b200.selfplay import SelfPlay
    from cchess_zero_b200.train import Trainer
    assert check_rules("reference", 16) == "reference" and check_rules("strict") == "strict"
    for bad in ("Strict", "full", None, 1):
        with pytest.raises(ValueError, match="rules must be"):
            check_rules(bad)
    with pytest.raises(ValueError, match="one-leaf engine"):
        SelfPlay(2, lambda x: None, 8, search_threads=16, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(2, leaves=4, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(2, search_threads=16, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(2, search_threads=1, rules="strict")        # search_threads = 1 still builds the FIFO engine
    with pytest.raises(ValueError, match="rules must be"):
        Engine(2, rules="chess")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Match(None, None, 2, 8, search_threads=16, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Trainer(None, 2, 8, search_threads=16, rules="strict")
    with pytest.raises(ValueError, match="rules must be"):
        random_openings(2, 2, rules="xiangqi")
    with pytest.raises(ValueError, match="plays by the 'strict' rules"):
        SelfPlay(2, lambda x: None, 8, engine=StrictStandIn(2, "hash_pos"))


def test_trainer_refuses_a_saved_run_of_other_rules(tmp_path):
    from cchess_zero_b200.train import Trainer, _savez

    class SP:
        _mt = np.zeros((2, 626), np.uint32)
    t = Trainer.__new__(Trainer)
    t.sp, t.n_games, t.rules = SP(), 2, "reference"
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt, rules=np.asarray("strict"))
    with pytest.raises(ValueError, match="'strict' rules, this Trainer by 'reference'"):
        t.load(str(tmp_path))
    t.rules = "strict"
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt)                 # saved before the rules choice existed: reference rules
    with pytest.raises(ValueError, match="'reference' rules, this Trainer by 'strict'"):
        t.load(str(tmp_path))
