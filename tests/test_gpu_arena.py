"""Arena on the device: Engine.play_moves (cz_engine_play_moves) and arena.Match, checked against Engine.play, the rules kernels and
the C oracle (tests/arena_oracle.py)."""
import contextlib
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NO_MOVE = 0xFFFF
ILLEGAL = 32


def _engine(B, K, arena_words=1 << 18):
    from cchess_zero_b200.engine import Engine
    return Engine(B, arena_words, 0, search_threads=K) if K > 1 else Engine(B, arena_words, 0)


def _search(e, net, playouts, mask=None):
    rows = e.rows
    nn_in = torch.zeros((rows, 9, 10, 14), device="cuda")
    lo = torch.zeros((rows, 2086), device="cuda")
    va = torch.zeros((rows,), device="cuda")

    def fwd(x):
        a, b = net(x)
        lo.copy_(a)
        va.copy_(b)
    e.search(fwd, playouts, nn_in, lo, va, mask=mask)


def _positions(n, seed):
    from cchess_zero_b200.arena import random_openings
    return random_openings(n, 8, seed)


def _status_equal(a, b):
    for k in ("boards", "side", "terminal", "winner", "ply", "rr", "root_N"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["q"].view(np.uint32), b["q"].view(np.uint32))


@pytest.mark.parametrize("K", [1, 16])
def test_play_moves_equals_play_by_index(K):
    from cchess_zero_b200.fakenet import FakeNet
    B, P = 64, 200
    net = FakeNet("hash_signed")
    boards, sides, rr = _positions(B, 11)
    e1, e2 = _engine(B, K), _engine(B, K)
    for e in (e1, e2):
        e.reset(None, boards, sides, rr)
        _search(e, net, P)
        e.raise_on_error()
    rc = e1.root_children()
    assert np.array_equal(rc["visits"], e2.root_children()["visits"])
    choice = np.zeros(B, dtype=np.int32)
    kinds = set()
    for g in range(B):
        n = int(rc["n"][g])
        vis = np.nonzero(rc["visits"][g, :n] > 0)[0]
        unv = np.nonzero(rc["visits"][g, :n] == 0)[0]
        if g % 3 == 1 and len(vis):
            choice[g] = vis[(g // 3) % len(vis)]
        elif g % 3 == 2 and len(unv):
            choice[g] = unv[(g // 3) % len(unv)]
        kinds.add("first" if choice[g] == 0 else "visited" if rc["visits"][g, choice[g]] > 0 else "unvisited")
    assert kinds == {"first", "visited", "unvisited"}
    moves = rc["moves"][np.arange(B), choice]
    s1 = e1.play(choice)
    s2 = e2.play_moves(moves)
    _status_equal(s1, s2)
    assert e2.counters()["error"] == 0
    assert np.array_equal(e1.root_keys(), e2.root_keys())
    for g in range(B):
        assert np.array_equal(e1.tree_signature(g), e2.tree_signature(g)), g
    live = (s1["terminal"] == 0).astype(np.uint8)
    for e in (e1, e2):
        _search(e, net, P, mask=live)
        e.raise_on_error()
    for g in range(B):
        assert np.array_equal(e1.tree_signature(g), e2.tree_signature(g)), g


@pytest.mark.parametrize("K", [1, 16])
def test_play_moves_at_unexpanded_roots(K):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.fakenet import FakeNet
    from oracle import oracle as O
    B, P = 64, 60
    boards, sides, rr = _positions(B, 12)
    rr = rr.copy()
    rr[::8] = 59                                              # these games reach restrict_round 60 unless the move captures
    e = _engine(B, K)
    e.reset(None, boards, sides, rr)
    mv, cnt = rules.legal_moves_batch(boards, sides)
    rs = np.random.RandomState(5)
    moves = mv[np.arange(B), rs.randint(0, cnt)]
    st = e.play_moves(moves)
    assert e.counters()["error"] == 0
    nb, cap = rules.apply_moves_batch(boards, moves)
    nrr = np.where(cap == 0, rr + 1, 0)
    term = np.where((cap == 1) | (cap == 8), 1, np.where(nrr >= 60, 2, 0))
    win = np.where(cap == 1, 1, np.where(cap == 8, 0, -1))
    assert np.array_equal(st["boards"], nb)
    assert np.array_equal(st["side"], sides ^ 1)
    assert np.array_equal(st["rr"], nrr) and np.array_equal(st["ply"], np.ones(B))
    assert np.array_equal(st["terminal"], term) and np.array_equal(st["winner"], win)
    assert (st["q"] == 0).all() and (st["root_N"] == 0).all()
    assert (term == 2).any()
    ref = _engine(B, 1, 1 << 14)
    ref.reset(None, nb, sides ^ 1, nrr)
    assert np.array_equal(e.root_keys(), ref.root_keys())
    assert (e.root_children()["n"] == -1).all()
    live = term == 0
    _search(e, FakeNet("hash_signed"), P, mask=live.astype(np.uint8))
    e.raise_on_error()
    for g in np.nonzero(live)[0]:
        t = O.Tree()
        t.reload(nb[g])
        if K > 1:
            t.search_fifo(int(sides[g] ^ 1), int(nrr[g]), P, K, "hash_signed")
        else:
            t.search(int(sides[g] ^ 1), int(nrr[g]), P, "hash_signed")
        assert np.array_equal(e.tree_signature(int(g)), t.signature()), g


def _own_capture(board, side):
    """a move of one of the mover's pieces onto another of its own pieces: looks like a move, is never legal"""
    own = np.nonzero((board >= 1) & (board <= 7))[0] if side == 0 else np.nonzero(board >= 8)[0]
    return int(own[0]) | (int(own[1]) << 7)


@pytest.mark.parametrize("searched", [False, True])
def test_play_moves_rejects_illegal_input(searched):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.fakenet import FakeNet
    B = 8
    boards, sides, rr = _positions(B, 13)
    mv, cnt = rules.legal_moves_batch(boards, sides)
    omv, ocnt = rules.legal_moves_batch(boards, sides ^ 1)
    legal = mv[:, 0]
    bad = {
        "off_board": lambda g: 127 | (127 << 7),
        "wrong_side": lambda g: int(omv[g, 0]),
        "own_capture": lambda g: _own_capture(boards[g], sides[g]),
        "not_a_code": lambda g: 0xFFFE,
    }
    for k, (name, make) in enumerate(bad.items()):
        g = (3 * k + 1) % B
        e = _engine(B, 1, 1 << 16)
        e.reset(None, boards, sides, rr)
        if searched:
            _search(e, FakeNet("hash_pos"), 24)
        before, keys, sig = e.status(), e.root_keys(), e.tree_signature(g)
        moves = legal.copy()
        moves[(g + 1) % B] = NO_MOVE
        moves[g] = make(g)
        assert moves[g] not in set(mv[g, :cnt[g]].tolist()), name
        st = e.play_moves(moves)
        c = e.counters()
        assert c["error"] == ILLEGAL and c["first_error_game"] == g, name
        for key in ("boards", "side", "terminal", "winner", "ply", "rr", "root_N"):
            assert np.array_equal(st[key][g], before[key][g]), (name, key)
        assert e.root_keys()[g] == keys[g] and np.array_equal(e.tree_signature(g), sig), name
        played = np.ones(B, bool)
        played[[g, (g + 1) % B]] = False
        assert (st["ply"][played] == 1).all() and (st["side"][played] == sides[played] ^ 1).all(), name
        n = (g + 1) % B
        assert st["ply"][n] == 0 and np.array_equal(st["boards"][n], boards[n]), name


def test_play_moves_in_a_finished_game_is_illegal_and_no_move_is_silent():
    from cchess_zero_b200 import rules
    B = 8
    boards, sides, _ = _positions(B, 14)
    rr = np.full(B, 59, dtype=np.int32)
    mv, cnt = rules.legal_moves_batch(boards, sides)
    _, cap = rules.apply_moves_batch(boards, mv[:, 0])
    assert (cap == 0).any()
    e = _engine(B, 1, 1 << 16)
    e.reset(None, boards, sides, rr)
    st = e.play_moves(mv[:, 0])
    assert e.counters()["error"] == 0
    done = np.nonzero(st["terminal"] == 2)[0]
    assert len(done)
    st0 = e.play_moves(np.full(B, NO_MOVE, dtype=np.uint16))           # 0xFFFF: nothing happens, no flag
    assert e.counters()["error"] == 0
    _status_equal(st, dict(st0, q=st["q"]))
    mv2, _ = rules.legal_moves_batch(st["boards"], st["side"])
    moves = np.full(B, NO_MOVE, dtype=np.uint16)
    g = int(done[0])
    moves[g] = mv2[g, 0]                                                # legal on the board, but the game is over
    st2 = e.play_moves(moves)
    c = e.counters()
    assert c["error"] == ILLEGAL and c["first_error_game"] == g
    _status_equal(dict(st2, q=st["q"]), st)


@pytest.mark.parametrize("K", [1, 16])
def test_match_equals_oracle(K):
    from arena_oracle import match_game
    from cchess_zero_b200.arena import Match
    from cchess_zero_b200.fakenet import FakeNet
    n, P, T0, plies0, cap = 8, 60, 1.0, 6, 80
    m = Match(FakeNet("hash_signed"), FakeNet("mod17"), n, P, search_threads=K, seeds=range(n), opening_temperature=T0,
              opening_plies=plies0, max_plies=cap, arena_words=1 << 18)
    watch = {0: None, 5: None}
    for g in watch:
        red, black = ("hash_signed", "mod17") if g < n // 2 else ("mod17", "hash_signed")
        watch[g] = match_game(red, black, P, np.random.RandomState(g), plies0, T0, 1e-3, search_threads=K, max_plies=cap, signatures=True)
    ply, left = 0, n
    while left:
        left = m.step()
        for g, o in watch.items():
            if ply < o["plies"]:
                for colour in (0, 1):
                    assert np.array_equal(m.tree_signature(g, colour), o["sigs"][ply][colour]), (g, ply, colour)
        ply += 1
    r = m.result()
    for g in range(n):
        red, black = ("hash_signed", "mod17") if g < n // 2 else ("mod17", "hash_signed")
        o = watch.get(g) or match_game(red, black, P, np.random.RandomState(g), plies0, T0, 1e-3, search_threads=K, max_plies=cap)
        rec = r.games[g]
        assert rec["moves"] == o["moves"], g
        assert rec["winner"] == "wbt"[o["winner"]] and rec["adjudicated"] == o["adjudicated"] and rec["plies"] == o["plies"], g


def _pv(seed, tmp_path):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(7, precision="fp16", seed=seed, save_dir=str(tmp_path / ("net%d" % seed)))


def test_match_real_networks(tmp_path):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.arena import Match, random_openings
    cand, best = _pv(1, tmp_path), _pv(0, tmp_path)
    n = 64
    op = random_openings(n // 2, 4, seed=0)
    runs = [Match(cand, best, n, 50, seeds=range(n), openings=op, max_plies=60).run() for _ in range(2)]
    r = runs[0]
    assert [g["moves"] for g in r.games] == [g["moves"] for g in runs[1].games]
    assert [g["result"] for g in r.games] == [g["result"] for g in runs[1].games]
    assert r.wins + r.draws + r.losses == n
    assert sum(g["candidate_colour"] == "w" for g in r.games) == n // 2
    for c in "wb":
        assert sum(r.by_colour[c].values()) == n // 2
    for g in r.games:
        assert g["opening"] == r.games[(g["game"] + n // 2) % n]["opening"] == g["game"] % (n // 2)
        assert g["labels"] == [rules.move_to_label(m) for m in g["moves"]]
        assert 1 <= g["plies"] <= 60 and g["result"] in ("win", "draw", "loss")
        b = op[0][g["opening"]][None].copy()
        s = op[1][g["opening"]:g["opening"] + 1].copy()
        for mv in g["moves"]:
            lm, c = rules.legal_moves_batch(b, s)
            assert mv in set(lm[0, :c[0]].tolist())
            b, _ = rules.apply_moves_batch(b, [mv])
            s ^= 1
    assert r.score == (r.wins + 0.5 * r.draws) / n
    assert r.promote() == (r.score > 0.55)
    assert (r.elo > 0) == (r.score > 0.5) and (r.elo < 0) == (r.score < 0.5)
    lo, hi = r.elo_interval()
    assert lo <= r.elo <= hi


def test_policy_evaluate(tmp_path, capsys):
    from cchess_zero_b200.selfplay import cchess_main
    pv = _pv(0, tmp_path)
    cm = cchess_main(playout=20, network=pv, log_file=False)
    capsys.readouterr()
    w = cm.policy_evaluate(4)
    out = capsys.readouterr().out
    assert isinstance(w, float) and 0.0 <= w <= 1.0
    line = [ln for ln in out.splitlines() if ln.startswith("num_playouts:")]
    assert len(line) == 1 and line[0].startswith("num_playouts:20, win: ")
    win, lose, tie = (int(x.split(":")[-1]) for x in line[0].split(",")[1:])
    assert win + lose + tie == 4 and w == (win + 0.5 * tie) / 4
