"""Strict rules inside the device search (engines created with rules='strict': k_wave<T, true>, k_play_moves<true>, k_root_mate)
against the specification (tests/strict_search_oracle.c): trees, whole self-play games, root mates, matches, snapshots and a resumed
strict training run.  Bit-exact everywhere."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

import strict_search_support as S
from strict_support import oracle_strict

pytestmark = pytest.mark.gpu

ILLEGAL = 32


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


def _search(e, cases, nets):
    """Run every case's search on strict engine e (one game per case); nets[g] evaluates game g's leaves."""
    from cchess_zero_b200.fakenet import FakeNet
    fns = {n: FakeNet(n) for n in set(nets)}
    nn_in = torch.zeros((e.rows, 9, 10, 14), device="cuda")
    logits = torch.zeros((e.rows, 2086), device="cuda")
    value = torch.zeros((e.rows,), device="cuda")
    pl = np.array([c["playouts"] for c in cases])
    for p in np.unique(pl):
        e.begin_search(int(p), (pl == p).astype(np.uint8))

    def fwd():
        for n, fn in fns.items():
            rows = torch.tensor([g for g in range(len(cases)) if nets[g] == n], device="cuda")
            lo, v = fn(nn_in[rows])
            logits[rows] = lo
            value[rows] = v.reshape(-1)
    waves = 0
    while True:
        e.wave(nn_in, logits, value)
        waves += 1
        if e.unfinished() == 0:
            break
        fwd()
        assert waves < 5 * pl.max() + 50
    return e


def test_trees_equal_the_specification():
    from cchess_zero_b200.engine import Engine
    cases = S.random_cases(7, 100)
    assert len(cases) >= 90
    e = Engine(len(cases), arena_words=1 << 18, rules="strict")
    e.reset(None, np.stack([c["board"] for c in cases]), [c["side"] for c in cases], [c["rr"] for c in cases])
    _search(e, cases, [c["net"] for c in cases])
    cnt = e.raise_on_error()
    tot = dict(n_expand=0, n_playout=0, sum_L=0, sum_c=0, sum_C=0)
    mated_leaves = in_check = 0
    for g, c in enumerate(cases):
        t = S.StrictTree(c["board"])
        assert t.search(c["side"], c["rr"], c["playouts"], c["net"]) == 0
        sig = t.signature()
        assert np.array_equal(sig, e.tree_signature(g)), g
        mated_leaves += int((sig[:, 5] == -1).sum())
        in_check += S.in_check(c["board"], c["side"])
        for k, v in t.stats().items():
            if k in tot:
                tot[k] += v
    for k in tot:
        assert cnt[k] == tot[k], k
    assert mated_leaves > 20 and in_check >= 30, (mated_leaves, in_check)


@pytest.mark.parametrize("net", S.NETS)
def test_selfplay_games_equal_the_specification(net, O):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    B, P = 12, 24
    seeds = [700 + 31 * g for g in range(B)]
    sp = SelfPlay(B, FakeNet(net), P, seeds=seeds, arena_words=1 << 18, auto_reset=False, rules="strict")
    sp.capture_graph()
    out = sp.play_games()
    assert len(out) == B
    ends = []
    for slot, rec in out:
        with np.errstate(all="ignore"):
            r = S.selfplay_game(net, P, np.random.RandomState(seeds[slot]))
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot
        ends.append(r["end"])
        for b, p, a in zip(r["boards"], r["players"], r["actions"]):       # every move played is strictly legal
            assert O.move_from_str(a) in [int(m) for m in S.strict_moves(b, p)]
    assert 3 in ends, ends


def test_root_mate_after_reset_set_root_meta_play_and_play_moves(O):
    from cchess_zero_b200.engine import Engine
    name, state, side, mate, _ = S.MATE_IN_ONE[0]
    b, s = O.from_state(state), 0 if side == "w" else 1
    mated, _ = O.apply_move(b, O.move_from_str(mate))
    e = Engine(4, arena_words=1 << 16, rules="strict")
    assert e.rules == "strict"
    # reset with a mated board (game 1), the mating position itself (game 0, running)
    e.reset(None, np.stack([b, mated, b, b]), [s, s ^ 1, s, s], [0, 0, 0, 0])
    st = e.status()
    assert list(st["terminal"]) == [0, 3, 0, 0] and st["winner"][1] == s
    # game 1 reset to the mated board with the mating side to move (a running game); set_root_meta then gives the move to the
    # mated side
    e.reset(np.array([0, 1, 0, 0], np.uint8), np.stack([b, mated, b, b]), [s, s, s, s], [0, 0, 0, 0])
    assert e.status()["terminal"][1] == 0
    e.set_root_meta(sides=np.array([s, s ^ 1, s, s], np.uint8), mask=np.array([0, 1, 0, 0], np.uint8))
    st = e.status()
    assert st["terminal"][1] == 3 and st["winner"][1] == s
    # play_moves at an unexpanded root: the mating move ends game 0; a pseudo-legal move that leaves the king attacked is refused
    bad = [int(m) for m in O.legal_moves(b, s) if int(m) not in [int(x) for x in S.strict_moves(b, s)]]
    assert bad                                         # (d9e9 would face the red king)
    before = e.status()
    sig2 = e.tree_signature(2)
    moves = np.full(4, 0xFFFF, np.uint16)
    moves[0] = O.move_from_str(mate)
    moves[2] = bad[0]
    st = e.play_moves(moves)
    assert st["terminal"][0] == 3 and st["winner"][0] == s and np.array_equal(st["boards"][0], mated)
    assert e.counters()["error"] == ILLEGAL
    for k in ("boards", "side", "terminal", "winner", "ply", "rr"):
        assert np.array_equal(st[k][2], before[k][2]), k
    assert np.array_equal(e.tree_signature(2), sig2)
    # play: search game 3, then play its mating child through the tree
    case = [dict(board=b, side=s, rr=0, playouts=200)] * 4
    e2 = Engine(4, arena_words=1 << 16, rules="strict")
    e2.reset(None, np.stack([b] * 4), [s] * 4, [0] * 4)
    _search(e2, case, ["hash_pos"] * 4)
    rc = e2.root_children(want_wpq=False)
    kids = [int(m) for m in rc["moves"][3, :rc["n"][3]]]
    st = e2.play(np.array([-1, -1, -1, kids.index(O.move_from_str(mate))], np.int32))
    assert st["terminal"][3] == 3 and st["winner"][3] == s and list(st["terminal"][:3]) == [0, 0, 0]
    assert e2.status()["terminal"][3] == 3
    e2.raise_on_error()


def test_strict_match_equals_the_specification():
    from cchess_zero_b200.arena import Match, random_openings
    from cchess_zero_b200.fakenet import FakeNet
    n, P, T0, plies0, cap = 8, 32, 1.0, 6, 300
    openings = random_openings(2, 4, seed=3, rules="strict")
    m = Match(FakeNet("hash_signed"), FakeNet("hash_pos"), n, P, seeds=range(n), opening_temperature=T0, opening_plies=plies0,
              max_plies=cap, arena_words=1 << 18, openings=openings, rules="strict")
    r = m.run()
    for g in range(n):
        red, black = ("hash_signed", "hash_pos") if g < n // 2 else ("hash_pos", "hash_signed")
        o = g % (n // 2) % 2
        with np.errstate(all="ignore"):
            x = S.match_game(red, black, P, np.random.RandomState(g), plies0, T0, 1e-3, board=openings[0][o], side=int(openings[1][o]),
                             rr=int(openings[2][o]), max_plies=cap)
        rec = r.games[g]
        assert rec["moves"] == x["moves"] and rec["winner"] == "wbt"[x["winner"]] and rec["plies"] == x["plies"], g
    # strict openings: every move drawn is strictly legal and the position reached is a running game
    mv, cnt, legal, _ = oracle_strict(openings[0], openings[1])
    assert (legal.any(axis=1)).all()


def test_snapshot_round_trip_with_mated_nodes_and_refusal_by_a_reference_engine():
    from cchess_zero_b200._lib import EngineError
    from cchess_zero_b200.engine import Engine
    cases = S.random_cases(11, 40)[:16]
    e = Engine(len(cases), arena_words=1 << 18, rules="strict")
    e.reset(None, np.stack([c["board"] for c in cases]), [c["side"] for c in cases], [c["rr"] for c in cases])
    nets = [c["net"] for c in cases]
    _search(e, cases, nets)
    assert sum(int((e.tree_signature(g)[:, 5] == -1).sum()) for g in range(len(cases))) > 0
    blob = e.snapshot()
    assert int(blob[8:12].view(np.uint32)[0]) == 2                               # format 2: strict rules
    f = Engine(len(cases), arena_words=1 << 19, rules="strict")
    f.restore(blob)
    ref = Engine(len(cases), arena_words=1 << 19)
    with pytest.raises(EngineError, match="rules differ"):
        ref.restore(blob)
    with pytest.raises(EngineError, match="rules differ"):
        f.restore(ref.snapshot())
    for ply in range(3):
        for x in (e, f):
            rc = x.root_children(want_wpq=False)
            vis = np.where(np.arange(128) < rc["n"][:, None], rc["visits"], -1)        # (entries past n are not written)
            ch = np.where(rc["n"] > 0, np.argmax(vis, axis=1), -1).astype(np.int32)
            x.play(ch)
        se, sf = e.status(), f.status()
        for k in ("boards", "terminal", "winner", "ply", "side"):
            assert np.array_equal(se[k], sf[k]), k
        assert all(np.array_equal(e.tree_signature(g), f.tree_signature(g)) for g in range(len(cases)))
        mask = (se["terminal"] == 0).astype(np.uint8)
        for x in (e, f):
            x.begin_search(60, mask)
        for x in (e, f):
            _search_masked(x, nets, mask)


def _search_masked(e, nets, mask):
    from cchess_zero_b200.fakenet import FakeNet
    fns = {n: FakeNet(n) for n in set(nets)}
    nn_in = torch.zeros((e.rows, 9, 10, 14), device="cuda")
    logits = torch.zeros((e.rows, 2086), device="cuda")
    value = torch.zeros((e.rows,), device="cuda")
    waves = 0
    while True:
        e.wave(nn_in, logits, value)
        waves += 1
        if e.unfinished() == 0:
            break
        for n, fn in fns.items():
            rows = torch.tensor([g for g in range(e.B) if nets[g] == n], device="cuda")
            lo, v = fn(nn_in[rows])
            logits[rows] = lo
            value[rows] = v.reshape(-1)
        assert waves < 2000
    e.raise_on_error()


def test_refusals_fifo_and_leaf_parallel():
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.selfplay import SelfPlay
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(4, search_threads=16, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(4, search_threads=1, rules="strict")        # the FIFO engine, even with one thread
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(4, leaves=8, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        Engine(4, leaves=-1, rules="strict")
    with pytest.raises(ValueError, match="one-leaf engine"):
        SelfPlay(4, lambda x: None, 8, search_threads=16, rules="strict")
    from cchess_zero_b200._lib import lib
    import ctypes as C
    h = C.c_void_p()
    assert lib().cz_engine_create_rules(4, 0, torch.cuda.current_device(), 2, C.byref(h)) != 0
    assert Engine(2).rules == "reference" and lib().cz_engine_rules(Engine(2, rules="strict").h) == 1


def _net(tmp, name, seed=0, blocks=2):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(blocks, seed=seed, save_dir=os.path.join(str(tmp), name))


def test_strict_trainer_resume_is_bit_identical(tmp_path, monkeypatch):
    from cchess_zero_b200.train import Trainer
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.chdir(tmp_path)
    run = str(tmp_path / "run")
    kw = dict(batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16, rules="strict")
    ta = Trainer(_net(tmp_path, "a"), 16, 8, seed=3, **kw)
    log_a, log_b = [], []
    with contextlib.redirect_stdout(io.StringIO()):
        while ta.updates < 1 and ta.plies < 3000:
            ta.ply()
        ta.save(run)
        for _ in range(12):
            ta.ply()
            log_a.append(ta.sp.engine.status()["boards"].copy())
        tb = Trainer(_net(tmp_path, "b", seed=5), 16, 8, seed=9, **kw)
        tb.load(run)
        for _ in range(12):
            tb.ply()
            log_b.append(tb.sp.engine.status()["boards"].copy())
        tr = Trainer(_net(tmp_path, "c", seed=5), 16, 8, seed=9, **dict(kw, rules="reference"))
        with pytest.raises(ValueError, match="'strict' rules"):
            tr.load(run)
    assert all(np.array_equal(x, y) for x, y in zip(log_a, log_b))
    assert all(np.array_equal(ta.sp.engine.tree_signature(g), tb.sp.engine.tree_signature(g)) for g in range(16))
    for name in ("boards", "n", "idx", "prob", "z"):
        assert torch.equal(getattr(ta.buffer, name), getattr(tb.buffer, name)), name
    assert (ta.games, ta.positions, ta.updates, ta.plies) == (tb.games, tb.positions, tb.updates, tb.plies)
