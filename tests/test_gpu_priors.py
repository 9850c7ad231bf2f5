"""Softmax priors on the device (Engine(priors='softmax'): the SOFTMAX instantiations of k_wave, k_wave_fifo and k_wave_multi): root
priors after one expansion against the definition on adversarial logit rows for every engine kind, whole self-play games and arena
games against the specification (tests/priors_spec.py), invariance under a constant added to every logit for the schedules the
specification does not restate, exact resumes, the setter's refusals and the explicit default.  Bit-exact everywhere."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

import priors_spec as PS
import search_spec as S

pytestmark = pytest.mark.gpu


def _labels(moves, side):
    from oracle import oracle as O
    unf = O.unflipped_index()
    li = [O.label_index(int(m) & 127, int(m) >> 7) for m in moves]
    return [int(unf[i]) if side == 1 else i for i in li]


def _adversarial_row(kind, rng):
    row = (rng.randn(2086) * 3).astype(np.float32)
    if kind == 1:
        row[:] = np.float32(0.75)                                      # every child tied
    elif kind == 2:
        row = rng.choice(np.float32([-2.0, 0.5, 0.5, 3.0]), 2086).astype(np.float32)
    elif kind == 3:
        row = (rng.uniform(-1, 1, 2086) * 1e30).astype(np.float32)    # huge range: most e_i underflow to 0
    elif kind == 4:
        row[rng.rand(2086) < 0.5] = -np.inf
    elif kind == 5:
        row[rng.rand(2086) < 0.01] = np.nan                            # a child with a NaN logit makes every prior NaN
    elif kind == 6:
        row = (rng.uniform(-80, 80, 2086)).astype(np.float32)
    elif kind == 7:
        row[:] = -np.inf                                               # every prior NaN
    return row


ENGINES = [("reference", {}), ("strict", dict(rules="strict")), ("fifo16", dict(search_threads=16)), ("multi8", dict(leaves=8))]


@pytest.mark.parametrize("name,kw", ENGINES, ids=[e[0] for e in ENGINES])
def test_root_priors_after_one_expansion_are_the_definition(name, kw):
    from cchess_zero_b200.engine import Engine
    from strict_support import random_play
    B = 64
    boards, sides = random_play(11, 4000)
    live = np.nonzero([(b == 1).any() and (b == 8).any() for b in boards])[0]
    pick = np.random.RandomState(2).choice(live, B, replace=False)
    boards, sides = boards[pick], sides[pick]
    e = Engine(B, 1 << 16, priors="softmax", **kw)
    assert e.priors == "softmax"
    e.reset(None, boards, sides, np.zeros(B, np.int32))
    rows = e.rows
    nn_in = torch.zeros((rows, 9, 10, 14), dtype=torch.float32, device="cuda")
    logits = torch.zeros((rows, 2086), dtype=torch.float32, device="cuda")
    value = torch.zeros(rows, dtype=torch.float32, device="cuda")
    rng = np.random.RandomState(7)
    table = np.stack([_adversarial_row(g % 8, rng) for g in range(B)])
    logits.copy_(torch.from_numpy(np.repeat(table, rows // B, axis=0)))      # every row of game g holds game g's logit row
    e.begin_search(0)
    for _ in range(3):
        e.wave(nn_in, logits, value)
        if e.unfinished() == 0:
            break
    assert e.unfinished() == 0
    rc = e.root_children(want_wpq=True)
    checked = 0
    for g in range(B):
        n = int(rc["n"][g])
        if n <= 0:
            continue
        li = _labels(rc["moves"][g, :n], int(sides[g]))
        want = PS.softmax(table[g][li])
        got = rc["p"][g, :n]
        nan = np.isnan(want)                                  # (a NaN's sign and payload are the platform's, not the definition's)
        assert np.array_equal(np.isnan(got), nan), (g, g % 8)
        assert np.array_equal(got[~nan].view(np.int32), want[~nan].view(np.int32)), (g, g % 8)
        checked += 1
    assert checked >= B - 4
    assert e.raise_on_error() is not None


def _selfplay(kind, B, P, seeds, priors, net="hash_signed", noise=None, graph=True, auto_reset=False, shift=0.0, compact=None):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    kw = dict(search_threads=16) if kind == "fifo" else dict(rules="strict") if kind == "strict" else {}
    fn = FakeNet(net)
    fwd = fn if shift == 0.0 else (lambda x: tuple(t + shift if i == 0 else t for i, t in enumerate(fn(x))))
    sp = SelfPlay(B, fwd, P, seeds=seeds, arena_words=1 << 18, auto_reset=auto_reset, root_noise=noise, compact=compact,
                  **({} if priors is None else dict(priors=priors)), **kw)
    if graph:
        sp.capture_graph()
    return sp


def _records(out):
    return [(slot, rec.states, rec.actions, [tuple(int(v) for v in x) for x in rec.visits], rec.z.copy(), rec.dense_pi())
            for slot, rec in sorted(out, key=lambda t: t[0])]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x[:4] == y[:4] and np.array_equal(x[4], y[4]) and np.array_equal(x[5], y[5])


@pytest.mark.parametrize("kind,noise,graph", [("reference", None, True), ("reference", None, False), ("strict", None, True),
                                              ("reference", (0.25, 0.3), True), ("strict", (0.25, 0.3), False)])
def test_softmax_selfplay_games_equal_the_specification(kind, noise, graph):
    B, P, net = 8, 24, "hash_signed"
    seeds = [410 + 17 * g for g in range(B)]
    sp = _selfplay(kind, B, P, seeds, "softmax", net=net, noise=noise, graph=graph)
    with np.errstate(all="ignore"):
        out = sp.play_games()
    assert len(out) == B
    rules = "strict" if kind == "strict" else "reference"
    for slot, rec in out:
        rn = None if noise is None else noise + (np.random.RandomState([seeds[slot], 1]),)
        with np.errstate(all="ignore"):
            r = PS.selfplay_game(net, P, np.random.RandomState(seeds[slot]), rules=rules, root_noise=rn, priors="softmax")
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert [tuple(int(v) for v in x) for x in rec.visits] == r["visits"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot


@pytest.mark.parametrize("kind,compact", [("reference", None), ("fifo", True), ("fifo", False)])
def test_softmax_games_do_not_see_a_logit_shift(kind, compact):
    """hash_signed's logits lie on a 2^-23 grid in [-1, 1): adding 1.0 is exact, so softmax-prior games are identical; reference-prior
    games are not."""
    B, P = 8, 32
    seeds = [31 + g for g in range(B)]
    games = {}
    for priors in ("softmax", "reference"):
        for shift in (0.0, 1.0):
            sp = _selfplay(kind, B, P, seeds, priors, shift=shift, compact=compact if kind == "fifo" else None)
            with np.errstate(all="ignore"):
                games[priors, shift] = _records(sp.play_games(max_plies=60))
    _same(games["softmax", 0.0], games["softmax", 1.0])
    assert any(x[2] != y[2] for x, y in zip(games["reference", 0.0], games["reference", 1.0]))


def _openings(n, plies, seed):
    """n positions after `plies` uniformly random pseudo-legal moves from the start position (the C specification's move generator)"""
    from oracle import oracle as O
    rng = np.random.RandomState(seed)
    boards, sides = np.zeros((n, 90), np.uint8), np.zeros(n, np.uint8)
    for g in range(n):
        b, side = O.from_state(O.START), 0
        for _ in range(plies):
            mv = O.legal_moves(b, side)
            b, _ = O.apply_move(b, int(mv[rng.randint(len(mv))]))
            side ^= 1
        boards[g], sides[g] = b, side
    return boards, sides


ONE_LEAF = [("k_wave", {}), ("k_wave_fifo_K1", dict(search_threads=1)), ("k_wave_multi_1slot", dict(leaves=-1))]


@pytest.mark.parametrize("name,kw", ONE_LEAF, ids=[e[0] for e in ONE_LEAF])
@pytest.mark.parametrize("net", ["hash_signed", "mod17"])
def test_softmax_trees_of_every_kernel_family_equal_the_specification(name, kw, net):
    """Whole trees after three searched and played plies against the one-leaf softmax specification, for the three wave kernels: the
    search_threads = 1 engine runs k_wave_fifo (its event loop with one task is the one-leaf search, so every expansion after the
    root goes through the loop's own expand_write), and leaves = -1 runs k_wave_multi with one slot."""
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.fakenet import FakeNet
    boards, sides = _openings(12, 6, 21)
    b2, s2 = _openings(12, 16, 22)
    keep = [g for g in range(12) if (b2[g] == 1).any() and (b2[g] == 8).any()]
    boards, sides = np.concatenate([boards, b2[keep]]), np.concatenate([sides, s2[keep]])
    B, P = len(boards), 80
    e = Engine(B, 1 << 18, priors="softmax", **kw)
    assert (e.fifo, e.leaves) == ((True, 1) if "search_threads" in kw else (False, 1))
    e.reset(None, boards, sides, np.zeros(B, np.int32))
    fn = FakeNet(net)
    x = torch.zeros((B, 9, 10, 14), dtype=torch.float32, device="cuda")
    lo = torch.zeros((B, 2086), dtype=torch.float32, device="cuda")
    v = torch.zeros(B, dtype=torch.float32, device="cuda")

    def fwd(inp):
        a, b = fn(inp)
        lo.copy_(a)
        v.copy_(b)
    from oracle import oracle as O
    trees = [PS.SoftmaxTree(boards[g]) for g in range(B)]
    board, side, rr = boards.copy(), sides.astype(np.int64), np.zeros(B, np.int64)
    for ply in range(3):
        e.search(fwd, P, x, lo, v)
        assert e.raise_on_error()["error"] == 0
        pick = np.full(B, -1, np.int32)
        for g, t in enumerate(trees):
            if not ((board[g] == 1).any() and (board[g] == 8).any()):
                continue                                     # a king was taken: the game is over, the engine searches it no more
            assert t.search(int(side[g]), int(rr[g]), P, net) == 0
            assert np.array_equal(e.tree_signature(g), t.signature()), (name, net, ply, g)
            mv, N = t.root_children()[:2]
            pick[g] = int(np.argmax(N))
            t.update(int(pick[g]))
            board[g], cap = O.apply_move(board[g], int(mv[pick[g]]))
            side[g] ^= 1
            rr[g] = rr[g] + 1 if cap == 0 else 0
        st = e.play(pick)
        assert np.array_equal(st["boards"], board)


def test_leaf_parallel_softmax_trees_do_not_see_a_logit_shift():
    """k_wave_multi, which the specification does not restate with softmax priors: trees, moves and error flags after three searched
    and played plies are identical with mod17's logits and with 1.0 added to them (exact: they are multiples of 1/16 in [-0.5, 0.5])."""
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.fakenet import FakeNet
    B, K = 16, 8
    boards, sides = _openings(B, 6, 3)
    net = FakeNet("mod17")
    runs = {}
    for priors in ("softmax", "reference"):
        for shift in (0.0, 1.0):
            e = Engine(B, 1 << 18, leaves=K, priors=priors)
            e.reset(None, boards, sides, np.zeros(B, np.int32))
            x = torch.zeros((B * K, 9, 10, 14), dtype=torch.float32, device="cuda")
            lo = torch.zeros((B * K, 2086), dtype=torch.float32, device="cuda")
            v = torch.zeros(B * K, dtype=torch.float32, device="cuda")

            def fwd(inp):
                a, b = net(inp)
                lo.copy_(a + shift)
                v.copy_(b)
            sigs, moves = [], []
            for _ in range(3):
                e.search(fwd, 96, x, lo, v)
                sigs.append([e.tree_signature(g) for g in range(B)])
                rc = e.root_children(want_wpq=False)
                pick = np.where(rc["n"] > 0, np.argmax(rc["visits"], axis=1), -1).astype(np.int32)
                moves.append(rc["moves"][np.arange(B), np.maximum(pick, 0)].copy())
                e.play(pick)
            runs[priors, shift] = (sigs, moves, e.counters()["error"])
    a, b = runs["softmax", 0.0], runs["softmax", 1.0]
    assert a[2] == b[2]
    assert all(np.array_equal(m, n) for m, n in zip(a[1], b[1]))
    assert all(np.array_equal(s, t) for p, q in zip(a[0], b[0]) for s, t in zip(p, q))
    r0, r1 = runs["reference", 0.0], runs["reference", 1.0]
    assert any(not np.array_equal(s, t) for p, q in zip(r0[0], r1[0]) for s, t in zip(p, q))


@pytest.mark.parametrize("rules", ["reference", "strict"])
def test_softmax_match_equals_the_specification(rules):
    from cchess_zero_b200.arena import Match
    from cchess_zero_b200.fakenet import FakeNet
    n, P, T0, plies0, cap = 4, 24, 1.0, 6, 60
    m = Match(FakeNet("hash_signed"), FakeNet("mod17"), n, P, seeds=range(n), opening_temperature=T0, opening_plies=plies0,
              max_plies=cap, arena_words=1 << 18, rules=rules, priors="softmax")
    with np.errstate(all="ignore"):
        r = m.run()
    for g in range(n):
        red, black = ("hash_signed", "mod17") if g < n // 2 else ("mod17", "hash_signed")
        with np.errstate(all="ignore"):
            o = PS.match_game(red, black, P, np.random.RandomState(g), plies0, T0, 1e-3, max_plies=cap, rules=rules, priors="softmax")
        rec = r.games[g]
        assert rec["moves"] == o["moves"], g
        assert rec["winner"] == "wbt"[o["winner"]] and rec["adjudicated"] == o["adjudicated"] and rec["plies"] == o["plies"], g


def test_explicit_reference_default_changes_nothing():
    B, P = 8, 24
    seeds = [5 + g for g in range(B)]
    with np.errstate(all="ignore"):
        a = _records(_selfplay("fifo", B, P, seeds, None).play_games(max_plies=40))
        b = _records(_selfplay("fifo", B, P, seeds, "reference").play_games(max_plies=40))
        c = _records(_selfplay("reference", B, P, seeds, None).play_games(max_plies=40))
        d = _records(_selfplay("reference", B, P, seeds, "reference").play_games(max_plies=40))
    _same(a, b)
    _same(c, d)


def test_setter_refusals_leave_the_engine_usable():
    from cchess_zero_b200._lib import check, lib
    from cchess_zero_b200.engine import Engine, EngineError
    from cchess_zero_b200.fakenet import FakeNet
    e = Engine(4, 1 << 16)
    assert lib().cz_engine_priors(e.h) == 0
    assert lib().cz_engine_set_priors(e.h, 2) == -1 and "mode" in lib().cz_last_error().decode()
    assert lib().cz_engine_set_priors(e.h, -1) == -1
    assert lib().cz_engine_priors(e.h) == 0
    check(lib().cz_engine_set_priors(e.h, 1))
    check(lib().cz_engine_set_priors(e.h, 0))              # before the first wave: may change again
    x = torch.zeros((4, 9, 10, 14), device="cuda")
    lo = torch.zeros((4, 2086), device="cuda")
    v = torch.zeros(4, device="cuda")
    net = FakeNet("hash_pos")

    def fwd(inp):
        a, b = net(inp)
        lo.copy_(a)
        v.copy_(b)
    e.search(fwd, 16, x, lo, v)
    for mode in (1, 0):
        assert lib().cz_engine_set_priors(e.h, mode) == -1 and "already run a wave" in lib().cz_last_error().decode()
    assert lib().cz_engine_set_priors(e.h, 7) == -1
    assert lib().cz_engine_priors(e.h) == 0
    with pytest.raises(EngineError):
        check(lib().cz_engine_set_priors(e.h, 1), "cz_engine_set_priors")
    e.search(fwd, 16, x, lo, v)                            # still searches
    assert int(e.root_children()["visits"].sum()) > 0 and e.raise_on_error()["error"] == 0
    assert lib().cz_engine_priors(None) == -1
    s = Engine(2, 1 << 16, priors="softmax")
    assert lib().cz_engine_priors(s.h) == 1


@pytest.mark.parametrize("kind", ["reference", "fifo"])
def test_softmax_selfplay_resumes_exactly(kind, tmp_path):
    B, P = 12, 32
    seeds = [60 + g for g in range(B)]
    a = _selfplay(kind, B, P, seeds, "softmax", auto_reset=True)
    log_a, log_b = [], []
    with np.errstate(all="ignore"):
        for _ in range(20):
            a.step()
        a.pop_finished()
        path = str(tmp_path / "games.npz")
        a.save_games(path)
        b = _selfplay(kind, B, P, [999] * B, "softmax", auto_reset=True)
        b.load_games(path)
        for sp, log in ((a, log_a), (b, log_b)):
            for _ in range(25):
                sp.step()
                log.append((sp.boards.copy(), [sp.engine.tree_signature(g) for g in range(B)]))
        r = _selfplay(kind, B, P, [999] * B, "reference", auto_reset=True)
        with pytest.raises(ValueError, match="priors"):
            r.load_games(path)
    for x, y in zip(log_a, log_b):
        assert np.array_equal(x[0], y[0]) and all(np.array_equal(s, t) for s, t in zip(x[1], y[1]))
    fa, fb = a.pop_finished(), b.pop_finished()
    assert [g for g, _ in fa] == [g for g, _ in fb]
    for (_, ra), (_, rb) in zip(fa, fb):
        assert ra.states == rb.states and np.array_equal(ra.dense_pi(), rb.dense_pi()) and np.array_equal(ra.z, rb.z)


def _net(tmp, name, seed=0, blocks=2):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(blocks, seed=seed, save_dir=os.path.join(str(tmp), name))


def test_softmax_trainer_resume_is_bit_identical(tmp_path, monkeypatch):
    from cchess_zero_b200.train import Trainer
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.chdir(tmp_path)
    run = str(tmp_path / "run")
    kw = dict(batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16, priors="softmax")
    ta = Trainer(_net(tmp_path, "a"), 16, 8, seed=3, **kw)
    assert ta.sp.priors == "softmax" and ta.sp.engine.priors == "softmax"
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
        tn = Trainer(_net(tmp_path, "c", seed=5), 16, 8, seed=9, **dict(kw, priors="reference"))
        with pytest.raises(ValueError, match="priors"):
            tn.load(run)
    assert all(np.array_equal(x, y) for x, y in zip(log_a, log_b))
    assert all(np.array_equal(ta.sp.engine.tree_signature(g), tb.sp.engine.tree_signature(g)) for g in range(16))
    for name in ("boards", "n", "idx", "prob", "z"):
        assert torch.equal(getattr(ta.buffer, name), getattr(tb.buffer, name)), name
