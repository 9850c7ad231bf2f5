"""Engine snapshots on the GPU: a round trip into a fresh engine with another arena size, an in-place restore under a captured CUDA
graph, refusals that leave the engine untouched, and a Trainer run that is interrupted, saved, resumed and still equals the
uninterrupted run bit for bit."""
import contextlib
import io
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF


def _selfplay(B, P, K, arena_words, **kw):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    return SelfPlay(B, FakeNet("hash_signed"), P, seeds=[40 + g for g in range(B)], arena_words=arena_words, search_threads=K, **kw)


def _state(e):
    """Everything a game exposes: tree signatures, root keys, status records, counters."""
    st = e.status()
    return dict(sig=[e.tree_signature(g) for g in range(e.B)], keys=e.root_keys(), counters=e.counters(),
                **{k: v for k, v in st.items() if k != "q"})


def _assert_same(a, b):
    assert all(np.array_equal(x, y) for x, y in zip(a["sig"], b["sig"])), "tree signatures differ"
    for k in a:
        if k != "sig":
            assert np.array_equal(a[k], b[k]) if isinstance(a[k], np.ndarray) else a[k] == b[k], k


def _play_same(engines, plies, sp_search):
    """Search every running game of every engine, then play its most visited root child (the same index everywhere)."""
    for _ in range(plies):
        running = engines[0].status()["terminal"] == 0
        for sp in sp_search:
            sp.search(running)
        choice = None
        for e in engines:
            rc = e.root_children(want_wpq=False)
            visits = np.where(np.arange(128)[None, :] < rc["n"][:, None], rc["visits"], -1)     # entries past n are not written
            c = np.where(running & (rc["n"] > 0), np.argmax(visits, axis=1), -1).astype(np.int32)
            assert choice is None or np.array_equal(c, choice), [x.counters() for x in engines]
            choice = c
        for e in engines:
            e.play(choice)


@pytest.mark.parametrize("K", [1, 16])
def test_round_trip_into_a_fresh_engine_with_another_arena_size(K):
    B, P = 12, 40
    a = _selfplay(B, P, K, 1 << 18, hashing=True)
    for _ in range(5):
        a.step()
    a.pop_finished()
    blob = a.engine.snapshot()
    assert blob.dtype == np.uint8 and blob.ndim == 1
    b = _selfplay(B, P, K, 1 << 17, hashing=True)                     # half the arena: the trees kept between plies still fit
    b.engine.restore(blob)
    _assert_same(_state(a.engine), _state(b.engine))
    assert np.array_equal(b.engine.snapshot(), blob)
    _play_same([a.engine, b.engine], 4, [a, b])
    _assert_same(_state(a.engine), _state(b.engine))
    assert a.engine.counters()["error"] == 0 and a.engine.counters()["max_arena_words"] < 1 << 17


def test_in_place_restore_under_a_captured_graph(tmp_path):
    sp = _selfplay(16, 32, 1, 1 << 18, auto_reset=True)
    sp.capture_graph()
    for _ in range(4):
        sp.step()
    sp.pop_finished()
    path = str(tmp_path / "games.npz")
    sp.save_games(path)
    runs = []
    for attempt in range(2):
        if attempt:
            sp.pop_finished()
            sp.load_games(path)                                       # the same engine, the graph captured before the save
        log = []
        for _ in range(4):
            out = sp.step()
            log.append((out["choice"].copy(), out["status"]["boards"].copy(), out["status"]["ply"].copy()))
        log.append([sp.engine.tree_signature(g) for g in range(sp.B)])
        runs.append(log)
    a, b = runs
    for x, y in zip(a[:-1], b[:-1]):
        assert all(np.array_equal(u, v) for u, v in zip(x, y))
    assert all(np.array_equal(u, v) for u, v in zip(a[-1], b[-1]))


def test_save_games_refuses_undrained_records(tmp_path):
    sp = _selfplay(4, 8, 1, 1 << 16, auto_reset=False)
    sp.finished.append((0, None))
    with pytest.raises(ValueError):
        sp.save_games(str(tmp_path / "g.npz"))


def test_snapshot_mid_search_is_refused():
    import torch
    from cchess_zero_b200._lib import EngineError
    from cchess_zero_b200.engine import Engine
    e = Engine(4, arena_words=1 << 16)
    nn, lo, va = torch.zeros((4, 9, 10, 14), device="cuda"), torch.zeros((4, 2086), device="cuda"), torch.zeros((4,), device="cuda")
    assert len(e.snapshot()) > 0                                       # a fresh engine is at rest
    e.begin_search(16)
    e.wave(nn, lo, va)
    with pytest.raises(EngineError, match="not at rest"):
        e.snapshot()


def _root_child_words(blob, g):
    """Word index (in blob viewed as uint32) of the CHILD array of game g's root block, its child count and the game's alloc
    (a one-leaf engine's blob: 52 words precede the arena)."""
    w = blob.view(np.uint32)
    off = int(blob[48 + 8 * g:56 + 8 * g].view(np.int64)[0])
    cnt, base, alloc = int(np.int32(w[off + 5])), int(w[off + 6]), int(w[off + 7])
    return off + 52 + base + 8 + 4 * ((cnt + 7) & ~7), cnt, alloc


def test_corrupt_blobs_and_arenas_too_small_are_refused_with_the_engine_unchanged():
    from cchess_zero_b200._lib import EngineError
    a = _selfplay(8, 200, 1, 1 << 18)
    for _ in range(3):
        a.step()
    blob = a.engine.snapshot()
    b = _selfplay(8, 200, 1, 1 << 18)
    for _ in range(2):
        b.step()                                                       # b holds trees of its own
    before = _state(b.engine)

    bad = blob.copy()
    w = bad.view(np.uint32)
    g, i = next((g, i) for g in range(8) for i in range(max(0, _root_child_words(bad, g)[1]))
                if w[_root_child_words(bad, g)[0] + i] != NONE)
    child, _, alloc = _root_child_words(bad, g)
    w[child + i] = alloc + 64                                          # a child pointer past the game's alloc
    with pytest.raises(EngineError, match="game %d: block outside" % g):
        b.engine.restore(bad)
    _assert_same(before, _state(b.engine))

    bad = blob.copy()
    bad[: 8] ^= 0xFF
    with pytest.raises(EngineError, match="magic"):
        b.engine.restore(bad)
    with pytest.raises(EngineError, match="truncated"):
        b.engine.restore(blob[:-4])
    _assert_same(before, _state(b.engine))

    assert max(_root_child_words(blob, g)[2] for g in range(8)) > 4096   # a retained tree larger than the smallest arena
    small = _selfplay(8, 200, 1, 4096)
    small_before = _state(small.engine)
    with pytest.raises(EngineError, match="exceeds the engine's arena words"):
        small.engine.restore(blob)
    _assert_same(small_before, _state(small.engine))
    b.engine.restore(blob)                                             # the intact blob still restores
    _assert_same(_state(a.engine), _state(b.engine))


# ---- the Trainer ----------------------------------------------------------------------------------------------------------
def _net(tmp, name, seed=0, blocks=2):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(blocks, seed=seed, save_dir=os.path.join(str(tmp), name))


@pytest.fixture
def deterministic(monkeypatch):
    import torch
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)


def _params(pv):
    return [p.detach().clone() for p in pv.net.state_dict().values()]


def _record(tr):
    """Log every ply's choices and statuses and every finished game's tuples of a Trainer's self-play."""
    log, fin = [], []
    step, pop = tr.sp.step, tr.sp.pop_finished

    def rec_step():
        out = step()
        st = out["status"]
        log.append((out["choice"].copy(), st["boards"].copy(), st["terminal"].copy(), st["winner"].copy(), st["ply"].copy()))
        return out

    def rec_pop():
        out = pop()
        fin.extend((g, list(r.states), r.dense_pi(), np.asarray(r.z)) for g, r in out)
        return out
    tr.sp.step, tr.sp.pop_finished = rec_step, rec_pop
    return log, fin


def test_trainer_resume_continues_the_interrupted_run_exactly(tmp_path, monkeypatch, deterministic):
    import torch
    from cchess_zero_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    run = str(tmp_path / "run")
    kw = dict(batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16)
    pa = _net(tmp_path, "a", seed=0)
    ta = Trainer(pa, 16, 8, seed=3, **kw)
    with contextlib.redirect_stdout(io.StringIO()):
        while ta.updates < 1 and ta.plies < 3000:
            ta.ply()
        ta.save(run)
        assert os.path.isfile(os.path.join(run, "games.npz"))
        log_a, fin_a = _record(ta)
        games0, m = ta.games, 0
        while (m < 12 or ta.games < games0 + 2) and m < 1000:          # on past a few finished games (and their updates)
            ta.ply()
            m += 1
        pb = _net(tmp_path, "b", seed=5)
        tb = Trainer(pb, 16, 8, seed=9, **kw)
        tb.load(run)
        log_b, fin_b = _record(tb)
        for _ in range(m):
            tb.ply()
    assert len(log_a) == len(log_b) == m
    for x, y in zip(log_a, log_b):
        assert all(np.array_equal(u, v) for u, v in zip(x, y))
    assert len(fin_a) == len(fin_b) >= 2
    for (ga, sa, pa_, za), (gb, sb, pb_, zb) in zip(fin_a, fin_b):
        assert ga == gb and sa == sb and np.array_equal(pa_, pb_) and np.array_equal(za, zb)
    assert all(np.array_equal(ta.sp.engine.tree_signature(g), tb.sp.engine.tree_signature(g)) for g in range(16))
    for name in ("boards", "n", "idx", "prob", "z"):
        assert torch.equal(getattr(ta.buffer, name), getattr(tb.buffer, name)), name
    assert (ta.games, ta.positions, ta.updates, ta.train_steps, ta.plies) == (tb.games, tb.positions, tb.updates, tb.train_steps, tb.plies)
    assert ta.updates > 1 and all(bool((x == y).all()) for x, y in zip(_params(pa), _params(pb)))
    assert ta.rng.getstate() == tb.rng.getstate() and np.array_equal(ta.sp._mt, tb.sp._mt)

    # a directory without games.npz (saved before games in flight were kept) resumes with fresh games
    os.remove(os.path.join(run, "games.npz"))
    pc = _net(tmp_path, "c", seed=7)
    tc = Trainer(pc, 16, 8, seed=1, **kw)
    with contextlib.redirect_stdout(io.StringIO()):
        tc.load(run)
        st = tc.sp.engine.status()
        assert (st["ply"] == 0).all() and (st["side"] == 0).all() and all(len(r.players) == 0 for r in tc.sp.records)
        assert all(len(tc.sp.engine.tree_signature(g)) == 0 for g in range(16))
        tc.ply()


def test_cli_saves_the_games_in_flight_and_resumes_them(tmp_path):
    d = str(tmp_path / "run")
    base = [sys.executable, "-m", "cchess_zero_b200.train", "--games", "8", "--playouts", "8", "--batch-size", "16", "--buffer-size", "128",
            "--res-block-nums", "2", "--report-every", "50", "--save-dir", d, "--checkpoint-every", "0"]
    plies = []
    for extra in (["--max-plies", "20"], ["--max-plies", "5", "--resume"]):
        r = subprocess.run(base + extra, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        assert json.loads(r.stdout.splitlines()[-1])["plies"] == (20 if not plies else 25)
        with np.load(os.path.join(d, "games.npz"), allow_pickle=False) as g:
            plies.append(int(g["plies"]))
    assert plies[1] == plies[0] + 8 * 5                                # the saved games' ply count continued: they were loaded
    shutil.rmtree(d)
