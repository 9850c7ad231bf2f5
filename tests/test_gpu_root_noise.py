"""Root exploration noise on the device (SelfPlay(root_noise=(eps, alpha)): a root-expansion pre-pass, cz_host_dirichlet and
k_root_noise): the kernel against the formula word for word, the pre-pass's transparency at eps = 0, whole self-play games against the
specification trees (tests/search_spec.py) under both rules and both search schedules, and exact resumes.  Bit-exact everywhere."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

import search_spec as S

pytestmark = pytest.mark.gpu


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


def _root_p_words(blob, B, narr):
    """word indices (into the blob as uint32) of every game's root P array, from the snapshot layout of include/cchess_b200.h"""
    w = blob.view(np.uint32)
    off = blob[48:48 + 8 * (B + 1)].view(np.int64)
    F = 52 if narr == 5 else 80
    out = {}
    for g in range(B):
        s = int(off[g])
        hdr = w[s:s + 16]
        cnt, base = int(np.int32(hdr[5])), int(hdr[6])
        out[g] = s + F + base + 8 + np.arange(max(cnt, 0))
    return out


def _selfplay(kind, B, P, seeds, noise, net="hash_signed", auto_reset=False, graph=True):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    kw = dict(search_threads=16) if kind == "fifo" else dict(rules="strict") if kind == "strict" else {}
    sp = SelfPlay(B, FakeNet(net), P, seeds=seeds, arena_words=1 << 18, auto_reset=auto_reset, root_noise=noise, **kw)
    if graph:
        sp.capture_graph()
    return sp


@pytest.mark.parametrize("kind", ["reference", "fifo", "strict"])
def test_kernel_equals_the_formula_and_changes_nothing_else(kind):
    B, eps = 24, 0.25
    sp = _selfplay(kind, B, 40, range(B), None, auto_reset=True)
    for _ in range(5):                                     # mid-game trees whose roots carry visits
        sp.step()
    e = sp.engine
    rng = np.random.RandomState(3)
    mask = (rng.rand(B) < 0.7) & sp.live
    e.begin_search(0, mask.astype(np.uint8))
    sp._run_waves(0, graph=False)                         # the pre-pass: expands the roots reached by an unvisited move
    assert e.unfinished() == 0
    n = e.root_counts()
    rc = e.root_children(want_wpq=True)
    assert np.array_equal(n, rc["n"]) and (n[mask] > 0).sum() >= 8 and (~mask).sum() >= 3
    before_sig = [e.tree_signature(g) for g in range(B)]
    before = e.snapshot()
    eta = np.zeros((B, 128))
    for g in range(B):
        if n[g] > 0:
            eta[g, :n[g]] = rng.dirichlet(0.3 * np.ones(n[g]))
    e.root_noise(mask.astype(np.uint8), eta, eps)
    after = e.snapshot()
    p = e.root_children(want_wpq=True)["p"]
    for g in range(B):
        k = max(int(n[g]), 0)                              # (-1: a root that was not searched and is not expanded)
        want = S.mix(rc["p"][g, :k], eta[g, :k], eps) if mask[g] else rc["p"][g, :k]
        assert np.array_equal(p[g, :k].view(np.uint32), want.view(np.uint32)), g
        sig = e.tree_signature(g)
        roots = _root_records(sig)
        assert np.array_equal(sig[roots, 3], want.view(np.uint32).astype(np.int64)), g
        keep = np.ones(len(sig), bool)
        keep[roots] = False
        assert np.array_equal(np.delete(sig, 3, axis=1), np.delete(before_sig[g], 3, axis=1)), g
        assert np.array_equal(sig[keep], before_sig[g][keep]), g
    # every word of the engine state outside the root P arrays of the masked games is unchanged
    words = _root_p_words(before, B, 6 if kind == "fifo" else 5)
    changed = np.nonzero(before.view(np.uint32) != after.view(np.uint32))[0]
    allowed = np.concatenate([words[g] for g in range(B) if mask[g]])
    assert np.isin(changed, allowed).all() and len(changed) > 0
    # eps = 1 puts eta in place
    e.root_noise(mask.astype(np.uint8), eta, 1.0)
    p1 = e.root_children(want_wpq=True)["p"]
    for g in np.nonzero(mask)[0]:
        assert np.array_equal(p1[g, :n[g]], eta[g, :n[g]].astype(np.float32)), g
    with pytest.raises(ValueError, match="eps"):
        e.root_noise(mask.astype(np.uint8), eta, 1.5)


def _run(sp, plies):
    log = []
    for _ in range(plies):
        out = sp.step()
        rc = sp.engine.root_children(want_wpq=True)
        vis = np.where(np.arange(128) < rc["n"][:, None], rc["visits"], -1)       # (entries past n are not written)
        log.append((out["choice"].copy(), vis, rc["n"].copy(),
                    [sp.engine.tree_signature(g) for g in range(sp.B)]))
        if not sp.live.any():
            break
    return log


@pytest.mark.parametrize("kind,graph", [("reference", True), ("reference", False), ("fifo", True), ("fifo", False), ("strict", True)])
def test_prepass_is_transparent_at_eps_zero(kind, graph):
    B, P = 16, 48 if kind == "fifo" else 32
    seeds = [70 + 3 * g for g in range(B)]
    a = _selfplay(kind, B, P, seeds, None, graph=graph, auto_reset=True)
    b = _selfplay(kind, B, P, seeds, (0.0, 0.3), graph=graph, auto_reset=True)
    with np.errstate(all="ignore"):
        la, lb = _run(a, 40), _run(b, 40)
    for x, y in zip(la, lb):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and np.array_equal(x[2], y[2])
        for sx, sy in zip(x[3], y[3]):
            sx, sy = sx.copy(), sy.copy()
            for s in (sx, sy):
                s[s[:, 3] == 0x80000000, 3] = 0                 # -0.0 -> +0.0: the one bit a mix with eps = 0 can change
            assert np.array_equal(sx, sy)
    assert a.plies == b.plies
    fa, fb = a.pop_finished(), b.pop_finished()
    assert [g for g, _ in fa] == [g for g, _ in fb]
    for (_, ra), (_, rb) in zip(fa, fb):
        assert ra.states == rb.states and ra.actions == rb.actions and np.array_equal(ra.z, rb.z)
        assert np.array_equal(ra.dense_pi(), rb.dense_pi())
    assert b.engine.raise_on_error() is not None


@pytest.mark.parametrize("kind", ["reference", "fifo", "strict"])
def test_noisy_selfplay_games_equal_the_specification(kind):
    B, P, eps, alpha, net = 8, 24 if kind != "fifo" else 40, 0.25, 0.3, "hash_signed"
    seeds = [300 + 13 * g for g in range(B)]
    sp = _selfplay(kind, B, P, seeds, (eps, alpha), net=net)
    with np.errstate(all="ignore"):
        out = sp.play_games()
    assert len(out) == B
    for slot, rec in out:
        with np.errstate(all="ignore"):
            r = S.selfplay_game(net, P, np.random.RandomState(seeds[slot]), rules="strict" if kind == "strict" else "reference",
                                search_threads=16 if kind == "fifo" else 1,
                                root_noise=(eps, alpha, np.random.RandomState([seeds[slot], 1])))
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert [tuple(int(v) for v in x) for x in rec.visits] == r["visits"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot


@pytest.mark.parametrize("kind", ["reference", "fifo"])
def test_noisy_selfplay_resumes_exactly(kind, tmp_path):
    B, P = 12, 32
    seeds = [50 + g for g in range(B)]
    a = _selfplay(kind, B, P, seeds, (0.25, 0.3), auto_reset=True)
    with np.errstate(all="ignore"):
        _run(a, 25)
        a.pop_finished()
        path = str(tmp_path / "games.npz")
        a.save_games(path)
        b = _selfplay(kind, B, P, [999] * B, (0.25, 0.3), auto_reset=True)
        b.load_games(path)
        la, lb = _run(a, 30), _run(b, 30)
    for x, y in zip(la, lb):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        assert all(np.array_equal(s, t) for s, t in zip(x[3], y[3]))
    assert np.array_equal(a._noise_mt, b._noise_mt) and np.array_equal(a._mt, b._mt)
    fa, fb = a.pop_finished(), b.pop_finished()
    assert len(fa) == len(fb)
    for (_, ra), (_, rb) in zip(fa, fb):
        assert ra.states == rb.states and np.array_equal(ra.dense_pi(), rb.dense_pi()) and np.array_equal(ra.z, rb.z)


def _net(tmp, name, seed=0, blocks=2):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(blocks, seed=seed, save_dir=os.path.join(str(tmp), name))


def test_noisy_trainer_resume_is_bit_identical(tmp_path, monkeypatch):
    from cchess_zero_b200.train import Trainer
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)
    monkeypatch.chdir(tmp_path)
    run = str(tmp_path / "run")
    kw = dict(batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16, root_noise=(0.25, 0.3))
    ta = Trainer(_net(tmp_path, "a"), 16, 8, seed=3, **kw)
    assert ta.sp.root_noise == (0.25, 0.3)
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
        tn = Trainer(_net(tmp_path, "c", seed=5), 16, 8, seed=9, **dict(kw, root_noise=None))
        with pytest.raises(ValueError, match="root noise"):
            tn.load(run)
    assert all(np.array_equal(x, y) for x, y in zip(log_a, log_b))
    assert all(np.array_equal(ta.sp.engine.tree_signature(g), tb.sp.engine.tree_signature(g)) for g in range(16))
    for name in ("boards", "n", "idx", "prob", "z"):
        assert torch.equal(getattr(ta.buffer, name), getattr(tb.buffer, name)), name
    assert (ta.games, ta.positions, ta.updates, ta.plies) == (tb.games, tb.positions, tb.updates, tb.plies)
    assert np.array_equal(ta.sp._noise_mt, tb.sp._noise_mt)


def test_gate_matches_stay_noise_free(tmp_path, monkeypatch):
    import cchess_zero_b200.arena as A
    from cchess_zero_b200.train import Trainer
    seen = []

    def spy(real):
        def make(*a, **kw):
            seen.append(kw.get("root_noise"))
            return real(*a, **kw)
        return make
    monkeypatch.setattr(A, "SelfPlay", spy(A.SelfPlay))
    monkeypatch.setattr(A, "network_selfplay", spy(A.network_selfplay))
    monkeypatch.chdir(tmp_path)
    with contextlib.redirect_stdout(io.StringIO()):
        t = Trainer(_net(tmp_path, "a"), 4, 8, eval_every=1, eval_games=2, batch_size=8, buffer_size=64, checkpoint_every=0,
                    arena_words=1 << 16, root_noise=(0.25, 0.3))
        t.gate()
    assert seen and all(x is None for x in seen)
