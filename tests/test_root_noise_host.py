"""Root exploration noise, host side: cz_host_dirichlet against numpy's RandomState.dirichlet, argument validation, the SelfPlay
search loop over CPU stand-in trees (draw order, which games draw, whole games against the specification), and the refusals of
save / load files and Trainer runs saved with another root noise setting.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import root_noise_support as R

MT_WORDS = 626


def _mt(seeds):
    mt = np.zeros((len(seeds), MT_WORDS), np.uint32)
    for g, sd in enumerate(seeds):
        st = np.random.RandomState([int(sd), 1]).get_state()
        mt[g, :624], mt[g, 624] = st[1], st[2]
    return mt


def _rs(row):
    rs = np.random.RandomState()
    rs.set_state(("MT19937", row[:624].copy(), int(row[624]), 0, 0.0))
    return rs


def _dirichlet(mask, n, alpha, mt, eta, threads=1):
    from cchess_zero_b200._lib import lib
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    return lib().cz_host_dirichlet(len(n), vp(mask), vp(n), C.byref(C.c_double(alpha)), vp(mt), vp(eta), threads)


@pytest.mark.parametrize("alpha", [0.03, 0.15, 0.3, 0.9])
@pytest.mark.parametrize("threads", [1, 4])
def test_host_dirichlet_is_numpy_bit_for_bit(alpha, threads):
    n = np.concatenate([np.arange(1, 129), [0, -1, 5, 7]]).astype(np.int32)
    B = len(n)
    mask = np.ones(B, np.uint8)
    mask[[3, 64, 130]] = 0                                  # masked out games and n <= 0 games draw nothing
    mt = _mt(range(1000, 1000 + B))
    before = mt.copy()
    eta = np.full((B, 128), -7.0)
    for rep in range(2):                                    # the second round continues each stream
        assert _dirichlet(mask, n, alpha, mt, eta, threads) == 0
        for g in range(B):
            if not mask[g] or n[g] <= 0:
                assert np.array_equal(mt[g], before[g]) and (eta[g] == -7.0).all(), g
                continue
            rs = _rs(before[g])
            for _ in range(rep + 1):
                want = rs.dirichlet(alpha * np.ones(int(n[g])))
            assert np.array_equal(eta[g, :n[g]], want), (g, rep)
            assert (eta[g, n[g]:] == -7.0).all()
            st = rs.get_state()
            assert np.array_equal(mt[g, :624], st[1]) and int(mt[g, 624]) == st[2], g


def test_host_dirichlet_refusals_leave_the_streams_alone():
    n = np.array([3, 129, 4], np.int32)
    mt = _mt([1, 2, 3])
    before = mt.copy()
    eta = np.zeros((3, 128))
    assert _dirichlet(None, n, 0.3, mt, eta) != 0                       # n > 128
    assert _dirichlet(np.array([1, 0, 1], np.uint8), n, 0.3, mt, eta) == 0   # ... unless that game is masked out
    assert not np.array_equal(mt[0], before[0]) and np.array_equal(mt[1], before[1])
    mt = before.copy()
    for bad in (0.0, 1.0, -0.3, 1.5, float("nan")):
        assert _dirichlet(None, np.array([3, 3, 3], np.int32), bad, mt, eta) != 0
    assert np.array_equal(mt, before)


def test_cz_host_choose_moves_is_unchanged():
    """The exploration mix of get_action still draws Dirichlet(0.3) (the shared sampler took alpha as a parameter)."""
    from cchess_zero_b200.selfplay import sample_moves
    rng = np.random.RandomState(5)
    B = 64
    n = rng.randint(1, 129, B).astype(np.int32)
    visits = rng.randint(0, 30, (B, 128)).astype(np.int32)
    visits[np.arange(B), 0] += 1
    mt = _mt(range(B))
    before = mt.copy()
    ch = sample_moves(n, visits, np.ones(B, bool), 1.0, mt, True, 4)
    with np.errstate(divide="ignore"):
        for g in range(B):
            rs = _rs(before[g])
            v = visits[g, :n[g]]
            lv = np.log(v.astype(np.int64)) * 1.0
            pr = np.exp(lv - np.max(lv)); pr /= np.sum(pr)
            p = 0.75 * pr + 0.25 * rs.dirichlet(0.3 * np.ones(int(n[g])))
            assert ch[g] == rs.choice(int(n[g]), p=p), g
            assert np.array_equal(mt[g, :624], rs.get_state()[1])


def test_root_noise_argument_is_validated():
    from cchess_zero_b200.selfplay import SelfPlay, check_root_noise
    from cchess_zero_b200.train import Trainer
    assert check_root_noise(None) is None
    assert check_root_noise((0.25, 0.3)) == (0.25, 0.3) and check_root_noise([0, 0.03]) == (0.0, 0.03)
    assert check_root_noise((1, 0.999)) == (1.0, 0.999)
    for bad in ((-0.01, 0.3), (1.01, 0.3), (0.25, 0.0), (0.25, 1.0), (0.25, -1), (float("nan"), 0.3), (0.25, float("nan"))):
        with pytest.raises(ValueError, match="root_noise: (eps|alpha)"):
            check_root_noise(bad)
    for bad in (0.25, (0.25,), (0.25, 0.3, 1), ("a", 0.3)):
        with pytest.raises(ValueError, match="root_noise must be"):
            check_root_noise(bad)
    with pytest.raises(ValueError, match="alpha"):
        SelfPlay(2, lambda x: None, 8, engine=R.StandIn(2, "hash_pos"), root_noise=(0.25, 1.5))
    with pytest.raises(ValueError, match="eps"):
        Trainer(None, 2, 8, root_noise=(2.0, 0.3))


def test_search_draws_in_slot_order_for_searched_live_games_with_children():
    from cchess_zero_b200.selfplay import SelfPlay
    B, eps, alpha = 6, 0.25, 0.3
    seeds = [40 + 7 * g for g in range(B)]
    e = R.StandIn(B, "hash_pos")
    sp = SelfPlay(B, lambda x: None, 16, seeds=seeds, engine=e, root_noise=(eps, alpha))
    rn = [np.random.RandomState([s, 1]) for s in seeds]
    sp.live[4] = False                                      # a game that is not running
    mask = np.array([1, 1, 0, 1, 1, 1], bool)               # a game that is not searched
    for rnd in range(3):
        e.log.clear()
        if rnd == 2:                                        # a root without children (a mated root under strict rules)
            counts = e.root_counts
            e.root_counts = lambda: np.where(np.arange(B) == 5, 0, counts()).astype(np.int32)
        sp.search(mask)
        calls = [c[0] for c in e.log]
        assert calls == ["begin_search", "root_counts", "root_noise", "begin_search"], calls
        assert e.log[0][1] == 0 and np.array_equal(e.log[0][2], mask)        # the pre-pass: 0 playouts, the searched games
        n = e.log[1][1] if rnd < 2 else np.where(np.arange(B) == 5, 0, e.log[1][1])
        sel = mask & sp.live & (n > 0)
        assert np.array_equal(e.log[2][1], sel)
        eta = e.log[2][2]
        for g in range(B):
            if sel[g]:
                assert np.array_equal(eta[g, :n[g]], rn[g].dirichlet(alpha * np.ones(int(n[g])))), (rnd, g)
        for g in range(B):
            st = rn[g].get_state()
            assert np.array_equal(sp._noise_mt[g, :624], st[1]) and sp._noise_mt[g, 624] == st[2], (rnd, g)
        assert e.log[2][3] == eps
    assert not e.log[2][1][5]
    e.root_counts = counts
    # a search of games none of which has a root with children draws nothing and launches no mix
    e.log.clear()
    sp.search(np.zeros(B, bool))
    assert [c[0] for c in e.log] == ["begin_search", "root_counts"]


@pytest.mark.parametrize("kind", ["reference", "strict"])
def test_selfplay_host_loop_with_noise_equals_the_specification(kind):
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net, eps, alpha = 3, 16, "hash_signed", 0.25, 0.3
    seeds = [900 + 11 * g for g in range(B)]
    sp = SelfPlay(B, lambda x: None, P, seeds=seeds, auto_reset=False, engine=R.StandIn(B, net, kind), rules=sp_rules(kind),
                  root_noise=(eps, alpha))
    with np.errstate(all="ignore"):
        out = sp.play_games(max_plies=120)
    for slot, rec in out:
        with np.errstate(all="ignore"):
            r = R.selfplay_game(kind, net, P, seeds[slot], eps, alpha)
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot


def sp_rules(kind):
    return "strict" if kind == "strict" else "reference"


def test_noise_changes_the_search_below_a_visited_root():
    """With eps > 0 the visit counts differ from the noise-free search once the root has visits of its own (a root reached by play:
    the tree's root N never grows during a search, so at a fresh root N = 0, U = 0 and the priors do not steer its children)."""
    from oracle import oracle as O
    b = O.from_state(O.START)
    plain, noisy = R.Tree("reference", b), R.Tree("reference", b)
    for t in (plain, noisy):
        assert t.search(0, 0, 200, "hash_pos") == 0
    R.noisy_search(plain, 0, 0, 0, "hash_pos", np.random.RandomState([1, 1]), 0.5, 0.03)     # noise at N = 0: no effect
    assert np.array_equal(plain.root_children()[2], noisy.root_children()[2])
    best = int(np.argmax(plain.root_children()[2]))
    for t in (plain, noisy):
        t.update(best)
    assert plain.search(1, 0, 200, "hash_pos") == 0
    R.noisy_search(noisy, 1, 0, 200, "hash_pos", np.random.RandomState([1, 1]), 0.5, 0.03)
    assert not np.array_equal(plain.root_children()[2], noisy.root_children()[2])


def test_games_file_refusals(tmp_path):
    from cchess_zero_b200.selfplay import SelfPlay
    B = 2

    def mk(noise):
        return SelfPlay(B, lambda x: None, 8, seeds=[3, 4], engine=R.StandIn(B, "hash_pos"), root_noise=noise)
    on, off = mk((0.25, 0.3)), mk(None)
    on.step()
    off.step()
    p_on, p_off = str(tmp_path / "on.npz"), str(tmp_path / "off.npz")
    on.pop_finished(); off.pop_finished()
    on.save_games(p_on)
    off.save_games(p_off)
    with np.load(p_on) as d:
        assert np.array_equal(d["noise_mt"], on._noise_mt)
    with np.load(p_off) as d:
        assert "noise_mt" not in d.files
    fresh_off, fresh_on = mk(None), mk((0.25, 0.3))
    keep_off, keep_on = (fresh_off._mt.copy(), fresh_off.plies), (fresh_on._mt.copy(), fresh_on._noise_mt.copy(), fresh_on.plies)
    with pytest.raises(ValueError, match="saved with root noise, this SelfPlay runs without"):
        fresh_off.load_games(p_on)
    with pytest.raises(ValueError, match="saved without root noise, this SelfPlay runs with"):
        fresh_on.load_games(p_off)
    assert np.array_equal(fresh_off._mt, keep_off[0]) and fresh_off.plies == keep_off[1]
    assert np.array_equal(fresh_on._mt, keep_on[0]) and np.array_equal(fresh_on._noise_mt, keep_on[1]) and fresh_on.plies == keep_on[2]
    fresh_on.load_games(p_on)
    assert np.array_equal(fresh_on._noise_mt, on._noise_mt) and np.array_equal(fresh_on._mt, on._mt)


def test_trainer_refuses_a_saved_run_with_another_root_noise_setting(tmp_path):
    from cchess_zero_b200.train import Trainer, _savez

    class SP:
        _mt = np.zeros((2, 626), np.uint32)
    t = Trainer.__new__(Trainer)
    t.sp, t.n_games, t.rules, t.root_noise = SP(), 2, "reference", None
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt, rules=np.asarray("reference"), root_noise=np.asarray([0.25, 0.3]),
           noise_mt=SP._mt)
    with pytest.raises(ValueError, match=r"root noise \(0.25, 0.3\), this Trainer None"):
        t.load(str(tmp_path))
    t.root_noise = (0.25, 0.15)
    with pytest.raises(ValueError, match=r"root noise \(0.25, 0.3\), this Trainer \(0.25, 0.15\)"):
        t.load(str(tmp_path))
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt, rules=np.asarray("reference"), root_noise=np.zeros(0))
    with pytest.raises(ValueError, match=r"root noise None, this Trainer \(0.25, 0.15\)"):
        t.load(str(tmp_path))
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt)                # saved before root noise existed: off
    with pytest.raises(ValueError, match=r"root noise None, this Trainer"):
        t.load(str(tmp_path))


def test_train_command_line_takes_root_noise(monkeypatch, tmp_path):
    import cchess_zero_b200.train as T
    seen = {}

    class Stop(Exception):
        pass

    def fake_trainer(*a, **kw):
        seen.update(kw)
        raise Stop
    monkeypatch.setattr(T, "Trainer", fake_trainer)
    monkeypatch.setattr("cchess_zero_b200.net.policy_value_network", lambda *a, **kw: type("N", (), {"save_dir": ""})())
    with pytest.raises(Stop):
        T.main(["--save-dir", str(tmp_path), "--root-noise", "0.25", "0.3"])
    assert seen["root_noise"] == [0.25, 0.3]
    with pytest.raises(Stop):
        T.main(["--save-dir", str(tmp_path)])
    assert seen["root_noise"] is None
