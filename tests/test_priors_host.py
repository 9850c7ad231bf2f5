"""Softmax priors, host side: csrc/cz_exp.h compiled for the host against numpy, the specification's priors against numpy's softmax,
shift invariance of softmax-prior trees, argument validation, the SelfPlay host loop over CPU stand-in trees against the specification,
games-file and Trainer refusals, and the command-line and UCCI plumbing.  No GPU needed."""
import io

import numpy as np
import pytest

import priors_spec as PS
import search_spec as S


def _ulps64(a, b):
    return np.abs(a.view(np.int64) - b.view(np.int64))


def test_cz_exp_is_within_one_ulp_of_numpy():
    x = np.concatenate([np.linspace(-760.0, 0.0, 2_000_001), -np.random.RandomState(0).rand(200_000) * 0.75,
                        np.linspace(-745.0, -708.0, 50_001)])             # the last range: subnormal results
    y, ref = PS.cz_exp(x), np.exp(x)
    assert (y >= 0).all()
    assert _ulps64(y, ref).max() <= 1
    sub = ref < np.finfo(np.float64).tiny
    assert sub.sum() > 10_000 and _ulps64(y[sub], ref[sub]).max() <= 1


def test_cz_exp_special_values():
    y = PS.cz_exp(np.array([0.0, -0.0, -np.inf, np.nan, -1e300, -746.5]))
    assert y[0] == 1.0 and y[1] == 1.0 and y[2] == 0.0 and np.isnan(y[3]) and y[4] == 0.0 and y[5] == 0.0


def _numpy_softmax(lg):
    l64 = np.asarray(lg, dtype=np.float32).astype(np.float64)
    e = np.exp(l64 - l64.max())
    return (e / e.sum()).astype(np.float32)


def _rows(seed, count):
    rng = np.random.RandomState(seed)
    for k in range(count):
        n = int(rng.choice([1, 2, 3, 17, 44, 90, 128]))
        kind = k % 5
        if kind == 0:
            lg = rng.randn(n) * rng.choice([0.01, 1.0, 8.0])
        elif kind == 1:                                          # ties, the maximum included
            lg = rng.choice([-1.5, 0.25, 2.0], n)
        elif kind == 2:                                          # +-80
            lg = rng.choice([-80.0, 80.0], n) + rng.randn(n) * 0.5
        elif kind == 3:
            lg = np.full(n, rng.randn())
        else:
            lg = rng.uniform(-80, 80, n)
        yield lg.astype(np.float32)


def test_specification_priors_are_the_softmax():
    for lg in _rows(1, 3000):
        P = PS.softmax(lg)
        ref = _numpy_softmax(lg)
        assert (P >= 0).all()
        assert np.abs(P.view(np.int32).astype(np.int64) - ref.view(np.int32)).max() <= 1, lg
        n = len(lg)
        assert abs(float(P.astype(np.float64).sum()) - 1.0) <= n * np.spacing(np.float32(1.0)), lg
    assert PS.softmax(np.array([3.5], np.float32))[0] == 1.0


def test_product_net_player_ranks_by_the_same_softmax():
    from cchess_zero_b200.selfplay import softmax_priors
    for lg in _rows(2, 400):
        a, b = softmax_priors(lg), PS.softmax(lg)
        assert np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32)).max() <= 1


def _sig_after(tree_cls, board, side, net, shift, plies=3, playouts=60):
    t = tree_cls(board)
    sigs = []
    for _ in range(plies):
        assert t.search(side, 0, playouts, net, shift) == 0
        sigs.append(t.signature())
        N = t.root_children()[1]
        t.update(int(np.argmax(N)))
        side ^= 1
    return sigs


@pytest.mark.parametrize("net", ["hash_signed", "mod17"])
def test_softmax_trees_do_not_see_a_logit_shift(net):
    """The stand-ins' logits lie on a 2^-23 grid in [-1, 1), so adding 1.0 is exact: the softmax is unchanged to the last bit, and with
    it every tree.  The reference priors change (the point of the feature)."""
    from strict_support import random_play
    from oracle import oracle as O
    boards, sides = random_play(5, 400)
    cases = [(O.from_state(O.START), 0)] + [(boards[i], int(sides[i])) for i in (50, 150, 390)]
    differ = 0
    for b, s in cases:
        if not ((b == 1).any() and (b == 8).any()):
            continue
        a0, a1 = _sig_after(PS.SoftmaxTree, b, s, net, 0.0), _sig_after(PS.SoftmaxTree, b, s, net, 1.0)
        assert all(np.array_equal(x, y) for x, y in zip(a0, a1))
        r0, r1 = _sig_after(PS.ReferenceTree, b, s, net, 0.0), _sig_after(PS.ReferenceTree, b, s, net, 1.0)
        differ += not all(np.array_equal(x, y) for x, y in zip(r0, r1))
    assert differ >= 2


@pytest.mark.parametrize("rules", ["reference", "strict"])
def test_reference_tree_of_the_softmax_spec_is_search_spec(rules):
    """ReferenceTree (shift 0) is search_spec.Tree: the softmax specification changes only the priors."""
    from oracle import oracle as O
    b = O.from_state(O.START)
    a, r = PS.ReferenceTree(b, rules), S.Tree(b, rules)
    for side in (0, 1):
        assert a.search(side, 0, 40, "hash_pos") == 0 and r.search(side, 0, 40, "hash_pos") == 0
        assert np.array_equal(a.signature(), r.signature())
        k = int(np.argmax(r.root_children()[1]))
        a.update(k), r.update(k)


def test_softmax_root_priors_are_the_softmax_of_the_root_logits():
    from oracle import oracle as O
    b = O.from_state(O.START)
    t = PS.SoftmaxTree(b)
    assert t.search(0, 0, 0, "hash_signed") == 0
    mv, _, _, P, _ = t.root_children()
    logits = O.fake_forward("hash_signed", O.encode(b, 0))[0][0]
    li = [O.label_index(int(m) & 127, int(m) >> 7) for m in mv]
    assert len(mv) == 44 and np.array_equal(P.view(np.int32), PS.softmax(logits[li]).view(np.int32))


def test_priors_argument_is_validated():
    from cchess_zero_b200.arena import Match
    from cchess_zero_b200.engine import Engine, check_priors
    from cchess_zero_b200.selfplay import SelfPlay
    from cchess_zero_b200.train import Trainer
    from cchess_zero_b200.ucci import UcciEngine
    assert check_priors("reference") == "reference" and check_priors("softmax") == "softmax"
    for bad in ("Softmax", "logits", None, 1):
        with pytest.raises(ValueError, match="priors must be 'reference' or 'softmax'"):
            check_priors(bad)
    with pytest.raises(ValueError, match="priors"):
        Engine(2, priors="soft")
    with pytest.raises(ValueError, match="priors"):
        SelfPlay(2, lambda x: None, 8, engine=S.StandIn(2, "hash_pos"), priors="soft")
    with pytest.raises(ValueError, match="uses the 'reference' priors, not 'softmax'"):
        SelfPlay(2, lambda x: None, 8, engine=S.StandIn(2, "hash_pos"), priors="softmax")
    with pytest.raises(ValueError, match="uses the 'softmax' priors, not 'reference'"):
        SelfPlay(2, lambda x: None, 8, engine=PS.StandIn(2, "hash_pos", priors="softmax"))
    with pytest.raises(ValueError, match="priors"):
        Match(None, None, 2, 8, priors="soft")
    with pytest.raises(ValueError, match="priors"):
        Trainer(None, 2, 8, priors="soft")
    with pytest.raises(ValueError, match="priors"):
        UcciEngine(lambda o: None, priors="soft")


@pytest.mark.parametrize("rules", ["reference", "strict"])
@pytest.mark.parametrize("noise", [None, (0.25, 0.3)])
def test_selfplay_host_loop_with_softmax_priors_equals_the_specification(rules, noise):
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net = 3, 16, "hash_signed"
    seeds = [700 + 7 * g for g in range(B)]
    sp = SelfPlay(B, lambda x: None, P, seeds=seeds, auto_reset=False, engine=PS.StandIn(B, net, rules, priors="softmax"),
                  rules=rules, root_noise=noise, priors="softmax")
    with np.errstate(all="ignore"):
        out = sp.play_games()
    assert len(out) == B
    for slot, rec in out:
        rn = None if noise is None else noise + (np.random.RandomState([seeds[slot], 1]),)
        with np.errstate(all="ignore"):
            r = PS.selfplay_game(net, P, np.random.RandomState(seeds[slot]), rules=rules, root_noise=rn, priors="softmax")
            ref = PS.selfplay_game(net, P, np.random.RandomState(seeds[slot]), rules=rules, root_noise=rn)
        assert rec.states == r["states"] and rec.actions == r["actions"], slot
        assert np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"]), slot
        assert rec.actions != ref["actions"] or not np.array_equal(rec.dense_pi(), ref["pis"]), slot


def test_games_file_refusals(tmp_path):
    from cchess_zero_b200.selfplay import SelfPlay
    B = 2

    def mk(priors):
        return SelfPlay(B, lambda x: None, 8, seeds=[3, 4], engine=PS.StandIn(B, "hash_pos", priors=priors), priors=priors)
    soft, ref = mk("softmax"), mk("reference")
    for sp in (soft, ref):
        sp.step()
        sp.pop_finished()
    p_soft, p_ref = str(tmp_path / "soft.npz"), str(tmp_path / "ref.npz")
    soft.save_games(p_soft)
    ref.save_games(p_ref)
    with np.load(p_soft) as d:
        assert str(d["priors"]) == "softmax"
    with np.load(p_ref) as d:
        assert "priors" not in d.files                         # a default run's file is as it was
    fresh_ref, fresh_soft = mk("reference"), mk("softmax")
    keep = fresh_ref._mt.copy(), fresh_soft._mt.copy()
    with pytest.raises(ValueError, match="saved with 'softmax' priors, this SelfPlay uses 'reference'"):
        fresh_ref.load_games(p_soft)
    with pytest.raises(ValueError, match="saved with 'reference' priors, this SelfPlay uses 'softmax'"):
        fresh_soft.load_games(p_ref)
    assert np.array_equal(fresh_ref._mt, keep[0]) and np.array_equal(fresh_soft._mt, keep[1])
    fresh_soft.load_games(p_soft)
    assert np.array_equal(fresh_soft._mt, soft._mt) and fresh_soft.plies == soft.plies


def test_trainer_refuses_a_saved_run_with_other_priors(tmp_path):
    from cchess_zero_b200.train import Trainer, _savez

    class SP:
        _mt = np.zeros((2, 626), np.uint32)
    t = Trainer.__new__(Trainer)
    t.sp, t.n_games, t.rules, t.root_noise, t.priors = SP(), 2, "reference", None, "reference"
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt, rules=np.asarray("reference"), root_noise=np.zeros(0), priors=np.asarray("softmax"))
    with pytest.raises(ValueError, match="saved run uses the 'softmax' priors, this Trainer 'reference'"):
        t.load(str(tmp_path))
    _savez(str(tmp_path / "trainer.npz"), mt=SP._mt, rules=np.asarray("reference"), root_noise=np.zeros(0))
    t.priors = "softmax"
    with pytest.raises(ValueError, match="saved run uses the 'reference' priors, this Trainer 'softmax'"):
        t.load(str(tmp_path))


class _Stop(Exception):
    pass


def _spy(seen):
    def make(*a, **kw):
        seen.update(kw)
        raise _Stop
    return make


def test_train_command_line_takes_priors(monkeypatch, tmp_path):
    import cchess_zero_b200.train as T
    seen = {}
    monkeypatch.setattr(T, "Trainer", _spy(seen))
    monkeypatch.setattr("cchess_zero_b200.net.policy_value_network", lambda *a, **kw: type("N", (), {"save_dir": ""})())
    with pytest.raises(_Stop):
        T.main(["--save-dir", str(tmp_path), "--priors", "softmax"])
    assert seen["priors"] == "softmax"
    with pytest.raises(_Stop):
        T.main(["--save-dir", str(tmp_path)])
    assert seen["priors"] == "reference"
    with pytest.raises(SystemExit):
        T.main(["--save-dir", str(tmp_path), "--priors", "logits"])


def test_arena_command_line_takes_priors(monkeypatch):
    import cchess_zero_b200.arena as A
    seen = {}
    monkeypatch.setattr(A, "Match", _spy(seen))
    monkeypatch.setattr(A, "_network", lambda *a, **kw: None)
    with pytest.raises(_Stop):
        A.main(["--priors", "softmax", "--games", "2"])
    assert seen["priors"] == "softmax"
    with pytest.raises(_Stop):
        A.main(["--games", "2"])
    assert seen["priors"] == "reference"


def test_play_command_line_takes_priors(monkeypatch):
    import cchess_zero_b200.play as P
    seen = {}
    monkeypatch.setattr(P, "ChessGame", _spy(seen))
    monkeypatch.setattr("sys.argv", ["play", "--priors", "softmax"])
    with pytest.raises(_Stop):
        P.main()
    assert seen["priors"] == "softmax"


def test_ucci_priors_option_rebuilds_the_driver(monkeypatch):
    from cchess_zero_b200 import ucci
    made = []

    def make(options):
        made.append(dict(options))
        return type("D", (), {"playout_counts": options["playouts"]})()
    eng = ucci.UcciEngine(make, out=io.StringIO(), priors="softmax")
    eng.out = io.StringIO()
    assert eng.handle("ucci")
    assert "option priors type combo default softmax var reference var softmax" in eng.out.getvalue().splitlines()
    assert eng.handle("isready") and made[-1]["priors"] == "softmax"
    eng.out = io.StringIO()
    assert eng.handle("setoption name priors value reference")
    assert eng._driver is None and eng.options["priors"] == "reference"
    assert eng.handle("isready") and made[-1]["priors"] == "reference" and len(made) == 2
    eng.out = io.StringIO()
    assert eng.handle("setoption name priors value logits")
    assert "priors must be reference or softmax" in eng.out.getvalue() and eng.options["priors"] == "reference"
    assert eng._driver is not None
    seen = {}
    monkeypatch.setattr(ucci, "UcciEngine", _spy(seen))
    monkeypatch.setattr("sys.argv", ["ucci", "--priors", "softmax"])
    with pytest.raises(_Stop):
        ucci.main()
    assert seen["priors"] == "softmax"


@pytest.mark.parametrize("priors", ["reference", "softmax"])
def test_cchess_main_batched_paths_search_with_its_priors(monkeypatch, priors):
    """selfplay_many (SelfPlay) and policy_evaluate (arena.Match) build their engines with the instance's priors."""
    import cchess_zero_b200.arena as A
    import cchess_zero_b200.selfplay as SP
    seen = {}

    def spy(name):
        def make(*a, **kw):
            seen[name] = kw
            raise _Stop
        return make
    monkeypatch.setattr(SP, "SelfPlay", spy("selfplay_many"))
    monkeypatch.setattr(A, "Match", spy("policy_evaluate"))
    m = SP.cchess_main.__new__(SP.cchess_main)
    m.policy_value_netowrk = type("N", (), {"plan": lambda self: None})()
    m.playout_counts, m.exploration, m.temperature, m.search_threads, m.priors = 8, False, 1, 1, priors
    with pytest.raises(_Stop):
        m.selfplay_many(2)
    with pytest.raises(_Stop):
        m.policy_evaluate(2)
    assert seen["selfplay_many"]["priors"] == priors and seen["policy_evaluate"]["priors"] == priors
