"""GPU tests of the reference-shaped surface: policy_value_network (forward / train_step / save / restore),
MCTS_tree and cchess_main drop-ins against the reference's golden vectors, and the real-network self-play path."""
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu


def sha(b):
    return hashlib.sha256(b).hexdigest()[:16]


def _positions(n, seed=0):
    from oracle import oracle as O
    rng = np.random.RandomState(seed)
    xs, b, side = [], O.from_state(O.START), 0
    while len(xs) < n:
        xs.append(O.encode(b, side))
        mv = O.legal_moves(b, side)
        b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
        if cap in (1, 8):
            b, side = O.from_state(O.START), 0
    return np.stack(xs)


@pytest.mark.parametrize("blocks", [7, 19])
def test_network_within_1e3_of_fp64(blocks):
    """north_star: NN outputs match within 1e-3 of an fp32/fp64 evaluation.  Tolerance 1e-3 absolute on
    logits and value; bf16 is measured too and is expected to miss it (that is why it is not the default)."""
    from cchess_zero_b200.net import InferencePlan, PolicyValueNet
    torch.manual_seed(0)
    net = PolicyValueNet(blocks).eval()
    x = torch.from_numpy(_positions(96))
    with torch.no_grad():
        rl, rv = net.double()(x.double())
    net = net.float().cuda().to(memory_format=torch.channels_last)
    err = {}
    for prec in ("fp32", "tf32", "fp16", "bf16"):
        plan = InferencePlan(net, prec)
        l, v = plan(x.cuda().to(plan.dtype))
        err[prec] = max((l.double().cpu() - rl).abs().max().item(), (v.double().cpu().reshape(-1) - rv.reshape(-1)).abs().max().item())
    print("max abs error vs fp64:", err)
    assert err["fp32"] < 1e-5
    assert err["tf32"] < 1e-3
    assert err["fp16"] < 1e-3      # the default inference precision


def test_policy_value_network_surface(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200.net import policy_value_network
    pv = policy_value_network(res_block_nums=2)
    x = _positions(12)
    lo, v = pv.forward(list(x))                      # the reference passes python lists (main.py:1170)
    assert lo.shape == (12, 2086) and lo.dtype == np.float32 and v.shape == (12, 1) and v.dtype == np.float32
    assert np.all(np.abs(v) <= 1)
    lo1, v1 = pv.forward(x[:1])
    assert np.allclose(lo1, lo[:1], atol=2e-3)
    pi = np.zeros((12, 2086), dtype=np.float32)
    pi[np.arange(12), np.arange(12) * 7] = 1
    z = np.where(np.arange(12) % 2 == 0, 1.0, -1.0).reshape(12, 1)
    losses = []
    for _ in range(8):
        acc, loss, step = pv.train_step(x, pi, z, 0.01)
        losses.append(loss)
    assert step == 8 and np.isfinite(losses).all() and losses[-1] < losses[0]
    lo2, v2 = pv.forward(x)
    path = pv.save(step)
    assert os.path.exists(path)
    pv2 = policy_value_network(res_block_nums=2)     # train_restore picks the checkpoint up (policy_value_network.py:164-174)
    assert pv2.global_step == 8
    lo3, v3 = pv2.forward(x)
    assert np.array_equal(lo2, lo3) and np.array_equal(v2, v3)


def test_mcts_tree_dropin_against_reference_vectors():
    from cchess_zero_b200.mcts import MCTS_tree
    from oracle.fakenets_np import FAKE_NETS
    for c in load_golden("tree.json")["cases"]:
        if c["playouts"] > 300:
            continue
        t = MCTS_tree(c["state"], FAKE_NETS[c["net"]], 1)          # the goldens are search_threads=1 runs of the reference
        t._set_position(c["state"], c["player"], c["rr"])
        t.main(c["state"], c["player"], c["rr"], c["playouts"])
        got = [[a, n.N] for a, n in t.root.child.items()]
        assert got == [[r[0], r[1]] for r in c["root"]], c["note"]
        for (a, n), r in zip(t.root.child.items(), c["root"]):
            q = np.float32(n.Q)
            assert (0x7FC00000 if np.isnan(q) else int(q.view(np.uint32))) == r[4]
        assert t.Q(c["root"][0][0]) == t.root.child[c["root"][0][0]].Q


def test_cchess_main_selfplay_dropin_against_reference_vectors(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200.selfplay import cchess_main
    from oracle.fakenets_np import FAKE_NETS

    class Net:
        def __init__(self, f):
            self.forward = f

    for g in load_golden("selfplay.json")["games"][:2]:
        m = cchess_main(playout=g["playouts"], in_search_threads=1, network=Net(FAKE_NETS[g["net"]]), log_file=False)
        np.random.seed(g["seed"])
        import contextlib, io
        with contextlib.redirect_stdout(io.StringIO()):
            data, n = m.selfplay()
        data = list(data)
        assert n == g["n"]
        assert [d[0] for d in data] == g["states"]
        assert [float(d[2]) for d in data] == g["z"]
        assert sha(np.asarray([d[1] for d in data], dtype=np.float64).tobytes()) == g["sha_pi"]
        ended, who = m.check_end()
        assert ended and who in ("w", "b", "t")


@pytest.mark.parametrize("precision,graph", [("fp16", True), ("tf32", False)])
def test_selfplay_with_real_network(precision, graph, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import SelfPlay
    pv = policy_value_network(res_block_nums=2, precision=precision)
    plan = pv.plan()
    B, P = 64, 24
    sp = SelfPlay(B, None, P, seeds=range(B), nn_dtype=plan.dtype, arena_words=1 << 18)
    sp.forward = lambda x: plan(x, sp.logits, sp.value)
    if graph:
        sp.capture_graph()
    for _ in range(6):
        sp.step()
    c = sp.engine.raise_on_error()
    assert c["n_playout"] == 6 * B * P
    assert 0 < c["n_expand"] <= c["n_playout"] + 6 * B
    st = sp.engine.status()
    assert (st["ply"] <= 6).all() and st["ply"].max() == 6


@pytest.mark.parametrize("blocks,first_conv", [(2, "gather"), (7, "gather"), (2, "tc"), (7, "tc"), (2, "mma"), (7, "mma")])
def test_native_network_ends_match_library_plan(blocks, first_conv, tmp_path, monkeypatch):
    """csrc/cz_net.cu (first conv from board bytes, fused heads) against the cuDNN/cuBLAS plan and against fp64.  The gather-add is
    the only first-convolution kernel: native_plan builds it for first_conv="gather" and refuses the removed "tc" / "mma" variants."""
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200 import rules
    from cchess_zero_b200.net import InferencePlan, NativePlan, PolicyValueNet, policy_value_network
    from cchess_zero_b200.selfplay import _flip_board
    from oracle import oracle as O
    torch.manual_seed(1)
    net = PolicyValueNet(blocks).eval()
    with torch.no_grad():   # non-trivial biases / BN statistics so that every folded term is exercised
        for m in net.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                m.bias.uniform_(-0.1, 0.1)
            if hasattr(m, "running_var"):
                m.running_var.uniform_(0.5, 1.5); m.running_mean.uniform_(-0.2, 0.2)
    rng = np.random.RandomState(3)
    boards, sides = [], []
    b, side = O.from_state(O.START), 0
    while len(boards) < 203:     # odd batch: exercises the tails of every kernel
        boards.append(b.copy()); sides.append(side)
        mv = O.legal_moves(b, side)
        b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
        if cap in (1, 8):
            b, side = O.from_state(O.START), 0
    enc = rules.encode_batch(np.stack(boards), sides)
    canon = np.zeros((len(boards), 96), dtype=np.uint8)
    for i, (bb, s) in enumerate(zip(boards, sides)):
        canon[i, :90] = _flip_board(bb) if s == 1 else bb
    with torch.no_grad():
        rl, rv = net.double()(torch.from_numpy(enc).double())
    net = net.float().cuda().to(memory_format=torch.channels_last)
    B = len(boards)
    lib_l, lib_v = InferencePlan(net, "fp16")(torch.from_numpy(enc).cuda().half())
    nat = NativePlan(net, 256)
    assert nat.first_conv == "gather"
    lo = torch.zeros((B, 2086), device="cuda"); vo = torch.zeros((B,), device="cuda")
    nat(torch.from_numpy(canon).cuda(), lo, vo)
    torch.cuda.synchronize()
    e_nat = max((lo.double().cpu() - rl).abs().max().item(), (vo.double().cpu() - rv.reshape(-1)).abs().max().item())
    e_lib = max((lib_l.double().cpu() - rl).abs().max().item(), (lib_v.double().cpu().reshape(-1) - rv.reshape(-1)).abs().max().item())
    print("max abs err vs fp64: native %.3g library %.3g" % (e_nat, e_lib))
    assert e_nat < 1e-3
    assert (lo - lib_l).abs().max().item() < 2e-3
    pv = policy_value_network(res_block_nums=1)
    if first_conv == "gather":
        assert pv.native_plan(8, first_conv).first_conv == "gather"
    else:
        with pytest.raises(ValueError):
            pv.native_plan(8, first_conv)


def test_selfplay_native_plan_board_mode(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import SelfPlay
    pv = policy_value_network(res_block_nums=2, precision="fp16")
    B, P = 96, 20
    sp = SelfPlay(B, None, P, seeds=range(B), arena_words=1 << 18, plan=pv.native_plan(B))
    sp.capture_graph()
    for _ in range(5):
        sp.step()
    c = sp.engine.raise_on_error()
    assert c["n_playout"] == 5 * B * P
    # the canonical boards handed to the network are the flipped root boards of the reference
    sp2 = SelfPlay(B, None, P, seeds=range(B), arena_words=1 << 18, plan=pv.plan())
    for _ in range(5):
        sp2.step()
    # same seeds + (numerically close) network: the opening plies normally coincide; at least the engines agree on ply counts
    assert (sp.engine.status()["ply"] == sp2.engine.status()["ply"]).all()


def test_mcts_tree_with_package_network_and_move_latency(tmp_path, monkeypatch):
    """BASELINE config 5 shape: one tree, the package's own network, select_move('mcts') for both sides."""
    monkeypatch.chdir(tmp_path)
    import contextlib, io, time
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import cchess_main
    pv = policy_value_network(res_block_nums=7)
    m = cchess_main(playout=200, in_search_threads=1, network=pv, exploration=False, log_file=False)
    np.random.seed(0)
    lat = []
    with contextlib.redirect_stdout(io.StringIO()):
        for _ in range(4):
            t0 = time.perf_counter()
            (sx, sy, dx, dy), win = m.select_move("mcts")
            lat.append(time.perf_counter() - t0)
            assert 0 <= sx < 9 and 0 <= sy < 10 and -1 <= float(win) <= 1
    visits = [n.N for n in m.mcts.root.child.values()]
    assert m.game_borad.round == 5 and m.game_borad.current_player == "w"
    assert sum(visits) <= 200 + m.mcts.root.N
    print("move latency (200 playouts, 7 blocks): %s" % ["%.3f" % x for x in lat])
    assert min(lat) < 5.0


def test_headless_play_mode_ai_vs_ai(tmp_path, monkeypatch):
    """--mode play --ai_count 2 of the reference (ChessGame.game_mode_2) without tkinter."""
    monkeypatch.chdir(tmp_path)
    import contextlib, io
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.play import ChessGame
    np.random.seed(3)
    with contextlib.redirect_stdout(io.StringIO()):
        g = ChessGame(2, "mcts", 64, network=policy_value_network(res_block_nums=2))
        who = g.start(max_moves=12)
    assert who in ("", "w", "b", "t")
    assert g.cchess_engine.game_borad.round >= 2 and len(g.move_times) >= 1
    with contextlib.redirect_stdout(io.StringIO()):
        g2 = ChessGame(2, "net", 64, network=g.cchess_engine.policy_value_netowrk)
        g2.start(max_moves=4)
    assert g2.cchess_engine.game_borad.round == 5


def test_play_mode_surface_against_reference_vectors(tmp_path, monkeypatch):
    """select_move / get_hint / human_move / check_end (main.py:1278-1329, 1380-1491) replayed against what the reference
    itself returned (tests/golden/play.json), for human_color 'b' and 'w' (the rank-flip convention) and the 'net' branches."""
    monkeypatch.chdir(tmp_path)
    import contextlib, io
    from cchess_zero_b200.selfplay import cchess_main
    from oracle.fakenets_np import FAKE_NETS

    class Net:
        def __init__(self, f):
            self.forward = f

    for sc in load_golden("play.json")["scripts"]:
        m = cchess_main(playout=sc["playouts"], in_search_threads=1, network=Net(FAKE_NETS[sc["net"]]), exploration=False,
                        human_color=sc["human_color"], log_file=False)
        if sc["seed"] is not None:
            np.random.seed(sc["seed"])
        with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
            for i, st in enumerate(sc["steps"]):
                op = st["op"]
                if op in ("select_move_mcts", "select_move_net"):
                    mv, wr = m.select_move("mcts" if op.endswith("mcts") else "net")
                    assert [int(x) for x in mv] == st["move"], (sc["human_color"], i)
                    assert float(wr).hex() == st["win_rate"], (sc["human_color"], i)
                    assert m.game_borad.state == st["state"]
                    if "player" in st:
                        assert m.game_borad.current_player == st["player"] and m.game_borad.restrict_round == st["rr"]
                elif op in ("get_hint_mcts", "get_hint_net"):
                    hint = m.get_hint("mcts" if op.endswith("mcts") else "net", op.endswith("mcts"), lambda: None)
                    assert [[a, float(p).hex()] for a, p in hint] == st["hint"], (sc["human_color"], i, op)
                elif op == "human_move_mcts":
                    wr = m.human_move(tuple(st["coord"]), "mcts")
                    assert float(wr).hex() == st["win_rate"], (sc["human_color"], i)
                    assert m.game_borad.state == st["state"] and m.game_borad.current_player == st["player"]
                    assert m.game_borad.restrict_round == st["rr"]
                elif op == "check_end":
                    ended, who = m.check_end()
                    assert bool(ended) == st["ended"] and who == st["who"]


def test_leaf_parallel_move_latency_mode(tmp_path, monkeypatch):
    """cchess_main(..., leaf_parallel=8): same API, up to 8 leaves of the one tree per network call."""
    monkeypatch.chdir(tmp_path)
    import contextlib, io, time
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import cchess_main
    pv = policy_value_network(res_block_nums=7)
    lat = {}
    for K in (1, 8):
        m = cchess_main(playout=400, in_search_threads=1, network=pv, exploration=False, log_file=False, leaf_parallel=K)
        np.random.seed(0)
        ts = []
        with contextlib.redirect_stdout(io.StringIO()):
            for _ in range(5):
                t0 = time.perf_counter()
                m.select_move("mcts")
                ts.append(time.perf_counter() - t0)
        lat[K] = min(ts[1:])
        assert m.game_borad.round == 6
    print("move latency 400 playouts: K=1 %.4f s, K=8 %.4f s" % (lat[1], lat[8]))
    assert lat[8] < lat[1]
