"""The training loop on the GPU (cchess_zero_b200/train.py): cz_replay_batch against the host path and the C oracle, Trainer.policy_update
against cchess_main.policy_update, a small end-to-end loop with its gate, resume, and the CLI."""
import contextlib
import ctypes as C
import io
import json
import os
import random
import subprocess
import sys
from collections import deque

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu


def _net(tmp, name, seed=0, blocks=2):
    from cchess_zero_b200.net import policy_value_network
    with contextlib.redirect_stdout(io.StringIO()):
        return policy_value_network(blocks, seed=seed, save_dir=os.path.join(str(tmp), name))


@pytest.fixture(scope="module")
def games(tmp_path_factory):
    """A few dozen whole games of real self-play (2-block network, 16 playouts) packed as the loop packs them."""
    from cchess_zero_b200.distributed import pack_records
    from cchess_zero_b200.selfplay import network_selfplay
    pv = _net(tmp_path_factory.mktemp("net"), "models")
    sp = network_selfplay(pv, 32, 16, seeds=range(32), auto_reset=False, arena_words=1 << 16)
    sp.capture_graph()
    recs = [rec for _, rec in sp.play_games()]
    buf, n, _ = pack_records(recs)
    assert n == sum(len(r) for r in recs) and n > 200
    return recs, buf


def _tb(buf, lo=0, hi=None):
    from cchess_zero_b200.distributed import TupleBatch
    return TupleBatch(buf[lo:hi])


def _mirror_board(b):
    return np.ascontiguousarray(np.asarray(b).reshape(10, 9)[:, ::-1]).reshape(90)


@pytest.fixture
def deterministic(monkeypatch):
    import torch
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", False)


def test_replay_batch_is_bit_exact_with_the_host_path_and_the_oracle(games):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.train import ReplayBuffer, mirror_labels
    from oracle import oracle as O
    recs, buf = games
    n = len(buf)
    cap = (2 * n) // 3                                                     # small enough to wrap
    rb = ReplayBuffer(cap)
    cut = n // 2
    rb.add(_tb(buf, 0, cut))
    rb.add(_tb(buf, cut))
    assert len(rb) == cap and rb.ring.head == n % cap                     # wrapped once
    states = [s for r in recs for s in r.states]
    pis = np.concatenate([r.dense_pi() for r in recs]).astype(np.float32)
    zs = np.concatenate([np.asarray(r.z, dtype=np.float64) for r in recs])
    keep = np.arange(n - cap, n)                                           # what deque(maxlen=cap) keeps
    rows = rb.ring.slots(np.arange(cap))
    planes, pi, z = (t.cpu().numpy() for t in rb.batch(rows))
    boards = np.stack([rules.state_to_board(states[i]) for i in keep])
    want = rules.encode_batch(boards, np.zeros(cap, np.uint8))
    assert np.array_equal(planes, want)
    assert all(np.array_equal(planes[i], O.encode(boards[i], 0)) for i in range(0, cap, 7))
    assert np.array_equal(pi, pis[keep])
    assert np.array_equal(z[:, 0], zs[keep].astype(np.float32))

    # mirror augmentation on half the rows
    mirror = (np.arange(cap) % 2).astype(np.uint8)
    mp, mpi, mz = (t.cpu().numpy() for t in rb.batch(rows, mirror))
    ml = mirror_labels()
    labels = rules.create_uci_labels()
    for i in range(cap):
        if not mirror[i]:
            assert np.array_equal(mp[i], planes[i]) and np.array_equal(mpi[i], pi[i])
            continue
        mb = _mirror_board(boards[i])
        assert np.array_equal(mp[i], O.encode(mb, 0))
        w = np.zeros(2086, np.float32)
        nz = np.nonzero(pi[i])[0]
        w[ml[nz]] = pi[i, nz]
        assert np.array_equal(mpi[i], w)
        if i % 5 == 1:
            legal = set(int(m) for m in O.legal_moves(mb, 0))
            assert all(rules.label_to_move(labels[l]) in legal for l in np.nonzero(mpi[i] > 0)[0])
    assert np.array_equal(mz, z)


def test_replay_batch_rejects_bad_rows_and_records(games):
    import torch
    from cchess_zero_b200._lib import lib
    from cchess_zero_b200.train import ReplayBuffer
    _, buf = games
    rb = ReplayBuffer(64)
    rb.add(_tb(buf, 0, 40))
    for rows in ([40], [-1], [0, 63]):
        with pytest.raises(ValueError):
            rb.batch(np.asarray(rows))
    with pytest.raises(ValueError):
        rb.batch(np.asarray([0, 1]), mirror=np.ones(3, np.uint8))
    bad = _tb(buf, 40, 50)
    bad.idx[3, 0] = 2086
    with pytest.raises(ValueError):
        rb.add(bad)
    assert len(rb) == 40 and rb.added == 40                               # nothing of the bad batch went in
    L = lib()
    out = [torch.empty((1, 9, 10, 14), device="cuda"), torch.empty((1, 2086), device="cuda"), torch.empty((1,), device="cuda")]
    rows = torch.zeros((1,), dtype=torch.int32, device="cuda")
    args = [rb.boards.data_ptr(), rb.n.data_ptr(), rb.idx.data_ptr(), rb.prob.data_ptr(), rb.z.data_ptr()]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert L.cz_replay_batch(*args, 64, rows.data_ptr(), None, -1, *[t.data_ptr() for t in out], st) == -1
    assert L.cz_replay_batch(*args, -1, rows.data_ptr(), None, 1, *[t.data_ptr() for t in out], st) == -1
    assert L.cz_replay_batch(None, *args[1:], 64, rows.data_ptr(), None, 1, *[t.data_ptr() for t in out], st) == -1
    assert L.cz_replay_batch(*args, 64, None, None, 1, *[t.data_ptr() for t in out], st) == -1
    assert L.cz_replay_batch(*args, 64, rows.data_ptr(), None, 1, out[0].data_ptr(), None, out[2].data_ptr(), st) == -1
    assert L.cz_replay_batch(*args, 64, rows.data_ptr(), None, 0, None, None, None, st) == 0
    torch.cuda.synchronize()


def _params(pv):
    return [p.detach().clone() for p in pv.net.state_dict().values()]


def _same(a, b):
    return all(x.shape == y.shape and bool((x == y).all()) for x, y in zip(a, b))


def test_trainer_policy_update_equals_cchess_main_policy_update(games, tmp_path, monkeypatch, deterministic):
    """Same tuples in a deque and in the ReplayBuffer, same random state, identical seed-0 networks: k updates of each path give the
    same rows, KL values (hence early stops), lr_multiplier, loss / accuracy and bit-identical weights."""
    from cchess_zero_b200 import train as T
    from cchess_zero_b200.selfplay import cchess_main
    monkeypatch.chdir(tmp_path)
    recs, buf = games
    pa, pb = _net(tmp_path, "a"), _net(tmp_path, "b")
    assert _same(_params(pa), _params(pb))
    k, cap = 64, min(300, len(buf))
    with contextlib.redirect_stdout(io.StringIO()):
        cm = cchess_main(playout=8, in_batch_size=k, network=pa, log_file=False)
    cm.data_buffer = deque(maxlen=cap)
    for r in recs:
        cm.data_buffer.extend((cm.mcts.state_to_positions(s), p, w) for s, p, w in r.tuples())
    tr = T.Trainer(pb, 2, 8, batch_size=k, buffer_size=cap, checkpoint_every=0, arena_words=1 << 14)
    tr.buffer.add(_tb(buf))
    assert len(tr.buffer) == len(cm.data_buffer) == cap
    random.seed(11)
    tr.rng.seed(11)
    kls = []
    real_kl = T.policy_kl
    monkeypatch.setattr(T, "policy_kl", lambda o, n: kls.append(real_kl(o, n)) or kls[-1])
    for _ in range(4):
        probe = random.Random()
        probe.setstate(random.getstate())
        want_rows = probe.sample(range(cap), k)
        kls.clear()
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            cm.policy_update()
        kl_ref = list(kls)
        kls.clear()
        st = tr.policy_update()
        assert [int(v) for v in (st["rows"] - (tr.buffer.ring.head - tr.buffer.ring.size)) % cap] == want_rows
        assert kls == kl_ref and st["steps"] == len(kl_ref)
        msg = [l for l in out.getvalue().splitlines() if l.startswith("kl:")][0]
        fields = dict(f.split(":", 1) for f in msg.split(","))
        assert fields["loss"] == str(st["loss"]) and fields["accuracy"] == str(st["accuracy"])
        assert cm.lr_multiplier == tr.lr_multiplier and cm.global_step == pb.global_step
        assert _same(_params(pa), _params(pb)), "weights differ after an update"


def _root_priors(sp):
    """Root priors of game 0 after a search from the start position (the engine is reset first)."""
    sp.engine.reset()
    sp.search()
    rc = sp.engine.root_children()
    n = int(rc["n"][0])
    return rc["moves"][0, :n].copy(), rc["p"][0, :n].copy()


def test_small_loop_trains_gates_and_promotes(tmp_path, monkeypatch):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    rules._init_tables()
    pv = _net(tmp_path, "net")
    tr = Trainer(pv, 16, 16, batch_size=32, buffer_size=512, checkpoint_every=0, arena_words=1 << 16, eval_every=4, eval_games=2,
                 eval_playouts=8, gate_threshold=1.0)
    best0 = _params(tr.best)
    with contextlib.redirect_stdout(io.StringIO()):
        while (tr.updates < 2 or tr.gates < 1) and tr.plies < 3000:
            tr.ply()
    assert tr.games >= 4 and len(tr.buffer) > 32 and tr.updates >= 2 and tr.train_steps >= 2
    assert tr.gates >= 1 and tr.promotions == 0 and tr.last_gate["promote"] is False
    assert _same(_params(tr.best), best0)                                  # threshold 1.0 never promotes
    assert not _same(_params(pv), best0)                                   # the candidate was trained
    rep = tr.report()
    assert rep["updates"] == tr.updates and rep["gate"]["games"] == 2 and set(rep["seconds"]) == {"selfplay", "ingest", "train", "gate"}

    tr.gate_threshold = -1.0
    with contextlib.redirect_stdout(io.StringIO()):
        r = tr.gate()
    assert r.promote(-1.0) and tr.promotions == 1
    assert _same(_params(tr.best), _params(pv))                            # best = candidate, bit for bit
    assert os.path.isfile(os.path.join(tr.best.save_dir, "checkpoint"))

    # self-play (driven by best) now searches with the promoted weights: priors = legal logits / their sum (expand, main.py:176-187)
    moves, p = _root_priors(tr.sp)
    lo, _ = pv.forward(rules.encode_batch(rules.state_to_board(rules.START_STATE)[None], [0]))
    lg = lo[0, [rules.label2i[rules.move_to_label(m)] for m in moves]].astype(np.float64)
    assert np.allclose(p, lg / (1e-8 + lg.sum()), rtol=2e-2, atol=2e-3)


def test_self_play_without_gate_follows_the_trained_network(tmp_path, monkeypatch):
    from cchess_zero_b200 import rules
    from cchess_zero_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    rules._init_tables()
    pv = _net(tmp_path, "net")
    tr = Trainer(pv, 16, 16, batch_size=32, buffer_size=512, checkpoint_every=0, arena_words=1 << 16)
    assert tr.best is None
    _, p0 = _root_priors(tr.sp)
    tr.sp.engine.reset()
    with contextlib.redirect_stdout(io.StringIO()):
        while tr.updates < 1 and tr.plies < 3000:
            tr.ply()
    assert tr.updates >= 1
    moves, p1 = _root_priors(tr.sp)
    assert not np.array_equal(p0, p1), "self-play searched with the pre-training weights"
    lo, _ = pv.forward(rules.encode_batch(rules.state_to_board(rules.START_STATE)[None], [0]))
    lg = lo[0, [rules.label2i[rules.move_to_label(m)] for m in moves]].astype(np.float64)
    assert np.allclose(p1, lg / (1e-8 + lg.sum()), rtol=2e-2, atol=2e-3)


def test_resume_restores_the_run_exactly(tmp_path, monkeypatch, deterministic):
    import torch
    from cchess_zero_b200.train import Trainer
    monkeypatch.chdir(tmp_path)
    pa = _net(tmp_path, "a", seed=0)
    ta = Trainer(pa, 16, 8, batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16, seed=3)
    with contextlib.redirect_stdout(io.StringIO()):
        while ta.updates < 2 and ta.plies < 3000:
            ta.ply()
        ta.save(str(tmp_path / "run"))
        pb = _net(tmp_path, "b", seed=5)
        tb = Trainer(pb, 16, 8, batch_size=32, buffer_size=256, checkpoint_every=0, arena_words=1 << 16, seed=9)
        tb.load(str(tmp_path / "run"))
    for name in ("boards", "n", "idx", "prob", "z"):
        assert torch.equal(getattr(ta.buffer, name), getattr(tb.buffer, name)), name
    assert (ta.buffer.ring.head, ta.buffer.ring.size, ta.buffer.added) == (tb.buffer.ring.head, tb.buffer.ring.size, tb.buffer.added)
    assert _same(_params(pa), _params(pb)) and pa.global_step == pb.global_step
    sa, sb = pa.opt.state_dict(), pb.opt.state_dict()
    assert sa["param_groups"] == sb["param_groups"] and sa["state"].keys() == sb["state"].keys()
    assert all(torch.equal(sa["state"][i]["momentum_buffer"], sb["state"][i]["momentum_buffer"]) for i in sa["state"])
    assert ta.lr_multiplier == tb.lr_multiplier and ta.rng.getstate() == tb.rng.getstate()
    assert np.array_equal(ta.sp._mt, tb.sp._mt)
    assert (ta.games, ta.positions, ta.updates, ta.train_steps) == (tb.games, tb.positions, tb.updates, tb.train_steps)
    ra, rb = ta.policy_update(), tb.policy_update()
    assert np.array_equal(ra["rows"], rb["rows"]) and ra["loss"] == rb["loss"]
    assert _same(_params(pa), _params(pb))
    with contextlib.redirect_stdout(io.StringIO()):
        tb.ply()                                                           # the resumed run plays on (fresh games)


def test_cli_prints_json_lines_and_resumes(tmp_path):
    d = str(tmp_path / "run")
    base = [sys.executable, "-m", "cchess_zero_b200.train", "--games", "8", "--playouts", "8", "--batch-size", "16", "--buffer-size", "128",
            "--res-block-nums", "2", "--report-every", "20", "--save-dir", d, "--eval-every", "4", "--eval-games", "2", "--eval-playouts", "4",
            "--checkpoint-every", "5", "--mirror"]
    keys = {"plies", "games", "positions", "buffer", "buffer_capacity", "updates", "train_steps", "loss", "accuracy", "kl", "lr_multiplier",
            "explained_var_old", "explained_var_new", "seconds", "gate", "promotions"}
    lines = []
    for extra in (["--max-plies", "150"], ["--max-plies", "10", "--resume"]):
        r = subprocess.run(base + extra, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        out = [json.loads(l) for l in r.stdout.splitlines()]
        assert out and all(keys <= set(o) for o in out)
        lines.append(out)
    assert lines[0][-1]["plies"] == 150 and lines[1][-1]["plies"] == 160            # the counters continue
    assert lines[1][-1]["games"] >= lines[0][-1]["games"]
    assert os.path.isfile(os.path.join(d, "trainer.npz")) and os.path.isfile(os.path.join(d, "network", "checkpoint"))
