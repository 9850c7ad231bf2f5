"""CPU-only tests: the C-ABI library loads and exports every declared symbol, the host-only entry points
work without a GPU, compute entry points fail loudly without one, and the host-side logic (tuple packing,
flip helpers, multi-rank gather over gloo) is correct."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from search_spec import StandIn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol():
    from cchess_zero_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "cchess_b200.h")).read()
    names = sorted(set(re.findall(r"\b(cz_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), "missing symbol %s" % n
    assert L.cz_version() >= 1


def test_ctypes_binding_matches_the_header_prototypes():
    """Every prototype of include/cchess_b200.h against the ctypes signature cchess_zero_b200/_lib.py binds it with: same number of
    parameters, pointers bound as pointers, integers as 32- / 64-bit integers (an ABI drift between the header and the binding would
    otherwise show up as a crash on the GPU box only)."""
    import ctypes as C
    from cchess_zero_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "cchess_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    protos = re.findall(r"\b(?:int|int64_t|const char \*|void)\s*\*?\s*(cz_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", hdr)
    assert len(protos) >= 45
    checked = 0
    for name, params in protos:
        params = params.strip()
        plist = [] if params in ("", "void") else [q.strip() for q in params.split(",")]
        at = getattr(getattr(L, name), "argtypes", None)
        if at is None:
            assert not plist, "%s: %d parameters in the header, no argtypes bound" % (name, len(plist))
            continue
        assert len(at) == len(plist), "%s: header has %d parameters, binding %d" % (name, len(plist), len(at))
        for q, t in zip(plist, at):
            is_ptr = "*" in q or "[" in q
            bound_ptr = t in (C.c_void_p, C.c_char_p) or hasattr(t, "contents") or getattr(t, "_type_", None) == "P" or "LP_" in getattr(t, "__name__", "")
            assert is_ptr == bound_ptr, "%s: parameter '%s' bound as %s" % (name, q, t)
            if not is_ptr:
                want64 = bool(re.search(r"\b(int64_t|long long|size_t|uint64_t)\b", q))
                assert (C.sizeof(t) == 8) == want64, "%s: parameter '%s' bound as %s" % (name, q, t)
        checked += 1
    assert checked >= 40


def test_host_only_entry_points_match_oracle():
    from cchess_zero_b200 import rules
    from oracle import oracle as O
    rules._init_tables()
    assert rules.labels_array == O.labels()
    assert rules.unflipped_index == O.unflipped_index()
    assert rules.labels_len == 2086 and rules.label2i["e0e9"] == 916 and rules.i2label[2056] == "c0e2"
    b = rules.state_to_board(rules.START_STATE)
    assert np.array_equal(b, O.from_state(O.START))
    assert rules.board_to_state(b) == rules.START_STATE
    with pytest.raises(Exception):
        rules.state_to_board("9/9/9")
    assert rules.flipped_uci_labels(["a0b9"]) == ["a9b0"]
    assert rules.is_kill_move("RNBAKABNR/9", "RNBAKABN1/9") == 1
    assert rules.GameBoard.board_to_pos_name("4K4/9")[0] == "1111K1111"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_compute_fails_loudly_without_gpu():
    from cchess_zero_b200 import rules
    from cchess_zero_b200._lib import EngineError
    from cchess_zero_b200.engine import Engine
    with pytest.raises(EngineError):
        Engine(4)
    with pytest.raises(EngineError):
        rules.GameBoard.get_legal_moves(rules.START_STATE, "w")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "cchess_zero_b200")
    for dp, _, fns in os.walk(pkg):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), fn
                assert "liboracle" not in src and "cchess_oracle" not in src, fn


def test_flip_helpers_and_record_packing():
    from cchess_zero_b200 import rules
    from cchess_zero_b200.distributed import pack_records, unpack_records, shard_seeds
    from cchess_zero_b200.selfplay import GameRecord, _flip_board, _flip_move_label_index
    from oracle import oracle as O
    rules._init_tables()
    b = O.from_state("R1BAKAB1R/9/1C2C1N2/P1P1P1P1P/2N6/6p2/p1p1p3p/1c2c1n2/9/rnbakab1r")
    assert np.array_equal(_flip_board(b), O.flip_board(b))
    for m in ("a0a1", "h9g7", "e9e0"):
        mv = O.move_from_str(m)
        assert _flip_move_label_index(mv) == rules.label2i[O.flip_label(m)]
    with np.errstate(all="ignore"):
        g = O.selfplay_game("hash_pos", 12, np.random.RandomState(4))
    nz = [np.nonzero(p)[0] for p in g["pis"]]
    rec = GameRecord.from_tuples(g["states"], nz, [p[ix] for p, ix in zip(g["pis"], nz)], g["z"])
    buf, k, left = pack_records([rec], 4096)
    assert k == len(g["states"]) and not left
    back = unpack_records(buf, k)
    for (s, pi, z), s0, p0, z0 in zip(back, g["states"], g["pis"], g["z"]):
        assert s == s0 and z == z0 and np.array_equal(pi, p0)
    _, k2, left2 = pack_records([rec, rec], len(g["states"]) + 3)      # a cap never splits or drops a game: the second one is handed back whole
    assert k2 == len(g["states"]) and len(left2) == 1 and left2[0] is rec
    from cchess_zero_b200.distributed import TupleBatch
    tb = TupleBatch(buf[:k])
    assert len(tb) == k and np.array_equal(tb.dense_pi(), np.stack(g["pis"])) and np.array_equal(tb.z, np.asarray(g["z"], dtype=np.float64))
    assert shard_seeds(4, 0) == [0, 1, 2, 3] and shard_seeds(4, 2, 10) == [18, 19, 20, 21]


_GLOO = r'''
import os, sys
sys.path.insert(0, %r)
import numpy as np, torch, torch.distributed as dist
from cchess_zero_b200.distributed import all_gather_tuples
from cchess_zero_b200.selfplay import GameRecord
from oracle import oracle as O
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
def game(seed):
    with np.errstate(all="ignore"):
        g = O.selfplay_game("hash_pos", 10, np.random.RandomState(seed))
    nz = [np.nonzero(p)[0] for p in g["pis"]]
    return g, GameRecord.from_tuples(g["states"], nz, [p[ix] for p, ix in zip(g["pis"], nz)], g["z"])
mine = [game(100 + rank * 2 + i) for i in range(2 if rank == 0 else 1)]     # ragged: rank 0 two games, rank 1 one
out = all_gather_tuples([r for _, r in mine], torch.device("cpu"), cap=1024)
exp = []
for rk in range(world):
    for i in range(2 if rk == 0 else 1):
        g, _ = game(100 + rk * 2 + i)
        exp += list(zip(g["states"], g["pis"], g["z"]))
assert len(out) == len(exp), (len(out), len(exp))
for (s, p, z), (s0, p0, z0) in zip(out, exp):
    assert s == s0 and z == z0 and np.array_equal(p, p0)
# the pipelined form: three rounds in flight (one of them empty on rank 1), nothing lost, nothing duplicated, round-major order
from cchess_zero_b200.distributed import AsyncTupleGather
ag = AsyncTupleGather(torch.device("cpu"))
rounds = [[game(200 + rank)], [] if rank == 1 else [game(210)], [game(220 + rank), game(230 + rank)]]
got = []
for rd in rounds:
    ag.start([r for _, r in rd])
    tb = ag.finish()
    if tb is not None: got += tb.tuples()
got += ag.drain().tuples()
exp2 = []
for i, rd in enumerate(rounds):
    for rk in range(world):
        gs = [[game(200 + rk)], [] if rk == 1 else [game(210)], [game(220 + rk), game(230 + rk)]][i]
        for g, _ in gs: exp2 += list(zip(g["states"], g["pis"], g["z"]))
assert len(got) == len(exp2), (len(got), len(exp2))
for (s, p, z), (s0, p0, z0) in zip(got, exp2):
    assert s == s0 and z == z0 and np.array_equal(p, p0)
if rank == 0: print("GLOO_OK", len(out), len(got))
dist.destroy_process_group()
'''


def test_all_gather_tuples_world_size_2_gloo(tmp_path):
    script = tmp_path / "g.py"
    script.write_text(_GLOO % ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29517", str(script)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "GLOO_OK" in r.stdout


def test_bench_reference_arm_prints_contract_line():
    """--impl reference times the UNMODIFIED reference (search_threads=16, one process per core) when it is present / staged."""
    env = dict(os.environ, CCHESS_REF_SECONDS="8")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1"],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    import json
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "mcts_node_expansions_per_sec" and line["value"] > 0
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import stage_reference as S
    cb = line["cpu_baseline"]
    if S.staged_dir() and S.verify():
        assert cb["kind"] == "reference" and cb["search_threads"] == 16 and cb["cores"] >= 1 and cb["tree_only_value"] > cb["value"]
        assert cb["port_value"]["kind"] == "port"
    else:
        assert cb["kind"] == "port"
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["steps"] == 2 and line["config"]["search_threads"] == 16


def test_staged_reference_is_byte_identical_and_loads_from_the_staged_copy(tmp_path):
    """oracle/stage_reference.py: the copy that travels to the GPU box hashes to the committed manifest and is importable
    through the harness without /root/reference (CCHESS_REFERENCE_DIR points at the staged directory)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import stage_reference as S
    if not os.path.isdir(S.DST):
        if not os.path.isdir(S.SRC):
            pytest.skip("neither the reference nor a staged copy is present")
        S.stage()
    assert S.verify(S.DST)
    code = ("import os, sys; sys.path.insert(0, %r); import ref_harness as H; ref = H.load_reference(); "
            "assert os.path.dirname(ref.__file__) == %r, ref.__file__; "
            "t = H.make_mcts(H.FAKE_NETS['mod17'], 16); t.main(t.root.state, 'w', 0, 64); "
            "print('STAGED_OK', sorted((a, c.N) for a, c in t.root.child.items() if c.N)[:2])") % (os.path.join(ROOT, "oracle"), S.DST)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=dict(os.environ, CCHESS_REFERENCE_DIR=S.DST))
    assert r.returncode == 0 and "STAGED_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]
    assert "('a0a1', 47), ('a0a2', 17)" in r.stdout          # SURVEY Appendix B: K=16, 64 playouts, mod17 net


_DP = r'''
import sys
sys.path.insert(0, %r)
import torch, torch.distributed as dist
from cchess_zero_b200.net import PolicyValueNet, train_step_module
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
torch.manual_seed(0)
net = PolicyValueNet(1)                               # same initial weights on every rank
opt = torch.optim.SGD(net.parameters(), lr=1e-2, momentum=0.9, nesterov=True)
g = torch.Generator().manual_seed(100 + rank)         # a different mini-batch ("tower") per rank
x = (torch.rand(6, 9, 10, 14, generator=g) < 0.03).float()
pi = torch.softmax(torch.randn(6, 2086, generator=g), 1)
z = torch.sign(torch.randn(6, 1, generator=g))
before = torch.cat([p.detach().reshape(-1) for p in net.parameters()]).clone()
for _ in range(3):
    acc, loss = train_step_module(net, opt, x, pi, z, 1e-2)
after = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
allp = [torch.empty_like(after) for _ in range(world)]
dist.all_gather(allp, after)
assert torch.isfinite(after).all() and not torch.equal(before, after)
assert all(torch.equal(allp[0], q) for q in allp), "replicas diverged"
if rank == 0: print("DP_OK", float(loss))
dist.destroy_process_group()
'''


def test_data_parallel_train_step_keeps_replicas_in_sync_gloo(tmp_path):
    script = tmp_path / "dp.py"
    script.write_text(_DP % ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29533", str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "DP_OK" in r.stdout


def test_train_step_matches_written_out_reference_update_rule():
    """train_step_module against a float64 restatement of policy_value_network.py:76-126: softmax-CE + MSE + 1e-4*sum(w^2)/2,
    tf.clip_by_global_norm(100), MomentumOptimizer(momentum 0.9, use_nesterov=True): accum = m*accum + g; w -= lr*(g + m*accum)."""
    from cchess_zero_b200.net import PolicyValueNet, train_step_module
    torch.manual_seed(3)
    net = PolicyValueNet(1)
    ref = PolicyValueNet(1).double()
    ref.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9, nesterov=True)
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(10, 9, 10, 14, generator=g) < 0.03).float()
    pi = torch.softmax(torch.randn(10, 2086, generator=g) * 3, 1)
    z = torch.sign(torch.randn(10, 1, generator=g))
    lr, m, c = 0.02, 0.9, 1e-4
    accum = [torch.zeros_like(p) for p in ref.parameters()]
    for step in range(3):
        acc, loss = train_step_module(net, opt, x, pi, z, lr)
        ref.train()
        lo, v = ref(x.double())
        rloss = (-(pi.double() * torch.log_softmax(lo, 1)).sum(1)).mean() + ((v - z.double()) ** 2).mean() \
            + c * sum((p ** 2).sum() / 2 for p in ref.parameters())
        grads = torch.autograd.grad(rloss, list(ref.parameters()))
        gn = torch.sqrt(sum((gr ** 2).sum() for gr in grads))
        scale = min(1.0, 100.0 / float(gn))
        with torch.no_grad():
            for p, gr, a in zip(ref.parameters(), grads, accum):
                gr = gr * scale
                a.mul_(m).add_(gr)
                p.sub_(lr * (gr + m * a))
        assert abs(loss - float(rloss)) < 1e-4 * max(1.0, abs(float(rloss)))
    for p, q in zip(net.parameters(), ref.parameters()):
        assert torch.allclose(p.double(), q, atol=2e-5, rtol=1e-4)


def test_replay_persistence_round_trip_and_rng_resume(tmp_path):
    import random
    from collections import deque
    from cchess_zero_b200.selfplay import load_replay, save_replay
    buf = deque(maxlen=50)
    rng = np.random.RandomState(0)
    for i in range(60):
        buf.append((rng.rand(9, 10, 14).astype(np.float32), rng.rand(2086), float(i % 3 - 1)))
    np.random.seed(11); random.seed(12)
    np.random.rand(5); random.random()
    p = str(tmp_path / "replay.pkl")
    save_replay(p, buf, dict(lr_multiplier=1.5, global_step=7))
    expect_np, expect_py = np.random.rand(3), random.random()       # what the run would have drawn next
    np.random.seed(999); random.seed(999)
    buf2, extra = load_replay(p)
    assert extra == dict(lr_multiplier=1.5, global_step=7) and buf2.maxlen == 50 and len(buf2) == 50
    for a, b in zip(buf, buf2):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
    assert np.array_equal(np.random.rand(3), expect_np) and random.random() == expect_py


def test_selfplay_host_loop_on_cpu_stand_in_engine_matches_reference_vectors():
    """SelfPlay.step's host side (softmax(log N), Dirichlet mix, choice, tuple recording, z, game end) against the reference's
    own self-play tuples, with the device engine replaced by the oracle trees."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conftest import load_golden
    from cchess_zero_b200.selfplay import SelfPlay
    import hashlib
    games = [g for g in load_golden("selfplay.json")["games"] if g["net"] == "hash_pos"]
    eng = StandIn(len(games), "hash_pos")
    sp = SelfPlay(len(games), lambda x: None, [g["playouts"] for g in games], seeds=[g["seed"] for g in games], auto_reset=False, engine=eng)
    with np.errstate(all="ignore"):
        out = sp.play_games()
    assert len(out) == len(games)
    for (slot, rec), g in zip(out, games):
        assert rec.states == g["states"] and [float(z) for z in rec.z] == g["z"]
        assert hashlib.sha256(rec.dense_pi().tobytes()).hexdigest()[:16] == g["sha_pi"]
    assert len(sp.pop_finished()) == len(games) and sp.finished == [] and sp.pop_finished() == []


def test_device_rule_source_compiled_for_host_matches_reference_vectors(tmp_path):
    """The product's own per-lane rule code (csrc/cz_rules.cuh: gen_piece, warp_encode) compiled for the HOST by nvcc and run
    against the golden vectors of the reference -- a CPU-tier check of the very source the kernels are built from."""
    import ctypes as C
    import shutil
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conftest import load_golden
    from oracle import oracle as O
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    so = str(tmp_path / "libhostrules.so")
    r = subprocess.run([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-shared", "-o", so,
                        os.path.join(ROOT, "tests", "host_rules_harness.cu")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    L = C.CDLL(so)
    recs = load_golden("movegen.json.gz")["records"]
    out = np.zeros(160, dtype=np.uint16)
    enc = np.zeros((9, 10, 14), dtype=np.float32)
    for r_ in recs[::3]:
        b = O.from_state(r_["state"])
        side = 0 if r_["player"] == "w" else 1
        n = L.hr_legal_moves(b.ctypes.data_as(C.c_void_p), side, out.ctypes.data_as(C.c_void_p))
        assert " ".join(O.move_str(m) for m in out[:n]) == r_["moves"], r_["state"]
        L.hr_encode_f32(b.ctypes.data_as(C.c_void_p), side, enc.ctypes.data_as(C.c_void_p))
        assert [int(i) for i in np.nonzero(enc.reshape(-1))[0]] == r_["enc"]


def test_selfplay_auto_reset_path_on_cpu_stand_in_engine():
    """The bench's mode: finished games are emitted with z and their slots restart from the start position; every finished
    game must equal what the oracle plays with the same slot RNG stream continued across games."""
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net = 6, 8, "hash_pos"
    eng = StandIn(B, net)
    sp = SelfPlay(B, lambda x: None, P, seeds=[40 + i for i in range(B)], auto_reset=True, engine=eng)
    with np.errstate(all="ignore"):
        for _ in range(260):
            sp.step()
    done = sp.pop_finished()
    assert len(done) >= B                      # every slot finished at least one game (60-ply rule bounds game length)
    first = {}
    for slot, rec in done:
        first.setdefault(slot, rec)
        assert rec.z is not None and len(rec.z) == len(rec) and rec.winner in ("w", "b", "t")
        assert rec.states[0] == "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"
    from oracle import oracle as O
    for slot, rec in first.items():            # first game of each slot == the oracle's game with that seed
        with np.errstate(all="ignore"):
            r = O.selfplay_game(net, P, np.random.RandomState(40 + slot))
        assert rec.states == r["states"] and np.array_equal(rec.z, r["z"]) and np.array_equal(rec.dense_pi(), r["pis"])


def test_torch_stand_in_nets_match_oracle_on_cpu():
    """cchess_zero_b200/fakenet.py (torch integer ops, used on the device in the GPU tests) evaluated on CPU tensors against
    the oracle's C restatement and the numpy original."""
    from cchess_zero_b200.fakenet import FakeNet
    from oracle import oracle as O
    from oracle.fakenets_np import FAKE_NETS
    rng = np.random.RandomState(1)
    xs, b, side = [], O.from_state(O.START), 0
    for _ in range(40):
        xs.append(O.encode(b, side))
        mv = O.legal_moves(b, side)
        b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
    x = np.stack(xs)
    for kind in ("hash_signed", "hash_pos", "mod17"):
        lo, v = FakeNet(kind, device="cpu")(torch.from_numpy(x))
        olo, ov = O.fake_forward(kind, x)
        nlo, nv = FAKE_NETS[kind](x)
        assert np.array_equal(lo.numpy(), olo) and np.array_equal(v.numpy(), ov.reshape(-1))
        assert np.array_equal(nlo, olo) and np.array_equal(nv, ov)


def test_pytorch_network_matches_independent_numpy_restatement_of_the_tf_graph():
    """cchess_zero_b200.net.PolicyValueNet (CPU, fp64) against oracle/net_numpy.py, a separately written NHWC / TF-layout
    evaluation of policy_value_network.py:45-74, 151-162 (SAME padding, BN without gamma/beta, (h,w,c) flatten, logits, tanh)."""
    from cchess_zero_b200.net import PolicyValueNet
    from oracle import net_numpy as NN
    from oracle import oracle as O
    torch.manual_seed(2)
    net = PolicyValueNet(3).double().eval()
    with torch.no_grad():   # non-trivial biases and moving statistics
        for m in net.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                m.bias.uniform_(-0.2, 0.2)
            if hasattr(m, "running_var"):
                m.running_var.uniform_(0.5, 2.0); m.running_mean.uniform_(-0.3, 0.3)
    rng = np.random.RandomState(0)
    xs, b, side = [], O.from_state(O.START), 0
    for _ in range(12):
        xs.append(O.encode(b, side))
        mv = O.legal_moves(b, side)
        b, _ = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
    x = np.stack(xs).astype(np.float64)
    with torch.no_grad():
        tl, tv = net(torch.from_numpy(x))
    nl, nv = NN.forward(x, NN.tf_params_from_torch(net), 3)
    assert nl.shape == (12, 2086) and nv.shape == (12, 1)
    assert np.abs(tl.numpy() - nl).max() < 1e-10 and np.abs(tv.numpy() - nv).max() < 1e-10


def test_tf32x3_split_algebra_is_fp32_accurate():
    """net.py: tf32_hi / split_weights / split_acts -- with EVERY operand rounded as the tensor cores see it (TF32 for the hi*hi
    product, fp16 operands and an fp16-rounded result for the two cross terms), the three-product convolution
    conv_tf32(hi, hi) + 2^-11 conv_fp16({ lo 2^11 | hi }, { hi | lo 2^11 }) is ~1e-6 from the exact one where a single TF32 product
    is ~1e-3 (what precision="tf32x3" rests on; the GPU tier measures the whole network against fp64, accumulator truncation included)."""
    import torch
    import torch.nn.functional as F
    from cchess_zero_b200.net import SPLIT_SCALE, tf32_hi, split_weights, split_acts
    torch.manual_seed(0)
    x = torch.relu(torch.randn(4, 128, 9, 10)) * 3.0
    w = torch.randn(128, 128, 3, 3) * 0.03
    h = tf32_hi(x)
    assert int((h.view(torch.int32) & 0x1FFF).abs().max()) == 0                       # representable in TF32
    assert float(((x - h).abs() / x.abs().clamp_min(1e-30)).max()) <= 2.0 ** -11 + 1e-9   # nearest
    assert torch.equal(tf32_hi(-x), -h)                                                # sign-symmetric (ties away from zero)
    ref = F.conv2d(x.double(), w.double(), padding=1)
    one = F.conv2d(tf32_hi(x).double(), tf32_hi(w).double(), padding=1)
    (xh, x2), (wh, w2) = split_acts(x), split_weights(w)
    assert x2.dtype == torch.float16 and w2.dtype == torch.float16
    assert torch.equal(xh, h) and torch.equal(x2[:, 128:].float(), h)                   # hi is exact in fp16
    assert float((x2[:, :128].double() / SPLIT_SCALE - (x - h).double()).abs().max()) <= 2.0 ** -11 * float((x - h).abs().max())   # 13-bit residue rounded to 11 bits
    cross = F.conv2d(x2.double(), w2.double(), padding=1).to(torch.float16).double() / SPLIT_SCALE
    three = F.conv2d(xh.double(), wh.double(), padding=1) + cross
    e1, e3 = float((one - ref).abs().max()), float((three - ref).abs().max())
    assert e1 > 5e-4 and e3 < 4e-6, (e1, e3)
