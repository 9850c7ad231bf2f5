#!/usr/bin/env python
"""Training-loop throughput on one GPU (cchess_zero_b200/train.py).

  python tools/train_bench.py [--games 1024 --playouts 400 --blocks 7 --batch 512 --rounds 3 --plies 8] [--out FILE]

(a) Mini-batch assembly.  cz_replay_batch timed by CUDA events at 512 and 4096 rows (a full 10000-position ring of synthetic valid
    records, random rows, half of them mirrored), with the algorithmic bytes per row: 90 + 1 + 256 + 512 + 4 in, 5040 + 8344 + 4 out
    (achieved GB/s and the share of the H100's 3.35 TB/s).  Beside it, the host path the reference's run() / policy_update takes for
    the same rows: MCTS_tree.state_to_positions per state, the dense pi vectors, and train_step's float32 conversion + H2D copies.
(b) The loop.  A Trainer (n games x playouts, a `blocks`-block fp16 network, batch `batch`, no gate) first plays until it has run one
    policy_update; then `rounds` x (`plies` Trainer plies, `plies` plies of a SelfPlay-only run of the same size and network depth),
    alternated in this one process.  Reports plies/s, games/hour and train steps/s of the loop, the loop's wall-time split, and the
    SelfPlay-only ply time.
Prints one JSON line (card name and power limit read in the same run)."""
import argparse
import contextlib
import json
import os
import random
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from arena_bench import card, timed  # noqa: E402

BYTES_IN, BYTES_OUT = 90 + 1 + 256 + 512 + 4, 5040 + 8344 + 4
HBM_PEAK = 3.35e12


def synthetic_records(n, seed=0):
    """n valid ring records: random piece codes, 20..60 distinct labels with probabilities summing to 1, z in {-1, 0, 1}."""
    from cchess_zero_b200.distributed import REC_BYTES, TupleBatch
    rs = np.random.RandomState(seed)
    tb = TupleBatch(np.zeros((n, REC_BYTES), dtype=np.uint8))
    tb.boards[:] = rs.randint(0, 15, size=(n, 90))
    tb.n = rs.randint(20, 61, size=n).astype(np.int64)
    for i in range(n):
        k = int(tb.n[i])
        tb.idx[i, :k] = rs.choice(2086, k, replace=False)
        tb.prob[i, :k] = rs.dirichlet(np.ones(k))
    tb.z[:] = rs.choice([-1.0, 0.0, 1.0], n)
    return tb


def kernel_part(iters=200):
    import ctypes as C
    from cchess_zero_b200 import rules
    from cchess_zero_b200._lib import lib
    from cchess_zero_b200.mcts import MCTS_tree
    from cchess_zero_b200.train import ReplayBuffer
    rules._init_tables()
    tb = synthetic_records(10000)
    rb = ReplayBuffer(10000)
    rb.add(tb)
    tree = MCTS_tree(rules.START_STATE, None, 1, arena_words=1 << 12)
    out = {}
    for m in (512, 4096):
        rows = np.asarray(rb.sample_rows(random.Random(m), m))
        mirror = (np.arange(m) % 2).astype(np.uint8)
        rb.batch(rows, mirror)                                  # warm-up (first mirror call uploads the table)
        rows_d = torch.from_numpy(rows.astype(np.int32)).cuda()
        mir_d = torch.from_numpy(mirror).cuda()
        planes = torch.empty((m, 9, 10, 14), device="cuda")
        pi = torch.empty((m, 2086), device="cuda")
        z = torch.empty((m,), device="cuda")
        L, st = lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
        args = (rb.boards.data_ptr(), rb.n.data_ptr(), rb.idx.data_ptr(), rb.prob.data_ptr(), rb.z.data_ptr(), rb.capacity, rows_d.data_ptr(),
                mir_d.data_ptr(), m, planes.data_ptr(), pi.data_ptr(), z.data_ptr(), st)
        for _ in range(10):
            L.cz_replay_batch(*args)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            L.cz_replay_batch(*args)
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / 1e3 / iters
        nbytes = m * (BYTES_IN + BYTES_OUT)
        # the host path of the same rows: deque tuples hold state strings (selfplay) -> state_to_positions at ingest, dense pi
        states = [rules.board_to_state(tb.boards[r]) for r in rows]
        sub = type(tb).__new__(type(tb))
        sub.boards, sub.n, sub.idx, sub.prob, sub.z = tb.boards[rows], tb.n[rows], tb.idx[rows], tb.prob[rows], tb.z[rows]
        t0 = time.perf_counter()
        pos = [tree.state_to_positions(s) for s in states]
        t1 = time.perf_counter()
        dense = list(sub.dense_pi())
        t2 = time.perf_counter()
        x = torch.as_tensor(np.asarray(pos, dtype=np.float32)).reshape(-1, 9, 10, 14).to("cuda")
        p = torch.as_tensor(np.asarray(dense, dtype=np.float32)).to("cuda")
        w = torch.as_tensor(np.asarray(sub.z, dtype=np.float32)).reshape(-1, 1).to("cuda")
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        out[str(m)] = dict(kernel_us=1e6 * t, bytes=nbytes, gb_per_s=nbytes / t / 1e9, share_of_3_35_tb_s=nbytes / t / HBM_PEAK,
                           host_path_ms=dict(state_to_positions=1e3 * (t1 - t0), dense_pi=1e3 * (t2 - t1), f32_and_h2d=1e3 * (t3 - t2),
                                             total=1e3 * (t3 - t0)))
        del x, p, w
    return out


def loop_part(n, playouts, blocks, batch, rounds, plies):
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import network_selfplay
    from cchess_zero_b200.train import Trainer
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        net = policy_value_network(blocks, precision="fp16", seed=0, save_dir=d)
        ref = policy_value_network(blocks, precision="fp16", seed=0, save_dir=d)
    tr = Trainer(net, n, playouts, batch_size=batch, buffer_size=10000, checkpoint_every=0, arena_words=1 << 20)
    sp = network_selfplay(ref, n, playouts, seeds=range(n), auto_reset=True, keep_records=True, arena_words=1 << 20)
    sp.capture_graph()
    t0 = time.perf_counter()
    warm = 0
    while tr.updates == 0:
        tr.ply()
        sp.step()
        sp.pop_finished()
        warm += 1
    warm_s = time.perf_counter() - t0
    base = dict(games=tr.games, steps=tr.train_steps, updates=tr.updates, seconds=dict(tr.seconds))
    t_loop, t_self = [], []
    for _ in range(rounds):
        for _ in range(plies):
            t_loop.append(timed(tr.ply))
        for _ in range(plies):
            t_self.append(timed(sp.step))
            sp.pop_finished()
    T = sum(t_loop)
    games, steps, updates = tr.games - base["games"], tr.train_steps - base["steps"], tr.updates - base["updates"]
    split = {k: tr.seconds[k] - base["seconds"][k] for k in tr.seconds}
    return dict(warmup_plies=warm, warmup_s=warm_s, timed_plies=len(t_loop), loop_ply_ms_median=1e3 * float(np.median(t_loop)),
                selfplay_only_ply_ms_median=1e3 * float(np.median(t_self)), loop_ply_ms=[round(1e3 * t, 1) for t in t_loop],
                selfplay_only_ply_ms=[round(1e3 * t, 1) for t in t_self], loop_plies_per_s=len(t_loop) / T,
                selfplay_only_plies_per_s=len(t_self) / sum(t_self), loop_games=games, loop_games_per_hour=games * 3600.0 / T,
                loop_updates=updates, loop_train_steps=steps, train_steps_per_s=steps / T,
                loop_split_s={k: round(v, 3) for k, v in split.items()}, loop_split_share={k: round(v / T, 3) for k, v in split.items()},
                buffer=len(tr.buffer))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--plies", type=int, default=8)
    ap.add_argument("--skip-loop", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    line = dict(tool="train_bench", card=card(), replay_batch=kernel_part())
    if not a.skip_loop:
        line["loop"] = dict(games=a.games, playouts=a.playouts, blocks=a.blocks, batch=a.batch, precision="fp16 self-play, fp32 training",
                            **loop_part(a.games, a.playouts, a.blocks, a.batch, a.rounds, a.plies))
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
