#!/usr/bin/env python
"""Size and cost of saving and restoring the games in flight (cz_engine_snapshot / cz_engine_restore, SelfPlay.save_games).

  python tools/snapshot_bench.py [--games 1024 --playouts 400 --blocks 7 --plies 30 --repeats 5] [--out FILE]

Self-play of `games` x `playouts` with a `blocks`-block fp16 network (CUDA graph, auto reset) for `plies` plies, then at rest:
  * blob bytes and the retained tree per game (alloc words: mean, max) -- the tree kept between plies, not a mid-search high-water mark;
  * Engine.snapshot() wall time (header fetch, pack kernel, device->host copy, each call ending in a synchronisation) and
    Engine.restore() wall time (host validation, host->device copy, unpack kernel), `repeats` times each, medians;
  * cz_snapshot_check alone (the host validator restore runs);
  * the kernels and copies alone from torch.profiler (CUDA activity records of one snapshot and one restore);
  * SelfPlay.save_games / load_games wall time (np.savez to a temporary directory, read back without pickle);
and checks that every tree signature is unchanged by the save / restore cycle.  Prints one JSON line (card name and power limit read
in the same run)."""
import argparse
import contextlib
import ctypes as C
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from arena_bench import card, timed  # noqa: E402


def allocs(blob):
    """alloc words of every game section (offset differences minus the section head)."""
    w = blob.view(np.uint32)
    B, narr = int(w[6]), int(w[8])
    off = blob[48:48 + 8 * (B + 1)].view(np.int64)
    return np.diff(off) - (80 if narr == 6 else 52)


def profiled(fn):
    """CUDA time (us) of the snapshot kernels and copies in one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        if "k_snapshot" in name or "Memcpy" in name:
            key = "k_snapshot_pack" if "k_snapshot_pack" in name else "k_snapshot_unpack" if "k_snapshot_unpack" in name else name
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = getattr(ev, "cuda_time_total", 0.0)
            out[key] = round(out.get(key, 0.0) + float(t), 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--plies", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    from cchess_zero_b200._lib import lib
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import network_selfplay
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        net = policy_value_network(a.blocks, precision="fp16", seed=0, save_dir=d)
    sp = network_selfplay(net, a.games, a.playouts, seeds=range(a.games), auto_reset=True, keep_records=True, arena_words=1 << 20)
    sp.capture_graph()
    t0 = time.perf_counter()
    for _ in range(a.plies):
        sp.step()
        sp.pop_finished()
    play_s = time.perf_counter() - t0
    e = sp.engine
    sig0 = [e.tree_signature(g) for g in range(a.games)]

    blob = e.snapshot()                                                # warm-up: staging allocation
    e.restore(blob)
    t_snap = [timed(e.snapshot) for _ in range(a.repeats)]
    t_rest = [timed(lambda: e.restore(blob)) for _ in range(a.repeats)]
    ptr = blob.ctypes.data_as(C.c_void_p)
    t_check = []
    for _ in range(a.repeats):
        t1 = time.perf_counter()
        assert lib().cz_snapshot_check(ptr, blob.nbytes, a.games, 1, 5, 1 << 20) == 0, lib().cz_last_error().decode()
        t_check.append(time.perf_counter() - t1)
    prof_snap, prof_rest = profiled(e.snapshot), profiled(lambda: e.restore(blob))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "games.npz")
        t_save = [timed(lambda: sp.save_games(path)) for _ in range(a.repeats)]
        t_load = [timed(lambda: sp.load_games(path)) for _ in range(a.repeats)]
        file_bytes = os.path.getsize(path)
    unchanged = all(np.array_equal(s, e.tree_signature(g)) for g, s in enumerate(sig0))
    al = allocs(blob)
    ms = lambda ts: round(1e3 * float(np.median(ts)), 3)  # noqa: E731
    line = dict(tool="snapshot_bench", card=card(), games=a.games, playouts=a.playouts, blocks=a.blocks, plies=a.plies,
                play_s=round(play_s, 1), blob_bytes=int(blob.nbytes), alloc_words_mean=float(al.mean()), alloc_words_max=int(al.max()),
                snapshot_ms=ms(t_snap), restore_ms=ms(t_rest), check_ms=ms(t_check), profile_snapshot_us=prof_snap,
                profile_restore_us=prof_rest, save_games_ms=ms(t_save), load_games_ms=ms(t_load), games_file_bytes=file_bytes,
                signatures_unchanged=unchanged)
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
