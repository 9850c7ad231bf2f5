#!/usr/bin/env python
"""Cost of root exploration noise: SelfPlay without noise against SelfPlay(root_noise=(0.25, 0.3)) in the training configuration
(1024 games, 7-block fp16 network on its native plan, CUDA-graph search), at 400 and 1200 playouts, the two alternating in one run.

  python tools/root_noise_bench.py [--games 1024 --playouts 400 1200 --plies 8 --rounds 3 --split-plies 4] [--out FILE]

Per playout count, setting and round: `plies` self-play plies (auto reset, after one warm-up ply), timed one by one with CUDA events.
The added time is split on `split-plies` further noisy plies whose pre-pass runs step by step, each step closed by a device
synchronise and timed on the host clock: begin_search(0) + the pre-pass waves (with their network passes; the engine launches they
made and the roots they had to expand are listed per ply), the root-count read, the host Dirichlet draws, the upload of eta, and
k_root_noise (CUDA events).  Prints one JSON line (card name and power limit read in the same run)."""
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
from arena_bench import card  # noqa: E402


def ply_times(sp, n):
    """n plies, each timed by CUDA events -> ms per ply"""
    ms = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sp.step()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        sp.pop_finished()
    return ms


def split_plies(sp, n):
    """n noisy plies whose pre-pass (SelfPlay._noise_roots, the same calls) is timed step by step -> {step: [ms per ply]}"""
    from cchess_zero_b200._lib import lib
    e = sp.engine
    eps, alpha = sp.root_noise
    out = dict(pending_roots=[], prepass_waves=[], prepass_launches=[], count_read=[], host_draws=[], upload=[], k_root_noise=[])
    eta_dev = torch.zeros((sp.B, 128), dtype=torch.float64, device="cuda")
    vp = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731

    def timed_noise_roots(m):
        out["pending_roots"].append(int((m & (e.root_counts() < 0)).sum()))   # roots the pre-pass has to expand (outside the timing)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        l0 = e.launches
        e.begin_search(0, m.astype(np.uint8))
        sp.waves += sp._run_waves(0, graph=False)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        out["prepass_launches"].append(e.launches - l0)
        n = np.ascontiguousarray(e.root_counts(), dtype=np.int32)
        t2 = time.perf_counter()
        sel = (m & sp.live & (n > 0)).astype(np.uint8)
        assert lib().cz_host_dirichlet(sp.B, vp(sel), vp(n), C.byref(C.c_double(alpha)), vp(sp._noise_mt), vp(sp._eta), sp._threads) == 0
        t3 = time.perf_counter()
        eta_dev.copy_(torch.from_numpy(sp._eta))
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        e.root_noise(sel, eta_dev, eps)
        b.record()
        b.synchronize()
        out["prepass_waves"].append(1e3 * (t1 - t0))
        out["count_read"].append(1e3 * (t2 - t1))
        out["host_draws"].append(1e3 * (t3 - t2))
        out["upload"].append(1e3 * (t4 - t3))
        out["k_root_noise"].append(a.elapsed_time(b))
    sp._noise_roots = timed_noise_roots
    try:
        for _ in range(n):
            sp.step()
            sp.pop_finished()
    finally:
        del sp._noise_roots
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, nargs="+", default=[400, 1200])
    ap.add_argument("--plies", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--split-plies", type=int, default=4)
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--eps", type=float, default=0.25)
    ap.add_argument("--alpha", type=float, default=0.3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import network_selfplay
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        net = policy_value_network(a.blocks, precision="fp16", seed=0, save_dir=d)
    out = dict(card=card(), games=a.games, blocks=a.blocks, precision="fp16", root_noise=[a.eps, a.alpha], plies_per_round=a.plies,
               rounds=a.rounds)
    for p in a.playouts:
        sps = {}
        for name, noise in (("off", None), ("on", (a.eps, a.alpha))):
            sps[name] = network_selfplay(net, a.games, p, seeds=range(a.games), arena_words=1 << 20, auto_reset=True, root_noise=noise)
            sps[name].capture_graph()
            ply_times(sps[name], 1)                                    # warm-up ply
        acc = {k: [] for k in sps}
        for _ in range(a.rounds):
            for name, sp in sps.items():
                acc[name] += ply_times(sp, a.plies)
        split = split_plies(sps["on"], a.split_plies)
        r = {k: dict(ply_ms_median=float(np.median(v)), ply_ms_min=float(np.min(v)), plies=len(v)) for k, v in acc.items()}
        r["added_ms_median"] = r["on"]["ply_ms_median"] - r["off"]["ply_ms_median"]
        r["added_share"] = r["added_ms_median"] / r["off"]["ply_ms_median"]
        r["split_ms_median"] = {k: float(np.median(v)) for k, v in split.items() if k not in ("pending_roots", "prepass_launches")}
        r["split_pending_roots"], r["split_prepass_launches"] = split["pending_roots"], split["prepass_launches"]
        out["playouts_%d" % p] = r
        del sps
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
