#!/usr/bin/env python
"""Cost of softmax priors: SelfPlay(priors='reference') against SelfPlay(priors='softmax') in the training configuration (1024 games,
7-block fp16 network on its native plan, CUDA-graph search), at 400 and 1200 playouts, the two alternating in one run.

  python tools/priors_bench.py [--games 1024 --playouts 400 1200 --plies 8 --rounds 3 --wave-launches 0] [--out FILE]

Per playout count, round and setting (the settings alternating): `plies` self-play plies (auto reset, after one warm-up ply), timed
one by one with CUDA events.  Then, in as many alternating rounds, one eager search per setting on the trees the plies left, whose
k_wave launches are timed one by one with CUDA events (all of them, or the first `wave-launches`; the network passes between them
untimed; the search plays no move).  Prints one JSON line (card name and power limit read in the same
run)."""
import argparse
import contextlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from arena_bench import card  # noqa: E402
from root_noise_bench import ply_times  # noqa: E402


def wave_times(sp, playouts, n):
    """k_wave launches of one eager search, each timed by CUDA events -> ms per launch (n > 0: the first n launches only; the search
    runs to its end either way)"""
    e = sp.engine
    e.begin_search(playouts, sp.live.astype(np.uint8))
    ms, waves = [], 0
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        e.wave(sp.nn_in, sp.logits, sp.value)
        b.record()
        b.synchronize()
        waves += 1
        if n <= 0 or len(ms) < n:
            ms.append(a.elapsed_time(b))
        if waves > playouts and e.unfinished() == 0:
            break
        sp.forward(sp.nn_in)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, nargs="+", default=[400, 1200])
    ap.add_argument("--plies", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--wave-launches", type=int, default=0, help="k_wave launches timed per search (0: all)")
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import network_selfplay
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        net = policy_value_network(a.blocks, precision="fp16", seed=0, save_dir=d)
    out = dict(card=card(), games=a.games, blocks=a.blocks, precision="fp16", plies_per_round=a.plies, rounds=a.rounds)
    for p in a.playouts:
        sps = {}
        for name in ("reference", "softmax"):
            sps[name] = network_selfplay(net, a.games, p, seeds=range(a.games), arena_words=1 << 20, auto_reset=True, priors=name)
            sps[name].capture_graph()
            ply_times(sps[name], 1)                                    # warm-up ply
        acc, waves = {k: [] for k in sps}, {k: [] for k in sps}
        for _ in range(a.rounds):
            for name, sp in sps.items():
                acc[name] += ply_times(sp, a.plies)
        for _ in range(a.rounds):                                      # after the timed plies: an eager search plays no move
            for name, sp in sps.items():
                waves[name] += wave_times(sp, p, a.wave_launches)
        r = {k: dict(ply_ms_median=float(np.median(v)), ply_ms_min=float(np.min(v)), plies=len(v),
                     k_wave_ms_median=float(np.median(waves[k])), k_wave_ms_mean=float(np.mean(waves[k])),
                     k_wave_launches=len(waves[k])) for k, v in acc.items()}
        r["added_ply_ms_median"] = r["softmax"]["ply_ms_median"] - r["reference"]["ply_ms_median"]
        r["added_ply_share"] = r["added_ply_ms_median"] / r["reference"]["ply_ms_median"]
        r["added_k_wave_ms_median"] = r["softmax"]["k_wave_ms_median"] - r["reference"]["k_wave_ms_median"]
        r["added_k_wave_ms_mean"] = r["softmax"]["k_wave_ms_mean"] - r["reference"]["k_wave_ms_mean"]
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
