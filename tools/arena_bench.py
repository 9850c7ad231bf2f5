#!/usr/bin/env python
"""Arena throughput: a match of two 7-block fp16 networks (seeds 1 vs 0) over 1024 concurrent games (512 colour-swapped pairs) at
400 playouts per move, beside self-play of the same game count and playouts on the same card.

  python tools/arena_bench.py [--games 1024 --playouts 400 --rounds 4 --plies 2 --max-plies 150] [--out FILE]

1. Alternated per-ply times: `rounds` x (`plies` match plies, then `plies` SelfPlay plies), both from the start position, CUDA
   synchronised around every ply.  A match ply searches the same number of trees as a self-play ply, split over two engines of
   half the batch (the candidate's and the best network's).
2. The match is then played out (draw adjudicated after --max-plies plies): plies/s and games/hour of the whole match.
Prints one JSON line (card name and power limit read in the same run)."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    out = dict(name=torch.cuda.get_device_name(0), power_limit_w=None)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        f = [x.strip() for x in r.stdout.strip().split(",")]
        out["name"], out["power_limit_w"] = f[0], float(f[1])
    except Exception as e:  # the card name from torch stays
        out["power_limit_error"] = str(e)
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--plies", type=int, default=2)
    ap.add_argument("--max-plies", type=int, default=150)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from cchess_zero_b200.arena import Match
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import SelfPlay
    torch.cuda.set_device(0)
    info = card()
    with contextlib.redirect_stdout(io.StringIO()), tempfile.TemporaryDirectory() as d:
        best = policy_value_network(7, precision="fp16", seed=0, save_dir=d)
        cand = policy_value_network(7, precision="fp16", seed=1, save_dir=d)
    n, P = a.games, a.playouts
    m = Match(cand, best, n, P, seeds=range(n), max_plies=a.max_plies)
    sp = SelfPlay(n, None, P, seeds=range(n), auto_reset=True, keep_records=False, plan=best.native_plan(n), arena_words=1 << 20)
    sp.capture_graph()
    t_match, t_self = [timed(m.step)], [timed(sp.step)]          # first plies: graph warm-up, reported apart
    first = dict(match_s=t_match[0], selfplay_s=t_self[0])
    t_match, t_self = [], []
    for _ in range(a.rounds):
        t_match += [timed(m.step) for _ in range(a.plies)]
        t_self += [timed(sp.step) for _ in range(a.plies)]
    sp_hw = sp.engine.counters()["max_arena_words"]
    del sp
    torch.cuda.empty_cache()
    t_rest, plies = 0.0, 1 + a.rounds * a.plies
    while m.live.any():
        t_rest += timed(m.step)
        plies += 1
    total = first["match_s"] + sum(t_match) + t_rest
    r = m.result()
    moves = int(sum(g["plies"] for g in r.games))
    hw = max(c["max_arena_words"] for c in m.counters())
    line = dict(tool="arena_bench", card=info, games=n, playouts=P, networks="7 residual blocks fp16, seeds 1 (candidate) vs 0",
                search_threads=1, max_plies=a.max_plies,
                match_ply_ms_median=1e3 * float(np.median(t_match)), selfplay_ply_ms_median=1e3 * float(np.median(t_self)),
                match_ply_ms=[round(1e3 * t, 2) for t in t_match], selfplay_ply_ms=[round(1e3 * t, 2) for t in t_self],
                first_ply_s=first, match_plies=plies, match_seconds=total, plies_per_s=plies / total, moves_per_s=moves / total,
                games_per_hour=n * 3600.0 / total, mean_game_plies=moves / n, adjudicated=sum(g["adjudicated"] for g in r.games),
                wins=r.wins, draws=r.draws, losses=r.losses, score=r.score,
                arena_high_water_words=dict(match=hw, selfplay=sp_hw))
    s = json.dumps(line)
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
