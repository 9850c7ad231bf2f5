#!/usr/bin/env python
"""Cost of strict rules inside the device search: SelfPlay with rules='reference' against rules='strict' in the training
configuration (1024 games x 400 playouts, 7-block fp16 network on its native plan, CUDA-graph search), the two alternating in one run.

  python tools/strict_search_bench.py [--games 1024 --playouts 400 --plies 12 --rounds 2 --wave-plies 2] [--out FILE]

Per rules and round: `plies` self-play plies (auto reset, after one warm-up ply), timed one by one with CUDA events; expansions/s =
expansions (engine counters) / summed ply time.  k_wave per launch: `wave-plies` further plies run eagerly (no graph) with CUDA events
around every wave launch (the network is outside them).  Finished games are counted by outcome: from the start position no strictly
legal move ever takes a king, so a decisive strict game ended by mate (checkmate or stalemate), a decisive reference game by a king
capture.  Prints one JSON line (card name and power limit read in the same run)."""
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


def ply_times(sp, n):
    """n plies, each timed by CUDA events; -> (ms per ply, expansions, finished records)"""
    e = sp.engine
    x0 = e.counters()["n_expand"]
    ms, fin = [], []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        sp.step()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        fin += [rec for _, rec in sp.pop_finished()]
    return ms, e.counters()["n_expand"] - x0, fin


def wave_times(sp, n):
    """n eager plies with CUDA events around every k_wave launch; -> ms per launch"""
    e, graph = sp.engine, sp.graph
    sp.graph = None
    wave, ev = e.wave, []

    def timed(*args):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        wave(*args)
        b.record()
        ev.append((a, b))
    e.wave = timed
    try:
        for _ in range(n):
            sp.step()
            sp.pop_finished()
    finally:
        e.wave, sp.graph = wave, graph
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games", type=int, default=1024)
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--plies", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--wave-plies", type=int, default=2)
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    from cchess_zero_b200.net import policy_value_network
    from cchess_zero_b200.selfplay import network_selfplay
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        net = policy_value_network(a.blocks, precision="fp16", seed=0, save_dir=d)
    sps = {}
    for rules in ("reference", "strict"):
        sps[rules] = network_selfplay(net, a.games, a.playouts, seeds=range(a.games), arena_words=1 << 19, auto_reset=True, rules=rules)
        sps[rules].capture_graph()
        ply_times(sps[rules], 1)                                        # warm-up ply
    acc = {r: dict(ms=[], exp=0, fin=[], wave_ms=[]) for r in sps}
    for _ in range(a.rounds):
        for rules, sp in sps.items():
            ms, x, fin = ply_times(sp, a.plies)
            acc[rules]["ms"] += ms
            acc[rules]["exp"] += x
            acc[rules]["fin"] += fin
            acc[rules]["wave_ms"] += wave_times(sp, a.wave_plies)
    out = dict(card=card(), games=a.games, playouts=a.playouts, blocks=a.blocks, precision="fp16", plies_per_round=a.plies, rounds=a.rounds)
    for rules, v in acc.items():
        wins = sum(1 for r in v["fin"] if r.winner in ("w", "b"))
        out[rules] = dict(ply_ms_median=float(np.median(v["ms"])), expansions_per_s=v["exp"] / (sum(v["ms"]) / 1e3),
                          k_wave_us_median=1e3 * float(np.median(v["wave_ms"])), k_wave_launches=len(v["wave_ms"]),
                          finished=len(v["fin"]), decisive=wins, draws=len(v["fin"]) - wins,
                          decisive_share=wins / max(1, len(v["fin"])))
    out["ply_time_ratio_strict_over_reference"] = out["strict"]["ply_ms_median"] / out["reference"]["ply_ms_median"]
    out["k_wave_ratio_strict_over_reference"] = out["strict"]["k_wave_us_median"] / out["reference"]["k_wave_us_median"]
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
