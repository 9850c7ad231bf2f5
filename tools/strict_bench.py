#!/usr/bin/env python
"""Cost of strict legality on the device: k_strict_moves (move list + 128-bit mask of strictly legal moves + in-check / mated flags)
against k_legal_moves (move list only) on the same mid-game positions.

  python tools/strict_bench.py [--sizes 1024 65536 --plies 30 --launches 200 --repeats 7] [--out FILE]

Positions: `plies` uniformly random pseudo-legal plies from the start position (seeded), games that lost a king dropped.  Each kernel
is timed by CUDA events around `launches` back-to-back launches through its device-pointer entry point (cz_*_dev: no copies, no
allocation), the two kernels alternating, `repeats` rounds, medians.  Algorithmic bytes per position: 91 in (board, side) and
260 out (128 moves, count) for k_legal_moves, 277 out (+ 16 mask + 1 flags) for k_strict_moves.  Prints one JSON line (card name
and power limit read in the same run)."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from arena_bench import card  # noqa: E402

BYTES_IN, BYTES_OUT_LEGAL, BYTES_OUT_STRICT = 91, 260, 277


def midgame(n, plies, seed):
    from cchess_zero_b200 import rules
    rng = np.random.RandomState(seed)
    boards = np.tile(rules.state_to_board(rules.START_STATE), (n + n // 4, 1))
    sides = np.zeros(len(boards), np.uint8)
    for _ in range(plies):
        mv, cnt = rules.legal_moves_batch(boards, sides)
        pick = (rng.random_sample(len(boards)) * cnt).astype(np.int64)
        boards, _ = rules.apply_moves_batch(boards, mv[np.arange(len(boards)), pick])
        sides ^= 1
    keep = ((boards == 1).sum(1) == 1) & ((boards == 8).sum(1) == 1)
    boards, sides = boards[keep][:n], sides[keep][:n]
    assert len(boards) == n, "too many games lost a king"
    return boards, sides


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1024, 65536])
    ap.add_argument("--plies", type=int, default=30)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    from cchess_zero_b200._lib import check, lib
    L = lib()
    results = []
    for n in a.sizes:
        hb, hs = midgame(n, a.plies, 0)
        boards, sides = torch.from_numpy(hb).cuda(), torch.from_numpy(hs).cuda()
        moves = torch.zeros((n, 128), dtype=torch.int16, device="cuda")
        counts = torch.zeros(n, dtype=torch.int32, device="cuda")
        mask = torch.zeros((n, 4), dtype=torch.int32, device="cuda")
        flags = torch.zeros(n, dtype=torch.uint8, device="cuda")
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def legal():
            check(L.cz_legal_moves_dev(p(boards), p(sides), n, p(moves), p(counts), st), "cz_legal_moves_dev")

        def strict():
            check(L.cz_strict_moves_dev(p(boards), p(sides), n, p(moves), p(counts), p(mask), p(flags), st), "cz_strict_moves_dev")

        def us_per_launch(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.launches):
                fn()
            e1.record()
            e1.synchronize()
            return 1e3 * e0.elapsed_time(e1) / a.launches

        for fn in (legal, strict):                      # warm-up: module load, clocks
            for _ in range(20):
                fn()
        torch.cuda.synchronize()
        t_legal, t_strict = [], []
        for _ in range(a.repeats):
            t_legal.append(us_per_launch(legal))
            t_strict.append(us_per_launch(strict))
        fl = flags.cpu().numpy()
        ml, ms = float(np.median(t_legal)), float(np.median(t_strict))
        results.append(dict(positions=n, mean_moves=round(float(counts.float().mean()), 2), in_check=int((fl & 1).sum()), mated=int((fl & 2).sum()),
                            legal_us=round(ml, 2), strict_us=round(ms, 2), legal_us_min_max=[round(min(t_legal), 2), round(max(t_legal), 2)],
                            strict_us_min_max=[round(min(t_strict), 2), round(max(t_strict), 2)], ratio=round(ms / ml, 3),
                            legal_ns_per_position=round(1e3 * ml / n, 3), strict_ns_per_position=round(1e3 * ms / n, 3),
                            legal_gb_s=round(n * (BYTES_IN + BYTES_OUT_LEGAL) / ml / 1e3, 1),
                            strict_gb_s=round(n * (BYTES_IN + BYTES_OUT_STRICT) / ms / 1e3, 1)))
    s = json.dumps(dict(tool="strict_bench", card=card(), plies=a.plies, launches=a.launches, repeats=a.repeats,
                        bytes_per_position=dict(read=BYTES_IN, legal_written=BYTES_OUT_LEGAL, strict_written=BYTES_OUT_STRICT), results=results))
    print(s, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
