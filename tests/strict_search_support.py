"""TEST INFRASTRUCTURE shared by test_strict_search_host.py and test_gpu_strict_search.py: the strict-rules search specification
(tests/strict_search_oracle.c, compiled together with oracle/cchess_oracle.c and tests/strict_oracle.c), a self-play game loop and an
arena game loop over it, hand-made positions with a mate in one, and the search cases the tree tests use."""
import ctypes as C
import os
import subprocess

import numpy as np

from strict_support import ROOT, _dir, _p, oracle_lib, random_play

_lib = None
NETS = ("hash_signed", "hash_pos", "mod17")
NET_IDS = {"hash_signed": 0, "hash_pos": 1, "mod17": 2}


def lib():
    global _lib
    if _lib is None:
        oracle_lib()                                      # (creates the build directory)
        so = os.path.join(_dir(), "libstrictsearch.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "strict_search_oracle.c"), os.path.join(ROOT, "tests", "strict_oracle.c"),
                               os.path.join(ROOT, "oracle", "cchess_oracle.c"), "-lm", "-lpthread"])
        L = C.CDLL(so)
        L.ss_tree_new.restype = C.c_void_p
        L.ss_tree_new.argtypes = [C.c_void_p]
        L.ss_tree_free.argtypes = [C.c_void_p]
        L.ss_tree_search_fake.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.ss_tree_root_children.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        L.ss_tree_update.argtypes = [C.c_void_p, C.c_int]
        L.ss_tree_root_mated.argtypes = [C.c_void_p]
        L.ss_tree_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.ss_tree_signature.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
        L.ss_tree_signature.restype = C.c_long
        L.so_in_check.argtypes = [C.c_void_p, C.c_int]
        L.so_strict_moves.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class StrictTree:
    """One game's search tree under the strict rules (the specification of k_wave<T, true>)."""

    def __init__(self, board):
        self.h = lib().ss_tree_new(_p(np.ascontiguousarray(board, dtype=np.uint8)))

    def __del__(self):
        try:
            lib().ss_tree_free(self.h)
        except Exception:
            pass

    def search(self, side, rr, playouts, net):
        return lib().ss_tree_search_fake(self.h, int(side), int(rr), int(playouts), NET_IDS[net])

    def root_children(self):
        mv, N = np.zeros(128, np.uint16), np.zeros(128, np.int32)
        W, P, Q = np.zeros(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.float32)
        n = max(lib().ss_tree_root_children(self.h, _p(mv), _p(N), _p(W), _p(P), _p(Q)), 0)
        return mv[:n].copy(), N[:n].copy(), W[:n].copy(), P[:n].copy(), Q[:n].copy()

    def update(self, idx):
        if lib().ss_tree_update(self.h, int(idx)) != 0:
            raise KeyError(idx)

    def root_mated(self):
        return bool(lib().ss_tree_root_mated(self.h))

    def stats(self):
        s = np.zeros(6, np.int64)
        lib().ss_tree_stats(self.h, _p(s))
        return dict(n_expand=int(s[0]), n_playout=int(s[1]), sum_L=int(s[2]), sum_c=int(s[3]), sum_C=int(s[4]), error=int(s[5]))

    def signature(self, cap=1 << 16):
        out = np.zeros((cap, 6), np.int64)
        n = lib().ss_tree_signature(self.h, _p(out), cap)
        if n > cap:
            return self.signature(int(n))
        return out[:n].copy()


def strict_moves(board, side):
    """The strictly legal moves (u16 codes, move-generation order, first 128 pseudo-legal moves) by the brute-force definition."""
    mv, ok = np.zeros(512, np.uint16), np.zeros(512, np.uint8)
    n = lib().so_strict_moves(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side), _p(mv), _p(ok))
    n = min(n, 128)
    return mv[:n][ok[:n].astype(bool)].copy()


def in_check(board, side):
    return bool(lib().so_in_check(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side)))


def game_end(board, side, rr):
    """The end test after a move, in the engine's order: a king taken -> (1, winner), rr >= 60 -> (2, -1), the side to move without a
    strictly legal move -> (3, the side that just moved); (0, -1) while the game runs."""
    hasK, hask = (board == 1).any(), (board == 8).any()
    if not hasK or not hask:
        return 1, (1 if not hasK else 0) if hask else 0
    if rr >= 60:
        return 2, -1
    if len(strict_moves(board, side)) == 0:
        return 3, side ^ 1
    return 0, -1


def selfplay_game(net, playouts, rs, temperature=1, board=None, max_plies=10000):
    """oracle.selfplay_game (cchess_main.selfplay + get_action) over the strict specification tree: the strict rules' SelfPlay game.
    -> dict(states, pis (dense [n,2086] f64), z, actions, visits, end (terminal code), boards (every position played from))."""
    from oracle import oracle as O
    lab = O.labels()
    l2i = {m: i for i, m in enumerate(lab)}
    board = O.from_state(O.START) if board is None else np.array(board, dtype=np.uint8)
    tree = StrictTree(board)
    side, rr = 0, 0
    states, pis, players, actions, all_visits, boards = [], [], [], [], [], []
    z, end = None, 0
    with np.errstate(divide="ignore"):
        while True:
            err = tree.search(side, rr, playouts, net)
            if err:
                raise RuntimeError("strict specification tree error %d" % err)
            mv, N, W, P, Q = tree.root_children()
            visits = tuple(int(v) for v in N)
            probs = O.softmax(1.0 / temperature * np.log(visits))
            p = 0.75 * probs + 0.25 * rs.dirichlet(0.3 * np.ones(len(probs)))
            acts = [O.move_str(m) for m in mv]
            act = rs.choice(acts, p=p)
            idx = acts.index(act)
            tree.update(idx)
            boards.append(board.copy())
            sboard = O.flip_board(board) if side == 1 else board
            states.append(O.to_state(sboard))
            prob = np.zeros(O.NLABEL)
            for a, pr in zip(acts, probs):
                prob[l2i[O.flip_label(a) if side == 1 else a]] = pr
            pis.append(prob)
            players.append(side)
            actions.append(act)
            all_visits.append(visits)
            board, cap = O.apply_move(board, mv[idx])
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            end, winner = game_end(board, side, rr)
            if end in (1, 3):
                z = np.where(np.array(players) == winner, 1.0, -1.0)
                break
            if end == 2 or len(states) >= max_plies:
                z = np.zeros(len(players))
                break
    return dict(states=states, pis=np.array(pis), z=z, actions=actions, visits=all_visits, end=end, boards=boards, players=players)


def match_game(net_red, net_black, playouts, rs, opening_plies, opening_T, T, board=None, side=0, max_plies=None, rr=0):
    """tests/arena_oracle.match_game over the strict specification trees (one per player; the other player's tree follows the move,
    or starts afresh when its root is not expanded).  -> dict(moves, winner 0 'w' / 1 'b' / 2 draw, plies, adjudicated, end)."""
    from oracle import oracle as O
    board = O.from_state(O.START) if board is None else np.array(board, dtype=np.uint8)
    trees = [StrictTree(board), StrictTree(board)]
    nets = [net_red, net_black]
    moves = []
    winner, adjudicated, end = -1, False, 0
    with np.errstate(divide="ignore"):
        while True:
            me = trees[side]
            if me.search(side, rr, playouts, nets[side]):
                raise RuntimeError("strict specification tree error")
            mv, N, _, _, _ = me.root_children()
            visits = tuple(int(v) for v in N)
            temp = opening_T if len(moves) < opening_plies else T
            probs = O.softmax(1.0 / temp * np.log(visits))
            acts = [O.move_str(m) for m in mv]
            idx = acts.index(rs.choice(acts, p=probs))
            move = int(mv[idx])
            me.update(idx)
            board, cap = O.apply_move(board, move)
            other = trees[side ^ 1]
            omv = other.root_children()[0]
            if len(omv):
                other.update(list(omv).index(move))
            else:
                trees[side ^ 1] = StrictTree(board)
            moves.append(move)
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            end, w = game_end(board, side, rr)
            if end:
                winner = 2 if end == 2 else w
                break
            if max_plies is not None and len(moves) >= max_plies:
                winner, adjudicated = 2, True
                break
    return dict(moves=moves, winner=winner, plies=len(moves), adjudicated=adjudicated, end=end)


# Hand-made positions with a mate in one for the side to move: (name, state (rank 0 = Red's back rank first), side to move, the
# mating move, True when the position it leaves is a stalemate rather than a checkmate)
MATE_IN_ONE = [
    # the rook on b1 holds rank 1; a5a0 checks along rank 0 and the red king has no square left
    ("checkmate_by_rook", "4K4/1r7/9/9/9/r8/9/9/9/3k5", "b", "a5a0", False),
    # i5i1 takes rank 1 from the red king; d0e0 would face the black king: no check, no move
    ("stalemate_by_rook", "3K5/9/9/9/9/8r/9/9/9/4k4", "b", "i5i1", True),
]


def random_cases(seed, n):
    """About n search cases (board, side, rr, playouts, net) from random play, over-weighted towards positions in check and positions
    with a mated position among their children or grandchildren (mates near the root)."""
    rng = np.random.RandomState(seed)
    boards, sides = random_play(seed, 60000)
    live = np.array([(b == 1).any() and (b == 8).any() for b in boards])
    boards, sides = boards[live], sides[live]
    chk = np.array([in_check(b, s) for b, s in zip(boards, sides)])
    near = []
    for i in rng.choice(len(boards), 3000, replace=False):
        b, s = boards[i], int(sides[i])
        mv = strict_moves(b, s)
        if len(mv) == 0:
            continue
        from oracle import oracle as O
        if any(len(strict_moves(O.apply_move(b, int(m))[0], s ^ 1)) == 0 for m in mv):
            near.append(i)
    pick = list(rng.choice(np.nonzero(chk)[0], n // 3, replace=False)) + near[: n // 3]
    pick += list(rng.choice(len(boards), n - len(pick), replace=False))
    return [dict(board=boards[i], side=int(sides[i]), rr=int(rng.choice([0, 56, 58])), playouts=int(rng.choice([50, 150, 250])),
                 net=NETS[k % 3]) for k, i in enumerate(pick) if len(strict_moves(boards[i], int(sides[i])))]
