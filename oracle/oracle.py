"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/liboracle.so (cchess_oracle.c).

Importers allowed: tests/, __graft_entry__.smoke(), bench.py (cpu_baseline / --impl reference).
The product package cchess_zero_b200/ must never import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "liboracle.so")
NLABEL = 2086
START = "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"
NET_IDS = {"hash_signed": 0, "hash_pos": 1, "mod17": 2}


def build(force=False):
    src = os.path.join(_HERE, "cchess_oracle.c")
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return _LIB


_lib = None
FWD_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float))


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        L.co_tree_new.restype = C.c_void_p
        L.co_tree_new.argtypes = [C.c_void_p]
        L.co_tree_free.argtypes = [C.c_void_p]
        L.co_tree_reload.argtypes = [C.c_void_p, C.c_void_p]
        L.co_tree_search.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, FWD_FN, C.c_void_p]
        L.co_tree_search_fake.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.co_tree_search_multi.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.co_tree_search_fifo.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.co_tree_root_children.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        L.co_tree_update.argtypes = [C.c_void_p, C.c_int]
        L.co_tree_root_board.argtypes = [C.c_void_p, C.c_void_p]
        L.co_tree_root_N.argtypes = [C.c_void_p]
        L.co_tree_stats.argtypes = [C.c_void_p, C.c_void_p]
        L.co_tree_signature.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
        L.co_tree_signature.restype = C.c_long
        L.co_tree_step_select.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_long, C.c_void_p]
        L.co_tree_step_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_float]
        L.co_tree_reset_playouts.argtypes = [C.c_void_p]
        L.co_batch_select.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_int]
        L.co_batch_finish.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.co_batch_fake_forward.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.co_legal_moves.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.co_apply_move.argtypes = [C.c_void_p, C.c_int]
        L.co_encode.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.co_flip_board.argtypes = [C.c_void_p, C.c_void_p]
        L.co_from_state.argtypes = [C.c_char_p, C.c_void_p]
        L.co_to_state.argtypes = [C.c_void_p, C.c_char_p]
        L.co_fake_forward.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.co_labels.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def labels():
    buf = np.zeros((NLABEL, 4), dtype=np.uint8)
    lib().co_labels(_p(buf))
    return [bytes(r).decode() for r in buf]


def label_index(src, dst):
    return lib().co_label_index(int(src), int(dst))


def unflipped_index():
    return [lib().co_unflipped_index(i) for i in range(NLABEL)]


def from_state(s):
    b = np.zeros(90, dtype=np.uint8)
    if lib().co_from_state(s.encode(), _p(b)) != 0:
        raise ValueError("bad state string: %r" % s)
    return b


def to_state(b):
    out = C.create_string_buffer(128)
    lib().co_to_state(_p(np.ascontiguousarray(b, dtype=np.uint8)), out)
    return out.value.decode()


def move_str(mv):
    s, d = int(mv) & 127, int(mv) >> 7
    return "abcdefghi"[s % 9] + str(s // 9) + "abcdefghi"[d % 9] + str(d // 9)


def move_from_str(m):
    s = int(m[1]) * 9 + (ord(m[0]) - 97)
    d = int(m[3]) * 9 + (ord(m[2]) - 97)
    return s | (d << 7)


def legal_moves(board, side):
    out = np.zeros(136, dtype=np.uint16)
    n = lib().co_legal_moves(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side), _p(out))
    return out[:n].copy()


def apply_move(board, mv):
    b = np.array(board, dtype=np.uint8, copy=True)
    cap = lib().co_apply_move(_p(b), int(mv))
    return b, cap


def encode(board, side):
    out = np.zeros((9, 10, 14), dtype=np.float32)
    lib().co_encode(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side), _p(out))
    return out


def flip_board(board):
    o = np.zeros(90, dtype=np.uint8)
    lib().co_flip_board(_p(np.ascontiguousarray(board, dtype=np.uint8)), _p(o))
    return o


def fake_forward(net, x):
    x = np.ascontiguousarray(x, dtype=np.float32).reshape(-1, 1260)
    lo = np.zeros((x.shape[0], NLABEL), dtype=np.float32)
    v = np.zeros((x.shape[0], 1), dtype=np.float32)
    lib().co_batch_fake_forward(NET_IDS[net] if isinstance(net, str) else int(net), x.shape[0], _p(x), _p(lo), _p(v), 1)
    return lo, v


class Tree:
    """One game's search tree (MCTS_tree + the root leaf_node, main.py:234-276)."""

    def __init__(self, board=None):
        self.b0 = from_state(START) if board is None else np.ascontiguousarray(board, dtype=np.uint8)
        self.h = lib().co_tree_new(_p(self.b0))
        self._cb = None

    def __del__(self):
        try:
            lib().co_tree_free(self.h)
        except Exception:
            pass

    def reload(self, board=None):
        b = from_state(START) if board is None else np.ascontiguousarray(board, dtype=np.uint8)
        lib().co_tree_reload(self.h, _p(b))

    def search(self, side, rr, playouts, net):
        """net: stand-in net name/id, or a python callable (x[1,9,10,14]) -> (logits[1,2086], value[1,1])."""
        if callable(net):
            def cb(ctx, x, lo, v):
                xa = np.ctypeslib.as_array(x, shape=(1, 9, 10, 14))
                l, val = net(xa)
                np.ctypeslib.as_array(lo, shape=(NLABEL,))[:] = np.asarray(l, dtype=np.float32).reshape(-1)
                v[0] = float(np.asarray(val).reshape(-1)[0])
            self._cb = FWD_FN(cb)
            return lib().co_tree_search(self.h, side, rr, playouts, self._cb, None)
        nid = NET_IDS[net] if isinstance(net, str) else int(net)
        return lib().co_tree_search_fake(self.h, side, rr, playouts, nid)

    def search_multi(self, side, rr, playouts, K, net):
        """cchess_zero_b200's own leaf-parallel schedule (K leaves per wave), serial specification; see cchess_oracle.c."""
        return lib().co_tree_search_multi(self.h, side, rr, playouts, int(K), NET_IDS[net] if isinstance(net, str) else int(net))

    def search_fifo(self, side, rr, playouts, K, net):
        """The reference's search_threads = K schedule in canonical (deterministic FIFO) form; see cchess_oracle.c / detloop.py."""
        return lib().co_tree_search_fifo(self.h, side, rr, playouts, int(K), NET_IDS[net] if isinstance(net, str) else int(net))

    def root_children(self):
        mv = np.zeros(136, dtype=np.uint16)
        N = np.zeros(136, dtype=np.int32)
        W = np.zeros(136, dtype=np.float32)
        P = np.zeros(136, dtype=np.float32)
        Q = np.zeros(136, dtype=np.float32)
        n = lib().co_tree_root_children(self.h, _p(mv), _p(N), _p(W), _p(P), _p(Q))
        n = max(n, 0)
        return mv[:n].copy(), N[:n].copy(), W[:n].copy(), P[:n].copy(), Q[:n].copy()

    def update(self, idx):
        if lib().co_tree_update(self.h, int(idx)) != 0:
            raise KeyError(idx)

    def root_board(self):
        b = np.zeros(90, dtype=np.uint8)
        lib().co_tree_root_board(self.h, _p(b))
        return b

    def root_N(self):
        return lib().co_tree_root_N(self.h)

    def stats(self):
        s = np.zeros(5, dtype=np.int64)
        lib().co_tree_stats(self.h, _p(s))
        return dict(n_expand=int(s[0]), n_playout=int(s[1]), sum_L=int(s[2]), sum_c=int(s[3]), error=int(s[4]))

    def signature(self, cap=1 << 20):
        out = np.zeros((cap, 6), dtype=np.int64)
        n = lib().co_tree_signature(self.h, _p(out), cap)
        if n > cap:
            return self.signature(int(n))
        return out[:n].copy()


def softmax(x):
    """main.py:1111-1116"""
    probs = np.exp(x - np.max(x))
    probs /= np.sum(probs)
    return probs


def flip_label(m):
    """flipped_uci_labels, main.py:23-27"""
    return "".join(str(9 - int(a)) if a.isdigit() else a for a in m)


def game_end(board, side, rr):
    """The reference's end test after a move (main.py:1380-1392, in the engine's order): a king taken -> (1, winner), rr >= 60 ->
    (2, -1); (0, -1) while the game runs."""
    hasK, hask = (board == 1).any(), (board == 8).any()
    if not hasK or not hask:
        return 1, (1 if not hasK else 0) if hask else 0
    return (2, -1) if rr >= 60 else (0, -1)


def selfplay_game(net, playouts, rs, exploration=True, temperature=1, max_plies=10000, search_threads=1, tree=None, search=None,
                  end=game_end):
    """cchess_main.selfplay (main.py:1493-1554) + get_action (1332-1358) over the C tree.

    rs: np.random.RandomState standing in for the global np.random of the reference.
    search_threads > 1: every search runs the reference's K-coroutine schedule in canonical form (co_tree_search_fifo).
    tree, search, end: another specification's tree at the start position, its search(side, rr) -> error and its end test
    end(board, side, rr) -> (code, winner) (tests/search_spec.py: strict rules, root noise) instead of this module's.
    Returns dict(states, pis (dense [n,2086] f64), z, actions, visits, end (the end code), boards (every position played from), players).
    """
    if tree is None:
        tree = Tree()
        search = (lambda side, rr: tree.search(side, rr, playouts, net)) if search_threads <= 1 else \
            (lambda side, rr: tree.search_fifo(side, rr, playouts, search_threads, net))
    l2i = {m: i for i, m in enumerate(labels())}
    board = from_state(START)
    side, rr = 0, 0
    states, pis, players, actions, all_visits, boards = [], [], [], [], [], []
    with np.errstate(divide="ignore"):
        while True:
            err = search(side, rr)
            if err:
                raise RuntimeError("oracle tree error %d" % err)
            mv, N, W, P, Q = tree.root_children()
            visits = tuple(int(v) for v in N)
            probs = softmax(1.0 / temperature * np.log(visits))
            if exploration:
                p = 0.75 * probs + 0.25 * rs.dirichlet(0.3 * np.ones(len(probs)))
            else:
                p = probs
            acts = [move_str(m) for m in mv]
            act = rs.choice(acts, p=p)
            idx = acts.index(act)
            tree.update(idx)
            boards.append(board.copy())
            sboard = flip_board(board) if side == 1 else board
            states.append(to_state(sboard))
            prob = np.zeros(NLABEL)
            for a, pr in zip(acts, probs):
                prob[l2i[flip_label(a) if side == 1 else a]] = pr
            pis.append(prob)
            players.append(side)
            actions.append(act)
            all_visits.append(visits)
            board, cap = apply_move(board, mv[idx])
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            code, winner = end(board, side, rr)
            if code in (1, 3):
                z = np.where(np.array(players) == winner, 1.0, -1.0)
                break
            if code == 2 or len(states) >= max_plies:
                z = np.zeros(len(players))
                break
    return dict(states=states, pis=np.array(pis), z=z, actions=actions, visits=all_visits, end=code, boards=boards, players=players)
