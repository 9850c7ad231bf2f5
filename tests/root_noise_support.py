"""TEST INFRASTRUCTURE shared by test_root_noise_host.py and test_gpu_root_noise.py: the specification of root exploration noise over
the C trees (tests/root_noise_oracle.c and tests/root_noise_strict_oracle.c: the reference-rules tree at K = 1 and in the K-coroutine
schedule, and the strict-rules tree, each with a root-prior setter), a self-play game loop over them, and an engine-interface stand-in
that drives SelfPlay's host loop on the CPU.

A noisy search of one game, as SelfPlay(root_noise=(eps, alpha)) defines it: expand the root (a search of 0 playouts); when it has
n >= 1 children, eta = RandomState([seed, 1]).dirichlet(alpha * ones(n)) and P' = f32((1 - eps) * f64(P) + eps * eta); then the
search's playouts."""
import ctypes as C
import os
import subprocess

import numpy as np

from strict_support import ROOT, _dir, _p

_lib = None
NET_IDS = {"hash_signed": 0, "hash_pos": 1, "mod17": 2}


def lib():
    global _lib
    if _lib is None:
        so = os.path.join(_dir(), "librootnoise.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "root_noise_oracle.c"), os.path.join(ROOT, "tests", "root_noise_strict_oracle.c"),
                               os.path.join(ROOT, "tests", "strict_oracle.c"), "-lm", "-lpthread"])
        L = C.CDLL(so)
        vp, i32 = C.c_void_p, C.c_int
        for pre in ("co", "ss"):
            getattr(L, pre + "_tree_new").restype = vp
            getattr(L, pre + "_tree_new").argtypes = [vp]
            getattr(L, pre + "_tree_free").argtypes = [vp]
            getattr(L, pre + "_tree_search_fake").argtypes = [vp, i32, i32, i32, i32]
            getattr(L, pre + "_tree_root_children").argtypes = [vp] + [vp] * 5
            getattr(L, pre + "_tree_update").argtypes = [vp, i32]
            getattr(L, "rn_%s_set_root_P" % pre).argtypes = [vp, vp]
        L.co_tree_search_fifo.argtypes = [vp, i32, i32, i32, i32, i32]
        L.co_tree_signature.argtypes = [vp, vp, C.c_long]
        L.co_tree_signature.restype = C.c_long
        L.ss_tree_signature.argtypes = [vp, vp, C.c_long]
        L.ss_tree_signature.restype = C.c_long
        _lib = L
    return _lib


class Tree:
    """One game's specification tree: kind 'reference' (co_tree_search), 'fifo' (co_tree_search_fifo, K coroutines) or 'strict'."""

    def __init__(self, kind, board, K=16):
        self.kind, self.K = kind, K
        self.pre = "ss" if kind == "strict" else "co"
        L = lib()
        self.h = getattr(L, self.pre + "_tree_new")(_p(np.ascontiguousarray(board, dtype=np.uint8)))

    def __del__(self):
        try:
            getattr(lib(), self.pre + "_tree_free")(self.h)
        except Exception:
            pass

    def search(self, side, rr, playouts, net):
        L = lib()
        if self.kind == "fifo":
            return L.co_tree_search_fifo(self.h, int(side), int(rr), int(playouts), int(self.K), NET_IDS[net])
        return getattr(L, self.pre + "_tree_search_fake")(self.h, int(side), int(rr), int(playouts), NET_IDS[net])

    def root_children(self):
        """-> (n (-1: not expanded), moves, N, W, P, Q)"""
        mv, N = np.zeros(128, np.uint16), np.zeros(128, np.int32)
        W, P, Q = np.zeros(128, np.float32), np.zeros(128, np.float32), np.zeros(128, np.float32)
        n = getattr(lib(), self.pre + "_tree_root_children")(self.h, _p(mv), _p(N), _p(W), _p(P), _p(Q))
        k = max(n, 0)
        return n, mv[:k].copy(), N[:k].copy(), W[:k].copy(), P[:k].copy(), Q[:k].copy()

    def set_root_P(self, P):
        assert getattr(lib(), "rn_%s_set_root_P" % self.pre)(self.h, _p(np.ascontiguousarray(P, dtype=np.float32))) == 0

    def update(self, idx):
        if getattr(lib(), self.pre + "_tree_update")(self.h, int(idx)) != 0:
            raise KeyError(idx)

    def signature(self, cap=1 << 16):
        out = np.zeros((cap, 6), np.int64)
        n = getattr(lib(), self.pre + "_tree_signature")(self.h, _p(out), cap)
        if n > cap:
            return self.signature(int(n))
        return out[:n].copy()


def mix(P, eta, eps):
    """The noised priors: f32((1 - eps) * f64(P) + eps * eta), each operation rounded once in float64."""
    return ((1.0 - eps) * np.asarray(P, dtype=np.float32).astype(np.float64) + eps * eta).astype(np.float32)


def noisy_search(tree, side, rr, playouts, net, rn, eps, alpha):
    """One search with root noise from RandomState rn; returns the eta drawn (None when the root has no child)."""
    assert tree.search(side, rr, 0, net) == 0
    n, _, _, _, P, _ = tree.root_children()
    eta = None
    if n >= 1:
        eta = rn.dirichlet(alpha * np.ones(n))
        tree.set_root_P(mix(P, eta, eps))
    assert tree.search(side, rr, playouts, net) == 0
    return eta


def selfplay_game(kind, net, playouts, seed, eps, alpha, temperature=1, K=16, max_plies=10000):
    """cchess_main.selfplay + get_action over the specification tree with root noise: the move stream RandomState(seed), the noise
    stream RandomState([seed, 1]).  -> dict(states, pis (dense [n,2086] f64), z, actions, visits)."""
    from oracle import oracle as O
    import strict_search_support as S
    lab = O.labels()
    l2i = {m: i for i, m in enumerate(lab)}
    rs, rn = np.random.RandomState(seed), np.random.RandomState([seed, 1])
    board = O.from_state(O.START)
    tree = Tree(kind, board, K)
    side, rr = 0, 0
    states, pis, players, actions, all_visits = [], [], [], [], []
    with np.errstate(divide="ignore"):
        while True:
            noisy_search(tree, side, rr, playouts, net, rn, eps, alpha)
            _, mv, N, _, _, _ = tree.root_children()
            visits = tuple(int(v) for v in N)
            probs = O.softmax(1.0 / temperature * np.log(visits))
            p = 0.75 * probs + 0.25 * rs.dirichlet(0.3 * np.ones(len(probs)))
            acts = [O.move_str(m) for m in mv]
            idx = acts.index(rs.choice(acts, p=p))
            tree.update(idx)
            sboard = O.flip_board(board) if side == 1 else board
            states.append(O.to_state(sboard))
            prob = np.zeros(O.NLABEL)
            for a, pr in zip(acts, probs):
                prob[l2i[O.flip_label(a) if side == 1 else a]] = pr
            pis.append(prob)
            players.append(side)
            actions.append(acts[idx])
            all_visits.append(visits)
            board, cap = O.apply_move(board, mv[idx])
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            if kind == "strict":
                end, winner = S.game_end(board, side, rr)
            else:
                hasK, hask = (board == 1).any(), (board == 8).any()
                end, winner = (1, 0 if not hask else 1) if not (hasK and hask) else ((2, -1) if rr >= 60 else (0, -1))
            if end in (1, 3):
                z = np.where(np.array(players) == winner, 1.0, -1.0)
                break
            if end == 2 or len(states) >= max_plies:
                z = np.zeros(len(players))
                break
    return dict(states=states, pis=np.array(pis), z=z, actions=actions, visits=all_visits)


class StandIn:
    """Engine-interface stand-in over the specification trees (one per game) with root_counts / root_noise: SelfPlay's host loop on
    the CPU.  root_noise applies mix() to the root priors, as k_root_noise does on the device.  Test infrastructure only."""
    torch_device = "cpu"

    def __init__(self, n, net, kind="reference"):
        from oracle import oracle as O
        self.O, self.B, self.net, self.kind, self.device, self.launches = O, n, net, kind, 0, 0
        self.rules = "strict" if kind == "strict" else "reference"
        self.boards = np.tile(O.from_state(O.START), (n, 1))
        self.trees = [Tree(kind, self.boards[g]) for g in range(n)]
        self.side = np.zeros(n, np.uint8); self.rr = np.zeros(n, np.int32); self.ply = np.zeros(n, np.int32)
        self.terminal = np.zeros(n, np.uint8); self.winner = -np.ones(n, np.int8)
        self.target = np.zeros(n, np.int64); self.pending = np.zeros(n, bool)
        self.log = []                                       # (call, arguments) of every begin_search / root_counts / root_noise

    def reset(self, mask=None, boards=None, sides=None, rr=None):
        for g in range(self.B):
            if mask is None or mask[g]:
                self.boards[g] = self.O.from_state(self.O.START)
                self.side[g] = 0; self.rr[g] = 0; self.ply[g] = 0; self.terminal[g] = 0; self.winner[g] = -1
                self.trees[g] = Tree(self.kind, self.boards[g])

    def begin_search(self, playouts, mask=None):
        self.log.append(("begin_search", int(playouts), None if mask is None else np.array(mask, dtype=bool)))
        for g in range(self.B):
            if (mask[g] if mask is not None else not self.terminal[g]):
                self.target[g] = playouts; self.pending[g] = True

    def wave(self, nn_in, logits, value):
        for g in np.nonzero(self.pending)[0]:
            assert self.trees[g].search(int(self.side[g]), int(self.rr[g]), int(self.target[g]), self.net) == 0
        self.pending[:] = False

    def unfinished(self):
        return int(self.pending.sum())

    def root_counts(self):
        n = np.array([t.root_children()[0] for t in self.trees], dtype=np.int32)
        self.log.append(("root_counts", n.copy()))
        return n

    def root_noise(self, mask, eta, eps):
        self.log.append(("root_noise", np.array(mask, dtype=bool), np.array(eta, dtype=np.float64), float(eps)))
        for g in np.nonzero(mask)[0]:
            n, _, _, _, P, _ = self.trees[g].root_children()
            if n > 0:
                self.trees[g].set_root_P(mix(P, eta[g, :n], eps))

    def root_children(self, want_wpq=True):
        n = np.zeros(self.B, np.int32); m = np.zeros((self.B, 128), np.uint16); v = np.zeros((self.B, 128), np.int32)
        for g, t in enumerate(self.trees):
            k, a, N = t.root_children()[:3]
            n[g] = k; m[g, :len(a)] = a; v[g, :len(a)] = N
        return dict(n=n, moves=m, visits=v, w=None, p=None, q=None)

    def play(self, choice, want_status=True):
        import strict_search_support as S
        for g, c in enumerate(choice):
            if c < 0:
                continue
            move = self.trees[g].root_children()[1][c]
            self.trees[g].update(int(c))
            self.boards[g], cap = self.O.apply_move(self.boards[g], int(move))
            self.side[g] ^= 1; self.rr[g] = self.rr[g] + 1 if cap == 0 else 0; self.ply[g] += 1
            if cap == 1: self.terminal[g], self.winner[g] = 1, 1
            elif cap == 8: self.terminal[g], self.winner[g] = 1, 0
            elif self.rr[g] >= 60: self.terminal[g] = 2
            elif self.kind == "strict" and len(S.strict_moves(self.boards[g], int(self.side[g]))) == 0:
                self.terminal[g], self.winner[g] = 3, self.side[g] ^ 1
        return self.status()

    def status(self, boards=True):
        return dict(terminal=self.terminal.copy(), winner=self.winner.copy(), ply=self.ply.copy(), rr=self.rr.copy(),
                    side=self.side.copy(), boards=self.boards.copy(), q=np.zeros(self.B, np.float32))

    def counters(self):
        return dict(error=0)

    def raise_on_error(self):
        return self.counters()

    def snapshot(self):
        return np.zeros(8, np.uint8)

    def restore(self, blob):
        pass
