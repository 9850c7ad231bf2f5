"""TEST INFRASTRUCTURE: the specification of softmax priors (Engine(priors='softmax'), DESIGN 3k).

tests/priors_oracle.c (built here with tests/strict_oracle.c, the flags of strict_support.oracle_lib) adds to the search specification
pz_softmax (the definition for one node), pz_exp (csrc/cz_exp.h compiled for the host) and pz_search (a one-leaf search of either rule
set whose expansions use softmax priors, over a stand-in net whose logits may be shifted by a constant).  SoftmaxTree is search_spec.Tree over that search; softmax_trees() makes search_spec's game
loops and engine stand-in (selfplay_game, match_game, StandIn) build SoftmaxTrees, so they specify priors='softmax' games."""
import contextlib
import ctypes as C
import os
import subprocess

import numpy as np

import search_spec
from strict_support import ROOT, _dir, _p

_lib = []


def lib():
    if not _lib:
        so = os.path.join(_dir(), "libpriorsspec.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "priors_oracle.c"), os.path.join(ROOT, "tests", "strict_oracle.c"),
                               "-lm", "-lpthread"])
        L = C.CDLL(so)
        vp, i32 = C.c_void_p, C.c_int
        L.pz_softmax.argtypes = [vp, i32, vp]
        L.pz_exp.argtypes = [vp, vp, C.c_long]
        L.pz_search.argtypes = [vp, i32, i32, i32, i32, i32, C.c_float, i32]
        L.co_tree_new.restype = L.ss_tree_new.restype = vp
        L.co_tree_new.argtypes = L.ss_tree_new.argtypes = [vp]
        L.co_tree_free.argtypes = [vp]
        L.co_tree_root_children.argtypes = [vp] * 6
        L.co_tree_update.argtypes = [vp, i32]
        L.rn_set_root_P.argtypes = [vp, vp]
        L.ss_tree_root_mated.argtypes = [vp]
        L.co_tree_stats.argtypes = L.ss_tree_stats.argtypes = [vp, vp]
        L.co_tree_signature.argtypes = L.ss_tree_signature.argtypes = [vp, vp, C.c_long]
        L.co_tree_signature.restype = L.ss_tree_signature.restype = C.c_long
        _lib.append(L)
    return _lib[0]


def cz_exp(x):
    """csrc/cz_exp.h on the host: float64 array -> float64 array"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty_like(x)
    lib().pz_exp(_p(x), _p(y), x.size)
    return y


def softmax(logits):
    """pz_softmax: the softmax priors of one node's logits (float32, 1..128 of them, move order)"""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    P = np.zeros(len(lg), np.float32)
    assert lib().pz_softmax(_p(lg), len(lg), _p(P)) == 0
    return P


class SoftmaxTree(search_spec.Tree):
    """search_spec.Tree whose searches expand with softmax priors (one-leaf searches of either rule set)."""

    def __init__(self, board, rules="reference", search_threads=1):
        if rules not in ("reference", "strict") or int(search_threads) != 1:
            raise ValueError("the softmax-prior specification covers the one-leaf searches: rules %r, search_threads %r"
                             % (rules, search_threads))
        self.rules, self.K = rules, 1
        b = _p(np.ascontiguousarray(board, dtype=np.uint8))
        self.h = lib().ss_tree_new(b) if rules == "strict" else lib().co_tree_new(b)

    def __del__(self):
        try:
            lib().co_tree_free(self.h)
        except Exception:
            pass

    softmax = True

    def search(self, side, rr, playouts, net, shift=0.0):
        """shift: a constant added to every logit of the stand-in net (reference rules)"""
        return lib().pz_search(self.h, int(self.rules == "strict"), int(side), int(rr), int(playouts), search_spec.NET_IDS[net],
                               float(shift), int(self.softmax))

    def count(self):
        return lib().co_tree_root_children(self.h, None, None, None, None, None)

    def root_children(self):
        mv, N = np.zeros(136, np.uint16), np.zeros(136, np.int32)
        W, P, Q = np.zeros(136, np.float32), np.zeros(136, np.float32), np.zeros(136, np.float32)
        n = max(lib().co_tree_root_children(self.h, _p(mv), _p(N), _p(W), _p(P), _p(Q)), 0)
        return mv[:n].copy(), N[:n].copy(), W[:n].copy(), P[:n].copy(), Q[:n].copy()

    def set_root_P(self, P):
        assert lib().rn_set_root_P(self.h, _p(np.ascontiguousarray(P, dtype=np.float32))) == 0

    def update(self, idx):
        if lib().co_tree_update(self.h, int(idx)) != 0:
            raise KeyError(idx)

    def root_mated(self):
        assert self.rules == "strict"
        return bool(lib().ss_tree_root_mated(self.h))

    def stats(self):
        s = np.zeros(6, np.int64)
        if self.rules == "strict":
            lib().ss_tree_stats(self.h, _p(s))
            keys = ("n_expand", "n_playout", "sum_L", "sum_c", "sum_C", "error")
        else:
            lib().co_tree_stats(self.h, _p(s))
            keys = ("n_expand", "n_playout", "sum_L", "sum_c", "error")
        return {k: int(v) for k, v in zip(keys, s)}

    def signature(self, cap=1 << 16):
        out = np.zeros((cap, 6), np.int64)
        fn = lib().ss_tree_signature if self.rules == "strict" else lib().co_tree_signature
        n = fn(self.h, _p(out), cap)
        if n > cap:
            return self.signature(int(n))
        return out[:n].copy()


class ReferenceTree(SoftmaxTree):
    """The same one-leaf search with the reference priors (search_spec.Tree's trees, plus the logit shift)."""
    softmax = False


@contextlib.contextmanager
def softmax_trees():
    """search_spec's game loops and StandIn build SoftmaxTrees inside this block."""
    old = search_spec.Tree
    search_spec.Tree = SoftmaxTree
    try:
        yield
    finally:
        search_spec.Tree = old


def selfplay_game(net, playouts, rs, rules="reference", search_threads=1, root_noise=None, priors="reference"):
    if priors != "softmax":
        return search_spec.selfplay_game(net, playouts, rs, rules, search_threads, root_noise)
    with softmax_trees():
        return search_spec.selfplay_game(net, playouts, rs, rules, search_threads, root_noise)


def match_game(*a, priors="reference", **kw):
    if priors != "softmax":
        return search_spec.match_game(*a, **kw)
    with softmax_trees():
        return search_spec.match_game(*a, **kw)


class StandIn(search_spec.StandIn):
    """search_spec.StandIn whose trees use the given priors (Engine interface: the `priors` attribute)."""

    def __init__(self, n, net, rules="reference", search_threads=1, priors="reference"):
        self.priors = priors
        if priors == "softmax":
            with softmax_trees():
                super().__init__(n, net, rules, search_threads)
        else:
            super().__init__(n, net, rules, search_threads)

    def reset(self, *a, **kw):
        with softmax_trees() if self.priors == "softmax" else contextlib.nullcontext():
            return super().reset(*a, **kw)

    def play_moves(self, *a, **kw):
        with softmax_trees() if self.priors == "softmax" else contextlib.nullcontext():
            return super().play_moves(*a, **kw)
