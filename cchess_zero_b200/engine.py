"""Python handle on the batched device engine (cz_engine_* in include/cchess_b200.h).

torch is used for device buffers and streams only; all tree / rules work happens in the
sm_90a kernels of csrc/cz_engine.cu."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import BF16, BOARD, F16, F32, MAXCHILD, PRIORS, RULES, STATUS_BYTES, EngineError, check, lib

_DT = {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16, torch.uint8: BOARD}


def _hp(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check_rules(rules, search_threads=1, leaves=1):
    """The engine rules `rules` names ('reference' or 'strict'); ValueError for another name, and for strict rules with more than one
    leaf per game and wave (leaf-parallel or search_threads > 1 engines play by the reference rules only).  search_threads as SelfPlay,
    Match and Trainer take it: 1 (or None) is the one-leaf engine."""
    if rules not in RULES:
        raise ValueError("rules must be 'reference' or 'strict', not %r" % (rules,))
    if rules == "strict" and (int(search_threads or 1) != 1 or int(leaves) != 1):
        raise ValueError("strict rules need the one-leaf engine (search_threads = 1, leaves = 1)")
    return rules


def check_priors(priors):
    """The prior mode `priors` names: 'reference' (P = logit / (1e-8 + the sum of the legal logits), the reference's expansion) or
    'softmax' (P = the softmax of the legal logits, DESIGN 3k); ValueError for another name.  Every engine kind takes either."""
    if priors not in PRIORS:
        raise ValueError("priors must be 'reference' or 'softmax', not %r" % (priors,))
    return priors


class Engine:
    def __init__(self, n_games, arena_words=0, device=None, leaves=1, search_threads=None, rules="reference", priors="reference"):
        """leaves > 1: leaf-parallel engine (up to `leaves` leaves per game per wave; network rows = n_games*leaves).
        leaves == -1: the leaf-parallel kernel with one slot (test hook).
        search_threads = K: the reference's search_threads schedule in canonical FIFO form (bit-exact with the reference's
        uvloop runs wherever those are reproducible); network rows = n_games*K.
        rules: 'reference' (pseudo-legal moves, a game ends when a king is taken) or 'strict' (strictly legal moves only; a side
        without one is mated, terminal code 3; cz_engine_create_rules).  Strict rules need the one-leaf engine: no search_threads
        (any search_threads value, 1 included, builds the FIFO engine) and leaves = 1.
        priors: 'reference' or 'softmax', how an expansion turns the network's logits into priors (check_priors;
        cz_engine_set_priors before the first wave)."""
        check_rules(rules, 1, leaves)
        check_priors(priors)
        if rules == "strict" and search_threads is not None:
            raise ValueError("strict rules need the one-leaf engine: search_threads = %r builds the search_threads schedule's (FIFO) "
                             "engine, which plays by the reference rules; leave search_threads unset" % (search_threads,))
        if not torch.cuda.is_available():
            raise EngineError("cchess_zero_b200 needs a CUDA device (no CPU fallback exists)")
        self.rules = rules
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.B = int(n_games)
        self.fifo = search_threads is not None
        self.leaves = int(search_threads) if self.fifo else abs(int(leaves))
        self.rows = self.B * self.leaves
        h = C.c_void_p()
        if self.fifo:
            check(lib().cz_engine_create_fifo(self.B, int(arena_words), self.device, int(search_threads), C.byref(h)), "cz_engine_create_fifo")
        elif rules == "strict":
            check(lib().cz_engine_create_rules(self.B, int(arena_words), self.device, RULES[rules], C.byref(h)), "cz_engine_create_rules")
        else:
            check(lib().cz_engine_create_ex(self.B, int(arena_words), self.device, int(leaves), C.byref(h)), "cz_engine_create_ex")
        self.h = h
        self.priors = priors
        if priors != "reference":
            check(lib().cz_engine_set_priors(h, PRIORS[priors]), "cz_engine_set_priors")
        self.launches = 0   # kernels of csrc/cz_engine.cu launched through this handle
        self._mate = 1 if rules == "strict" else 0          # k_root_mate after every root change of a strict engine
        self._count = torch.zeros(1, dtype=torch.int32, device="cuda:%d" % self.device)
        self._eta = None                                      # device copy of host root-noise draws (root_noise), made on first use

    def close(self):
        if getattr(self, "h", None):
            lib().cz_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- game state -------------------------------------------------------------------
    def reset(self, mask=None, boards=None, sides=None, rr=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        b = None if boards is None else np.ascontiguousarray(boards, dtype=np.uint8).reshape(self.B, 90)
        s = None if sides is None else np.ascontiguousarray(sides, dtype=np.uint8)
        r = None if rr is None else np.ascontiguousarray(rr, dtype=np.int32)
        self.launches += 1 + self._mate
        check(lib().cz_engine_reset(self.h, _stream(), _hp(m), _hp(b), _hp(s), _hp(r)), "cz_engine_reset")

    def set_root_meta(self, sides=None, rr=None, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        s = None if sides is None else np.ascontiguousarray(sides, dtype=np.uint8)
        r = None if rr is None else np.ascontiguousarray(rr, dtype=np.int32)
        self.launches += 1 + self._mate
        check(lib().cz_engine_set_root_meta(self.h, _stream(), _hp(m), _hp(s), _hp(r)), "cz_engine_set_root_meta")

    def begin_search(self, playouts, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self.launches += 1
        check(lib().cz_engine_begin_search(self.h, _stream(), _hp(m), int(playouts)), "cz_engine_begin_search")

    # ---- waves (device tensors) ---------------------------------------------------------
    def wave(self, nn_in, logits, value):
        self.launches += 1
        check(lib().cz_engine_wave(self.h, _stream(), nn_in.data_ptr(), _DT[nn_in.dtype], logits.data_ptr(), value.data_ptr()),
              "cz_engine_wave")

    def wave_compact(self, nn_stage, nn_dense, logits, value):
        """search_threads = K engines: a wave whose leaves are gathered densely into nn_dense (cz_engine_wave_compact); evaluate
        nn_dense[:live_rows()] into logits / value before the next call."""
        self.launches += 3           # k_wave_fifo, k_compact_scan, k_compact_rows
        check(lib().cz_engine_wave_compact(self.h, _stream(), nn_stage.data_ptr(), nn_dense.data_ptr(), _DT[nn_stage.dtype],
                                           logits.data_ptr(), value.data_ptr()), "cz_engine_wave_compact")

    def live_rows(self):
        out = C.c_int32(0)
        check(lib().cz_engine_live_rows(self.h, _stream(), C.byref(out)), "cz_engine_live_rows")
        return out.value

    # ---- board hashing (Zobrist keys of the pending leaves; never used by the search) -------
    def enable_hashing(self, on=True):
        check(lib().cz_engine_enable_hashing(self.h, 1 if on else 0), "cz_engine_enable_hashing")

    def leaf_hashes(self):
        """int64 view (device tensor, [rows]) of the 64-bit Zobrist keys of the positions in the network batch rows."""
        ptr = C.c_void_p()
        check(lib().cz_engine_leaf_hashes(self.h, C.byref(ptr)), "cz_engine_leaf_hashes")
        n = self.rows

        class _Arr:                                            # __cuda_array_interface__ view of engine-owned memory
            __cuda_array_interface__ = dict(shape=(n,), typestr="<i8", data=(ptr.value, False), version=2)
        return torch.as_tensor(_Arr(), device="cuda:%d" % self.device)

    def root_keys(self):
        out = np.zeros(self.B, dtype=np.uint64)
        check(lib().cz_engine_root_keys(self.h, _stream(), _hp(out)), "cz_engine_root_keys")
        return out

    def unfinished(self):
        out = C.c_int32(0)
        self.launches += 1
        check(lib().cz_engine_unfinished(self.h, _stream(), C.byref(out)), "cz_engine_unfinished")
        return out.value

    def unfinished_async(self):
        self.launches += 1
        check(lib().cz_engine_unfinished_async(self.h, _stream(), self._count.data_ptr()), "cz_engine_unfinished_async")
        return self._count

    # ---- root statistics / moves ----------------------------------------------------------
    def root_children(self, want_wpq=True):
        B = self.B
        n = np.zeros(B, dtype=np.int32)
        mv = np.zeros((B, MAXCHILD), dtype=np.uint16)
        vis = np.zeros((B, MAXCHILD), dtype=np.int32)
        w = np.zeros((B, MAXCHILD), dtype=np.float32) if want_wpq else None
        p = np.zeros((B, MAXCHILD), dtype=np.float32) if want_wpq else None
        q = np.zeros((B, MAXCHILD), dtype=np.float32) if want_wpq else None
        self.launches += 1
        check(lib().cz_engine_root_children(self.h, _stream(), _hp(n), _hp(mv), _hp(vis), _hp(w), _hp(p), _hp(q)),
              "cz_engine_root_children")
        return dict(n=n, moves=mv, visits=vis, w=w, p=p, q=q)

    def root_counts(self):
        """int32 [B]: the number of root children of every game (-1: root not expanded; 0: expanded without children, a mated root
        of a strict engine).  One copy of the header lines, no kernel."""
        n = np.zeros(self.B, dtype=np.int32)
        check(lib().cz_engine_root_counts(self.h, _stream(), _hp(n)), "cz_engine_root_counts")
        return n

    def root_noise(self, mask, eta, eps):
        """Root exploration noise: in every game with mask[g] that is in a search (begin_search) and has an expanded root of n > 0
        children, root prior i becomes f32((1 - eps) * f64(P_i) + eps * eta[g, i]) (k_root_noise; no renormalisation).  eta: float64
        [B, 128], a device tensor or a host array (copied to the device).  Expand the roots first: begin_search(0, mask) and waves
        until unfinished() is 0."""
        eps = float(eps)
        if not 0.0 <= eps <= 1.0:
            raise ValueError("root noise: eps must lie in [0, 1], not %r" % eps)
        if isinstance(eta, torch.Tensor) and eta.is_cuda:
            if eta.dtype != torch.float64 or tuple(eta.shape) != (self.B, MAXCHILD) or not eta.is_contiguous():
                raise ValueError("root noise: eta must be a contiguous float64 [%d, %d] tensor" % (self.B, MAXCHILD))
            dev = eta
        else:
            if self._eta is None:
                self._eta = torch.zeros((self.B, MAXCHILD), dtype=torch.float64, device="cuda:%d" % self.device)
            self._eta.copy_(torch.from_numpy(np.ascontiguousarray(eta, dtype=np.float64).reshape(self.B, MAXCHILD)))
            dev = self._eta
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        assert m.shape == (self.B,)
        self.launches += 1
        check(lib().cz_engine_root_noise(self.h, _stream(), _hp(m), C.c_void_p(dev.data_ptr()), C.byref(C.c_double(1.0 - eps)),
                                         C.byref(C.c_double(eps))), "cz_engine_root_noise")

    def play(self, child_index, want_status=True):
        """GameBoard update + update_tree for every game with child_index >= 0; returns the status of all games (see status())
        from the same call: one kernel, one device->host copy, one synchronisation."""
        ci = np.ascontiguousarray(child_index, dtype=np.int32)
        assert ci.shape == (self.B,)
        self.launches += 1 + self._mate
        rec = np.zeros((self.B, STATUS_BYTES), dtype=np.uint8) if want_status else None
        check(lib().cz_engine_play_status(self.h, _stream(), _hp(ci), _hp(rec)), "cz_engine_play_status")
        return self._unpack_status(rec) if want_status else None

    def play_moves(self, moves, want_status=True):
        """Play the given move (src | dst << 7; 0xFFFF = none) in every game, searched at the root or not: the opponent's move in a
        game where each player keeps its own tree (update_tree for a move the tree did not choose).  A move that is not legal at the
        root, or any move in a finished game, sets the ILLEGAL error flag and leaves that game unchanged (cz_engine_play_moves).  A strict
        engine accepts only strictly legal moves."""
        mv = np.ascontiguousarray(moves, dtype=np.uint16)
        assert mv.shape == (self.B,)
        self.launches += 1 + self._mate
        rec = np.zeros((self.B, STATUS_BYTES), dtype=np.uint8) if want_status else None
        check(lib().cz_engine_play_moves(self.h, _stream(), _hp(mv), _hp(rec)), "cz_engine_play_moves")
        return self._unpack_status(rec) if want_status else None

    @staticmethod
    def _unpack_status(rec):
        tail = np.ascontiguousarray(rec[:, 96:112]).view(np.int32)
        return dict(boards=np.ascontiguousarray(rec[:, :90]), side=rec[:, 90].copy(), terminal=rec[:, 91].copy(),
                    winner=rec[:, 92].copy().view(np.int8), ply=tail[:, 0].copy(), rr=tail[:, 1].copy(),
                    q=np.ascontiguousarray(tail[:, 2]).view(np.float32), root_N=tail[:, 3].copy())

    def status(self, boards=True):
        """terminal / winner / ply / restrict_round / side / boards of every game (check_end, main.py:1380-1392).  terminal: 0 running,
        1 king captured, 2 draw, 3 mated (strict engines; the winner is the side that just moved)."""
        rec = np.zeros((self.B, STATUS_BYTES), dtype=np.uint8)
        self.launches += 1
        check(lib().cz_engine_status_packed(self.h, _stream(), _hp(rec)), "cz_engine_status_packed")
        return self._unpack_status(rec)

    def counters(self):
        out = np.zeros(9, dtype=np.int64)
        check(lib().cz_engine_counters(self.h, _stream(), _hp(out)), "cz_engine_counters")
        return dict(n_expand=int(out[0]), n_playout=int(out[1]), sum_L=int(out[2]), sum_c=int(out[3]), error=int(out[4]),
                    max_arena_words=int(out[5]), first_error_game=int(out[6]), max_depth=int(out[7]), sum_C=int(out[8]))

    def raise_on_error(self):
        c = self.counters()
        if c["error"]:
            names = [v for k, v in _lib.ERR_NAMES.items() if c["error"] & k]
            raise EngineError("engine error flags %s (first game %d)" % ("|".join(names), c["first_error_game"]))
        return c

    def tree_signature(self, game, cap=1 << 16):
        out = np.zeros((cap, 6), dtype=np.int64)
        n = C.c_int64(0)
        check(lib().cz_engine_tree_signature(self.h, _stream(), int(game), _hp(out), cap, C.byref(n)), "cz_engine_tree_signature")
        if n.value > cap:
            return self.tree_signature(game, int(n.value))
        return out[: n.value].copy()

    # ---- snapshots of games at rest (cz_engine_snapshot / cz_engine_restore) ----------------
    def snapshot(self):
        """Every game's state as one self-describing uint8 blob; EngineError while a search is in progress."""
        n = C.c_int64(0)
        check(lib().cz_engine_snapshot_size(self.h, _stream(), C.byref(n)), "cz_engine_snapshot_size")
        out = np.empty(n.value, dtype=np.uint8)
        self.launches += 1
        check(lib().cz_engine_snapshot(self.h, _stream(), _hp(out), out.nbytes, C.byref(n)), "cz_engine_snapshot")
        return out

    def restore(self, blob):
        """Write a snapshot back in place (captured graphs stay valid).  The blob is validated first: a corrupt one, or one from an
        engine of another shape, raises EngineError and leaves the engine untouched."""
        b = np.ascontiguousarray(blob, dtype=np.uint8)
        if b.ndim != 1:
            raise ValueError("a snapshot is a 1-d uint8 array")
        if b.ctypes.data % 8:                      # the validator reads the blob as 64-bit words
            b = b.copy()
        self.launches += 1
        check(lib().cz_engine_restore(self.h, _stream(), _hp(b), b.nbytes), "cz_engine_restore")

    # ---- a whole search: MCTS_tree.main for every selected game ---------------------------
    def search(self, forward_dev, playouts, nn_in, logits, value, mask=None):
        """forward_dev(nn_in) must fill `logits` [B,2086] f32 and `value` [B] (or [B,1]) f32 in place
        (device tensors).  Runs waves until every selected game has finished `playouts` playouts."""
        self.begin_search(playouts, mask)
        return run_waves(self, lambda: self.wave(nn_in, logits, value), playouts // self.leaves, playouts,
                         evaluate=lambda: forward_dev(nn_in))


def run_waves(engine, step, min_waves, pmax, evaluate=None, may_stop=None, per_step=1):
    """The wave loop of every search (after begin_search).  step() runs `per_step` waves -- for a captured graph, together with their
    evaluations.  The search ends once more than `min_waves` waves have run, may_stop() (if given) holds and engine.unfinished() is 0;
    until then evaluate() (if given) runs the network on the leaves of the last step.  A search still running after 4 * pmax + 64
    waves (pmax: the largest playout count) raises EngineError: for the engine's error flags if any are set (raise_on_error), else
    for the missing convergence.  Returns the number of waves."""
    waves = 0
    while True:
        step()
        waves += per_step
        if waves > min_waves and (may_stop is None or may_stop()) and engine.unfinished() == 0:
            return waves
        if evaluate is not None:
            evaluate()
        if waves > 4 * pmax + 64:
            engine.raise_on_error()
            raise EngineError("search did not converge after %d waves" % waves)


def capture_cuda_graph(body, warm, warmup, pool=None):
    """body() captured into a new CUDA graph (on a fresh stream; pool: a memory pool shared with other graphs), after `warmup` runs
    of warm() on a side stream: the first launches load modules and let libraries pick algorithms, which a capture must not do."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            warm()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, pool=pool, stream=torch.cuda.Stream()):
        body()
    return g
