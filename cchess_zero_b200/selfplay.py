"""Batched self-play driver (many games in lock-step on one GPU) and the reference-shaped
`cchess_main` facade (main.py:1118-1554).

Move choice stays on the host in numpy, exactly as the reference does it (get_action,
main.py:1332-1358): pi = softmax(log(visits)/T) in float64 and
np.random.choice(p = 0.75*pi + 0.25*Dirichlet(0.3)) on a legacy MT19937 RandomState -- one
RandomState per game slot stands in for the reference's global np.random (SURVEY H3).  The device
produces the integer visit counts; everything before them (select / expand / backup / encode /
move generation / re-rooting) runs in csrc/cz_engine.cu."""
import ctypes as C
import os
import pickle
import random
import time
import types
from collections import defaultdict, deque

import numpy as np
import torch

from . import rules as _rules                        # (SelfPlay takes a `rules` argument)
from ._lib import MAXCHILD, MT_WORDS, NLABEL, NSQ, TERM_MATED, EngineError, lib
from .engine import Engine, capture_cuda_graph, check_priors, check_rules, run_waves


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _flip_board(b):
    """try_flip (main.py:560-574) for one board [90] or a stack [L,90]: reverse the rows, swap the colours; files are not mirrored."""
    f = b.reshape(-1, 10, 9)[:, ::-1].copy()
    red, blk = (f >= 1) & (f <= 7), f >= 8
    f[red] += 7
    f[blk] -= 7
    return f.reshape(b.shape)


def _flip_move_label_index(moves, flip=True):
    """Label index of every u16 move code in `moves`; where `flip` (broadcast against moves; by default every move) is set, of the
    rank-mirrored move (y -> 9 - y: flipped_uci_labels for black, main.py:23-27 / 1507-1512).  KeyError, as label2i[...] in the
    reference, when a move is not a label."""
    mv = np.asarray(moves).astype(np.int64)
    src, dst = mv & 127, (mv >> 7) & 127
    flip = np.asarray(flip, dtype=bool)
    src = np.where(flip, (9 - src // 9) * 9 + src % 9, src)
    dst = np.where(flip, (9 - dst // 9) * 9 + dst % 9, dst)
    li = _label_table()[src, dst]
    if (li < 0).any():
        raise KeyError("move outside the label table")
    return li


def visit_exp(n, visits, temperature):
    """The rows of pi = softmax(1/T * log(visits)) (main.py:1341, 1111-1116) before their sums: exp(lv - max(lv)) with
    lv = 1/T * log(visits) in float64, -inf (exp 0) past each row's n.  n [L], visits [L,128]; temperature: a scalar or one value per
    row.  log / exp / max are element-wise or exact, so they are taken over the whole batch at once; the order-sensitive row sums are
    cz_host_choose_moves', operation for operation what numpy does for `probs /= np.sum(probs)`."""
    inv_t = (1.0 / temperature) if np.ndim(temperature) == 0 else (1.0 / np.asarray(temperature, dtype=np.float64))[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        lv = inv_t * np.log(visits.astype(np.int64))
        lv[np.arange(MAXCHILD)[None, :] >= n[:, None]] = -np.inf
        return np.ascontiguousarray(np.exp(lv - np.max(lv, axis=1, keepdims=True)))


def mt_streams(seeds, key=None):
    """One legacy MT19937 stream per seed, RandomState(seed) (or RandomState([seed, key])), as raw numpy RandomState states
    uint32 [len(seeds), 626]: csrc/cz_host.cu draws from them exactly as RandomState.dirichlet / .choice would."""
    mt = np.zeros((len(seeds), MT_WORDS), dtype=np.uint32)
    for g, sd in enumerate(seeds):
        st = np.random.RandomState(int(sd) if key is None else [int(sd), key]).get_state()
        mt[g, :624], mt[g, 624] = st[1], st[2]
    return mt


_LABEL_OF = None


def _label_table():
    """(src_sq, dst_sq) -> label index as a numpy table (cz_label_index); -1 where the pair is not a label."""
    global _LABEL_OF
    if _LABEL_OF is None:
        L = lib()
        _LABEL_OF = np.array([[L.cz_label_index(s, d) for d in range(90)] for s in range(90)], dtype=np.int64)
    return _LABEL_OF


def check_root_noise(root_noise):
    """None (no root noise) or (eps, alpha) as two floats, with eps in [0, 1] and alpha in (0, 1) (AlphaZero: 0.25 and 0.3 for chess,
    0.15 for shogi, 0.03 for Go); ValueError otherwise."""
    if root_noise is None:
        return None
    try:
        eps, alpha = (float(v) for v in root_noise)
    except (TypeError, ValueError):
        raise ValueError("root_noise must be None or (eps, alpha), not %r" % (root_noise,))
    if not 0.0 <= eps <= 1.0:
        raise ValueError("root_noise: eps must lie in [0, 1], not %r" % eps)
    if not 0.0 < alpha < 1.0:
        raise ValueError("root_noise: alpha must lie in (0, 1), not %r" % alpha)
    return eps, alpha


def sample_moves(n_children, visits, live, temperature, mt_states, exploration, n_threads=1):
    """get_action's move choice (main.py:1339-1348) for a batch of games, bit-identical to the numpy calls: pi = softmax(1/T *
    log(visits)) in float64, then RandomState.choice(p = pi) -- with exploration, p = 0.75 * pi + 0.25 * RandomState.dirichlet(0.3).
    n_children [B] int32 / visits [B,128]: the root statistics; live [B]: the games that choose (others get -1); temperature: a
    scalar or one value per game; mt_states [B,626]: one legacy MT19937 state per game, advanced in place.  Returns choice [B] int32."""
    B = len(n_children)
    choice = np.full(B, -1, dtype=np.int32)
    # pi's rows (visit_exp); the row sums, the Dirichlet / choice draws and the cumulative sums happen per game in csrc/cz_host.cu,
    # operation for operation what numpy does for RandomState.dirichlet and RandomState.choice (main.py:1345-1348)
    ex = visit_exp(n_children, visits, temperature)
    probs = np.empty((B, MAXCHILD), dtype=np.float64)
    fallback = np.zeros(B, dtype=np.uint8)
    live8 = np.ascontiguousarray(live, dtype=np.uint8)
    nn = np.ascontiguousarray(n_children, dtype=np.int32)
    rcode = lib().cz_host_choose_moves(B, _vp(live8), _vp(nn), _vp(ex), 1 if exploration else 0, _vp(mt_states), _vp(choice), _vp(probs),
                                       _vp(fallback), n_threads)
    if rcode:
        raise EngineError("cz_host_choose_moves failed (%d)" % rcode)
    for g in np.nonzero(fallback)[0]:
        # a probability vector numpy would reject (NaN priors ...): let numpy raise exactly what the reference would raise
        n = int(nn[g])
        rs = np.random.RandomState()
        rs.set_state(("MT19937", mt_states[g, :624].copy(), int(mt_states[g, 624]), 0, 0.0))
        pr = ex[g, :n] / np.sum(ex[g, :n])
        choice[g] = int(rs.choice(n, p=pr))          # (the Dirichlet draws were consumed by the native sampler, as in the reference)
        st_ = rs.get_state()
        mt_states[g, :624], mt_states[g, 624] = st_[1], st_[2]
    return choice


# one log entry per ply (SelfPlay.step), for the whole batch: (field, shape per game, dtype)
_LOG = (("boards", (NSQ,), np.uint8), ("n", (), np.int32), ("moves", (MAXCHILD,), np.uint16), ("visits", (MAXCHILD,), np.int32),
        ("choice", (), np.int32))


class GameRecord:
    """(s, pi, z) tuples of one finished game in the reference's format (selfplay, main.py:1493-1554).

    During play nothing per game is recorded: SelfPlay keeps ONE log entry per ply for the whole batch (boards, root moves and
    visit counts, chosen indices); a record only remembers its slot, ply span, players and temperature.  positions() turns them into
    the game's training positions on first use; pi is recomputed from the integer visit counts with the very numpy operations
    get_action uses, so bit-identical."""

    def __init__(self, slot=None, logs=None, temperature=1):
        self._slot, self._logs, self._T = slot, logs if logs is not None else [], temperature
        self.players = []
        self.z = None
        self.winner = None
        self._log = self._pos = self._states = None

    def __len__(self):
        return len(self.players)

    def _log_arrays(self):
        """This slot's log span as arrays: boards [L,90], n [L], moves [L,128], visits [L,128], choice [L]."""
        if self._log is None:
            g, L = self._slot, len(self._logs)
            self._log = {k: np.array([lg[k][g] for lg in self._logs], dtype=dt).reshape((L,) + shp) for k, shp, dt in _LOG}
            self._logs = None
        return self._log

    def positions(self):
        """The game's training positions, in the fields of distributed.TupleBatch plus sides: boards u8 [L,90] (side to move
        canonical, main.py:1504-1505), sides u8 [L], n [L], idx i16 [L,128] (label indices, black's ranks flipped: main.py:1507-1512),
        prob f64 [L,128] (pi) and z f64 [L]; idx and prob are 0 past n."""
        if self._pos is None:
            r = self._log_arrays()
            n, L = r["n"], len(r["n"])
            sides = np.asarray(self.players, dtype=np.uint8)
            valid = np.arange(MAXCHILD)[None, :] < n[:, None]
            idx = np.zeros((L, MAXCHILD), dtype=np.int16)
            idx[valid] = _flip_move_label_index(r["moves"][valid], np.repeat(sides == 1, n))
            # pi = softmax(1/T * log(visits)) at this slot's temperature; the row sums are get_action's batch path (sample_moves)
            T = self._T if np.ndim(self._T) == 0 else np.asarray(self._T, dtype=np.float64)[self._slot]
            ex = visit_exp(n, r["visits"], T)
            prob = np.zeros((L, MAXCHILD), dtype=np.float64)
            mt = np.zeros((L, MT_WORDS), dtype=np.uint32); mt[:, 624] = 624          # scratch generators: the draws are discarded
            ch, fb = np.zeros(L, np.int32), np.zeros(L, np.uint8)
            lib().cz_host_choose_moves(L, None, _vp(n), _vp(ex), 0, _vp(mt), _vp(ch), _vp(prob), _vp(fb), 1)
            for i in np.nonzero(fb)[0]:                                               # (NaN rows: plain numpy, as get_action would)
                pr = ex[i, :n[i]].copy(); pr /= np.sum(pr); prob[i, :n[i]] = pr
            boards = np.where((sides == 1)[:, None], _flip_board(r["boards"]), r["boards"])
            self._pos = types.SimpleNamespace(boards=boards, sides=sides, n=n, idx=idx, prob=prob, z=np.asarray(self.z, dtype=np.float64))
        return self._pos

    @classmethod
    def from_tuples(cls, states, pi_idx, pi_val, z):
        """A record built from already materialised tuples (tests, gathered data); its sides are 0."""
        r = cls()
        r._states, r.z = list(states), z
        L = len(r._states)
        r.players = [0] * L
        n = np.fromiter((len(ix) for ix in pi_idx), dtype=np.int32, count=L)
        if (n > MAXCHILD).any():
            raise ValueError("more than %d moves in one position" % MAXCHILD)
        idx, prob = np.zeros((L, MAXCHILD), dtype=np.int16), np.zeros((L, MAXCHILD), dtype=np.float64)
        for i, (ix, pv) in enumerate(zip(pi_idx, pi_val)):
            idx[i, :n[i]], prob[i, :n[i]] = ix, pv
        boards = np.array([_rules.state_to_board(s) for s in r._states], dtype=np.uint8).reshape(L, NSQ)
        r._pos = types.SimpleNamespace(boards=boards, sides=np.zeros(L, dtype=np.uint8), n=n, idx=idx, prob=prob,
                                       z=np.asarray(z, dtype=np.float64))
        return r

    @property
    def states(self):
        if self._states is None:
            self._states = [_rules.board_to_state(b) for b in self.positions().boards]
        return self._states

    @property
    def pi_idx(self):
        p = self.positions()
        return [p.idx[i, :k] for i, k in enumerate(p.n)]

    @property
    def pi_val(self):
        p = self.positions()
        return [p.prob[i, :k] for i, k in enumerate(p.n)]

    @property
    def visits(self):
        r = self._log_arrays()
        return [v[:k] for v, k in zip(r["visits"], r["n"])]

    @property
    def actions(self):
        r = self._log_arrays()
        return [_rules.move_to_label(mv[c]) for mv, c in zip(r["moves"], r["choice"])]

    def dense_pi(self):
        p = self.positions()
        valid = np.arange(MAXCHILD)[None, :] < p.n[:, None]
        out = np.zeros((len(self), NLABEL))
        out[np.nonzero(valid)[0], p.idx[valid]] = p.prob[valid]
        return out

    def tuples(self):
        return zip(self.states, self.dense_pi(), self.z)


class SelfPlay:
    """n_games concurrent self-play games on one engine, advanced in lock-step plies by step().

    Evaluator: pass `plan` (an InferencePlan / NativePlan: it owns the input buffer layout and writes logits / value in
    place), or `forward` = a callable (nn_in) -> (logits [B,2086] f32, value [B] f32) device tensors, which are copied
    into the static buffers the engine reads.  Finished games accumulate in `finished` (slot, GameRecord); long runs
    should drain them with pop_finished()."""

    def __init__(self, n_games, forward, playouts, seeds=None, exploration=True, temperature=1,
                 nn_dtype=torch.float32, arena_words=0, auto_reset=True, device=None, keep_records=True, plan=None,
                 plan_factory=None, lanes=1, engine=None, hashing=False, search_threads=1, compact=None, rules="reference",
                 root_noise=None, priors="reference"):
        """plan: an InferencePlan / NativePlan (defines the input buffer, writes logits/value in place); plan_factory(rows) builds
        one when `plan` is not given.  lanes: 1 is the only value.  rules: 'reference' or 'strict' (the search expands strictly legal
        moves only and a side without one is mated: the game ends with terminal code 3, won by the side that moved last); strict
        rules need search_threads = 1.  root_noise: None (off) or (eps, alpha): every search() first mixes Dirichlet noise into the
        root priors of its games, P' = (1 - eps) P + eps Dir(alpha) (see search).  priors: 'reference' or 'softmax', how the search
        turns the network's logits into priors (Engine priors; the noise mixes into either)."""
        if lanes != 1:
            raise ValueError("SelfPlay: lanes must be 1")
        self.rules = check_rules(rules, search_threads)
        self.root_noise = check_root_noise(root_noise)
        self.priors = check_priors(priors)
        if engine is not None and getattr(engine, "priors", "reference") != priors:
            raise ValueError("SelfPlay: the engine uses the %r priors, not %r" % (getattr(engine, "priors", "reference"), priors))
        if engine is not None and getattr(engine, "rules", "reference") != rules:
            raise ValueError("SelfPlay: the engine plays by the %r rules, not %r" % (getattr(engine, "rules", "reference"), rules))
        self.B = n_games
        # search_threads = K > 1: every game runs the reference's K-coroutine schedule (k_wave_fifo); the network batch has K rows per game
        self.K = max(1, int(search_threads))
        # ... of which only the rows that carry a leaf are evaluated (row compaction, cz_engine_wave_compact): default for K > 1
        self.compact = (self.K > 1 and engine is None) if compact is None else bool(compact)
        assert not self.compact or self.K > 1, "row compaction belongs to the search_threads = K engine"
        # `engine`: an object with the Engine interface (tests drive the host loop with a CPU stand-in); the product
        # always constructs the CUDA engine here
        self.engine = engine if engine is not None else (Engine(n_games, arena_words, device, search_threads=self.K, priors=priors)
                                                         if self.K > 1 else Engine(n_games, arena_words, device, rules=rules, priors=priors))
        if hashing:                              # Zobrist keys of the pending leaves (must be on before a graph is captured)
            self.engine.enable_hashing(True)
        dev = torch.device("cuda", self.engine.device) if engine is None else torch.device(getattr(engine, "torch_device", "cpu"))
        rows = n_games * self.K
        if plan is None and plan_factory is not None:
            plan = plan_factory(rows)
        self.logits = torch.zeros((rows, NLABEL), dtype=torch.float32, device=dev)
        self.value = torch.zeros((rows,), dtype=torch.float32, device=dev)
        if plan is not None:
            self.nn_in = plan.make_input(rows)
            forward = lambda x: plan(x, self.logits, self.value)  # noqa: E731
        else:
            self.nn_in = torch.zeros((rows, 9, 10, 14), dtype=nn_dtype, device=dev)
        if self.compact:                                   # the engine writes every slot's row here; the leaves go densely to nn_in
            self.nn_stage = torch.zeros_like(self.nn_in)
            self._bucket_graphs, self._use_graphs, self._pool = {}, False, None
            self.rows_evaluated = 0
            # batch sizes the network is run at: multiples of the game count (K sizes, one lazily captured CUDA graph each).  Finer
            # buckets evaluate 3.5 % fewer rows but a search then meets dozens of sizes, and capturing their graphs costs more
            # than it saves in anything but a very long run (measured: 2.32 -> 1.81 M exp/s over 6 plies with 256-row buckets)
            self.bucket_rows = n_games
        self.lanes = None                                  # one engine and one network batch (bench.py reads the attribute)
        self.plan = plan
        self.forward = forward
        self.playouts = np.broadcast_to(np.asarray(playouts, dtype=np.int64), (n_games,)).copy()
        self.exploration = exploration
        self.temperature = temperature
        self.auto_reset = auto_reset
        self.keep_records = keep_records
        self._start_board = _rules.state_to_board(_rules.START_STATE)
        # one legacy MT19937 stream per game slot (stands in for the reference's global np.random, SURVEY H3); with root noise a
        # second one, RandomState([seed, 1]), so that the move choice draws stay those of a run without noise
        seeds = range(n_games) if seeds is None else seeds
        self._eta = None if self.root_noise is None else np.zeros((n_games, MAXCHILD), dtype=np.float64)   # one search's draws
        self._start_games(mt_streams(seeds), None if self.root_noise is None else mt_streams(seeds, 1))
        self.plies = 0
        self.waves = 0
        self.graph = None
        self._threads = max(1, min(16, (len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else 4)))
        _rules._init_tables()

    def _start_games(self, mt, noise_mt):
        """Host state of a fresh game in every slot: start position, red to move, live, empty records, move streams mt and, with root
        noise, noise streams noise_mt (uint32 [B, 626] each, see mt_streams)."""
        B = self.B
        if (noise_mt is None) != (self.root_noise is None):
            raise ValueError("noise streams are given if and only if root noise is on")
        self._mt = np.array(mt, dtype=np.uint32).reshape(B, MT_WORDS)
        self._noise_mt = None if noise_mt is None else np.array(noise_mt, dtype=np.uint32).reshape(B, MT_WORDS)
        self._span = [[] for _ in range(B)]             # the log entries of each slot's current game
        self.records = [GameRecord(g, None, self.temperature) for g in range(B)]
        self.boards = np.tile(self._start_board, (B, 1))
        self.sides = np.zeros(B, dtype=np.uint8)
        self.live = np.ones(B, dtype=bool)
        self.finished = []

    def restart_games(self, mt, noise_mt=None):
        """Every slot starts a fresh game from the start position (the engine is reset), drawing its moves from the stream mt[slot]
        and, with root noise, its noise from noise_mt[slot]."""
        self.engine.reset()
        self._start_games(mt, noise_mt)

    # -- evaluation step ---------------------------------------------------------------------
    def _eval(self, nn_in):
        out = self.forward(nn_in)
        if out is not None:
            lo, v = out
            self.logits.copy_(lo.reshape(self.B * self.K, NLABEL))
            self.value.copy_(v.reshape(self.B * self.K))

    # -- search_threads = K with row compaction ---------------------------------------------------
    def _eval_rows(self, n):
        """Evaluate the first n rows of the dense batch into logits[:n] / value[:n]."""
        x = self.nn_in[:n]
        if self.plan is not None:
            self.plan(x, self.logits[:n], self.value[:n])
            return
        lo, v = self.forward(x)
        self.logits[:n].copy_(lo.reshape(n, NLABEL))
        self.value[:n].copy_(v.reshape(n))

    def _eval_bucket(self, n_live):
        """The network on n_live rows rounded up to the bucket size (one lazily captured CUDA graph per size, sharing a memory pool)."""
        n = min(self.B * self.K, -(-n_live // self.bucket_rows) * self.bucket_rows)
        self.rows_evaluated += n
        if not self._use_graphs:
            return self._eval_rows(n)
        g = self._bucket_graphs.get(n)
        if g is None:
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            g = self._bucket_graphs[n] = capture_cuda_graph(lambda: self._eval_rows(n), lambda: self._eval_rows(n), 2, self._pool)
        g.replay()

    def capture_graph(self, warmup=3):
        """Capture (wave kernel -> network) into one CUDA graph; the search loop then replays it."""
        if self.compact:                                    # the wave runs eagerly (the host reads the row count); the network is one
            self._use_graphs = True                         # graph per bucket size, captured on first use
            return

        def body():
            self.engine.wave(self.nn_in, self.logits, self.value)
            self._eval(self.nn_in)
        self.graph = capture_cuda_graph(body, lambda: self._eval(self.nn_in), warmup)

    def search(self, mask=None):
        """MCTS_tree.main for every live game (or every game with mask[g], e.g. the games where one player of a match is to move):
        `playouts[g]` playouts each.  With root noise, the roots are expanded and noised first (_noise_roots)."""
        m = self.live if mask is None else np.asarray(mask, dtype=bool)
        e = self.engine
        if self.plan is not None and hasattr(self.plan, "refresh_if_stale"):
            self.plan.refresh_if_stale()       # weights trained / restored since the last search (the graph reads them in place)
        if self.root_noise is not None:
            self._noise_roots(m)
        for p in np.unique(self.playouts[m]):
            e.begin_search(int(p), (m & (self.playouts == p)).astype(np.uint8))
        pmax = int(self.playouts[m].max()) if m.any() else 0
        waves = self._run_waves(pmax)
        self.waves += waves
        return waves

    def _run_waves(self, pmax, graph=True):
        """The wave loop after begin_search, in the engine's mode: row compaction, the captured graph (graph=True) or eager waves."""
        e = self.engine
        if self.compact:
            n = 0

            def step():
                nonlocal n
                e.wave_compact(self.nn_stage, self.nn_in, self.logits, self.value)
                n = e.live_rows()                           # stream sync: the host picks the bucket

            def evaluate():
                if n > 0:
                    self._eval_bucket(n)
            # done when nothing is left to evaluate and every search is complete
            return run_waves(e, step, 0, pmax, evaluate, may_stop=lambda: n == 0)
        if graph and self.graph is not None:
            def step():
                self.graph.replay()
                e.launches += 1          # the captured k_wave launch
            return run_waves(e, step, pmax // self.K, pmax)
        # (K leaves per game and wave in the search_threads = K schedule: pmax // K waves at least)
        return run_waves(e, lambda: e.wave(self.nn_in, self.logits, self.value), pmax // self.K, pmax,
                         evaluate=lambda: self._eval(self.nn_in))

    def _noise_roots(self, m):
        """Root exploration noise for the games in mask m.  A search of 0 playouts expands every pending root and runs no playout
        (k_wave / k_wave_fifo stop at the target; a root expanded before is left alone): the network evaluates exactly the roots the
        search itself would evaluate first.  Eager waves, not the captured graph, so that no network pass runs without a leaf.  Then,
        for every searched, live game with n >= 1 root children, in slot order: eta = RandomState([seed, 1]).dirichlet(alpha * ones(n))
        (cz_host_dirichlet) and P' = f32((1 - eps) f64(P) + eps eta) on the device (k_root_noise).  The noised root block is dropped
        by the next play (only the chosen subtree is kept), so games at rest never hold noised priors."""
        e = self.engine
        e.begin_search(0, m.astype(np.uint8))
        self.waves += self._run_waves(0, graph=False)
        n = np.ascontiguousarray(e.root_counts(), dtype=np.int32)
        sel = (m & self.live & (n > 0)).astype(np.uint8)
        if not sel.any():
            return
        eps, alpha = self.root_noise
        rc = lib().cz_host_dirichlet(self.B, _vp(sel), _vp(n), C.byref(C.c_double(alpha)), _vp(self._noise_mt), _vp(self._eta), self._threads)
        if rc:
            raise EngineError("cz_host_dirichlet failed (%d)" % rc)
        e.root_noise(sel, self._eta, eps)

    # -- one ply for every live game ------------------------------------------------------------
    def step(self):
        e = self.engine
        self.search()
        rc = e.root_children(want_wpq=False)                      # n, moves, visits: what get_action reads (main.py:1339)
        live = np.nonzero(self.live)[0]
        if (rc["n"][live] <= 0).any():
            e.raise_on_error()
            raise EngineError("game %d has no root children" % int(live[np.argmax(rc["n"][live] <= 0)]))
        nn = np.ascontiguousarray(rc["n"], dtype=np.int32)
        choice = sample_moves(nn, rc["visits"], self.live, self.temperature, self._mt, self.exploration, self._threads)
        if self.keep_records:
            entry = dict(boards=self.boards, n=nn, moves=rc["moves"], visits=rc["visits"], choice=choice)
            for g in live:
                self._span[g].append(entry)
        sides_now = self.sides
        for g in live:
            self.records[g].players.append(int(sides_now[g]))
        st = e.play(choice)                                          # board update + re-root + status, one synchronisation
        win_rate = np.where(choice >= 0, st["q"], 0.0).astype(np.float32)                 # mcts.Q(act), main.py:1350
        self.boards, self.sides = st["boards"], st["side"]
        self.plies += int(self.live.sum())
        done_now = []
        for g in np.nonzero(self.live & (st["terminal"] != 0))[0]:
            rec = self.records[g]
            players = np.asarray(rec.players)
            if st["terminal"][g] in (1, TERM_MATED):                                     # main.py:1532-1541; mated: strict rules
                w = int(st["winner"][g])
                rec.z = np.where(players == w, 1.0, -1.0)
                rec.winner = "w" if w == 0 else "b"
            else:                                                                        # main.py:1542-1545
                rec.z = np.zeros(len(players))
                rec.winner = "t"
            rec._logs, rec._T = self._span[g], self.temperature
            self._span[g] = []
            done_now.append((int(g), rec))
            self.finished.append((int(g), rec))
            self.records[g] = GameRecord(int(g), None, self.temperature)
        if done_now:
            idx = [g for g, _ in done_now]
            if self.auto_reset:
                mask = np.zeros(self.B, dtype=np.uint8)
                mask[idx] = 1
                e.reset(mask)                                                            # GameBoard.reload + mcts.reload
                st = {k: v.copy() for k, v in st.items()}
                st["boards"][idx] = self._start_board                                    # what reload() leaves: no second status read
                st["side"][idx] = 0
                st["terminal"][idx] = 0
                st["winner"][idx] = -1
                st["ply"][idx] = 0
                st["rr"][idx] = 0
                self.boards, self.sides = st["boards"], st["side"]
            else:
                self.live[idx] = False
        return dict(choice=choice, win_rate=win_rate, finished=done_now, status=st)

    def pop_finished(self):
        """Hand over (and forget) the games finished so far: keeps memory flat in long self-play runs."""
        out, self.finished = self.finished, []
        return out

    # -- games in flight: save and restore between plies ------------------------------------------------
    def save_games(self, path):
        """Every game in flight into one np.savez file (written to a temporary file, then renamed): the engine's trees and game state
        (Engine.snapshot) and the host state -- boards, sides, live, the per-slot MT19937 states (and, with root noise, the noise
        streams' states under 'noise_mt'; with softmax priors, priors='softmax'), plies, temperature and each slot's unfinished record (its players and log span).  load_games
        continues exactly where this left off.  The finished games must have been handed over with pop_finished first."""
        if self.finished:
            raise ValueError("save_games: %d finished games were not drained with pop_finished()" % len(self.finished))
        from .train import _savez
        blob = self.engine.snapshot()
        rows = [(lg, g) for g in range(self.B) for lg in self._span[g]]
        log = {"log_" + k: np.asarray([lg[k][g] for lg, g in rows], dtype=dt).reshape((len(rows),) + shp) for k, shp, dt in _LOG}
        players = [self.records[g].players for g in range(self.B)]
        if self.root_noise is not None:
            log["noise_mt"] = self._noise_mt
        if self.priors != "reference":                                 # (absent: reference priors, so older files stay as they were)
            log["priors"] = np.asarray(self.priors)
        _savez(path, engine=blob, boards=self.boards, sides=self.sides, live=self.live, mt=self._mt, plies=np.int64(self.plies),
               temperature=np.asarray(self.temperature, dtype=np.float64), span_len=np.asarray([len(s) for s in self._span], dtype=np.int64),
               players_len=np.asarray([len(p) for p in players], dtype=np.int64),
               players=np.asarray([p for ps in players for p in ps], dtype=np.uint8), **log)

    def load_games(self, path):
        """Restore what save_games wrote into this SelfPlay (same number of games and engine kind, root noise on in both or in neither;
        the same prior mode; the engine is restored in place, so a captured graph stays valid).  The file is read without pickle and checked; ValueError / EngineError leave everything as it
        was."""
        with np.load(path, allow_pickle=False) as d:
            a = {k: d[k] for k in d.files}
        B = self.B
        want = dict(engine=(None, np.uint8), boards=((B, NSQ), np.uint8), sides=((B,), np.uint8), live=((B,), np.bool_),
                    mt=((B, MT_WORDS), np.uint32), plies=((), np.int64), span_len=((B,), np.int64), players_len=((B,), np.int64),
                    players=(None, np.uint8), temperature=(None, np.float64))
        rows = int(a["span_len"].sum()) if "span_len" in a else -1
        for k, shp, dt in _LOG:
            want["log_" + k] = ((rows,) + shp, dt)
        if ("noise_mt" in a) != (self.root_noise is not None):        # the noise streams are part of an exact resume
            raise ValueError("games file: saved %s root noise, this SelfPlay runs %s" % (("with", "without") if "noise_mt" in a
                                                                                        else ("without", "with")))
        saved = str(a["priors"]) if "priors" in a else "reference"
        if saved != self.priors:                                       # the trees were searched with the saved file's priors
            raise ValueError("games file: saved with %r priors, this SelfPlay uses %r" % (saved, self.priors))
        if self.root_noise is not None:
            want["noise_mt"] = ((B, MT_WORDS), np.uint32)
        for k, (shp, dt) in want.items():
            if k not in a or a[k].dtype != dt or (shp is not None and a[k].shape != shp):
                raise ValueError("games file: '%s' missing or not %s %s" % (k, np.dtype(dt).name, shp))
        if a["engine"].ndim != 1 or a["players"].ndim != 1 or a["temperature"].shape not in ((), (B,)):
            raise ValueError("games file: bad engine / players / temperature shape")
        if a["span_len"].min() < 0 or a["players_len"].min() < 0 or int(a["players_len"].sum()) != len(a["players"]):
            raise ValueError("games file: bad span or player counts")
        if a["boards"].max() > 14 or a["sides"].max() > 1 or (len(a["players"]) and a["players"].max() > 1) or a["plies"] < 0:
            raise ValueError("games file: piece code, side or ply count out of range")
        n = a["log_n"]
        if len(n) and (n.min() < 0 or n.max() > MAXCHILD or (a["log_choice"] < 0).any() or (a["log_choice"] >= n).any()):
            raise ValueError("games file: logged move count or choice out of range")
        self.engine.restore(a["engine"])                     # validated as a whole before anything on the device is written
        spans = a["span_len"]
        L = int(spans.max()) if B else 0
        entries = [{k: np.zeros((B,) + shp, dtype=dt) for k, shp, dt in _LOG} for _ in range(L)]
        r = 0
        for g in range(B):                                   # a slot's span is the last span_len[g] plies: align them at the end
            for j in range(L - int(spans[g]), L):
                for k, _, _ in _LOG:
                    entries[j][k][g] = a["log_" + k][r]
                r += 1
        t = a["temperature"]
        self.temperature = float(t) if t.ndim == 0 else t.copy()
        self._span = [entries[L - int(spans[g]):] for g in range(B)]
        self.records = [GameRecord(g, None, self.temperature) for g in range(B)]
        ends = np.cumsum(a["players_len"])
        for g in range(B):
            self.records[g].players = [int(p) for p in a["players"][ends[g] - a["players_len"][g]:ends[g]]]
        self.boards, self.sides, self.live = a["boards"].copy(), a["sides"].copy(), a["live"].copy()
        self._mt[:] = a["mt"]
        if self.root_noise is not None:
            self._noise_mt[:] = a["noise_mt"]
        self.plies = int(a["plies"])

    def play_games(self, max_plies=100000):
        """Every slot plays ONE game to the end (auto_reset must be False)."""
        assert not self.auto_reset
        n = 0
        while self.live.any() and n < max_plies:
            self.step()
            n += 1
        self.engine.raise_on_error()
        return sorted(self.finished, key=lambda t: t[0])


def softmax_priors(logits):
    """The softmax priors of one node's legal-move logits (float32, in move order), as the engine computes them with
    priors='softmax' (DESIGN 3k) up to the last bit of the exponential: m = the largest logit (NaNs ignored), e_i = exp(f64(l_i) - m),
    s = the serial f64 sum of the e_i, P_i = f32(e_i / s).  float32 array."""
    lg = np.asarray(logits, dtype=np.float32).astype(np.float64)
    if lg.size == 0:
        return np.zeros(0, dtype=np.float32)
    e = np.exp(lg - np.fmax.reduce(lg))
    s = 0.0
    for v in e:
        s += v
    return (e / s).astype(np.float32)


def network_selfplay(network, n_games, playouts, **kw):
    """SelfPlay evaluated by a policy_value_network: an fp16 network runs its native plan (board bytes in, the hand-written first
    convolution and heads), any other precision its own inference plan.  Either plan follows the network's weights_version, so a
    search after train_step / restore sees the new weights."""
    if network.precision == "fp16":
        return SelfPlay(n_games, None, playouts, plan_factory=lambda r: network.native_plan(r), **kw)
    return SelfPlay(n_games, None, playouts, plan_factory=lambda r: network.plan(), **kw)


# =================================================================================================
# Reference-shaped facade: cchess_main (main.py:1118-1554).  One game at a time through MCTS_tree,
# exactly the call sequence of the reference, so main.py's train loop runs unchanged on top of it.
# For throughput use SelfPlay (thousands of games per GPU); `selfplay_many` bridges the two.
# =================================================================================================
def save_replay(path, data_buffer, extra=None):
    """Persist the replay deque (main.py:1138-1139 keeps it in memory only) together with the global numpy / python RNG
    states, so that a training run can resume exactly where it stopped (SURVEY 8(f)2).  Atomic: write + rename."""
    blob = dict(data=list(data_buffer), maxlen=getattr(data_buffer, "maxlen", None), np_state=np.random.get_state(),
                py_state=random.getstate(), extra=dict(extra or {}))
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        pickle.dump(blob, f, protocol=pickle.HIGHEST_PROTOCOL)
    os.replace(tmp, path)


def load_replay(path, restore_rng=True):
    """-> (deque, extra).  With restore_rng the numpy / python global RNGs continue from the saved point."""
    with open(path, "rb") as f:
        blob = pickle.load(f)
    if restore_rng:
        np.random.set_state(blob["np_state"])
        random.setstate(blob["py_state"])
    return deque(blob["data"], maxlen=blob["maxlen"]), blob["extra"]


class cchess_main(object):
    # strict=True plays by the full rules of xiangqi instead of the reference's (pseudo-legal moves, the game ends when a king is
    # captured): no move that leaves the own king attacked or is in banned_moves is played, a mated side has lost, and
    # human_move refuses such a move.  The search is the same either way; the filter is applied to its result.
    strict = False
    banned_moves = ()       # move labels the next get_action / select_move must not play (a GUI's perpetual-check ban)

    def __init__(self, playout=400, in_batch_size=128, exploration=True, in_search_threads=16, processor="cpu",
                 num_gpus=1, res_block_nums=7, human_color="b", network=None, log_file=True, leaf_parallel=1, strict=False,
                 priors="reference"):
        from .mcts import MCTS_tree
        from .net import policy_value_network, policy_value_network_gpus
        _rules._init_tables()
        self.epochs = 5
        self.playout_counts = playout
        self.temperature = 1
        self.batch_size = in_batch_size
        self.game_batch = 400
        self.top_steps = 30
        self.top_temperature = 1
        self.eta = 0.03
        self.learning_rate = 0.001
        self.lr_multiplier = 1.0
        self.buffer_size = 10000
        self.data_buffer = deque(maxlen=self.buffer_size)
        self.game_borad = _rules.GameBoard()
        if network is not None:
            self.policy_value_netowrk = network
        else:  # `processor` selected CPU/GPU TensorFlow in the reference (main.py:1142); both map to the CUDA net here
            self.policy_value_netowrk = policy_value_network(res_block_nums) if processor == "cpu" else policy_value_network_gpus(num_gpus, res_block_nums)
        self.search_threads = in_search_threads
        # priors='softmax': the search and the 'net' player use the softmax of the legal moves' logits (reference: logit / sum)
        self.priors = check_priors(priors)
        self.mcts = MCTS_tree(self.game_borad.state, self.policy_value_netowrk.forward, self.search_threads, leaf_parallel=leaf_parallel,
                              priors=priors)
        self.exploration = exploration
        self.resign_threshold = -0.8
        self.global_step = 0
        self.kl_targ = 0.025
        self.log_file = open(os.path.join(os.getcwd(), "log_file.txt"), "w") if log_file else None
        self.human_color = human_color
        self.strict = strict

    @staticmethod
    def flip_policy(prob):  # main.py:1152-1155
        prob = np.asarray(prob).flatten()
        return np.asarray([prob[i] for i in _rules.unflipped_index])

    # ---- training (main.py:1157-1205) ------------------------------------------------------------
    def policy_update(self):
        from .train import explained_variance, next_lr_multiplier, policy_kl
        mini_batch = random.sample(self.data_buffer, self.batch_size)
        state_batch = [d[0] for d in mini_batch]
        mcts_probs_batch = [d[1] for d in mini_batch]
        winner_batch = np.expand_dims([d[2] for d in mini_batch], 1)
        start_time = time.time()
        old_probs, old_v = self.mcts.forward(state_batch)
        kl, loss, accuracy, new_v = 0.0, 0.0, 0.0, old_v
        for _ in range(self.epochs):
            accuracy, loss, self.global_step = self.policy_value_netowrk.train_step(
                state_batch, mcts_probs_batch, winner_batch, self.learning_rate * self.lr_multiplier)
            new_probs, new_v = self.mcts.forward(state_batch)
            kl = policy_kl(old_probs, new_probs)
            if kl > self.kl_targ * 4:
                break
        self.policy_value_netowrk.save(self.global_step)
        print("train using time {} s".format(time.time() - start_time))
        self.lr_multiplier = next_lr_multiplier(kl, self.kl_targ, self.lr_multiplier)
        explained_var_old = explained_variance(winner_batch, old_v)
        explained_var_new = explained_variance(winner_batch, new_v)
        msg = "kl:{:.5f},lr_multiplier:{:.3f},loss:{},accuracy:{},explained_var_old:{:.3f},explained_var_new:{:.3f}".format(
            kl, self.lr_multiplier, loss, accuracy, explained_var_old, explained_var_new)
        print(msg)
        if self.log_file:
            self.log_file.write(msg + "\n")
            self.log_file.flush()

    def save_state(self, path):
        """Replay buffer + lr multiplier + step + RNG states (the reference checkpoints only the network weights)."""
        save_replay(path, self.data_buffer, dict(lr_multiplier=self.lr_multiplier, global_step=self.global_step))

    def load_state(self, path):
        self.data_buffer, extra = load_replay(path)
        self.lr_multiplier = extra.get("lr_multiplier", self.lr_multiplier)
        self.global_step = extra.get("global_step", self.global_step)

    def run(self, max_batches=None):  # main.py:1224-1248
        batch_iter = 0
        try:
            while max_batches is None or batch_iter < max_batches:
                batch_iter += 1
                play_data, episode_len = self.selfplay()
                print("batch i:{}, episode_len:{}".format(batch_iter, episode_len))
                extend_data = []
                for state, mcts_prob, winner in play_data:
                    extend_data.append((self.mcts.state_to_positions(state), mcts_prob, winner))
                self.data_buffer.extend(extend_data)
                if len(self.data_buffer) > self.batch_size:
                    self.policy_update()
        except KeyboardInterrupt:
            if self.log_file:
                self.log_file.close()
            self.policy_value_netowrk.save(self.global_step)

    # ---- move choice (main.py:1278-1358) -----------------------------------------------------------
    def _visit_probs(self):
        actions_visits = [(act, nod.N) for act, nod in self.mcts.root.child.items()]
        actions, visits = zip(*actions_visits)
        with np.errstate(divide="ignore"):
            probs = _rules.softmax(1.0 / self.temperature * np.log(visits))
        return actions, probs

    def get_hint(self, mcts_or_net, reverse, disp_mcts_msg_handler):
        act_prob_dict = defaultdict(float)
        if mcts_or_net == "mcts":
            if self.mcts.root.child == {}:
                disp_mcts_msg_handler()
                self.mcts.main(self.game_borad.state, self.game_borad.current_player, self.game_borad.restrict_round, self.playout_counts)
            actions, probs = self._visit_probs()
            for i in range(len(actions)):
                action = "".join(_rules.flipped_uci_labels(actions[i])) if self.human_color == "w" else actions[i]
                act_prob_dict[action] = probs[i]
        elif mcts_or_net == "net":
            moves, p, _ = self._net_priors()
            for action, mov_p in zip(moves, p):
                if self.human_color == "w":
                    action = "".join(_rules.flipped_uci_labels(action))
                act_prob_dict[action] = mov_p
        return sorted(act_prob_dict.items(), key=lambda item: item[1], reverse=reverse)

    def _net_priors(self):
        """The 'net' branches of get_hint / select_move (main.py:1300-1324, 1437-1459)."""
        positions = self.mcts.generate_inputs(self.game_borad.state, self.game_borad.current_player)
        action_probs, value = self.mcts.forward(np.expand_dims(positions, 0))
        if self.mcts.is_black_turn(self.game_borad.current_player):
            action_probs = cchess_main.flip_policy(action_probs)
        moves = _rules.GameBoard.get_legal_moves(self.game_borad.state, self.game_borad.current_player)
        action_probs = np.asarray(action_probs).flatten()
        if getattr(self, "priors", "reference") == "softmax":
            return moves, list(softmax_priors(action_probs[[_rules.label2i[a] for a in moves]])), value
        tot_p = 1e-8
        p = []
        for action in moves:
            mov_p = action_probs[_rules.label2i[action]]
            p.append(mov_p)
            tot_p += mov_p
        return moves, [x / tot_p for x in p], value

    # ---- strict legality (strict=True only) ----------------------------------------------------------
    def _strict_position(self):
        """(pseudo-legal move labels, their strict-legality flags, in check, mated) for the side to move on the board:
        one k_strict_moves launch."""
        gb = self.game_borad
        mv, cnt, legal, chk, mated = _rules.strict_moves_batch(_rules.state_to_board(gb.state)[None], [_rules.side_of(gb.current_player)])
        n = min(int(cnt[0]), mv.shape[1])
        return [_rules.move_to_label(m) for m in mv[0, :n]], legal[0, :n], bool(chk[0]), bool(mated[0])

    def _playable(self):
        """Labels of the moves that are strictly legal and not banned."""
        labels, legal, _, _ = self._strict_position()
        return {m for m, ok in zip(labels, legal) if ok and m not in self.banned_moves}

    def _strict_visits(self, actions, visits):
        """The root's visit counts with every child that may not be played set to 0.  When no playable child was visited, the
        playable child with the largest prior gets the only visit (first maximum wins)."""
        playable = self._playable()
        kept = tuple(v if a in playable else 0 for a, v in zip(actions, visits))
        if any(kept):
            return kept
        rest = [a for a in actions if a in playable]
        if not rest:
            raise ValueError("no move is both strictly legal and not banned")
        child = self.mcts.root.child
        best = max(rest, key=lambda a: child[a].P)
        return tuple(1 if a == best else 0 for a in actions)

    def get_action(self, state, temperature=1e-3):
        self.mcts.main(state, self.game_borad.current_player, self.game_borad.restrict_round, self.playout_counts)
        actions_visits = [(act, nod.N) for act, nod in self.mcts.root.child.items()]
        actions, visits = zip(*actions_visits)
        if self.strict:
            visits = self._strict_visits(actions, visits)
        with np.errstate(divide="ignore"):
            probs = _rules.softmax(1.0 / temperature * np.log(visits))
        move_probs = [[actions, probs]]
        if self.exploration and self.strict:      # the Dirichlet noise must not revive a filtered move
            p = np.where(np.asarray(visits) > 0, 0.75 * probs + 0.25 * np.random.dirichlet(0.3 * np.ones(len(probs))), 0.0)
            act = np.random.choice(actions, p=p / p.sum())
        elif self.exploration:
            act = np.random.choice(actions, p=0.75 * probs + 0.25 * np.random.dirichlet(0.3 * np.ones(len(probs))))
        else:
            act = np.random.choice(actions, p=probs)
        win_rate = self.mcts.Q(act)
        self.mcts.update_tree(act)
        return act, move_probs, win_rate

    # ---- game flow (main.py:1380-1554) -------------------------------------------------------------
    def check_end(self):
        st = self.game_borad.state
        if st.find("K") == -1 or st.find("k") == -1:
            if st.find("K") == -1:
                print("Green is Winner")
                return True, "b"
            print("Red is Winner")
            return True, "w"
        elif self.game_borad.restrict_round >= 60:
            print("TIE! No Winners!")
            return True, "t"
        elif self.strict and self._strict_position()[3]:      # checkmate or stalemate: the side to move has lost
            if self.game_borad.current_player == "w":
                print("Green is Winner")
                return True, "b"
            print("Red is Winner")
            return True, "w"
        return False, ""

    def _advance(self, action):
        """state / round / player / restrict_round bookkeeping shared by human_move, select_move, selfplay."""
        last_state = self.game_borad.state
        self.game_borad.state = _rules.GameBoard.sim_do_action(action, self.game_borad.state)
        self.game_borad.round += 1
        self.game_borad.current_player = "w" if self.game_borad.current_player == "b" else "b"
        if _rules.is_kill_move(last_state, self.game_borad.state) == 0:
            self.game_borad.restrict_round += 1
        else:
            self.game_borad.restrict_round = 0

    def human_move(self, coord, mcts_or_net):
        win_rate = 0
        action = "abcdefghi"[coord[0]] + str(coord[1]) + "abcdefghi"[coord[2]] + str(coord[3])
        if self.human_color == "w":
            action = "".join(_rules.flipped_uci_labels(action))
        if self.strict:
            labels, legal, _, _ = self._strict_position()
            if action not in {m for m, ok in zip(labels, legal) if ok}:
                raise ValueError("%s is not a legal move" % action)
        if mcts_or_net == "mcts":
            if self.mcts.root.child == {}:
                self.mcts.main(self.game_borad.state, self.game_borad.current_player, self.game_borad.restrict_round, self.playout_counts)
            win_rate = self.mcts.Q(action)
            self.mcts.update_tree(action)
        self._advance(action)
        return win_rate

    def select_move(self, mcts_or_net):
        if mcts_or_net == "mcts":
            action, probs, win_rate = self.get_action(self.game_borad.state, self.temperature)
        else:
            moves, p, value = self._net_priors()
            win_rate = value[0, 0]
            if self.strict:
                playable = self._playable()
                moves, p = zip(*[(m, q) for m, q in zip(moves, p) if m in playable])
            action = max(zip(moves, p), key=lambda t: t[1])[0]   # first maximum wins, main.py:1461
        print("Win rate for player {} is {:.4f}".format(self.game_borad.current_player, win_rate))
        print(self.game_borad.current_player, " now take a action : ", action, "[Step {}]".format(self.game_borad.round))
        self._advance(action)
        self.game_borad.print_borad(self.game_borad.state)
        if self.human_color == "w":
            action = "".join(_rules.flipped_uci_labels(action))
        sx, sy, dx, dy = ord(action[0]) - 97, int(action[1]), ord(action[2]) - 97, int(action[3])
        return (sx, sy, dx - sx, dy - sy), win_rate

    def selfplay(self):
        self.game_borad.reload()
        states, mcts_probs, current_players = [], [], []
        z = None
        game_over = False
        start_time = time.time()
        while not game_over:
            action, probs, win_rate = self.get_action(self.game_borad.state, self.temperature)
            black = self.mcts.is_black_turn(self.game_borad.current_player)
            state, _ = self.mcts.try_flip(self.game_borad.state, self.game_borad.current_player, black)
            states.append(state)
            prob = np.zeros(_rules.labels_len)
            for a, pr in zip(probs[0][0], probs[0][1]):
                prob[_rules.label2i["".join(_rules.flipped_uci_labels(a)) if black else a]] = pr
            mcts_probs.append(prob)
            current_players.append(self.game_borad.current_player)
            self._advance(action)
            st = self.game_borad.state
            if st.find("K") == -1 or st.find("k") == -1:
                winnner = "b" if st.find("K") == -1 else "w"
                z = np.zeros(len(current_players))
                z[np.array(current_players) == winnner] = 1.0
                z[np.array(current_players) != winnner] = -1.0
                game_over = True
                print("Game end. Winner is player : ", winnner, " In {} steps".format(self.game_borad.round - 1))
            elif self.game_borad.restrict_round >= 60:
                z = np.zeros(len(current_players))
                game_over = True
                print("Game end. Tie in {} steps".format(self.game_borad.round - 1))
            if game_over:
                self.mcts.reload()
        print("Using time {} s".format(time.time() - start_time))
        return zip(states, mcts_probs, z), len(z)

    # ---- evaluation (main.py:1207-1222, commented out in the reference; not called from run()) ---------------------------
    def policy_evaluate(self, n_games=10, opponent=None):
        """Plays n_games (even: colour-swapped pairs) of this network against `opponent` (another policy_value_network; None = a
        search-only opponent with zero logits and zero value -- the reference's stub used pure MCTS with random rollouts, which
        this engine does not have), self.playout_counts playouts per move and self.search_threads, all games at once
        (arena.Match, both sides searching with this instance's priors).  Prints the stub's line and returns win_ratio = (win + 0.5 tie)
        / n_games."""
        from .arena import Match, UniformEvaluator
        r = Match(self.policy_value_netowrk, UniformEvaluator() if opponent is None else opponent, n_games, self.playout_counts,
                  search_threads=self.search_threads, priors=getattr(self, "priors", "reference")).run()
        win_ratio = 1.0 * (r.wins + 0.5 * r.draws) / n_games
        print("num_playouts:{}, win: {}, lose: {}, tie:{}".format(self.playout_counts, r.wins, r.losses, r.draws))
        return win_ratio

    # ---- batched bridge: many games at once on this rank's GPU ---------------------------------------
    def selfplay_many(self, n_games, seeds=None, arena_words=0):
        """Plays n_games concurrent games with the engine's lock-step waves and returns a list of
        (zip(states, mcts_probs, z), n) -- the same tuples selfplay() yields, one entry per game.  The games search with this instance's
        priors."""
        net = self.policy_value_netowrk
        plan = net.plan()
        sp = SelfPlay(n_games, None, self.playout_counts, seeds=seeds, exploration=self.exploration, temperature=self.temperature,
                      arena_words=arena_words, auto_reset=False, plan=plan, priors=getattr(self, "priors", "reference"))
        return [(rec.tuples(), len(rec)) for _, rec in sp.play_games()]
