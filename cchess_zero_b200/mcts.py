"""Drop-in for the reference's MCTS_tree / leaf_node surface (main.py:93-206, 234-577) on top of a
one-game device engine.  Same constructor, same methods, same attribute names that main.py's callers
touch (`root.child[label].N/.Q`, `Q(move)`, `update_tree`, `reload`, `forward`, `generate_inputs`,
`try_flip`, `state_to_positions`, `is_black_turn`).

Semantics: `search_threads` is honoured.  1 = one playout at a time (SURVEY Appendix A.4), bit-exact with the reference.
K > 1 = the reference's coroutine schedule (semaphore of K playouts, now_expanding spins, prediction_worker batching,
main.py:337-470) in its canonical deterministic form -- the engine's k_wave_fifo, specified by oracle/detloop.py and pinned to
real uvloop runs of the reference: identical visit counts wherever the reference reproduces itself (it is timing-dependent on a
few per cent of positions, see DESIGN.md).  Up to K leaves are evaluated per network call.  `leaf_parallel=K` selects the
package's own virtual-loss batching schedule instead (not the reference's visit counts)."""
import os
from collections import OrderedDict

import numpy as np
import torch

from . import rules
from ._lib import NLABEL
from .engine import Engine, capture_cuda_graph, run_waves


class leaf_node(object):
    """Read-only view of one root child (the fields get_action / get_hint / Q read, main.py:1286, 1339)."""

    __slots__ = ("P", "Q", "N", "W", "U", "v", "parent", "child", "state")

    def __init__(self, P, Q, N, W):
        self.P, self.Q, self.N, self.W = P, Q, N, W
        self.U = 0
        self.v = 0
        self.parent = None
        self.child = {}
        self.state = None


class _Root(object):
    def __init__(self, tree):
        self._t = tree

    @property
    def state(self):
        return self._t._state

    @property
    def N(self):
        return self._t._root_N

    @property
    def child(self):
        return self._t._children()

    def is_leaf(self):
        return len(self.child) == 0


class MCTS_tree(object):
    def __init__(self, in_state, in_forward, search_threads, arena_words=1 << 21, leaf_parallel=1, priors="reference"):
        """leaf_parallel = K > 1 evaluates up to K leaves of this tree per network call (virtual-loss batching; faster moves,
        deterministic, but no longer the reference's search_threads=1 visit counts).  Default 1 = bit-exact mode."""
        self.noise_eps = 0.25
        self.dirichlet_alpha = 0.3
        # main.py:238 draws from np.random here (a 1-element Dirichlet is always [1.]); kept so that the
        # global RNG stream is consumed exactly like the reference's constructor does.
        self.p_ = (1 - self.noise_eps) * 1 + self.noise_eps * np.random.dirichlet([self.dirichlet_alpha])
        self.c_puct = 5
        self.forward = in_forward
        self.virtual_loss = 3
        self.search_threads = search_threads
        self.fifo = int(leaf_parallel) <= 1 and int(search_threads) > 1
        if self.fifo and int(search_threads) > 32:
            raise ValueError("search_threads > 32 is not supported by the device event loop")
        self.K = int(search_threads) if self.fifo else max(1, int(leaf_parallel))
        # priors: 'reference' (logit / sum, the reference's expansion) or 'softmax' (Engine priors)
        self.engine = (Engine(1, arena_words, search_threads=self.K, priors=priors) if self.fifo
                       else Engine(1, arena_words, leaves=self.K, priors=priors))
        dev = torch.device("cuda", self.engine.device)
        owner = getattr(in_forward, "__self__", None)
        K = self.K
        self._logits = torch.zeros((K, NLABEL), dtype=torch.float32, device=dev)
        self._value = torch.zeros((K,), dtype=torch.float32, device=dev)
        self._plan = self._graph = None
        if owner is not None and hasattr(owner, "native_plan") and getattr(owner, "precision", "") == "fp16":
            # the evaluator is this package's network: stay on the device (board bytes -> cz_net kernels -> tower) and
            # replay one CUDA graph per playout
            # (<= 16 rows per call: the one-launch cluster trunk of csrc/cz_tower.cu)
            small = K <= 16 and hasattr(owner, "small_plan")
            self._plan = owner.small_plan(K) if small else owner.native_plan(K)
            self._nn_in = self._plan.make_input(K)
            self._dev_forward = lambda x, lo, v: self._plan(x, lo, v)
        else:
            self._dev_forward = getattr(owner, "forward_device", None)
            dt = getattr(owner, "nn_dtype", torch.float32) if self._dev_forward else torch.float32
            self._nn_in = torch.zeros((K, 9, 10, 14), dtype=dt, device=dev)
        self._h_in = torch.zeros((K, 9, 10, 14), dtype=torch.float32).pin_memory()
        self._h_logits = torch.zeros((K, NLABEL), dtype=torch.float32).pin_memory()
        self._h_value = torch.zeros((K,), dtype=torch.float32).pin_memory()
        self.root = _Root(self)
        self._set_position(in_state, "w", 0)
        rules._init_tables()

    # ---- internals -------------------------------------------------------------------------------
    def _set_position(self, state, player, rr):
        self.engine.reset(None, rules.state_to_board(state)[None], [rules.side_of(player)], [rr])
        self._state, self._side, self._rr, self._root_N = state, rules.side_of(player), rr, 0
        self._cache = None

    def _eval(self, nn_in):
        if self._dev_forward is not None:
            self._dev_forward(nn_in, self._logits, self._value)
            return
        self._h_in.copy_(nn_in.float(), non_blocking=False)
        probs, value = self.forward(self._h_in.numpy())
        self._h_logits.copy_(torch.as_tensor(np.asarray(probs, dtype=np.float32).reshape(self.K, NLABEL)))
        self._h_value.copy_(torch.as_tensor(np.asarray(value, dtype=np.float32).reshape(self.K)))
        self._logits.copy_(self._h_logits, non_blocking=True)
        self._value.copy_(self._h_value, non_blocking=True)

    def _children(self):
        if self._cache is None:
            rc = self.engine.root_children()
            n = int(rc["n"][0])
            d = OrderedDict()
            for i in range(max(n, 0)):
                N = int(rc["visits"][0, i])
                d[rules.move_to_label(rc["moves"][0, i])] = leaf_node(rc["p"][0, i], rc["q"][0, i] if N else 0, N, rc["w"][0, i])
            self._cache = d
        return self._cache

    # ---- reference surface ---------------------------------------------------------------------
    def reload(self):  # main.py:255-258
        self._set_position(rules.START_STATE, "w", 0)

    def Q(self, move) -> float:  # main.py:261-270
        ch = self._children()
        if move in ch:
            return ch[move].Q
        print("{} not exist in the child".format(move))
        return 0.0

    def update_tree(self, act):  # main.py:272-276
        ch = self._children()
        idx = list(ch.keys()).index(act)   # KeyError/ValueError like root.child[act]
        self._root_N = ch[act].N
        st = self.engine.play(np.array([idx], dtype=np.int32))
        self._state = rules.board_to_state(st["boards"][0])
        self._side, self._rr = int(st["side"][0]), int(st["rr"][0])
        self._cache = None

    def is_expanded(self, key) -> bool:  # main.py:333-335
        return len(self._children()) > 0

    def main(self, state, current_player, restrict_round, playouts):  # main.py:473-493
        side = rules.side_of(current_player)
        if side != self._side or restrict_round != self._rr:
            self.engine.set_root_meta([side], [restrict_round])
            self._side, self._rr = side, restrict_round
        if self._plan is not None:
            self._plan.refresh_if_stale()      # the evaluator was trained / restored since the last search: new weights into the captured graph
            self._search_graph(playouts)
        else:
            self.engine.search(self._eval, playouts, self._nn_in, self._logits, self._value)
        self.engine.raise_on_error()
        self._cache = None

    def _search_graph(self, playouts):
        e = self.engine
        if self._graph is None:
            # one playout at a time: several (wave -> evaluation) pairs per graph, so that the gap between two graph launches is paid
            # once per REPS playouts (a wave of a completed search does nothing: at most REPS - 1 idle evaluations per move)
            self._reps = int(os.environ.get("CCHESS_WAVES_PER_GRAPH", "8")) if self.K == 1 else 1

            def body():
                for _ in range(self._reps):
                    e.wave(self._nn_in, self._logits, self._value)
                    self._plan(self._nn_in, self._logits, self._value)
            self._graph = capture_cuda_graph(body, lambda: self._plan(self._nn_in, self._logits, self._value), 3)
        e.begin_search(playouts)

        def step():
            self._graph.replay()
            e.launches += self._reps
        run_waves(e, step, playouts // self.K, playouts, per_step=self._reps)      # K leaves per wave: fewer waves needed

    def generate_inputs(self, in_state, current_player):  # main.py:531-533
        return rules.encode_batch(rules.state_to_board(in_state)[None], [rules.side_of(current_player)])[0]

    def state_to_positions(self, state):  # main.py:547-557 (no flip)
        return rules.encode_batch(rules.state_to_board(state)[None], [0])[0]

    def replace_board_tags(self, board):  # main.py:535-544
        return "".join(rules.GameBoard.board_to_pos_name(board))

    def try_flip(self, state, current_player, flip=False):  # main.py:560-574
        if not flip:
            return state, current_player
        rows = state.split("/")
        return "/".join(r.swapcase() for r in reversed(rows)), ("w" if current_player == "b" else "b")

    def is_black_turn(self, current_player):  # main.py:576-577
        return current_player == "b"
