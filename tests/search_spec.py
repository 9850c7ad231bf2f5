"""TEST INFRASTRUCTURE: the serial specification that the device search is checked against, for both rule sets, with and without root
exploration noise.  The C trees (tests/strict_search_oracle.c, built by strict_support.oracle_lib together with tests/strict_oracle.c),
the end test, a self-play game loop, an arena game loop, an engine-interface stand-in that drives the host loops of SelfPlay, Match
and Trainer on the CPU, hand-made positions with a mate in one and the search cases the strict tree tests use.

rules='reference' is the reference's search (co_tree_search; search_threads = K > 1: its K-coroutine schedule, co_tree_search_fifo);
rules='strict' is the strict-rules one-leaf search (ss_tree_search_fake).  priors='softmax' makes every expansion of the tree use
softmax priors (pz_softmax, the definition of Engine(priors='softmax'), DESIGN 3k) instead of the reference's logit / sum.  The names
mirror the product's rules=, search_threads= and priors=.

A noisy search of one game, as SelfPlay(root_noise=(eps, alpha)) defines it: expand the root (a search of 0 playouts); when it has
n >= 1 children, eta = RandomState([seed, 1]).dirichlet(alpha * ones(n)) and P' = f32((1 - eps) * f64(P) + eps * eta); then the
search's playouts."""
import numpy as np

from strict_support import _p, oracle_lib as lib, random_play

NETS = ("hash_signed", "hash_pos", "mod17")
NET_IDS = {"hash_signed": 0, "hash_pos": 1, "mod17": 2}


class Tree:
    """One game's specification tree."""

    def __init__(self, board, rules="reference", search_threads=1, priors="reference"):
        if rules not in ("reference", "strict") or (rules == "strict" and search_threads != 1) or priors not in ("reference", "softmax"):
            raise ValueError("rules %r with search_threads %r and priors %r" % (rules, search_threads, priors))
        self.rules, self.K = rules, int(search_threads)
        b = _p(np.ascontiguousarray(board, dtype=np.uint8))
        self.h = lib().ss_tree_new(b) if rules == "strict" else lib().co_tree_new(b)
        if priors == "softmax":
            lib().pz_tree_softmax(self.h)

    def __del__(self):
        try:
            lib().co_tree_free(self.h)
        except Exception:
            pass

    def search(self, side, rr, playouts, net, shift=0.0):
        """shift: a constant added to every logit of the stand-in net (reference rules, search_threads = 1)"""
        L, args = lib(), (self.h, int(side), int(rr), int(playouts))
        if shift != 0.0:
            if self.rules != "reference" or self.K != 1:
                raise ValueError("a logit shift needs reference rules and search_threads 1")
            return L.pz_search_shifted(*args, NET_IDS[net], float(shift))
        if self.rules == "strict":
            return L.ss_tree_search_fake(*args, NET_IDS[net])
        if self.K > 1:
            return L.co_tree_search_fifo(*args, self.K, NET_IDS[net])
        return L.co_tree_search_fake(*args, NET_IDS[net])

    def count(self):
        """the number of root children; -1 when the root is not expanded"""
        return lib().co_tree_root_children(self.h, None, None, None, None, None)

    def root_children(self):
        """-> (moves, N, W, P, Q) of the root's children, empty when the root is not expanded"""
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
        """(label index, N, W bits, P bits, Q bits, n_children) of every node in depth-first order; under strict rules n_children is
        -1 for a node expanded without children"""
        out = np.zeros((cap, 6), np.int64)
        fn = lib().ss_tree_signature if self.rules == "strict" else lib().co_tree_signature
        n = fn(self.h, _p(out), cap)
        if n > cap:
            return self.signature(int(n))
        return out[:n].copy()


def softmax(logits):
    """pz_softmax: the softmax priors of one node's logits (float32, 1..128 of them, move order)"""
    P = np.array(logits, dtype=np.float32)
    assert 1 <= len(P) <= 128
    lib().pz_softmax(_p(P), len(P))
    return P


def cz_exp(x):
    """csrc/cz_exp.h on the host: float64 array -> float64 array"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty_like(x)
    lib().pz_exp(_p(x), _p(y), x.size)
    return y


def strict_moves(board, side):
    """The strictly legal moves (u16 codes, move-generation order, first 128 pseudo-legal moves) by the brute-force definition."""
    mv, ok = np.zeros(512, np.uint16), np.zeros(512, np.uint8)
    n = lib().so_strict_moves(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side), _p(mv), _p(ok))
    n = min(n, 128)
    return mv[:n][ok[:n].astype(bool)].copy()


def in_check(board, side):
    return bool(lib().so_in_check(_p(np.ascontiguousarray(board, dtype=np.uint8)), int(side)))


def game_end(board, side, rr, rules):
    """oracle.game_end (a king taken -> (1, winner), rr >= 60 -> (2, -1)) and after it, under strict rules, the side to move without a
    strictly legal move -> (3, the side that just moved); (0, -1) while the game runs."""
    from oracle import oracle as O
    code, winner = O.game_end(board, side, rr)
    if code == 0 and rules == "strict" and len(strict_moves(board, side)) == 0:
        return 3, side ^ 1
    return code, winner


def mix(P, eta, eps):
    """The noised priors: f32((1 - eps) * f64(P) + eps * eta), each operation rounded once in float64."""
    return ((1.0 - eps) * np.asarray(P, dtype=np.float32).astype(np.float64) + eps * eta).astype(np.float32)


def noisy_search(tree, side, rr, playouts, net, rn, eps, alpha):
    """One search with root noise from RandomState rn; returns the eta drawn (None when the root has no child)."""
    assert tree.search(side, rr, 0, net) == 0
    _, _, _, P, _ = tree.root_children()
    eta = None
    if len(P) >= 1:
        eta = rn.dirichlet(alpha * np.ones(len(P)))
        tree.set_root_P(mix(P, eta, eps))
    assert tree.search(side, rr, playouts, net) == 0
    return eta


def selfplay_game(net, playouts, rs, rules="reference", search_threads=1, root_noise=None, priors="reference"):
    """oracle.selfplay_game (cchess_main.selfplay + get_action: one slot's SelfPlay game) over the specification tree of `rules`,
    `search_threads` and `priors`, ended by game_end.  rs: np.random.RandomState standing in for the global np.random of the reference.
    root_noise: None, or (eps, alpha, rn) with rn the noise stream RandomState([seed, 1]): every search is a noisy_search."""
    from oracle import oracle as O
    tree = Tree(O.from_state(O.START), rules, search_threads, priors)

    def search(side, rr):
        if root_noise is None:
            return tree.search(side, rr, playouts, net)
        eps, alpha, rn = root_noise
        noisy_search(tree, side, rr, playouts, net, rn, eps, alpha)
        return 0
    return O.selfplay_game(net, playouts, rs, tree=tree, search=search, end=lambda b, s, r: game_end(b, s, r, rules))


def match_game(net_red, net_black, playouts, rs, opening_plies, opening_T, T, board=None, side=0, rr=0, max_plies=None, rules="reference",
               search_threads=1, signatures=False, priors="reference"):
    """One arena game, the specification of cchess_zero_b200.arena.Match.  Each player keeps its own tree.  The player to move searches
    its tree, chooses with rs.choice(acts, p = softmax(1/T log visits)) (get_action with exploration off, main.py:1339-1348) and moves
    its root with update(idx); the other player's tree follows the same move when its root has children, and otherwise starts afresh
    at the new position.
    -> dict(moves [u16 codes], winner 0 'w' / 1 'b' / 2 draw, plies, adjudicated, end (game_end's code), sigs [(red tree, black tree)
    after every ply] when `signatures`).  net_*: stand-in net names (hash_signed, hash_pos, mod17)."""
    from oracle import oracle as O
    board = O.from_state(O.START) if board is None else np.array(board, dtype=np.uint8)
    trees = [Tree(board, rules, search_threads, priors), Tree(board, rules, search_threads, priors)]
    nets = [net_red, net_black]
    moves, sigs = [], []
    winner, adjudicated = -1, False
    with np.errstate(divide="ignore"):
        while True:
            me = trees[side]
            err = me.search(side, rr, playouts, nets[side])
            if err:
                raise RuntimeError("specification tree error %d" % err)
            mv, N, _, _, _ = me.root_children()
            visits = tuple(int(v) for v in N)
            temp = opening_T if len(moves) < opening_plies else T
            probs = O.softmax(1.0 / temp * np.log(visits))
            acts = [O.move_str(m) for m in mv]
            idx = acts.index(rs.choice(acts, p=probs))
            move = int(mv[idx])
            me.update(idx)
            board, cap = O.apply_move(board, move)
            omv = trees[side ^ 1].root_children()[0]
            if len(omv):
                trees[side ^ 1].update(list(omv).index(move))
            else:
                trees[side ^ 1] = Tree(board, rules, search_threads, priors)
            moves.append(move)
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            if signatures:
                sigs.append((trees[0].signature(), trees[1].signature()))
            end, w = game_end(board, side, rr, rules)
            if end:
                winner = 2 if end == 2 else w
                break
            if max_plies is not None and len(moves) >= max_plies:
                winner, adjudicated = 2, True
                break
    return dict(moves=moves, winner=winner, plies=len(moves), adjudicated=adjudicated, end=end, sigs=sigs)


class StandIn:
    """Engine-interface stand-in over the specification trees (one per game): SelfPlay's, Match's and Trainer's host loops on the CPU.
    The whole search of every selected game happens in the first wave.  A game ends as game_end says; under strict rules a reset to a
    position without a strictly legal move is mated at once, as on the device.  root_noise applies mix() to the root priors, as
    k_root_noise does.  `priors` is the trees' prior rule, as Engine's.  `log` records every begin_search / root_counts / root_noise
    call.  Test infrastructure only."""
    torch_device = "cpu"

    def __init__(self, n, net, rules="reference", search_threads=1, priors="reference"):
        from oracle import oracle as O
        self.O, self.B, self.net, self.rules, self.K, self.device, self.launches = O, n, net, rules, search_threads, 0, 0
        self.priors = priors
        self.boards = np.tile(O.from_state(O.START), (n, 1))
        self.trees = [Tree(self.boards[g], rules, search_threads, priors) for g in range(n)]
        self.side = np.zeros(n, np.uint8); self.rr = np.zeros(n, np.int32); self.ply = np.zeros(n, np.int32)
        self.terminal = np.zeros(n, np.uint8); self.winner = -np.ones(n, np.int8)
        self.target = np.zeros(n, np.int64); self.pending = np.zeros(n, bool)
        self.log = []

    def reset(self, mask=None, boards=None, sides=None, rr=None):
        for g in range(self.B):
            if mask is None or mask[g]:
                self.boards[g] = self.O.from_state(self.O.START) if boards is None else boards[g]
                self.side[g] = 0 if sides is None else sides[g]
                self.rr[g] = 0 if rr is None else rr[g]
                self.trees[g] = Tree(self.boards[g], self.rules, self.K, self.priors)
                self.ply[g] = 0; self.terminal[g] = 0; self.winner[g] = -1
                if self.rules == "strict" and len(strict_moves(self.boards[g], int(self.side[g]))) == 0:
                    self.terminal[g], self.winner[g] = 3, self.side[g] ^ 1

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
        n = np.array([t.count() for t in self.trees], dtype=np.int32)
        self.log.append(("root_counts", n.copy()))
        return n

    def root_noise(self, mask, eta, eps):
        self.log.append(("root_noise", np.array(mask, dtype=bool), np.array(eta, dtype=np.float64), float(eps)))
        for g in np.nonzero(mask)[0]:
            P = self.trees[g].root_children()[3]
            if len(P):
                self.trees[g].set_root_P(mix(P, eta[g, :len(P)], eps))

    def root_children(self, want_wpq=True):
        n = np.array([t.count() for t in self.trees], dtype=np.int32)
        out = dict(n=n, moves=np.zeros((self.B, 128), np.uint16), visits=np.zeros((self.B, 128), np.int32))
        for k in ("w", "p", "q"):
            out[k] = np.zeros((self.B, 128), np.float32)
        for g, t in enumerate(self.trees):
            for k, a in zip(("moves", "visits", "w", "p", "q"), t.root_children()):
                out[k][g, :len(a)] = a
        return out

    def _advance(self, g, move):
        self.boards[g], cap = self.O.apply_move(self.boards[g], int(move))
        self.side[g] ^= 1; self.rr[g] = self.rr[g] + 1 if cap == 0 else 0; self.ply[g] += 1
        self.terminal[g], self.winner[g] = game_end(self.boards[g], int(self.side[g]), int(self.rr[g]), self.rules)

    def play(self, choice, want_status=True):
        q = np.zeros(self.B, np.float32)
        for g, c in enumerate(choice):
            if c >= 0:
                mv, _, _, _, Q = self.trees[g].root_children()
                q[g] = Q[c]
                self.trees[g].update(int(c))
                self._advance(g, mv[c])
        return dict(self.status(), q=q) if want_status else None

    def play_moves(self, moves, want_status=True):
        legal = strict_moves if self.rules == "strict" else self.O.legal_moves
        for g, m in enumerate(moves):
            if m == 0xFFFF:
                continue
            assert self.terminal[g] == 0 and int(m) in [int(x) for x in legal(self.boards[g], int(self.side[g]))]
            kids = list(self.trees[g].root_children()[0])
            if kids:
                self.trees[g].update(kids.index(m))
                self._advance(g, m)
            else:
                self._advance(g, m)
                self.trees[g] = Tree(self.boards[g], self.rules, self.K, self.priors)
        return self.status() if want_status else None

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

    def tree_signature(self, g):
        return self.trees[g].signature()


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
