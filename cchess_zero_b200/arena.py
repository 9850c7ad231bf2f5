"""Batched arena: one network plays another over thousands of concurrent games on one GPU, each player searching its own trees.

The evaluation match the reference planned (cchess_main.policy_evaluate, main.py:1207-1222, commented out there) and the gate of
AlphaGo Zero: is the candidate network stronger than the one it would replace?

Layout.  n games (n even) form n/2 colour-swapped pairs: game i and game i + n/2 start from the same position, the candidate plays
red in the first half and black in the second.  Each player keeps its own tree of every game, so four engines of n/2 games hold the
trees: (candidate, first half), (best, first half), (candidate, second half), (best, second half).  At every ply only the engine of
the player to move searches a game; the other player's tree of that game follows the move with Engine.play_moves (update_tree for a
move the tree did not choose; an unexpanded root starts a fresh tree at the new position).  When all games have the side to move in
common, exactly one candidate engine and one best engine search per ply, each with a full batch of games.

Move choice is get_action with exploration off (main.py:1332-1358): np.random.choice(actions, p = softmax(1/T log visits)) on one
legacy MT19937 stream per game, at `opening_temperature` for the first `opening_plies` plies of a game and `temperature` after."""
import argparse
import contextlib
import json
import math
import sys

import numpy as np
import torch

from . import rules as _rules                        # (random_openings and Match take a `rules` argument)
from ._lib import NLABEL, TERM_MATED, EngineError
from .engine import check_priors, check_rules
from .selfplay import SelfPlay, mt_streams, network_selfplay, sample_moves

NO_MOVE = 0xFFFF


class UniformEvaluator:
    """Zero logits and zero value for every position: a search-only opponent.  The priors are the logits themselves (as in the
    reference's expand, main.py:175-187), so every prior is 0 and the search follows the backed-up values of terminal positions alone.
    The reference's pure-MCTS opponent used random rollouts; this engine has none."""

    @torch.no_grad()
    def __call__(self, x):
        n = x.shape[0]
        return torch.zeros((n, NLABEL), dtype=torch.float32, device=x.device), torch.zeros((n,), dtype=torch.float32, device=x.device)


def random_openings(n_pairs, plies, seed=0, rules="reference"):
    """n_pairs start positions reached by `plies` uniformly random legal moves from the start position (positions where a king was
    captured are drawn again).  -> (boards u8 [n_pairs, 90], sides u8 [n_pairs], restrict_round i32 [n_pairs]).
    rules='strict': the moves are drawn from the strictly legal ones, and an opening that reaches a position without one (mated) is
    drawn again, so every opening is a running game under the strict rules."""
    strict = check_rules(rules) == "strict"
    rs = np.random.RandomState(seed)
    start = _rules.state_to_board(_rules.START_STATE)
    boards = np.tile(start, (n_pairs, 1))
    sides = np.zeros(n_pairs, dtype=np.uint8)
    rr = np.zeros(n_pairs, dtype=np.int32)
    todo = np.arange(n_pairs)
    for _ in range(1000):
        if len(todo) == 0:
            return boards, sides, rr
        b = np.tile(start, (len(todo), 1))
        s = np.zeros(len(todo), dtype=np.uint8)
        r = np.zeros(len(todo), dtype=np.int32)
        dead = np.zeros(len(todo), dtype=bool)
        for _ in range(plies):
            if strict:                                   # the strictly legal moves, compacted in move-generation order
                mv, cnt, legal, _, _ = _rules.strict_moves_batch(b, s)
                order = np.argsort(~legal, axis=1, kind="stable")
                mv, cnt = np.take_along_axis(mv, order, axis=1), legal.sum(axis=1).astype(np.int32)
            else:
                mv, cnt = _rules.legal_moves_batch(b, s)
            dead |= cnt <= 0
            pick = rs.randint(0, np.maximum(cnt, 1))
            b, cap = _rules.apply_moves_batch(b, mv[np.arange(len(todo)), pick])
            dead |= (cap == 1) | (cap == 8)
            r = np.where(cap == 0, r + 1, 0).astype(np.int32)
            s ^= 1
        if strict:
            dead |= _rules.strict_moves_batch(b, s)[4]
        ok = ~dead
        boards[todo[ok]], sides[todo[ok]], rr[todo[ok]] = b[ok], s[ok], r[ok]
        todo = todo[dead]
    raise RuntimeError("random_openings: could not draw %d openings of %d plies" % (n_pairs, plies))


def _elo(score):
    if score <= 0.0:
        return -math.inf
    if score >= 1.0:
        return math.inf
    return -400.0 * math.log10(1.0 / score - 1.0)


class MatchResult:
    """Outcome of a match, from the candidate's side.  games: one dict per game (candidate colour 'w' / 'b', opening index, result
    'win' / 'draw' / 'loss', winner 'w' / 'b' / 't', plies, adjudicated = drawn by max_plies, moves as u16 codes and labels)."""

    def __init__(self, games):
        self.games = games
        self.n = len(games)
        res = [g["result"] for g in games]
        self.wins, self.draws, self.losses = res.count("win"), res.count("draw"), res.count("loss")
        self.by_colour = {}
        for c in ("w", "b"):
            rc = [g["result"] for g in games if g["candidate_colour"] == c]
            self.by_colour[c] = dict(wins=rc.count("win"), draws=rc.count("draw"), losses=rc.count("loss"))

    @property
    def score(self):
        return (self.wins + 0.5 * self.draws) / self.n

    @property
    def elo(self):
        """Elo difference candidate - best: -400 log10(1/score - 1) (+-inf at score 1 / 0)."""
        return _elo(self.score)

    def elo_interval(self, z=1.959964):
        """95 % interval of the Elo difference: score +- z * standard error of the mean per-game score (trinomial variance of
        {1, 1/2, 0}), mapped through the Elo curve (an end at score 0 / 1 is -inf / +inf)."""
        s = self.score
        var = (self.wins * (1.0 - s) ** 2 + self.draws * (0.5 - s) ** 2 + self.losses * s ** 2) / self.n
        half = z * math.sqrt(var / self.n)
        return _elo(max(0.0, s - half)), _elo(min(1.0, s + half))

    def promote(self, threshold=0.55):
        """AlphaGo Zero's gate: the candidate replaces the best network if it scores more than `threshold`."""
        return self.score > threshold

    def to_json(self, threshold=0.55, games=True):
        f = lambda v: v if math.isfinite(v) else ("inf" if v > 0 else "-inf")  # noqa: E731
        lo, hi = self.elo_interval()
        d = dict(games=self.n, wins=self.wins, draws=self.draws, losses=self.losses, by_colour=self.by_colour, score=self.score,
                 elo=f(self.elo), elo_95=[f(lo), f(hi)], threshold=threshold, promote=self.promote(threshold))
        if games:
            d["records"] = self.games
        return json.dumps(d)


class _Player:
    """One player's trees of one half of the games: an engine driven by a SelfPlay used for its search() only."""

    def __init__(self, evaluator, n, playouts, search_threads, arena_words, colour, lo, rules="reference", priors="reference"):
        self.colour, self.lo, self.hi = colour, lo, lo + n
        kw = dict(auto_reset=False, keep_records=False, search_threads=search_threads, arena_words=arena_words, rules=rules,
                  priors=priors)
        if hasattr(evaluator, "native_plan"):                       # a policy_value_network: its own plan and precision
            self.sp = network_selfplay(evaluator, n, playouts, **kw)
        else:                                                       # a device callable (nn_in) -> (logits, value)
            self.sp = SelfPlay(n, evaluator, playouts, **kw)
        self.sp.capture_graph()
        self.engine = self.sp.engine


class Match:
    """candidate vs best over n_games concurrent games; step() plays one ply of every running game, run() plays them all out."""

    def __init__(self, candidate, best, n_games, playouts, search_threads=1, seeds=None, temperature=1e-3, opening_temperature=1.0,
                 opening_plies=30, openings=None, max_plies=None, arena_words=1 << 20, rules="reference", priors="reference"):
        """rules: 'reference' or 'strict' (every engine searches strictly legal moves only; a side without one is mated and loses;
        needs search_threads = 1; openings should then come from random_openings(..., rules='strict')).  Under strict rules a game
        whose opening leaves the side to move without a strictly legal move is over before its first ply, won by the other side.
        priors: 'reference' or 'softmax', how all four engines turn the networks' logits into priors (Engine priors)."""
        if n_games <= 0 or n_games % 2:
            raise ValueError("n_games must be a positive even number (colour-swapped pairs), got %r" % (n_games,))
        self.rules = check_rules(rules, search_threads)
        self.priors = check_priors(priors)
        _rules._init_tables()
        self.n, self.half = int(n_games), int(n_games) // 2
        self.temperature, self.opening_temperature, self.opening_plies = temperature, opening_temperature, int(opening_plies)
        self.max_plies = max_plies
        h = self.half
        # players[k]: half k // 2, candidate for even k; the candidate is red ('w') in the first half and black in the second
        self.players = [_Player(candidate, h, playouts, search_threads, arena_words, 0, 0, self.rules, self.priors),
                        _Player(best, h, playouts, search_threads, arena_words, 1, 0, self.rules, self.priors),
                        _Player(candidate, h, playouts, search_threads, arena_words, 1, h, self.rules, self.priors),
                        _Player(best, h, playouts, search_threads, arena_words, 0, h, self.rules, self.priors)]
        self._mt = mt_streams(range(self.n) if seeds is None else seeds)
        if len(self._mt) != self.n:
            raise ValueError("Match: %d seeds for %d games" % (len(self._mt), self.n))
        if openings is None:
            ob = _rules.state_to_board(_rules.START_STATE)[None]
            os_, orr = np.zeros(1, np.uint8), np.zeros(1, np.int32)
        else:
            ob, os_, orr = (np.asarray(a) for a in openings)
            ob = ob.reshape(-1, 90).astype(np.uint8)
        self.opening = np.tile(np.arange(h) % len(ob), 2)             # opening index of every game (a pair shares it)
        boards, sides, rr = ob[self.opening[:h]], np.asarray(os_, np.uint8)[self.opening[:h]], np.asarray(orr, np.int32)[self.opening[:h]]
        for p in self.players:
            p.engine.reset(None, boards, sides, rr)
        self.sides = np.tile(sides, 2)
        self.live = np.ones(self.n, dtype=bool)
        self.plies = np.zeros(self.n, dtype=np.int64)
        self.moves = [[] for _ in range(self.n)]
        self.winner = np.full(self.n, -1, dtype=np.int64)              # 0 'w', 1 'b', 2 draw
        self.adjudicated = np.zeros(self.n, dtype=bool)
        self.ply = 0
        if self.rules == "strict":            # an opening whose side to move has no strictly legal move: reset marked it mated
            st = self.players[0].engine.status()
            over = np.tile(st["terminal"] == TERM_MATED, 2)
            self.winner[over] = np.tile(st["winner"].astype(np.int64), 2)[over]
            self.live[over] = False

    def _to_move(self, p):
        return self.live[p.lo:p.hi] & (self.sides[p.lo:p.hi] == p.colour)

    def step(self):
        """One ply of every running game; returns the number of games still running."""
        if not self.live.any():
            return 0
        n = self.n
        for p in self.players:                                   # the engines of the players to move search
            m = self._to_move(p)
            if m.any():
                p.sp.search(mask=m)
        nch = np.zeros(n, dtype=np.int32)
        visits = np.zeros((n, 128), dtype=np.int32)
        codes = np.zeros((n, 128), dtype=np.uint16)
        for p in self.players:
            m = self._to_move(p)
            if m.any():
                rc = p.engine.root_children(want_wpq=False)
                idx = p.lo + np.nonzero(m)[0]
                nch[idx], visits[idx], codes[idx] = rc["n"][m], rc["visits"][m], rc["moves"][m]
        live = self.live.copy()
        if (nch[live] <= 0).any():
            for p in self.players:
                p.engine.raise_on_error()
            raise EngineError("game %d has no root children" % int(np.nonzero(live & (nch <= 0))[0][0]))
        temp = np.where(self.plies < self.opening_plies, self.opening_temperature, self.temperature)
        choice = sample_moves(nch, visits, live, temp, self._mt, False)
        move = np.full(n, NO_MOVE, dtype=np.uint16)
        move[live] = codes[live, choice[live]]
        status = {}
        for k in (0, 2):                                         # the two halves: (candidate, best) engines of the same games
            pair = self.players[k], self.players[k + 1]
            lo, hi = pair[0].lo, pair[0].hi
            if not live[lo:hi].any():
                continue
            for p in pair:
                mine = self._to_move(p)
                other = live[lo:hi] & ~mine
                st = None
                if mine.any():
                    st = p.engine.play(np.where(mine, choice[lo:hi], -1))
                if other.any():
                    st = p.engine.play_moves(np.where(other, move[lo:hi], NO_MOVE))
                status[p.colour] = st
            a, b = status[0], status[1]
            for key in ("boards", "side", "terminal", "winner", "ply", "rr"):
                if not np.array_equal(a[key], b[key]):
                    raise EngineError("match: the two players' trees of games %d..%d disagree on %s after ply %d" % (lo, hi - 1, key, self.ply))
            self.sides[lo:hi] = a["side"]
            term = live[lo:hi] & (a["terminal"] != 0)
            gi = lo + np.nonzero(term)[0]
            won = (a["terminal"][term] == 1) | (a["terminal"][term] == TERM_MATED)           # a king taken, or mated (strict rules)
            self.winner[gi] = np.where(won, a["winner"][term], 2)
            self.live[gi] = False
        for p in self.players:
            p.engine.raise_on_error()
        for g in np.nonzero(live)[0]:
            self.moves[g].append(int(move[g]))
        self.plies[live] += 1
        if self.max_plies is not None:
            adj = self.live & (self.plies >= self.max_plies)
            self.winner[adj] = 2
            self.adjudicated[adj] = True
            self.live[adj] = False
        self.ply += 1
        return int(self.live.sum())

    def tree_signature(self, game, colour):
        """Signature of the tree the player of `colour` (0 'w', 1 'b') keeps for `game` (Engine.tree_signature)."""
        for p in self.players:
            if p.lo <= game < p.hi and p.colour == colour:
                return p.engine.tree_signature(game - p.lo)
        raise IndexError(game)

    def counters(self):
        """Engine counters of the four engines (max_arena_words: the high-water mark of tree storage per game and half)."""
        return [p.engine.counters() for p in self.players]

    def result(self):
        games = []
        for g in range(self.n):
            cc = 0 if g < self.half else 1
            w = int(self.winner[g])
            res = "running" if w < 0 else "draw" if w == 2 else ("win" if w == cc else "loss")
            games.append(dict(game=g, pair=g % self.half, opening=int(self.opening[g]), candidate_colour="wb"[cc], result=res,
                              winner="?" if w < 0 else "wbt"[w], plies=int(self.plies[g]), adjudicated=bool(self.adjudicated[g]),
                              moves=list(self.moves[g]), labels=[_rules.move_to_label(m) for m in self.moves[g]]))
        return MatchResult(games)

    def run(self):
        while self.step():
            pass
        return self.result()


def _network(ckpt, seed, res_block_nums, precision):
    import tempfile
    from .net import policy_value_network
    with contextlib.redirect_stdout(sys.stderr), tempfile.TemporaryDirectory() as d:
        pv = policy_value_network(res_block_nums, precision=precision, seed=seed, save_dir=d)   # no checkpoint is picked up from ./models
        if ckpt:
            pv.restore(ckpt)
    return pv


def main(argv=None):
    ap = argparse.ArgumentParser(description="Play a candidate network against the best one over many concurrent games; prints one JSON line.")
    ap.add_argument("--candidate", default=None, help="checkpoint of the candidate (policy_value_network.save)")
    ap.add_argument("--best", default=None, help="checkpoint of the best network so far")
    ap.add_argument("--candidate_seed", type=int, default=1, help="seed of a freshly initialised candidate (no --candidate)")
    ap.add_argument("--best_seed", type=int, default=0, help="seed of a freshly initialised best network (no --best)")
    ap.add_argument("--games", type=int, default=400)
    ap.add_argument("--playouts", type=int, default=400)
    ap.add_argument("--search_threads", type=int, default=None, help="default 16 (reference rules) or 1 (strict rules)")
    ap.add_argument("--rules", choices=("reference", "strict"), default="reference",
                    help="strict: both players search strictly legal moves only and a side without one is mated")
    ap.add_argument("--priors", choices=("reference", "softmax"), default="reference",
                    help="softmax: the searches use the softmax of the legal moves' logits as priors (reference: logit / sum)")
    ap.add_argument("--res_block_nums", type=int, default=7)
    ap.add_argument("--precision", default="fp16")
    ap.add_argument("--threshold", type=float, default=0.55)
    ap.add_argument("--seed", type=int, default=0, help="game g draws its moves from RandomState(seed + g)")
    ap.add_argument("--openings", type=int, default=0, help="number of random openings (0: every pair starts from the start position)")
    ap.add_argument("--opening_moves", type=int, default=4, help="random plies of each opening")
    ap.add_argument("--opening_plies", type=int, default=30)
    ap.add_argument("--opening_temperature", type=float, default=1.0)
    ap.add_argument("--temperature", type=float, default=1e-3)
    ap.add_argument("--max_plies", type=int, default=None)
    ap.add_argument("--json", default=None, help="also write the full result (with every game's moves) to this file")
    a = ap.parse_args(argv)
    cand = _network(a.candidate, a.candidate_seed, a.res_block_nums, a.precision)
    best = _network(a.best, a.best_seed, a.res_block_nums, a.precision)
    threads = a.search_threads if a.search_threads is not None else (1 if a.rules == "strict" else 16)
    openings = random_openings(a.openings, a.opening_moves, a.seed, rules=a.rules) if a.openings > 0 else None
    m = Match(cand, best, a.games, a.playouts, search_threads=threads, seeds=[a.seed + g for g in range(a.games)],
              temperature=a.temperature, opening_temperature=a.opening_temperature, opening_plies=a.opening_plies, openings=openings,
              max_plies=a.max_plies, rules=a.rules, priors=a.priors)
    r = m.run()
    if a.json:
        with open(a.json, "w") as f:
            f.write(r.to_json(a.threshold, games=True) + "\n")
    print(r.to_json(a.threshold, games=False), flush=True)
    return r


if __name__ == "__main__":
    main()
