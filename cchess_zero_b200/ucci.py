"""UCCI front-end: drives cchess_main's play surface (get_action / update_tree / check_end, main.py:1332-1392) from the
Universal Chinese Chess Interface text protocol instead of the reference's tkinter ChessGame/ChessView (ChessGame.py:55-204).

    python -m cchess_zero_b200.ucci [--playouts 1200] [--res_block_nums 7] [--leaf_parallel 8]

Commands understood: ucci, isready, setoption name <playouts|leaf_parallel|temperature|priors> value <v>, position {startpos | fen <fen>}
[moves m1 m2 ...], banmoves m1 m2 ... (the next go does not play them; the next position clears them), go [nodes N | depth D | time ms ...] (nodes = playouts; depth/time are accepted and
ignored -- the reference searches a fixed playout count, main.py:1336), stop (no-op: go is synchronous like the reference's
blocking forward), probe/d (print position), quit.

Coordinates: UCCI squares are file a-i, rank 0-9 counted from Red's back rank -- exactly the reference's move labels
(main.py:30-65), so moves pass through unchanged.  FEN rows run from rank 9 down to rank 0 while the reference's state string
starts at rank 0 (main.py:585), so the rows are reversed; H/E are accepted as aliases of N/B.

The search object is injected (`driver`): anything with cchess_main's attributes `game_borad`, `mcts`, `playout_counts`,
`get_action`, `check_end`, `banned_moves` -- tests drive the protocol on CPU with a stand-in, the module's main() builds the real
one with strict=True: it never answers with a move that leaves its own king attacked, and answers nobestmove when it is mated.
main() also checks the moves of `position` for strict legality (`legal_moves`) and refuses a list that holds an illegal one."""
import sys

from ._lib import PRIORS

START_STATE = "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"
START_FEN = "rnbakabnr/9/1c5c1/p1p1p1p1p/9/9/P1P1P1P1P/1C5C1/9/RNBAKABNR w - - 0 1"
_ALIAS = {"H": "N", "h": "n", "E": "B", "e": "b"}
_PIECES = set("KABNRCPkabnrcp")


class UcciError(ValueError):
    pass


def _rows(board_field):
    rows = board_field.split("/")
    if len(rows) != 10:
        raise UcciError("FEN needs 10 ranks, got %d" % len(rows))
    out = []
    for r in rows:
        cells = []
        for ch in r:
            ch = _ALIAS.get(ch, ch)
            if ch.isdigit():
                cells.extend("1" * int(ch))
            elif ch in _PIECES:
                cells.append(ch)
            else:
                raise UcciError("bad FEN character %r" % ch)
        if len(cells) != 9:
            raise UcciError("FEN rank %r does not have 9 files" % r)
        out.append(cells)
    return out


def _compress(cells):
    s, run = [], 0
    for c in cells:
        if c == "1":
            run += 1
        else:
            if run:
                s.append(str(run))
                run = 0
            s.append(c)
    if run:
        s.append(str(run))
    return "".join(s)


def fen_to_state(fen):
    """-> (reference state string, 'w'|'b', halfmove clock).  Red ('w' or 'r') moves first in the reference."""
    f = fen.split()
    if not f:
        raise UcciError("empty FEN")
    rows = _rows(f[0])
    state = "/".join(_compress(r) for r in reversed(rows))
    side = f[1].lower() if len(f) > 1 else "w"
    if side not in ("w", "r", "b"):
        raise UcciError("bad side to move %r" % side)
    half = int(f[4]) if len(f) > 4 and f[4].isdigit() else 0
    return state, ("b" if side == "b" else "w"), half


def state_to_fen(state, player="w", halfmove=0, fullmove=1):
    rows = _rows(state)
    return "%s %s - - %d %d" % ("/".join(_compress(r) for r in reversed(rows)), player, halfmove, fullmove)


def parse_move(m):
    if len(m) != 4 or m[0] not in "abcdefghi" or m[2] not in "abcdefghi" or not m[1].isdigit() or not m[3].isdigit():
        raise UcciError("bad move %r" % m)
    return m


def apply_move(state, move):
    """GameBoard.sim_do_action on the state string (main.py:647-702): dst <- src, src <- empty.  -> (state, captured piece or '')"""
    rows = _rows(state)
    sx, sy, dx, dy = ord(move[0]) - 97, int(move[1]), ord(move[2]) - 97, int(move[3])
    piece = rows[sy][sx]
    if piece == "1":
        raise UcciError("no piece on %s" % move[:2])
    cap = rows[dy][dx]
    rows[dy][dx], rows[sy][sx] = piece, "1"
    return "/".join(_compress(r) for r in rows), ("" if cap == "1" else cap)


class UcciEngine:
    """Protocol state machine.  `driver_factory(options) -> driver` is called lazily at the first isready/position/go, so that
    `ucci` answers immediately the way GUIs expect."""

    NAME = "cchess-zero-b200"

    def __init__(self, driver_factory, out=None, playouts=1200, leaf_parallel=1, legal_moves=None, priors="reference"):
        """legal_moves: (state, player) -> [move labels]; when given, every move of a `position` command must be in it."""
        self._factory = driver_factory
        self._legal_moves = legal_moves
        self._banned = ()
        self._driver = None
        self.out = out if out is not None else sys.stdout
        self.options = {"playouts": int(playouts), "leaf_parallel": int(leaf_parallel), "temperature": 1e-3,
                        "priors": priors}
        if priors not in PRIORS:
            raise ValueError("priors must be 'reference' or 'softmax', not %r" % (priors,))
        self._base = (START_STATE, "w", 0)
        self._moves = ()
        self._synced = None          # (base, moves) the driver's tree currently stands on

    # ---- plumbing ------------------------------------------------------------------------------------
    def _say(self, line):
        self.out.write(line + "\n")
        self.out.flush()

    def driver(self):
        if self._driver is None:
            self._driver = self._factory(dict(self.options))
            self._synced = None
        return self._driver

    def _position_now(self):
        """(state, player, restrict_round, round) after base + moves; restrict_round follows main.py:1529-1533."""
        state, player, rr = self._base
        for m in self._moves:
            state, cap = apply_move(state, m)
            rr = 0 if cap else rr + 1
            player = "b" if player == "w" else "w"
        return state, player, rr, 1 + len(self._moves)

    def _sync(self):
        """Bring the driver's board and tree to the commanded position, keeping the searched subtree when the new move list
        extends the old one by moves the tree already holds (MCTS_tree.update_tree, main.py:272-276)."""
        d = self.driver()
        want = (self._base, self._moves)
        if self._synced == want:
            return d
        state, player, rr, rnd = self._position_now()
        reused = False
        if self._synced is not None and self._synced[0] == self._base:
            old = self._synced[1]
            if len(self._moves) > len(old) and self._moves[:len(old)] == old:
                reused = True
                for m in self._moves[len(old):]:
                    if m in d.mcts.root.child:
                        d.mcts.update_tree(m)
                    else:
                        reused = False
                        break
        if not reused:
            d.mcts._set_position(state, player, rr)
        gb = d.game_borad
        gb.state, gb.current_player, gb.restrict_round, gb.round = state, player, rr, rnd
        self._synced = want
        return d

    # ---- commands ------------------------------------------------------------------------------------
    def cmd_ucci(self, args):
        self._say("id name %s" % self.NAME)
        self._say("id author cchess_zero_b200")
        self._say("option playouts type spin min 1 max 1000000 default %d" % self.options["playouts"])
        self._say("option leaf_parallel type spin min 1 max 16 default %d" % self.options["leaf_parallel"])
        self._say("option temperature type string default %g" % self.options["temperature"])
        self._say("option priors type combo default %s var reference var softmax" % self.options["priors"])
        self._say("ucciok")

    def cmd_isready(self, args):
        self.driver()
        self._say("readyok")

    def cmd_setoption(self, args):
        # setoption [name] <option> [value] <v>
        a = [t for t in args if t not in ("name", "value")]
        if len(a) < 2:
            raise UcciError("setoption needs an option and a value")
        key = a[0].lower()
        if key not in self.options:
            self._say("info string unknown option %s" % a[0])
            return
        if key == "priors":
            if a[1] not in PRIORS:
                self._say("info string priors must be reference or softmax, not %s" % a[1])
                return
            self.options[key] = a[1]
        else:
            self.options[key] = float(a[1]) if key == "temperature" else int(a[1])
        if key in ("leaf_parallel", "priors") and self._driver is not None:
            self._driver = None      # K and the priors are construction-time properties of the engine handle
        elif key == "playouts" and self._driver is not None:
            self._driver.playout_counts = self.options["playouts"]

    def cmd_position(self, args):
        if not args:
            raise UcciError("position needs startpos or fen")
        if "moves" in args:
            k = args.index("moves")
            head, moves = args[:k], tuple(parse_move(m) for m in args[k + 1:])
        else:
            head, moves = args, ()
        if head[0] == "startpos":
            base = (START_STATE, "w", 0)
        elif head[0] == "fen":
            base = fen_to_state(" ".join(head[1:]))
        else:
            raise UcciError("position needs startpos or fen")
        state, player, rr = base
        for k, m in enumerate(moves):                     # validate before committing
            if self._legal_moves is not None and m not in self._legal_moves(state, player):
                raise UcciError("illegal move %s (move %d)" % (m, k + 1))
            state, _ = apply_move(state, m)
            player = "b" if player == "w" else "w"
        self._base, self._moves, self._banned = base, moves, ()

    def cmd_banmoves(self, args):
        self._banned = tuple(parse_move(m) for m in args)

    def cmd_go(self, args):
        playouts = self.options["playouts"]
        if "nodes" in args:
            playouts = int(args[args.index("nodes") + 1])
        d = self._sync()
        d.playout_counts = playouts
        d.banned_moves = self._banned
        ended, who = d.check_end()
        if ended:
            self._say("info string game over (%s)" % who)
            self._say("nobestmove")
            return
        try:
            act, move_probs, win_rate = d.get_action(d.game_borad.state, self.options["temperature"])
        except ValueError as e:                           # strict rules: every legal move is banned
            if not getattr(d, "strict", False):
                raise
            self._say("info string %s" % e)
            self._say("nobestmove")
            return
        # get_action already re-rooted the tree on `act` (main.py:1351); mirror it in the protocol state so that the GUI's next
        # "position ... moves ... act reply" continues inside the same tree.
        state, player, rr, rnd = self._position_now()
        nstate, cap = apply_move(state, act)
        gb = d.game_borad
        gb.state, gb.current_player = nstate, ("b" if player == "w" else "w")
        gb.restrict_round, gb.round = (0 if cap else rr + 1), rnd + 1
        self._synced = (self._base, self._moves + (act,))
        actions, probs = move_probs[0]
        best = sorted(zip(actions, probs), key=lambda t: -t[1])[:3]
        self._say("info nodes %d score %d pv %s" % (playouts, int(round(float(win_rate) * 1000)), act))
        self._say("info string visits " + " ".join("%s:%.3f" % (a, p) for a, p in best))
        self._say("bestmove %s" % act)

    def cmd_stop(self, args):
        pass

    def cmd_probe(self, args):
        state, player, rr, rnd = self._position_now()
        self._say("info string fen %s" % state_to_fen(state, player, rr, (rnd + 1) // 2))

    cmd_d = cmd_probe

    def handle(self, line):
        """-> False when the session should end."""
        toks = line.split()
        if not toks:
            return True
        if toks[0] == "quit":
            self._say("bye")
            return False
        fn = getattr(self, "cmd_" + toks[0], None)
        if fn is None:
            self._say("info string unknown command %s" % toks[0])
            return True
        try:
            fn(toks[1:])
        except UcciError as e:
            self._say("info string error %s" % e)
        return True

    def loop(self, inp=None):
        inp = inp if inp is not None else sys.stdin
        for line in inp:
            if not self.handle(line.strip()):
                break


def _real_driver(res_block_nums):
    def make(options):
        from .selfplay import cchess_main
        return cchess_main(playout=options["playouts"], exploration=False, processor="gpu", res_block_nums=res_block_nums,
                           log_file=False, leaf_parallel=options["leaf_parallel"], strict=True, priors=options["priors"])
    return make


def main():
    import argparse
    import contextlib
    ap = argparse.ArgumentParser()
    ap.add_argument("--playouts", default=1200, type=int)
    ap.add_argument("--leaf_parallel", default=8, type=int)
    ap.add_argument("--res_block_nums", default=7, type=int)
    ap.add_argument("--priors", default="reference", choices=("reference", "softmax"),
                    help="softmax: search with the softmax of the legal moves' logits as priors (reference: logit / sum)")
    a = ap.parse_args()
    from .rules import GameBoard
    eng = UcciEngine(_real_driver(a.res_block_nums), out=sys.stdout, playouts=a.playouts, leaf_parallel=a.leaf_parallel,
                     legal_moves=GameBoard.get_strict_moves, priors=a.priors)
    real_out = sys.stdout
    eng.out = real_out
    with contextlib.redirect_stdout(sys.stderr):      # cchess_main prints progress lines; keep the protocol stream clean
        eng.loop(sys.stdin)


if __name__ == "__main__":
    main()
