"""TEST INFRASTRUCTURE ONLY -- one arena game restated over two C oracle trees (oracle/oracle.py), the specification that
cchess_zero_b200.arena.Match is checked against.

Each player keeps its own tree.  The player to move searches its tree (co_tree_search, or co_tree_search_fifo for
search_threads > 1), chooses with rs.choice(acts, p = softmax(1/T log visits)) (get_action with exploration off, main.py:1339-1348)
and moves its root with update(idx); the other player's tree follows the same move with update(index of the move) when its root
has children, and otherwise starts afresh at the new position (reload)."""
import numpy as np

from oracle import oracle as O


def match_game(net_red, net_black, playouts, rs, opening_plies, opening_T, T, board=None, side=0, search_threads=1, max_plies=None,
               rr=0, signatures=False):
    """-> dict(moves [u16 codes], winner 0 'w' / 1 'b' / 2 draw, plies, adjudicated, sigs [(red tree, black tree) after every ply]
    when `signatures`).  net_*: stand-in net names of the oracle (hash_signed, hash_pos, mod17)."""
    board = O.from_state(O.START) if board is None else np.array(board, dtype=np.uint8)
    trees = [O.Tree(board), O.Tree(board)]
    nets = [net_red, net_black]
    moves, sigs = [], []
    winner, adjudicated = -1, False
    with np.errstate(divide="ignore"):
        while True:
            me = trees[side]
            err = (me.search(side, rr, playouts, nets[side]) if search_threads <= 1
                   else me.search_fifo(side, rr, playouts, search_threads, nets[side]))
            if err:
                raise RuntimeError("oracle tree error %d" % err)
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
                other.reload(board)
            moves.append(move)
            side ^= 1
            rr = rr + 1 if cap == 0 else 0
            if signatures:
                sigs.append((trees[0].signature(), trees[1].signature()))
            if not (board == 1).any() or not (board == 8).any():
                winner = 1 if not (board == 1).any() else 0
                break
            if rr >= 60:
                winner = 2
                break
            if max_plies is not None and len(moves) >= max_plies:
                winner, adjudicated = 2, True
                break
    return dict(moves=moves, winner=winner, plies=len(moves), adjudicated=adjudicated, sigs=sigs)
