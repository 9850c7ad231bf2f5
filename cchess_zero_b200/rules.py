"""Host-side mirror of the reference's rules surface (module globals + GameBoard), backed by the
CUDA library -- same names, argument meaning and error behaviour as main.py:23-91, 208-232, 579-1109.

Every function that computes something (move lists, applied moves, encodes) launches the sm_90a
kernels through the C ABI (cz_*_batch); nothing here re-implements the rules on the CPU."""
import ctypes as C

import numpy as np

from ._lib import MAXCHILD, NLABEL, EngineError, check, lib

START_STATE = "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"  # main.py:585
pieces_order = "KARBNPCkarbnpc"  # main.py:208
ind = {pieces_order[i]: i for i in range(14)}
c_PUCT = 5          # main.py:230
virtual_loss = 3    # main.py:231


def _hp(a):
    return a.ctypes.data_as(C.c_void_p)


def _device():
    import torch

    if not torch.cuda.is_available():
        raise EngineError("cchess_zero_b200 needs a CUDA device (no CPU fallback exists)")
    return torch.cuda.current_device()


def create_uci_labels():
    buf = np.zeros((NLABEL, 4), dtype=np.uint8)
    check(lib().cz_labels(_hp(buf)), "cz_labels")
    return [bytes(r).decode() for r in buf]


def flipped_uci_labels(param):
    """main.py:23-27 (string utility: every digit d -> 9-d)."""
    def repl(x):
        return "".join([(str(9 - int(a)) if a.isdigit() else a) for a in x])
    return [repl(x) for x in param]


labels_len = NLABEL
_LAZY = ("labels_array", "unflipped_index", "i2label", "label2i")


def _init_tables():
    g = globals()
    if "labels_array" not in g:
        la = create_uci_labels()
        u = np.zeros(NLABEL, dtype=np.int32)
        check(lib().cz_unflipped_index(_hp(u)), "cz_unflipped_index")
        g["labels_array"] = la                                   # main.py:211
        g["unflipped_index"] = [int(v) for v in u]               # main.py:213-214
        g["i2label"] = {i: v for i, v in enumerate(la)}          # main.py:216
        g["label2i"] = {v: i for i, v in enumerate(la)}          # main.py:217


def __getattr__(name):  # lazy module globals: importing the package must not need the library yet
    if name in _LAZY:
        _init_tables()
        return globals()[name]
    raise AttributeError(name)


# ---- state strings / moves -----------------------------------------------------------------
def state_to_board(state):
    b = np.zeros(90, dtype=np.uint8)
    check(lib().cz_from_state(state.encode(), _hp(b)), "cz_from_state")
    return b


def board_to_state(board):
    out = C.create_string_buffer(128)
    check(lib().cz_to_state(_hp(np.ascontiguousarray(board, dtype=np.uint8)), out), "cz_to_state")
    return out.value.decode()


def move_to_label(mv):
    s, d = int(mv) & 127, (int(mv) >> 7) & 127
    return "abcdefghi"[s % 9] + str(s // 9) + "abcdefghi"[d % 9] + str(d // 9)


def label_to_move(m):
    return (int(m[1]) * 9 + ord(m[0]) - 97) | ((int(m[3]) * 9 + ord(m[2]) - 97) << 7)


def side_of(player):
    return 0 if player == "w" else 1


# ---- batched device rules (host buffers) ------------------------------------------------------
def legal_moves_batch(boards, sides):
    boards = np.ascontiguousarray(boards, dtype=np.uint8).reshape(-1, 90)
    sides = np.ascontiguousarray(sides, dtype=np.uint8)
    n = boards.shape[0]
    mv = np.zeros((n, MAXCHILD), dtype=np.uint16)
    cnt = np.zeros(n, dtype=np.int32)
    check(lib().cz_legal_moves_batch(_device(), _hp(boards), _hp(sides), n, _hp(mv), _hp(cnt)), "cz_legal_moves_batch")
    return mv, cnt


def strict_moves_batch(boards, sides):
    """legal_moves_batch plus strict legality (cz_strict_moves_batch, one launch): -> (moves, counts, legal bool [n, 128],
    in_check bool [n], mated bool [n]).  legal[g, i]: move i does not leave the mover's king attacked (flying general included);
    mated: no such move, checkmate or stalemate."""
    boards = np.ascontiguousarray(boards, dtype=np.uint8).reshape(-1, 90)
    sides = np.ascontiguousarray(sides, dtype=np.uint8)
    n = boards.shape[0]
    mv = np.zeros((n, MAXCHILD), dtype=np.uint16)
    cnt = np.zeros(n, dtype=np.int32)
    mask = np.zeros((n, 4), dtype=np.uint32)
    flags = np.zeros(n, dtype=np.uint8)
    check(lib().cz_strict_moves_batch(_device(), _hp(boards), _hp(sides), n, _hp(mv), _hp(cnt), _hp(mask), _hp(flags)), "cz_strict_moves_batch")
    legal = ((mask[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(n, MAXCHILD)
    return mv, cnt, legal, (flags & 1).astype(bool), (flags & 2).astype(bool)


def apply_moves_batch(boards, moves):
    boards = np.array(boards, dtype=np.uint8, copy=True).reshape(-1, 90)
    moves = np.ascontiguousarray(moves, dtype=np.uint16)
    cap = np.zeros(boards.shape[0], dtype=np.uint8)
    check(lib().cz_apply_moves_batch(_device(), _hp(boards), _hp(moves), boards.shape[0], _hp(cap)), "cz_apply_moves_batch")
    return boards, cap


def encode_batch(boards, sides):
    boards = np.ascontiguousarray(boards, dtype=np.uint8).reshape(-1, 90)
    sides = np.ascontiguousarray(sides, dtype=np.uint8)
    out = np.zeros((boards.shape[0], 9, 10, 14), dtype=np.float32)
    check(lib().cz_encode_batch(_device(), _hp(boards), _hp(sides), boards.shape[0], _hp(out)), "cz_encode_batch")
    return out


def get_pieces_count(state):  # main.py:219-224
    return sum(1 for s in state if s.isalpha())


def is_kill_move(state_prev, state_next):  # main.py:226-227
    return get_pieces_count(state_prev) - get_pieces_count(state_next)


def softmax(x):  # main.py:1111-1116
    probs = np.exp(x - np.max(x))
    probs /= np.sum(probs)
    return probs


class GameBoard(object):
    """main.py:579-1109 -- same attributes and static methods; the rules run on the GPU."""
    Ny = 10
    Nx = 9

    def __init__(self):
        self.state = START_STATE
        self.round = 1
        self.current_player = "w"
        self.restrict_round = 0

    def reload(self):
        self.state = START_STATE
        self.round = 1
        self.current_player = "w"
        self.restrict_round = 0

    @staticmethod
    def print_borad(board, action=None):  # main.py:611-643
        rows = GameBoard.board_to_pos_name(board)
        src_x = src_y = None
        if action is not None:
            src_x, src_y = ord(action[0]) - 97, int(action[1])
        print("  abcdefghi")
        for i, line in enumerate(rows):
            line = line.replace("1", " ")
            if action is not None and i == src_y:
                line = line[:src_x] + "x" + line[src_x + 1:]
            print(i, line)

    @staticmethod
    def board_to_pos_name(board):  # main.py:705-714
        for d in range(2, 10):
            board = board.replace(str(d), "1" * d)
        return board.split("/")

    @staticmethod
    def check_bounds(toY, toX):  # main.py:717-724
        return not (toY < 0 or toX < 0 or toY >= GameBoard.Ny or toX >= GameBoard.Nx)

    @staticmethod
    def sim_do_action(in_action, in_state):
        """main.py:647-702 -> cz_apply_moves_batch (n = 1)."""
        b, _ = apply_moves_batch(state_to_board(in_state)[None], [label_to_move(in_action)])
        return board_to_state(b[0])

    @staticmethod
    def get_legal_moves(state, current_player):
        """main.py:743-1109 -> cz_legal_moves_batch (n = 1); same move order."""
        mv, cnt = legal_moves_batch(state_to_board(state)[None], [side_of(current_player)])
        return [move_to_label(m) for m in mv[0, : cnt[0]]]

    @staticmethod
    def get_strict_moves(state, current_player):
        """The moves of get_legal_moves, in the same order, that do not leave the mover's own king attacked."""
        mv, cnt, legal, _, _ = strict_moves_batch(state_to_board(state)[None], [side_of(current_player)])
        return [move_to_label(m) for m, ok in zip(mv[0, : cnt[0]], legal[0]) if ok]

    @staticmethod
    def in_check(state, current_player):
        """Could the other side capture current_player's king if it were to move (flying general included)?"""
        return bool(strict_moves_batch(state_to_board(state)[None], [side_of(current_player)])[3][0])
