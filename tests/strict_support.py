"""TEST INFRASTRUCTURE shared by test_strict_host.py and test_gpu_strict.py: the brute-force strict-legality oracle
(tests/strict_oracle.c, compiled together with oracle/cchess_oracle.c), the host build of the product's own per-lane source
(tests/host_strict_harness.cu), seeded position generators and hand-made positions with known answers."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_tmp = None
_libs = {}


def _dir():
    global _tmp
    if _tmp is None:
        _tmp = tempfile.TemporaryDirectory(prefix="cz_strict_")
    return _tmp.name


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def oracle_lib():
    if "so" not in _libs:
        so = os.path.join(_dir(), "libstrictoracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-shared", "-o", so,
                               os.path.join(ROOT, "tests", "strict_oracle.c"), os.path.join(ROOT, "oracle", "cchess_oracle.c"), "-lm", "-lpthread"])
        L = C.CDLL(so)
        L.so_strict_moves_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4
        L.so_random_play.argtypes = [C.c_uint64, C.c_int, C.c_void_p, C.c_void_p]
        L.so_random_setup.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _libs["so"] = L
    return _libs["so"]


def host_lib():
    """None when nvcc is not available."""
    if "hr" not in _libs:
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        if not os.path.exists(nvcc):
            return None
        so = os.path.join(_dir(), "libhoststrict.so")
        r = subprocess.run([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-shared", "-o", so,
                            os.path.join(ROOT, "tests", "host_strict_harness.cu")], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        L = C.CDLL(so)
        L.hr_strict_moves_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4
        _libs["hr"] = L
    return _libs["hr"]


def _batch(fn, boards, sides):
    boards = np.ascontiguousarray(boards, dtype=np.uint8).reshape(-1, 90)
    sides = np.ascontiguousarray(sides, dtype=np.uint8)
    n = boards.shape[0]
    mv, cnt = np.zeros((n, 128), np.uint16), np.zeros(n, np.int32)
    legal, flags = np.zeros((n, 4), np.uint32), np.zeros(n, np.uint8)
    fn(_p(boards), _p(sides), n, _p(mv), _p(cnt), _p(legal), _p(flags))
    return mv, cnt, legal, flags


def oracle_strict(boards, sides):
    """(moves u16[n,128], counts, legal u32[n,4], flags) by the brute-force definition: cz_strict_moves_batch's layout."""
    return _batch(oracle_lib().so_strict_moves_batch, boards, sides)


def host_strict(boards, sides):
    return _batch(host_lib().hr_strict_moves_batch, boards, sides)


def mask_bits(legal):
    """u32[n,4] -> bool[n,128]"""
    return ((legal[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(-1, 128)


def random_play(seed, n):
    boards, sides = np.zeros((n, 90), np.uint8), np.zeros(n, np.uint8)
    oracle_lib().so_random_play(seed, n, _p(boards), _p(sides))
    return boards, sides


def random_setup(seed, n, density, narrow):
    boards, sides = np.zeros((n, 90), np.uint8), np.zeros(n, np.uint8)
    oracle_lib().so_random_setup(seed, n, density, int(narrow), _p(boards), _p(sides))
    return boards, sides


def setup_boards():
    """Set-up boards from sparse to the full piece set, anywhere on the board and crowded onto the palace files."""
    bs, ss = [], []
    for k, (density, narrow) in enumerate([(40, 0), (110, 0), (256, 0), (60, 1), (140, 1), (256, 1)]):
        b, s = random_setup(1000 + k, 5000, density, narrow)
        bs.append(b); ss.append(s)
    return np.concatenate(bs), np.concatenate(ss)


def strict_labels(state, player):
    """The oracle's strictly legal moves as labels: a CPU stand-in for GameBoard.get_strict_moves."""
    from oracle import oracle as O
    mv, cnt, legal, _ = oracle_strict(O.from_state(state)[None], [0 if player == "w" else 1])
    ok = mask_bits(legal)[0]
    return [O.move_str(m) for i, m in enumerate(mv[0, :cnt[0]]) if ok[i]]


# Hand-made positions with known answers: (name, state string (rank 0 = Red's back rank first), side to move, in check, mated,
# the strictly legal moves, the pseudo-legal moves that are not strictly legal), both in move-generation order.
HAND_MADE = [
    # the rook is the only piece between the kings: it may slide along the file but not leave it
    ("flying_general_pin", "4K4/9/9/9/4R4/9/9/9/9/4k4", "w", False, False,
     "e0d0 e0f0 e0e1 e4e3 e4e2 e4e1 e4e5 e4e6 e4e7 e4e8 e4e9",
     "e4d4 e4c4 e4b4 e4a4 e4f4 e4g4 e4h4 e4i4"),
    # the knight on c2 reaches d0 over its leg c1: a pawn there blocks the check (d0e0 would face the other king)
    ("knight_check_blocked_at_the_leg", "3K5/2P6/2n6/9/9/9/9/9/9/4k4", "w", False, False, "d0d1 c1c2", "d0e0"),
    ("knight_check_with_the_leg_open", "3K5/9/2n6/9/9/9/9/9/9/4k4", "w", True, False, "d0d1", "d0e0"),
    # cannon check over the pawn: a second screen (a1e1) or a king step answers it, advancing the screen does not
    ("cannon_check_answered_by_adding_a_screen", "4K4/R8/9/9/4P4/9/9/4c4/9/3k5", "w", True, False,
     "e0f0 a1e1",
     "e0d0 e0e1 a1b1 a1c1 a1d1 a1f1 a1g1 a1h1 a1i1 a1a0 a1a2 a1a3 a1a4 a1a5 a1a6 a1a7 a1a8 a1a9 e4e5"),
    # the screen is a knight: every knight move takes the screen away
    ("cannon_check_answered_by_removing_the_screen", "4K4/9/9/9/4N4/9/9/4c4/9/3k5", "w", True, False,
     "e0f0 e4d2 e4c3 e4f2 e4g3 e4d6 e4c5 e4f6 e4g5", "e0d0 e0e1"),
    # rook on the file and knight from f2: no rook move helps, only the king step to f0
    ("double_check_only_a_king_move", "4K4/9/5n3/9/9/4r4/9/R8/9/3k5", "w", True, False,
     "e0f0",
     "e0d0 e0e1 a7b7 a7c7 a7d7 a7e7 a7f7 a7g7 a7h7 a7i7 a7a6 a7a5 a7a4 a7a3 a7a2 a7a1 a7a0 a7a8 a7a9"),
    ("checkmate", "r3K4/1r7/9/9/9/9/9/9/9/3k5", "w", True, True, "", "e0d0 e0f0 e0e1"),
    ("stalemate", "3K5/8r/9/9/9/9/9/9/9/4k4", "w", False, True, "", "d0e0 d0d1"),
    # the side to move can take the king (e8e0): that move is strictly legal
    ("king_capture_is_legal", "4K4/9/9/9/9/9/9/9/4r4/3k5", "b", False, False,
     "e8d8 e8c8 e8b8 e8a8 e8f8 e8g8 e8h8 e8i8 e8e7 e8e6 e8e5 e8e4 e8e3 e8e2 e8e1 e8e0 e8e9 d9e9 d9d8", ""),
    # attackers that reach a king only on set-up boards: advisor and king step inside the attacker's palace, bishop inside
    # the attacker's half with an empty eye
    ("advisor_check_answered_by_capture", "3R5/9/9/9/9/9/9/3a5/4K4/3k5", "w", True, False,
     "d0d7", "d0c0 d0b0 d0a0 d0e0 d0f0 d0g0 d0h0 d0i0 d0d1 d0d2 d0d3 d0d4 d0d5 d0d6"),
    ("bishop_check", "9/9/9/9/9/4K4/9/6b2/9/3k5", "w", True, True, "", ""),
    ("bishop_check_blocked_at_the_eye", "9/9/9/9/9/4K4/5P3/6b2/9/3k5", "w", False, True, "", "f6f7 f6g6 f6e6"),
    ("bishop_does_not_cross_the_river", "9/9/9/9/4K4/9/6b2/9/9/3k5", "w", False, True, "", ""),
    ("king_step_check_inside_the_attackers_palace", "9/9/9/9/9/9/9/9/9/3Kk4", "w", True, True, "", ""),
    ("king_step_not_outside_the_own_palace", "9/9/9/9/9/9/9/9/9/3Kk4", "b", False, False, "e9d9 e9f9 e9e8", ""),
]


def hand_made_boards():
    from oracle import oracle as O
    return (np.stack([O.from_state(h[1]) for h in HAND_MADE]), np.array([0 if h[2] == "w" else 1 for h in HAND_MADE], np.uint8))


def check_hand_made(mv, cnt, legal, flags):
    """Asserts that a strict-moves result (cz_strict_moves_batch's layout) over hand_made_boards() gives the known answers."""
    from oracle import oracle as O
    ok = mask_bits(legal)
    for i, (name, _, _, chk, mated, good, bad) in enumerate(HAND_MADE):
        lab = [O.move_str(m) for m in mv[i, :cnt[i]]]
        assert [m for m, k in zip(lab, ok[i]) if k] == good.split(), name
        assert [m for m, k in zip(lab, ok[i]) if not k] == bad.split(), name
        assert (bool(flags[i] & 1), bool(flags[i] & 2)) == (chk, mated), name
