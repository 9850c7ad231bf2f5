"""cz_snapshot_check on the CPU: engine snapshots built by hand in the layout include/cchess_b200.h documents, one valid blob and one
corruption per check.  Restore runs exactly this validator before it writes anything to the device."""
import ctypes as C

import numpy as np
import pytest

MAGIC = 0x485350414E535A43
H_FLAGS, H_DONE, H_TARGET, H_RR, H_ROOTN, H_ROOTCNT, H_ROOTBASE, H_ALLOC = range(8)
F_ACTIVE, F_CUR = 1, 16
NONE = 0xFFFFFFFF
START = "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"


def zobrist_checksum():
    """FNV-1a 64 over the little-endian bytes of the 16 x 96 splitmix64 Zobrist keys (restated from the format description)."""
    M = (1 << 64) - 1
    x, h = 0x9E3779B97F4A7C15, 0xCBF29CE484222325
    for _ in range(16 * 96):
        x = (x + 0x9E3779B97F4A7C15) & M
        t = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
        t = ((t ^ (t >> 27)) * 0x94D049BB133111EB) & M
        v = t ^ (t >> 31)
        for i in range(8):
            h = ((h ^ ((v >> (8 * i)) & 0xFF)) * 0x100000001B3) & M
    return h


ZOB = zobrist_checksum()


def _lib():
    from cchess_zero_b200._lib import lib
    return lib()


def start_board():
    b = np.zeros(96, dtype=np.uint8)
    assert _lib().cz_from_state(START.encode(), b.ctypes.data_as(C.c_void_p)) == 0
    return b


def block(moves, children=None, ngc=None, narr=5):
    """A node block: 8-word header {n_children, 0...}, then P | W | N | META | CHILD (| Q) with stride roundup8(n)."""
    n = len(moves)
    cs = (n + 7) & ~7
    b = np.zeros(8 + narr * cs, dtype=np.uint32)
    b[0] = n
    children = children or [NONE] * n
    ngc = ngc or [0] * n
    for i, mv in enumerate(moves):
        b[8 + i] = np.float32(1.0 / n).view(np.uint32)
        b[8 + 2 * cs + i] = 1
        b[8 + 3 * cs + i] = mv | (ngc[i] << 16)
        b[8 + 4 * cs + i] = children[i]
    for i in range(n, cs):
        b[8 + 4 * cs + i] = NONE
    return b


def mv(src, dst):
    return src | (dst << 7)


def tree(narr=5):
    """root (3 children) at 0; child 0 -> block A (2) at 48; child 2 -> block B (1) at 96 -> block C (10) at 144.  Returns
    (arena words, {name: base})."""
    k = 8 + narr * 8
    base = dict(root=0, A=k, B=2 * k, C=3 * k)
    root = block([mv(1, 20), mv(7, 24), mv(64, 67)], [base["A"], NONE, base["B"]], [2, 0, 1], narr)
    a = block([mv(81, 63), mv(83, 75)], narr=narr)
    b = block([mv(82, 64)], [base["C"]], [10], narr)
    c = block([mv(i, i + 9) for i in range(10)], narr=narr)
    return np.concatenate([root, a, b, c]), base


def game(arena, rootcnt=3, narr=5, flags=F_CUR):
    hdr = np.zeros(16, dtype=np.uint32)
    hdr[H_FLAGS] = flags
    hdr[H_ROOTCNT] = np.uint32(rootcnt & 0xFFFFFFFF)
    hdr[H_ALLOC] = len(arena)
    hdr[H_ROOTN] = 9
    cnt = np.arange(1, 11, dtype=np.uint32)                        # 5 u64 counters as 10 words
    fifo = np.zeros(28 if narr == 6 else 0, dtype=np.uint32)
    return [hdr, start_board().view(np.uint32), cnt, np.zeros(2, np.uint32), fifo, arena.astype(np.uint32)]


def blob(games, K=1, narr=5):
    B = len(games)
    fixed = 80 if narr == 6 else 52
    hw = ((48 + 8 * (B + 1) + 15) & ~15) // 4
    off = [hw]
    for s in games:
        off.append(off[-1] + sum(len(p) for p in s))
    head = np.zeros(hw // 2, dtype=np.uint64)
    head[0], head[1], head[2] = MAGIC, 1 | (2 << 32), ZOB
    head[3] = B | (K << 32)
    head[4] = narr | (fixed << 32)
    head[6:6 + B + 1] = off
    return np.concatenate([head.view(np.uint32)] + [p for s in games for p in s]).view(np.uint8).copy()


def check(b, B=1, K=1, narr=5, arena_words=1 << 16):
    L = _lib()
    rc = L.cz_snapshot_check(b.ctypes.data_as(C.c_void_p), b.nbytes, B, K, narr, arena_words)
    return rc, L.cz_last_error().decode()


def words(b):
    return b.view(np.uint32)


def section(b, g=0):
    """word offset of game g's section in blob b"""
    return int(b[48 + 8 * g:56 + 8 * g].view(np.int64)[0])


def test_valid_blobs_pass():
    ar, _ = tree()
    assert check(blob([game(ar)]))[0] == 0
    # two games, one of them a fresh reset (unexpanded root, empty tree); leaves K = 4
    two = blob([game(ar), game(np.zeros(0, np.uint32), rootcnt=-1, flags=0)], K=4)
    assert check(two, B=2, K=4)[0] == 0
    # a FIFO engine's blob (6 arrays per block, FIFO words) and an active game whose search is complete
    ar6, _ = tree(6)
    g6 = game(ar6, narr=6, flags=F_CUR | F_ACTIVE)
    g6[0][H_DONE] = g6[0][H_TARGET] = 400
    assert check(blob([g6], K=16, narr=6), K=16, narr=6)[0] == 0
    # the arena may be smaller than the saving engine's, as long as every alloc fits
    assert check(blob([game(ar)]), arena_words=len(ar))[0] == 0


def _corrupt(fn, **kw):
    ar, base = tree()
    b = blob([game(ar)])
    fn(words(b), section(b), base, len(ar))
    rc, msg = check(b, **kw)
    assert rc == -1, "accepted"
    return msg


def _meta_child(w, s, base, blk, i, n=None):
    """(META index, CHILD index) words of child i in the block at `base[blk]` with n children"""
    n = n or int(w[s + 52 + base[blk]])
    cs = (n + 7) & ~7
    at = s + 52 + base[blk] + 8
    return at + 3 * cs + i, at + 4 * cs + i


def test_each_corruption_is_refused_with_its_own_message():
    msgs = {}

    def child_past_alloc(w, s, base, alloc):
        _, c = _meta_child(w, s, base, "root", 0)
        w[c] = alloc + 8
    msgs["child past alloc"] = (_corrupt(child_past_alloc), "outside [0, alloc)")

    def child_below_parent(w, s, base, alloc):
        _, c = _meta_child(w, s, base, "B", 0)
        w[c] = base["B"]
    msgs["child <= parent base"] = (_corrupt(child_below_parent), "not above its parent's base")

    def count_mismatch(w, s, base, alloc):
        w[s + 52 + base["A"]] = 3
    msgs["count mismatch"] = (_corrupt(count_mismatch), "header count differs")

    def too_many(w, s, base, alloc):
        m, _ = _meta_child(w, s, base, "B", 0)
        w[m] = (w[m] & 0xFFFF) | (200 << 16)
        w[s + 52 + base["C"]] = 200
    msgs["more than 128 children"] = (_corrupt(too_many), "more than 128 children")

    msgs["alloc > arena words"] = (_corrupt(lambda w, s, base, alloc: None, arena_words=64), "exceeds the engine's arena words")

    def pending(w, s, base, alloc):
        w[s + H_FLAGS] |= 2
    msgs["pending flag"] = (_corrupt(pending), "not at rest")

    def owed(w, s, base, alloc):
        w[s + H_FLAGS] |= F_ACTIVE
        w[s + H_TARGET] = 8
    assert "not at rest" in _corrupt(owed)

    def in_flight(w, s, base, alloc):
        m, _ = _meta_child(w, s, base, "A", 1)
        w[m] |= 1 << 24
    msgs["in-flight count"] = (_corrupt(in_flight), "META bits 24-31")

    def off_board(w, s, base, alloc):
        m, _ = _meta_child(w, s, base, "C", 4)
        w[m] = (int(w[m]) & ~0x7F) | 95
    msgs["move square"] = (_corrupt(off_board), "move square")

    def shared(w, s, base, alloc):
        _, c0 = _meta_child(w, s, base, "root", 0)
        m2, c2 = _meta_child(w, s, base, "root", 2)
        w[c2], w[m2] = w[c0], (w[m2] & 0xFFFF) | (2 << 16)
    msgs["block reached twice"] = (_corrupt(shared), "reached twice")

    def bad_piece(w, s, base, alloc):
        w[s + 16] = 15
    msgs["piece code"] = (_corrupt(bad_piece), "piece code")

    def rootcnt(w, s, base, alloc):
        w[s + H_ROOTCNT] = 129
    msgs["root count"] = (_corrupt(rootcnt), "root child count")

    def winner(w, s, base, alloc):
        w[s + H_FLAGS] |= 1 << 8                                      # king captured, no winner
    msgs["terminal / winner"] = (_corrupt(winner), "terminal / winner")

    ar, _ = tree()
    b = blob([game(ar)])
    msgs["truncated"] = (check(b[:-16])[1], "truncated")
    msgs["truncated head"] = (check(b[:40])[1], "shorter than its head")
    for i, what in ((0, "magic"), (2, "Zobrist")):
        c = b.copy()
        c.view(np.uint64)[i] ^= 1
        msgs[what] = (check(c)[1], what)
    c = b.copy()
    c.view(np.uint64)[1] += 1
    msgs["version"] = (check(c)[1], "format version")
    msgs["B"] = (check(b, B=2)[1], "n_games differs")
    msgs["K"] = (check(b, K=16)[1], "(K) differs")
    msgs["narr"] = (check(b, narr=6)[1], "(narr) differ")

    for case, (msg, want) in msgs.items():
        assert want in msg, "%s: %r" % (case, msg)
    texts = [m for m, _ in msgs.values()]
    assert len(set(texts)) == len(texts), "two checks share a message"
    assert all("game 0" in msgs[k][0] for k in ("child past alloc", "count mismatch", "pending flag", "alloc > arena words"))


def test_offsets_must_be_monotone_and_name_the_game():
    ar, _ = tree()
    b = blob([game(ar), game(ar)])
    assert check(b, B=2)[0] == 0
    c = b.copy()
    off = c[48:48 + 24].view(np.int64)
    off[1] = off[0] - 4                                                # game 1 starts before game 0
    rc, msg = check(c, B=2)
    assert rc == -1 and "not monotone" in msg
    c = b.copy()
    words(c)[section(c, 1) + H_ALLOC] -= 8                             # game 1's alloc disagrees with its section size
    rc, msg = check(c, B=2)
    assert rc == -1 and "game 1" in msg and "section size" in msg


def test_save_games_round_trips_the_host_state_of_every_slot(tmp_path):
    """SelfPlay.save_games / load_games on the CPU (the engine replaced by the specification trees, its blob by a marker): boards,
    sides, live, RNG states, plies and every slot's unfinished record come back, and the records materialise the same tuples."""
    from search_spec import StandIn
    from cchess_zero_b200.selfplay import SelfPlay

    class Eng(StandIn):
        def snapshot(self):
            return np.arange(40, dtype=np.uint8)

        def restore(self, blob):
            assert np.array_equal(blob, np.arange(40, dtype=np.uint8))
            self.restored = True

    B, P = 5, 8
    a = SelfPlay(B, lambda x: None, P, seeds=[7 + g for g in range(B)], auto_reset=True, engine=Eng(B, "hash_pos"))
    with np.errstate(all="ignore"):
        for _ in range(70):
            a.step()
            a.pop_finished()
    a.finished.append((0, None))
    with pytest.raises(ValueError):
        a.save_games(str(tmp_path / "g.npz"))
    a.finished = []
    path = str(tmp_path / "g.npz")
    a.save_games(path)
    b = SelfPlay(B, lambda x: None, P, seeds=[99] * B, auto_reset=True, engine=Eng(B, "hash_pos"))
    b.load_games(path)
    assert b.engine.restored
    for k in ("boards", "sides", "live", "_mt"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert a.plies == b.plies and a.temperature == b.temperature
    for g in range(B):
        ra, rb = a.records[g], b.records[g]
        assert ra.players == rb.players and len(a._span[g]) == len(b._span[g]) == len(ra.players)
        ra._logs, rb._logs = a._span[g], b._span[g]
        ra.z = rb.z = np.zeros(len(ra.players))
        assert ra.states == rb.states and np.array_equal(ra.dense_pi(), rb.dense_pi()) and ra.actions == rb.actions

    np.savez(str(tmp_path / "bad.npz"), **{k: v for k, v in np.load(path).items() if k != "mt"})
    with pytest.raises(ValueError, match="'mt' missing"):
        b.load_games(str(tmp_path / "bad.npz"))


def test_fifo_event_loop_mid_search_is_refused():
    ar, _ = tree(6)
    b = blob([game(ar, narr=6)], narr=6)
    assert check(b, narr=6)[0] == 0
    words(b)[section(b) + 52] = 3                                      # FI_ITER of an event loop that is still running
    rc, msg = check(b, narr=6)
    assert rc == -1 and "game 0: FIFO event loop" in msg
