"""GPU parity tests: the CUDA path (through the C ABI) against the golden vectors produced by the
reference and against the CPU oracle on seeded inputs.  Bit-exact everywhere (integer / f32-bit compares)."""
import hashlib

import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu


def sha(b):
    return hashlib.sha256(b).hexdigest()[:16]


def bits(v):
    """float32 bit pattern with NaN canonicalised (see oracle/ref_harness.py:f32_bits)"""
    v = np.float32(v)
    return 0x7FC00000 if np.isnan(v) else int(v.view(np.uint32))


@pytest.fixture(scope="module")
def O():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def R():
    from cchess_zero_b200 import rules
    rules._init_tables()
    return rules


def test_rules_against_reference_vectors(R):
    g = load_golden("movegen.json.gz")["records"]
    boards = np.stack([R.state_to_board(r["state"]) for r in g])
    sides = np.array([0 if r["player"] == "w" else 1 for r in g], dtype=np.uint8)
    mv, cnt = R.legal_moves_batch(boards, sides)
    enc = R.encode_batch(boards, sides)
    for i, r in enumerate(g):
        assert " ".join(R.move_to_label(m) for m in mv[i, : cnt[i]]) == r["moves"], r["state"]
        assert [int(k) for k in np.nonzero(enc[i].reshape(-1))[0]] == r["enc"]
    assert set(np.unique(enc)) <= {0.0, 1.0}
    have = [i for i, r in enumerate(g) if "move" in r]
    nb, cap = R.apply_moves_batch(boards[have], [R.label_to_move(g[i]["move"]) for i in have])
    for k, i in enumerate(have):
        assert R.board_to_state(nb[k]) == g[i]["next"]
        assert int(cap[k] != 0) == g[i]["kill"]


def test_gameboard_surface(R):
    gb = R.GameBoard()
    mv = R.GameBoard.get_legal_moves(gb.state, "w")
    assert len(mv) == 44 and mv[:4] == ["a0a1", "a0a2", "b0a2", "b0c2"]
    assert R.GameBoard.sim_do_action("h2e2", gb.state) == "RNBAKABNR/9/1C2C4/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakabnr"
    assert R.GameBoard.sim_do_action("b7b0", gb.state) == "RcBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/7c1/9/rnbakabnr"
    with pytest.raises(KeyError):
        R.label2i["a0a0"]


def _random_positions(O, n_games, seed, max_plies=160):
    rng = np.random.RandomState(seed)
    boards, sides = [], []
    for _ in range(n_games):
        b, side = O.from_state(O.START), 0
        for _ply in range(max_plies):
            boards.append(b.copy()); sides.append(side)
            mv = O.legal_moves(b, side)
            if len(mv) == 0:
                break
            b, cap = O.apply_move(b, mv[rng.randint(len(mv))])
            side ^= 1
            if cap in (1, 8):
                boards.append(b.copy()); sides.append(side)
                break
    return np.stack(boards), np.array(sides, dtype=np.uint8)


def test_rules_random_play_vs_oracle(O, R):
    boards, sides = _random_positions(O, 400, 123)
    assert len(boards) > 30000
    mv, cnt = R.legal_moves_batch(boards, sides)
    enc = R.encode_batch(boards, sides)
    for i in range(len(boards)):
        om = O.legal_moves(boards[i], int(sides[i]))
        assert cnt[i] == len(om) and np.array_equal(mv[i, : cnt[i]], om), i
    for i in range(0, len(boards), 7):
        assert np.array_equal(enc[i], O.encode(boards[i], int(sides[i])))


def test_encode_dtypes(O, R):
    from cchess_zero_b200._lib import lib, check, BF16, F16, F32
    boards, sides = _random_positions(O, 10, 5)
    n = len(boards)
    db = torch.from_numpy(boards).cuda()
    ds = torch.from_numpy(sides).cuda()
    ref = torch.from_numpy(R.encode_batch(boards, sides)).cuda()
    for dt, code in ((torch.float32, F32), (torch.bfloat16, BF16), (torch.float16, F16)):
        out = torch.full((n, 9, 10, 14), 7.0, dtype=dt, device="cuda")
        check(lib().cz_encode_dev(db.data_ptr(), ds.data_ptr(), n, out.data_ptr(), code, None))
        torch.cuda.synchronize()
        assert torch.equal(out.float(), ref)


def test_fakenets_match_oracle(O, R):
    from cchess_zero_b200.fakenet import FakeNet
    boards, sides = _random_positions(O, 6, 9)
    enc = R.encode_batch(boards, sides)
    x = torch.from_numpy(enc).cuda()
    for kind in ("hash_signed", "hash_pos", "mod17"):
        lo, v = FakeNet(kind)(x)
        olo, ov = O.fake_forward(kind, enc)
        assert np.array_equal(lo.cpu().numpy(), olo), kind
        assert np.array_equal(v.cpu().numpy(), ov.reshape(-1)), kind


def _run_cases(cases, net, R, graph=False, leaves=1):
    """cases: list of dict(board, side, rr, playouts).  Returns the engine after searching."""
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.fakenet import FakeNet
    B = len(cases)
    e = Engine(B, arena_words=1 << 20, leaves=leaves)
    e.reset(None, np.stack([c["board"] for c in cases]), [c["side"] for c in cases], [c["rr"] for c in cases])
    fn = FakeNet(net)
    nn_in = torch.zeros((e.rows, 9, 10, 14), device="cuda")
    logits = torch.zeros((e.rows, 2086), device="cuda")
    value = torch.zeros((e.rows,), device="cuda")
    pl = np.array([c["playouts"] for c in cases])
    for p in np.unique(pl):
        e.begin_search(int(p), (pl == p).astype(np.uint8))

    def fwd():
        lo, v = fn(nn_in)
        logits.copy_(lo); value.copy_(v)

    waves = 0
    while True:
        e.wave(nn_in, logits, value)
        waves += 1
        if e.unfinished() == 0:
            break
        fwd()
        assert waves < 5 * pl.max() + 50
    e.raise_on_error()
    return e


@pytest.mark.parametrize("net", ["mod17", "hash_signed", "hash_pos"])
def test_tree_against_reference_vectors(net, R):
    cases = [c for c in load_golden("tree.json")["cases"] if c["net"] == net]
    e = _run_cases([dict(board=R.state_to_board(c["state"]), side=0 if c["player"] == "w" else 1, rr=c["rr"],
                         playouts=c["playouts"]) for c in cases], net, R)
    rc = e.root_children()
    for g, c in enumerate(cases):
        sig = e.tree_signature(g)
        assert sig.shape[0] == c["n_nodes"], c["note"]
        assert sig[:40].tolist() == c["head"], c["note"]
        if sha(sig.tobytes()) != c["sha_sig"]:   # locate the first differing record with the oracle's help
            from oracle import oracle as OO
            t = OO.Tree(OO.from_state(c["state"]))
            t.search(0 if c["player"] == "w" else 1, c["rr"], c["playouts"], c["net"])
            osig = t.signature()
            d = np.nonzero((osig != sig).any(axis=1))[0]
            raise AssertionError("%s: first differing records %s: oracle %s cuda %s" % (c["note"], d[:3], osig[d[:3]], sig[d[:3]]))
        n = rc["n"][g]
        got = [[R.move_to_label(rc["moves"][g, i]), int(rc["visits"][g, i]), bits(rc["w"][g, i]), bits(rc["p"][g, i]), bits(rc["q"][g, i])] for i in range(n)]
        assert got == c["root"], c["note"]


@pytest.mark.parametrize("net", ["hash_signed", "hash_pos"])
def test_tree_many_positions_vs_oracle(net, O, R):
    boards, sides = _random_positions(O, 3, 77)
    sel = np.arange(0, len(boards), max(1, len(boards) // 96))[:96]
    rng = np.random.RandomState(1)
    cases = [dict(board=boards[i], side=int(sides[i]), rr=int(rng.choice([0, 5, 56, 58])), playouts=int(rng.choice([50, 150, 250])))
             for i in sel if (boards[i] == 1).any() and (boards[i] == 8).any()]
    e = _run_cases(cases, net, R)
    cnt = e.counters()
    tot = dict(n_expand=0, n_playout=0, sum_L=0, sum_c=0)
    for g, c in enumerate(cases):
        t = O.Tree(c["board"])
        assert t.search(c["side"], c["rr"], c["playouts"], net) == 0
        assert np.array_equal(t.signature(), e.tree_signature(g)), g
        s = t.stats()
        for k in tot:
            tot[k] += s[k]
    for k in tot:
        assert cnt[k] == tot[k], k


def _golden_selfplay_games(net):
    return [g for g in load_golden("selfplay.json")["games"] if g["net"] == net]


@pytest.mark.parametrize("net", ["hash_pos", "hash_signed", "mod17"])
def test_selfplay_tuples_against_reference_vectors(net, R):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    games = _golden_selfplay_games(net)
    sp = SelfPlay(len(games), FakeNet(net), [g["playouts"] for g in games], seeds=[g["seed"] for g in games],
                  arena_words=1 << 20, auto_reset=False)
    out = sp.play_games()
    assert len(out) == len(games)
    for (slot, rec), g in zip(out, games):
        assert len(rec) == g["n"]
        assert rec.states == g["states"]
        assert [float(z) for z in rec.z] == g["z"]
        pis = rec.dense_pi()
        assert sha(pis.tobytes()) == g["sha_pi"]
        for p, spv in zip(pis, g["pi_sparse"]):
            assert [[int(k), float(p[k]).hex()] for k in np.nonzero(p)[0]] == spv


@pytest.mark.parametrize("graph", [False, True])
def test_selfplay_many_games_vs_oracle(graph, O, R):
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    B, playouts, net = 48, 40, "hash_pos"
    sp = SelfPlay(B, FakeNet(net), playouts, seeds=[1000 + i for i in range(B)], arena_words=1 << 20, auto_reset=False)
    if graph:
        sp.capture_graph()
    out = sp.play_games()
    assert len(out) == B
    for slot, rec in out:
        with np.errstate(all="ignore"):
            r = O.selfplay_game(net, playouts, np.random.RandomState(1000 + slot))
        assert rec.states == r["states"], slot
        assert np.array_equal(rec.z, r["z"])
        assert np.array_equal(rec.dense_pi(), r["pis"])
        assert rec.actions == r["actions"]


def test_full_size_1024_games_1200_playouts_properties_and_samples(O, R):
    """BASELINE configs[1] size (1024 games x 1200 playouts).  Size-independent properties on every game, bit-exact
    comparison with the oracle on a sample of games, determinism (duplicate seeds -> identical trees)."""
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net = 1024, 1200, "hash_pos"
    seeds = [9000 + (g % 512) for g in range(B)]          # game g and g+512 share a seed
    sp = SelfPlay(B, FakeNet(net), P, seeds=seeds, auto_reset=False)
    sp.capture_graph()
    e = sp.engine
    # ply 1
    sp.search()
    rc1 = e.root_children()
    assert (rc1["n"] == 44).all()                                     # 44 pseudo-legal moves at the start position
    assert (rc1["visits"].sum(axis=1) == P).all()                     # root.N is never incremented, every playout passes a child
    sig0 = e.tree_signature(0)
    for g in (1, 511, 512, 1023):
        assert np.array_equal(e.tree_signature(g), sig0)              # same position, same net -> same tree, any slot
    t = O.Tree()
    assert t.search(0, 0, P, net) == 0
    assert np.array_equal(t.signature(), sig0)                        # ... and it is the oracle's tree, bit for bit
    # step() = search + host move choice; the search is done, choose the moves by hand (any legal child will do)
    choice = np.array([int(np.random.RandomState(s).randint(44)) for s in seeds], dtype=np.int32)
    N_chosen = rc1["visits"][np.arange(B), choice]
    st_play = e.play(choice)
    # ply 2 (tree re-use): children of the new root keep their statistics, then P more playouts are added
    st_read = e.status()
    for k in ("boards", "side", "terminal", "winner", "ply", "rr"):
        assert np.array_equal(st_play[k], st_read[k]), k               # play() returns the status a separate read would give
    assert np.array_equal(st_play["q"], rc1["q"][np.arange(B), choice]) and np.array_equal(st_play["root_N"], N_chosen)
    sp.boards, sp.sides = st_read["boards"], st_read["side"]
    sp.search()
    rc2 = e.root_children()
    tot = np.array([rc2["visits"][g, : rc2["n"][g]].sum() for g in range(B)])
    expect = np.where(N_chosen > 0, N_chosen - 1 + P, P)              # first visit of a node expands it, the rest descend
    assert np.array_equal(tot, expect)
    for g in range(0, 512, 37):
        assert choice[g] == choice[g + 512]
        assert np.array_equal(e.tree_signature(g), e.tree_signature(g + 512))
    for g in (3, 77, 300):                                            # oracle replay of the same two plies
        t = O.Tree()
        t.search(0, 0, P, net)
        t.update(int(choice[g]))
        b, cap = O.apply_move(O.from_state(O.START), int(rc1["moves"][g, choice[g]]))
        assert np.array_equal(t.root_board(), b)
        t.search(1, 1 if cap == 0 else 0, P, net)
        assert np.array_equal(t.signature(), e.tree_signature(g)), g
    c = e.raise_on_error()
    assert c["n_playout"] == 2 * B * P


def test_edge_cases_empty_batches_bad_arguments_and_loud_failures(R):
    import ctypes as C
    from cchess_zero_b200._lib import EngineError, lib
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.fakenet import FakeNet
    L = lib()
    # empty batches are fine
    mv, cnt = R.legal_moves_batch(np.zeros((0, 90), np.uint8), np.zeros(0, np.uint8))
    assert mv.shape == (0, 128) and cnt.shape == (0,)
    assert R.encode_batch(np.zeros((0, 90), np.uint8), np.zeros(0, np.uint8)).shape == (0, 9, 10, 14)
    # bad arguments return error codes with a message, never crash
    assert L.cz_legal_moves_batch(0, None, None, 3, None, None) < 0 and b"null" in L.cz_last_error()
    assert L.cz_label_index(-1, 200) == -1
    with pytest.raises(EngineError):
        R.state_to_board("9/9")
    h = C.c_void_p()
    assert L.cz_engine_create(0, 0, 0, C.byref(h)) < 0
    assert L.cz_engine_create(4, 100, 0, C.byref(h)) < 0            # arena too small to be meaningful
    # an empty board (no kings, no pieces): zero moves -> the engine flags it instead of hanging (reference: ValueError)
    e = Engine(2, arena_words=1 << 16)
    boards = np.zeros((2, 90), np.uint8)
    boards[1] = R.state_to_board(R.START_STATE)
    e.reset(None, boards, [0, 0], [0, 0])
    fn = FakeNet("hash_pos")
    nn_in = torch.zeros((2, 9, 10, 14), device="cuda"); lo = torch.zeros((2, 2086), device="cuda"); v = torch.zeros(2, device="cuda")

    def fwd(x):
        l, val = fn(x); lo.copy_(l); v.copy_(val)
    e.search(fwd, 20, nn_in, lo, v)
    with pytest.raises(EngineError, match="NOMOVES"):
        e.raise_on_error()
    assert e.counters()["first_error_game"] == 0
    # arena exhaustion is reported loudly, not silently truncated
    e2 = Engine(1, arena_words=4096)
    nn1 = torch.zeros((1, 9, 10, 14), device="cuda"); lo1 = torch.zeros((1, 2086), device="cuda"); v1 = torch.zeros(1, device="cuda")

    def fwd1(x):
        l, val = fn(x); lo1.copy_(l); v1.copy_(val)
    e2.search(fwd1, 400, nn1, lo1, v1)
    with pytest.raises(EngineError, match="ARENA"):
        e2.raise_on_error()


def test_selfplay_full_game_at_1200_playouts_against_reference_vectors(R):
    """A whole game at the BASELINE playout count, bit-exact against the reference's own (s, pi, z) output."""
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    g = load_golden("selfplay_1200.json")["games"][0]
    sp = SelfPlay(4, FakeNet(g["net"]), g["playouts"], seeds=[g["seed"]] * 4, auto_reset=False)
    sp.capture_graph()
    out = sp.play_games()
    for slot, rec in out:
        assert len(rec) == g["n"] and rec.states == g["states"]
        assert [float(z) for z in rec.z] == g["z"]
        assert sha(rec.dense_pi().tobytes()) == g["sha_pi"]


def _check_tree_invariants(sig):
    """sig: DFS records (label, N, Wbits, Pbits, Qbits, n_children).  For every expanded node entered through an edge with N
    visits: the first visit expanded it, every later visit went on to one child -> sum(children N) == N - 1; no leftover
    virtual loss anywhere (it would break the identity by multiples of 3)."""
    pos = 0

    def node(n_children):
        nonlocal pos
        tot = 0
        for _ in range(n_children):
            lab, N, _, _, _, nc = sig[pos]
            pos += 1
            tot += int(N)
            if nc > 0:
                s = node(int(nc))
                assert s == int(N) - 1, (lab, N, s)
        return tot

    # root: find its child count = number of top-level records
    top = 0
    i = 0
    def skip(i):
        nc = int(sig[i][5]); i += 1
        for _ in range(nc):
            i = skip(i)
        return i
    while i < len(sig):
        i = skip(i); top += 1
    return node(top)


def test_leaf_parallel_kernel_with_one_slot_equals_reference_vectors(R):
    """k_wave_multi with K = 1 must be the one-leaf kernel: same golden trees of the reference, bit for bit."""
    for net in ("hash_pos", "hash_signed", "mod17"):
        cases = [c for c in load_golden("tree.json")["cases"] if c["net"] == net and c["playouts"] <= 600]
        e = _run_cases([dict(board=R.state_to_board(c["state"]), side=0 if c["player"] == "w" else 1, rr=c["rr"],
                             playouts=c["playouts"]) for c in cases], net, R, leaves=-1)
        for g, c in enumerate(cases):
            assert sha(e.tree_signature(g).tobytes()) == c["sha_sig"], c["note"]


@pytest.mark.parametrize("K", [4, 16])
def test_leaf_parallel_search_conserves_visits_and_is_deterministic(K, O, R):
    boards, sides = _random_positions(O, 2, 31)
    sel = [i for i in range(0, len(boards), 9) if (boards[i] == 1).any() and (boards[i] == 8).any()][:24]
    cases = [dict(board=boards[i], side=int(sides[i]), rr=int(i % 50), playouts=300) for i in sel]
    sigs = []
    for rep in range(2):
        e = _run_cases(cases, "hash_pos", R, leaves=K)
        rc = e.root_children()
        for g in range(len(cases)):
            sig = e.tree_signature(g)
            assert rc["visits"][g, : rc["n"][g]].sum() == 300              # every playout passes exactly one root child
            assert _check_tree_invariants(sig) == 300
            if rep == 0:
                sigs.append(sig)
            else:
                assert np.array_equal(sig, sigs[g])                         # deterministic schedule
        c = e.counters()
        assert c["n_playout"] == 300 * len(cases)


@pytest.mark.parametrize("K", [2, 4, 16])
def test_leaf_parallel_kernel_equals_its_serial_specification(K, O, R):
    """k_wave_multi against oracle co_tree_search_multi (an independent serial implementation of the same schedule):
    full trees bit for bit, over positions with captures, draws and king captures in reach."""
    boards, sides = _random_positions(O, 3, 57)
    sel = [i for i in range(0, len(boards), 7) if (boards[i] == 1).any() and (boards[i] == 8).any()][:40]
    rng = np.random.RandomState(K)
    cases = [dict(board=boards[i], side=int(sides[i]), rr=int(rng.choice([0, 7, 55, 58])), playouts=int(rng.choice([100, 260, 400]))) for i in sel]
    for net in ("hash_pos", "hash_signed"):
        e = _run_cases(cases, net, R, leaves=K)
        for g, c in enumerate(cases):
            t = O.Tree(c["board"])
            assert t.search_multi(c["side"], c["rr"], c["playouts"], K, net) == 0
            assert np.array_equal(t.signature(), e.tree_signature(g)), (net, K, g)


def test_rules_flip_symmetry_on_a_quarter_million_positions(R):
    """Size-independent property of the CUDA rules at scale, no oracle involved: for every position reached by 4096 random
    games, moves(flip(board), other side) is the rank mirror of moves(board, side) as a set, encode(board, 'b') equals
    encode(flip(board), 'w'), and a move and its mirror capture alike."""
    from cchess_zero_b200.selfplay import _flip_board
    G, plies = 4096, 60
    rng = np.random.RandomState(2)
    boards = np.tile(R.state_to_board(R.START_STATE), (G, 1))
    sides = np.zeros(G, dtype=np.uint8)
    n_checked = 0

    def mirror(mv):
        s, d = mv & 127, mv >> 7
        return (((9 - s // 9) * 9 + s % 9) | (((9 - d // 9) * 9 + d % 9) << 7)).astype(np.uint16)

    def flip_all(b):
        f = b.reshape(-1, 10, 9)[:, ::-1, :].copy()
        red, blk = (f >= 1) & (f <= 7), f >= 8
        f[red] += 7; f[blk] -= 7
        return f.reshape(-1, 90)

    for ply in range(plies):
        mv, cnt = R.legal_moves_batch(boards, sides)
        fb = flip_all(boards)
        assert np.array_equal(fb[:3], np.stack([_flip_board(b) for b in boards[:3]]))
        fmv, fcnt = R.legal_moves_batch(fb, sides ^ 1)
        assert np.array_equal(cnt, fcnt)
        valid = np.arange(128)[None, :] < cnt[:, None]
        a = np.where(valid, mirror(mv), 0xFFFF); b = np.where(valid, fmv, 0xFFFF)
        assert np.array_equal(np.sort(a, axis=1), np.sort(b, axis=1))
        if ply % 10 == 0:
            black = sides == 1
            if black.any():
                assert np.array_equal(R.encode_batch(boards[black], sides[black]), R.encode_batch(fb[black], sides[black] ^ 1))
        n_checked += G
        pick = (rng.rand(G) * np.maximum(cnt, 1)).astype(np.int64)
        chosen = mv[np.arange(G), pick]
        nb, cap = R.apply_moves_batch(boards, chosen)
        nfb, fcap = R.apply_moves_batch(fb, mirror(chosen))
        assert np.array_equal(flip_all(nb), nfb) and np.array_equal(cap == 0, fcap == 0)
        dead = (cap == 1) | (cap == 8) | (cnt == 0)
        boards, sides = nb, sides ^ 1
        boards[dead] = R.state_to_board(R.START_STATE); sides[dead] = 0
    assert n_checked == G * plies


def test_board_hashing_keys_are_incremental_zobrist_and_never_touch_the_search(O, R):
    """north_star "board hashing": the engine maintains a 64-bit Zobrist key per root (updated by every played move) and per
    pending leaf (updated along the descent).  (1) the incrementally maintained root key equals the key computed from scratch
    for the same position and side to move; (2) equal positions <=> equal keys across games; (3) hashing on / off gives the
    same trees bit for bit; (4) leaf keys of games that evaluate the same position coincide, different positions differ."""
    from cchess_zero_b200.engine import Engine
    from cchess_zero_b200.fakenet import FakeNet
    from cchess_zero_b200.selfplay import SelfPlay
    B, P, net = 64, 24, "hash_pos"
    seeds = [7 + (i % 16) for i in range(B)]                         # 16 distinct games, each played 4 times
    sp = SelfPlay(B, FakeNet(net), P, seeds=seeds, arena_words=1 << 18, auto_reset=False, hashing=True)
    sp0 = SelfPlay(B, FakeNet(net), P, seeds=seeds, arena_words=1 << 18, auto_reset=False)
    for _ in range(6):
        sp.step(); sp0.step()
    for g in (0, 5, 17, 63):
        assert np.array_equal(sp.engine.tree_signature(g), sp0.engine.tree_signature(g))          # (3)
    keys = sp.engine.root_keys()
    st = sp.engine.status()
    e2 = Engine(B, 1 << 12)
    e2.reset(None, st["boards"], st["side"], st["rr"])
    assert np.array_equal(e2.root_keys(), keys)                                                    # (1)
    by_pos = {}
    for g in range(B):
        by_pos.setdefault((st["boards"][g].tobytes(), int(st["side"][g])), set()).add(int(keys[g]))
    assert all(len(v) == 1 for v in by_pos.values()) and len({next(iter(v)) for v in by_pos.values()}) == len(by_pos)   # (2)
    assert len(by_pos) >= 8
    # (4) one wave of the next search: rows of replicated games carry identical leaf keys
    sp.engine.begin_search(P)
    sp.engine.wave(sp.nn_in, sp.logits, sp.value)
    sp._eval(sp.nn_in)
    sp.engine.wave(sp.nn_in, sp.logits, sp.value)
    lk = sp.engine.leaf_hashes().cpu().numpy()
    assert (lk != 0).any()
    for g in range(16):
        assert len({int(lk[g + 16 * r]) for r in range(4)}) == 1
    e2.close()
