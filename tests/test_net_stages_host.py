"""CPU tier of tests/net_stages.py, the float64 statement of the hand-written network kernels: chained with rounding off, its stages are
the reference network (oracle/net_numpy.py, TF conventions), and its un-layout helpers invert the kernel layouts net.py builds."""
import types

import numpy as np
import pytest
import torch

import net_stages as S


def _positions(n, seed):
    """Random-play positions of both sides: (boards [n][90] as stored, sides, side-to-move canonical boards u8 [n][96])."""
    from oracle import oracle as O
    rng = np.random.RandomState(seed)
    boards, sides, canon = [], [], []
    b, side = O.from_state(O.START), 0
    while len(boards) < n:
        c = np.zeros(96, np.uint8)
        c[:90] = O.flip_board(b) if side == 1 else b
        boards.append(b.copy()); sides.append(side); canon.append(c)
        mv = O.legal_moves(b, side)
        b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
        if cap in (1, 8):
            b, side = O.from_state(O.START), 0
    return boards, sides, np.stack(canon)


def _folded(p, conv, bn):
    """BN folded into a TF kernel / bias: k * s, (b - mean) * s with s = 1 / sqrt(var + 1e-5)."""
    s = 1.0 / np.sqrt(p[bn + ".var"] + 1e-5)
    return p[conv + ".k"] * s, (p[conv + ".b"] - p[bn + ".mean"]) * s


@pytest.mark.parametrize("blocks", [1, 2, 3])
def test_stages_chained_are_the_reference_network(blocks):
    """first_conv -> blocks -> head_conv -> policy_fc / value_mlp with rounding off == net_numpy.forward(O.encode(board, side)) to 1e-10,
    with non-trivial biases and BN statistics: pins the board-byte -> image mapping and the flatten order of the reference itself."""
    from oracle import net_numpy as N
    from oracle import oracle as O
    from cchess_zero_b200.net import PolicyValueNet
    torch.manual_seed(blocks)
    net = PolicyValueNet(blocks).eval()
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                m.bias.uniform_(-0.3, 0.3)
            if hasattr(m, "running_var"):
                m.running_var.uniform_(0.5, 1.5); m.running_mean.uniform_(-0.2, 0.2)
        net.p_fc.weight.mul_(30.0)                                           # logits of a trained network's size
    p = N.tf_params_from_torch(net.double())
    boards, sides, canon = _positions(40, seed=blocks)
    x = np.stack([O.encode(b, s) for b, s in zip(boards, sides)]).astype(np.float64)
    assert np.array_equal(S.image(canon), x)                                 # the kernels' board reading is the engine's encoding
    rl, rv = N.forward(x, p, blocks)
    k_in, b_in = _folded(p, "conv_in", "bn_in")
    convs, biases = [], [b_in]
    for i in range(blocks):
        for c, b in (("c1", "b1"), ("c2", "b2")):
            k, bb = _folded(p, "b%d.%s" % (i, c), "b%d.%s" % (i, b))
            convs.append(k); biases.append(bb)
    kp, bp = _folded(p, "p_conv", "p_bn")
    kv, bv = _folded(p, "v_conv", "v_bn")
    wh = np.concatenate([kp.reshape(128, 2), kv.reshape(128, 1)], 1).T       # [3][128]
    bh = np.concatenate([bp, bv])
    v0, _ = S.first_conv(canon, k_in.reshape(9, 14, 128), b_in)
    hp, hv, trunk = S.tower(canon, k_in.reshape(9, 14, 128), convs, biases, wh, bh, round16=False)
    assert trunk.shape == (40, 90, 128) and np.abs(v0 - S.tower(canon, k_in.reshape(9, 14, 128), [], biases[:1], wh, bh, False)[2]).max() == 0
    logits = S.policy_fc(hp, p["p_fc.w"].T, p["p_fc.b"])
    value, _, _ = S.value_mlp(hv, p["v_fc1.w"], p["v_fc1.b"], p["v_fc2.w"], p["v_fc2.b"])
    assert np.abs(rl).max() > 1.0
    assert np.abs(logits - rl).max() < 1e-10 and np.abs(value - rv.reshape(-1)).max() < 1e-10
    assert not hp[:, 180:].any()


def test_rounding_helpers():
    assert S.ulp16(1.0) == 2.0 ** -10 and S.ulp16(0.0) == 2.0 ** -24 and S.ulp16(-3.0) == 2.0 ** -9
    assert S.r16(1.0 + 2.0 ** -11) == 1.0 and S.r16(1.0 + 3 * 2.0 ** -11) == 1.0 + 2.0 ** -9      # ties to even, from float64
    assert S.r16(1.0 + 2.0 ** -11 + 2.0 ** -40) == 1.0 + 2.0 ** -10                                 # no double rounding
    assert np.isnan(S.head_conv(np.full((1, 90, 128), np.nan), np.ones((3, 128)), np.zeros(3))[1]).all()   # NaN is not clipped


def _coded(shape, part):
    """Distinct values for a layout test that survive fp16: entry i holds (i + 1) % 2048 (part 0) or (i + 1) // 2048 (part 1), both
    exact in fp16, so that part1 * 2048 + part0 recovers i + 1 (0 only where a layout puts padding)."""
    i = torch.arange(1, int(np.prod(shape)) + 1, dtype=torch.int64).reshape(shape)
    return (i % 2048 if part == 0 else i // 2048).float()


def _decode(parts):
    return parts[1].astype(np.int64) * 2048 + parts[0].astype(np.int64)


def test_unlayout_inverts_the_native_plan_layouts():
    """NativePlan._derive's wgmma tiles of the policy FC weights (and its w1 / policy FC copies) on CPU tensors with distinct values:
    unlayout_wp_tiled gives back the [2112][192] zero-padded, label-major weights, element for element."""
    from cchess_zero_b200.net import NativePlan, PolicyValueNet
    net = PolicyValueNet(1).eval()
    got = {}
    for part in (0, 1):
        with torch.no_grad():
            net.p_fc.weight.copy_(_coded((2086, 180), part))
        w_in = _coded((128, 14, 3, 3), part).half()
        base = types.SimpleNamespace(w_in=(w_in, torch.zeros(128)), w_head=(torch.zeros(3, 128, 1, 1).half(), torch.zeros(3).half()))
        d = NativePlan._derive(types.SimpleNamespace(net=net, _base=base))
        for k in ("wp_tiled", "wp", "w1"):
            got.setdefault(k, []).append(d[k].float().numpy())
        assert d["bp_pad"].shape == (2176,) and d["wp_tiled"].shape == (17, 24, 128, 8)
    idx = np.arange(1, 2086 * 180 + 1).reshape(2086, 180)
    want = np.zeros((2176, 192), np.int64)
    want[:2086, :180] = idx
    assert np.array_equal(_decode([S.unlayout_wp_tiled(g) for g in got["wp_tiled"]]), want)
    assert np.array_equal(_decode(got["wp"]), want[:2112])
    # w1 [9 taps][14 pieces][128]: the TF kernel [kh][kw][cin][cout] of the torch weight [cout][cin][kh][kw]
    w = np.arange(1, 128 * 14 * 9 + 1).reshape(128, 14, 3, 3)
    assert np.array_equal(_decode(got["w1"]), w.transpose(2, 3, 1, 0).reshape(9, 14, 128))


@pytest.mark.parametrize("blocks", [1, 2])
def test_unlayout_inverts_the_small_tower_blob(blocks):
    """SmallTowerPlan._derive's TMA weight blob [conv][tap][rank][k-chunk][32][8] on CPU tensors with distinct values:
    unlayout_tower_blob gives back every convolution as a TF kernel [3][3][cin][cout], in execution order."""
    from cchess_zero_b200.net import PolicyValueNet, SmallTowerPlan
    net = PolicyValueNet(1).eval()
    n_conv = 2 * blocks
    got, bias = [], None
    for part in (0, 1):
        ws = _coded((n_conv, 128, 128, 3, 3), part).half()
        bs = torch.arange(n_conv * 128, dtype=torch.float32).reshape(n_conv, 128)
        blocks_ = [((ws[2 * i], bs[2 * i]), (ws[2 * i + 1], bs[2 * i + 1])) for i in range(blocks)]
        base = types.SimpleNamespace(w_in=(torch.zeros(128, 14, 3, 3).half(), -torch.ones(128)), blocks=blocks_,
                                     w_head=(torch.zeros(3, 128, 1, 1).half(), torch.zeros(3).half()))
        d = SmallTowerPlan._derive(types.SimpleNamespace(net=net, _base=base, CL=4))
        assert d["blob"].dtype == torch.float16 and d["blob"].numel() * 2 == n_conv * 9 * 128 * 256
        got.append(S.unlayout_tower_blob(d["blob"].float().numpy()))
        bias = d["bias"].numpy()
    w = np.arange(1, n_conv * 128 * 128 * 9 + 1).reshape(n_conv, 128, 128, 3, 3)      # [conv][cout][cin][kh][kw]
    assert np.array_equal(_decode(got), w.transpose(0, 3, 4, 2, 1))
    assert np.array_equal(bias, np.concatenate([-np.ones((1, 128)), np.arange(n_conv * 128).reshape(n_conv, 128)]))


def test_unlayout_inverts_the_tiled_head_features():
    """k_head_conv_mma<true> writes feature k of position pos at ((pos >> 7) * 24 + (k >> 3)) * 1024 + (pos & 127) * 8 + (k & 7)
    (halves); unlayout_hp_tiled reads that address formula back into [tiles * 128][192]."""
    B = 300
    tiles = (B + 127) // 128
    hp = np.arange(1, B * 192 + 1).reshape(B, 192)
    flat = np.zeros(tiles * 24 * 128 * 8, np.int64)
    pos, k = np.meshgrid(np.arange(B), np.arange(192), indexing="ij")
    flat[((pos >> 7) * 24 + (k >> 3)) * 1024 + (pos & 127) * 8 + (k & 7)] = hp
    back = S.unlayout_hp_tiled(flat.reshape(tiles, 24, 128, 8))
    assert np.array_equal(back[:B], hp) and not back[B:].any()


def test_image_reads_byte_r9_plus_f_and_never_82_to_95():
    b = np.zeros((2, 96), np.uint8)
    b[0, 81] = 14                                # cell (8, 9): the last byte read
    b[1, 82:] = 7                                # never read
    b[1, 9] = 3                                  # byte 9 is cell (0, 9) and cell (1, 0): the reference's quirk
    x = S.image(b)
    assert x[0, 8, 9, 13] == 1 and x[0].sum() == 1
    assert x[1].sum() == 2 and x[1, 0, 9, 2] == 1 and x[1, 1, 0, 2] == 1
