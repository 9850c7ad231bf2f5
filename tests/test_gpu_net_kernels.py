"""Each hand-written network kernel (csrc/cz_net.cu, csrc/cz_tower.cu) against tests/net_stages.py, the float64 statement of its own
arithmetic, called through its C entry point with the weights the plans derive.  Every output and scratch buffer carries canary
rows filled with a sentinel bit pattern: no row at or beyond the batch may be written.

Bounds are derived from the arithmetic, u = 2^-24 (f32 unit roundoff):
  * an f32 accumulation of n terms:  c * n * u * sum|terms|, c = 1 for round-to-nearest sums on the CUDA cores, c = 2 for the
    tensor cores, whose accumulator truncates (the project documents about -6.6e-9 relative per term, under one u; c = 2 allows a
    full f32 ulp per addition).  fp16 x fp16 products are exact in f32; an f32 product on the CUDA cores adds one rounding (c = 2
    for those sums, the library is built with --fmad=false);
  * an fp16 store: one fp16 ulp of the reference value on top.
Inputs are chosen so that each plausible kernel error (a dropped MMA, k-chunk, tap, skip or weight residue) misses its bound by
at least 10x; the tests print each stage's measured error next to its bound."""
import ctypes as C

import numpy as np
import pytest
import torch

import net_stages as S

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SENT16, SENT32 = 0x7E5A, 0x7FA5A5A5       # fp16 / f32 NaNs with a payload no kernel produces
EXTRA = 3                                 # canary rows beyond the batch


def _lib():
    from cchess_zero_b200._lib import lib
    return lib()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _canary(rows, *shape, dtype=torch.float32):
    """A device buffer of rows + EXTRA rows filled with the sentinel bit pattern."""
    if dtype == torch.float16:
        return torch.full((rows + EXTRA,) + shape, SENT16, dtype=torch.int16, device="cuda").view(torch.float16)
    return torch.full((rows + EXTRA,) + shape, SENT32, dtype=torch.int32, device="cuda").view(torch.float32)


def _untouched(t, B):
    """Rows >= B of a canary buffer still hold the sentinel."""
    bits = t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)[B:]
    return bool((bits == (SENT16 if t.dtype == torch.float16 else SENT32)).all())


def _np(t):
    return t.detach().float().cpu().numpy().astype(np.float64)


def _report(name, err, bound):
    """Largest error / bound ratio of a stage (NaN-free inputs), printed and returned."""
    r = float(np.max(err / bound)) if np.size(err) else 0.0
    print("%-44s max err %.3e  max bound %.3e  max err/bound %.3f" % (name, float(np.max(err)), float(np.max(bound)), r))
    return r


def _net(blocks, seed, exact_bn=False):
    """A network on the device with non-trivial biases and BN statistics; with exact_bn the BN folding is the identity (mean 0,
    var 1, eps 0), so that designed weights reach the plans unchanged."""
    from cchess_zero_b200.net import PolicyValueNet
    torch.manual_seed(seed)
    net = PolicyValueNet(blocks).eval()
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)):
                m.bias.uniform_(-0.2, 0.2)
            if hasattr(m, "running_var"):
                if exact_bn:
                    m.eps = 0.0
                else:
                    m.running_var.uniform_(0.5, 1.5); m.running_mean.uniform_(-0.2, 0.2)
        net.p_fc.bias.copy_(torch.arange(2086, dtype=torch.float32) * 2.0 ** -7 - 8.0)     # a distinct bias per label
        net.p_fc.weight.mul_(20.0)
    return net.cuda().to(memory_format=torch.channels_last)


def _boards(B, seed):
    """Random byte boards, codes 0..14 at every cell; row 0 empty and row 1 full when B > 2; bytes 82..95 hold piece codes
    (valid, so that a read of them would change the output without leaving the weight table) that must never be read."""
    rng = np.random.RandomState(seed)
    b = rng.randint(0, 15, (B, 96)).astype(np.uint8)
    if B >= 2:
        b[0, :82] = 0
        b[1, :82] = rng.randint(1, 15, 82)
    b[:, 82:] = rng.randint(1, 15, (B, 14))
    return b


# ---------------------------------------------------------------------------------------------------------------------------------
# k_first_conv
# ---------------------------------------------------------------------------------------------------------------------------------

def _first_conv(boards, w1, b1):
    B = len(boards)
    out = _canary(B, 90, 128, dtype=torch.float16)
    assert _lib().cz_net_first_conv(torch.from_numpy(boards).cuda().data_ptr(), B, w1.data_ptr(), b1.data_ptr(), out.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    assert _untouched(out, B)
    return out[:B]


@pytest.mark.parametrize("B", [1, 2, 7, 203, 1024])
def test_first_conv_against_fp64(B):
    """fp16 output within one fp16 ulp of fp16(fp64 sum) for the folded weights of a plan, and bit for bit with dyadic weights
    (multiples of 2^-8 below 1: every f32 partial sum is exact).  Skipping a tap or misreading a byte moves an output by a whole
    weight row, thousands of ulps."""
    from cchess_zero_b200.net import NativePlan
    boards = _boards(B, seed=B)
    net = _net(1, seed=B)
    plan = NativePlan(net, B)
    got = _np(_first_conv(boards, plan.w1, plan.b1))
    v, v16 = S.first_conv(boards, _np(plan.w1).reshape(9, 14, 128), _np(plan.b1))
    assert np.abs(v).max() > 0.5 and (v == 0).any()
    _report("first_conv B=%d |k - fp16(fp64)| / ulp" % B, np.abs(got - v16), S.ulp16(v16))
    assert (np.abs(got - v16) <= S.ulp16(v16)).all()
    rng = np.random.RandomState(7)
    w1 = torch.from_numpy(rng.randint(-255, 256, (9, 14, 128)) / 256.0).half().cuda()
    b1 = torch.from_numpy(rng.randint(-255, 256, 128) / 256.0).float().cuda()
    got = _first_conv(boards, w1, b1)
    _, v16 = S.first_conv(boards, _np(w1).reshape(9, 14, 128), _np(b1))
    assert np.array_equal(_np(got), v16)
    if B >= 2:
        assert np.array_equal(_np(got[0]), S.r16(np.maximum(np.broadcast_to(_np(b1), (90, 128)), 0)))    # empty board: fp16(relu(b1))


def test_first_conv_nan_weight_row_reaches_only_positions_with_that_piece():
    """A NaN row of w1 for piece code 5 (every tap) makes NaN exactly the cells whose 3x3 neighbourhood holds a 5, and leaves every
    other cell and position bit-identical (the gather-add never touches the rows of absent pieces).  fmaxf-ReLU kernels clip it to 0."""
    B = 64
    boards = _boards(B, seed=11)
    boards[: B // 2, :82][boards[: B // 2, :82] == 5] = 6                      # first half: no piece 5
    boards[B // 2:, 40] = 5                                                    # second half: at least one
    rng = np.random.RandomState(3)
    w1 = torch.from_numpy(rng.randn(9, 14, 128) * 0.3).half().cuda()
    b1 = torch.from_numpy(rng.randn(128) * 0.1).float().cuda()
    clean = _first_conv(boards, w1, b1).clone()
    w1[:, 4, :] = float("nan")
    got = _first_conv(boards, w1, b1)
    img = S.image(boards)[..., 4]                                              # [B][9][10]: piece 5 present
    pad = np.pad(img, ((0, 0), (1, 1), (1, 1)))
    near = sum(pad[:, i:i + 9, j:j + 10] for i in range(3) for j in range(3)).reshape(B, 90) > 0
    nan = torch.isnan(got).cpu().numpy()
    assert near[B // 2:].any(axis=1).all() and not near[: B // 2].any()
    assert np.array_equal(nan.all(axis=2), near) and np.array_equal(nan.any(axis=2), near)
    keep = torch.from_numpy(~near).cuda()
    assert torch.equal(got[keep].view(torch.int16), clean[keep].view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------------------
# heads: k_head_conv_mma<false / true>, k_value_mlp, k_policy_fc, k_policy_fc_tc
# ---------------------------------------------------------------------------------------------------------------------------------

def _head_weights(seed):
    """f32 head weights whose residue below fp16 is large and of one sign: w = h + (7/16) ulp16(h), h an fp16 value just above a
    power of two, so that hi = fp16(w) = h and lo = w - h is exact in fp16 and ~4.2e-4 of w.  The value channel is positive; a
    kernel that drops the lo half errs by ~4.2e-4 of the sum of |terms|, coherently.  bh is dyadic."""
    rng = np.random.RandomState(seed)
    h = (1.0 + rng.randint(0, 16, (3, 128)) / 1024.0) * 2.0 ** rng.randint(-6, -1, (3, 128))
    h[:2] *= rng.choice([-1.0, 1.0], (2, 128))
    w = h + np.sign(h) * (7.0 / 16.0) * S.ulp16(h)
    assert np.array_equal(S.r16(w), h)
    bh = np.array([0.25, -0.125, 2.0 ** -6])
    return torch.from_numpy(w).float().cuda(), torch.from_numpy(bh).float().cuda()


def _trunk_out(B, seed):
    """Head-conv input x fp16 [B][90][128]: positive, channel scales spread over four decades (a channel or cell off by one is
    large), every fifth cell negated so that its head sums are negative and the ReLU clips them; cells 88, 89 (features
    176..179, the last k-chunk of the policy FC) are not small."""
    rng = np.random.RandomState(seed)
    scale = 10.0 ** np.linspace(-2.5, 1.5, 128)[rng.permutation(128)]
    x = rng.uniform(0.5, 1.5, (B, 90, 128)) * scale
    x[:, ::5] *= -1.0
    x[:, 88:] *= 3.0
    return torch.from_numpy(x).half().cuda()


def _head_bounds(x, wh, bh):
    """(reference hp [B][192], hv [B][90], bound hp, bound hv): tensor-core sums of 2 x 128 exact products + the bias (c = 2,
    n = 257), then the fp16 store of hp (+ one ulp)."""
    hp, hv = S.head_conv(x, wh, bh)
    t = np.abs(x) @ np.abs(wh).T + np.abs(bh)                                # [B][90][3]
    acc = 2 * 257 * U * t
    bhp = np.zeros_like(hp)
    bhp[:, :180] = acc[..., :2].reshape(len(x), 180)
    return hp, hv, bhp + S.ulp16(hp), acc[..., 2]


def _fc_bound(hp, wp, bp):
    """Policy FC: 192 exact fp16 products accumulated on the tensor cores, + the bias (c = 2, n = 193)."""
    return 2 * 193 * U * (np.abs(hp[:, :180]) @ np.abs(wp[:2086, :180]).T + np.abs(bp[:2086]))


def _value_bound(hv, w1t, b1, w2, b2):
    """k_value_mlp: hidden h_j = b1_j + sum_k w1t[k][j] hv[k] (90 f32 products + 91 sums, c = 2, n = 91); z = b2 + sum_j w2_j relu(h_j)
    by a per-term product, a 5-level shuffle tree, an 8-way sum and the bias (each term sees <= 15 roundings: c = 2, n = 15), carrying
    the hidden errors through |w2|; tanhf adds 2 f32 ulps and has slope <= 1."""
    v, z, h = S.value_mlp(hv, w1t, b1, w2, b2)
    eh = 2 * 91 * U * (np.abs(hv[:, :90]) @ np.abs(w1t) + np.abs(b1))
    ez = eh @ np.abs(w2) + 2 * 15 * U * ((np.maximum(h, 0) + eh) @ np.abs(w2) + abs(float(b2)))
    return v, z, ez + 2 * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)


def _plan_fc(plan):
    return (_np(plan.wp), _np(plan.bp), _np(plan.w1t), _np(plan.bv1), _np(plan.w2), float(plan.b2t.item()))


def _heads(plan, x, wh, bh, tc, hp_buf=None):
    """One call of cz_net_heads (tc False) or cz_net_heads_tc (tc True) on canary buffers -> (hp [B][192], hv, logits, value) on the host."""
    B = x.shape[0]
    L = _lib()
    hv = _canary(B, 96)
    logits, value = _canary(B, 2086), _canary(B)
    if tc:
        tiles = (B + 127) // 128
        hp = hp_buf if hp_buf is not None else torch.full((tiles + 1, 24, 128, 8), SENT16, dtype=torch.int16, device="cuda").view(torch.float16)
        rc = L.cz_net_heads_tc(x.data_ptr(), B, wh.data_ptr(), bh.data_ptr(), plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(),
                               plan.b2t.data_ptr(), plan.wp_tiled.data_ptr(), plan.bp_pad.data_ptr(), hp.data_ptr(), hv.data_ptr(),
                               logits.data_ptr(), value.data_ptr(), _st())
    else:
        hp = _canary(B, 192, dtype=torch.float16)
        rc = L.cz_net_heads(x.data_ptr(), B, wh.data_ptr(), bh.data_ptr(), plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(),
                            plan.b2t.data_ptr(), plan.wp.data_ptr(), plan.bp.data_ptr(), hp.data_ptr(), hv.data_ptr(), logits.data_ptr(),
                            value.data_ptr(), _st())
    assert rc == 0
    torch.cuda.synchronize()
    assert _untouched(hv, B) and _untouched(logits, B) and _untouched(value, B)
    if tc:
        rows = S.unlayout_hp_tiled(hp.view(torch.int16).cpu().numpy())
        assert (rows[B:] == np.int16(SENT16)).all() if hp_buf is None else True   # positions >= B of every tile untouched
        hp_rows = torch.from_numpy(rows[:B].copy()).view(torch.float16)
    else:
        assert _untouched(hp, B)
        hp_rows = hp[:B].cpu()
    return hp_rows.double().numpy(), _np(hv[:B]), _np(logits[:B]), _np(value[:B])


def _check_heads(tag, x, wh, bh, plan, got):
    hp_k, hv_k, lo_k, v_k = got
    wp, bp, w1t, b1, w2, b2 = _plan_fc(plan)
    hp, hv, bhp, bhv = _head_bounds(_np(x), _np(wh), _np(bh))
    assert (hv[:, ::5] == 0).all() and (hv > 0).mean() > 0.7                 # clipped cells and live ones
    assert not hp_k[:, 180:].any() and not np.signbit(hp_k[:, 180:]).any()   # K padding: +0 exactly
    assert _report(tag + " head conv hv (hi+lo split)", np.abs(hv_k[:, :90] - hv), bhv) <= 1
    assert _report(tag + " head conv hp", np.abs(hp_k - hp), bhp) <= 1
    lo = S.policy_fc(hp_k, wp, bp)
    assert _report(tag + " policy FC logits", np.abs(lo_k - lo), _fc_bound(hp_k, wp, bp)) <= 1
    v, _, bv = _value_bound(hv_k, w1t, b1, w2, b2)
    assert _report(tag + " value MLP", np.abs(v_k - v), bv) <= 1


@pytest.mark.parametrize("B", [1, 2, 63, 64, 65, 127])
def test_heads_mma_against_fp64(B):
    """cz_net_heads (k_head_conv_mma<false>, k_policy_fc on mma.sync, k_value_mlp) at the 64-row tile edges of the policy FC:
    hv to the f32-weight fp64 dot product (a missing lo MMA errs by ~14x the bound), hp within one fp16 ulp, zero K padding, every
    one of the 2086 labels (distinct biases) and the value against fp64 of the kernel's own features, nothing written past B."""
    from cchess_zero_b200.net import NativePlan
    plan = NativePlan(_net(1, seed=20 + B), max(B, 8))
    x = _trunk_out(B, seed=B)
    wh, bh = _head_weights(seed=B)
    _check_heads("mma B=%d" % B, x, wh, bh, plan, _heads(plan, x, wh, bh, tc=False))


@pytest.mark.parametrize("B", [128, 129, 255, 256, 257, 1023, 1024])
def test_heads_tc_against_fp64(B):
    """cz_net_heads_tc (k_head_conv_mma<true> writing wgmma tiles, k_policy_fc_tc, k_value_mlp): the tiled features un-tiled, the
    label tile 16 with its 38 valid labels, positions >= B of every tile untouched, against fp64 like the mma.sync path."""
    from cchess_zero_b200.net import NativePlan
    plan = NativePlan(_net(1, seed=B), B)
    assert np.array_equal(S.unlayout_wp_tiled(_np(plan.wp_tiled))[:2112], _np(plan.wp))
    x = _trunk_out(B, seed=B)
    wh, bh = _head_weights(seed=B)
    _check_heads("tc B=%d" % B, x, wh, bh, plan, _heads(plan, x, wh, bh, tc=True))


def test_heads_tc_stale_rows_of_a_larger_batch_reach_no_logit():
    """The tiled feature scratch keeps rows of an earlier, larger batch: a call with B = 257 and then one with B = 129 on the same
    scratch.  The second call's logits and value equal those of a fresh scratch, bit for bit."""
    from cchess_zero_b200.net import NativePlan
    plan = NativePlan(_net(1, seed=5), 257)
    wh, bh = _head_weights(seed=5)
    x = _trunk_out(257, seed=5)
    hp = torch.zeros((4, 24, 128, 8), dtype=torch.float16, device="cuda")
    _heads(plan, x, wh, bh, tc=True, hp_buf=hp)
    stale = _heads(plan, x[128:].contiguous(), wh, bh, tc=True, hp_buf=hp)    # rows 129.. of tile 1 and tile 2 stay from the first call
    fresh = _heads(plan, x[128:].contiguous(), wh, bh, tc=True)
    for a, b in zip(stale[1:], fresh[1:]):
        assert np.array_equal(a, b, equal_nan=True)                          # hv columns 90..95 hold the (NaN) sentinel
    _check_heads("tc stale B=129", x[128:], wh, bh, plan, stale)


def _heads_fc(plan, hp, hv):
    B = hp.shape[0]
    logits, value = _canary(B, 2086), _canary(B)
    assert _lib().cz_net_heads_fc(hp.data_ptr(), hv.data_ptr(), B, plan.w1t.data_ptr(), plan.bv1.data_ptr(), plan.w2.data_ptr(), plan.b2t.data_ptr(),
                                  plan.wp.data_ptr(), plan.bp.data_ptr(), logits.data_ptr(), value.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    assert _untouched(logits, B) and _untouched(value, B)
    return logits[:B], value[:B]


def _value_inputs(B, w1t, b1, w2, seed):
    """Synthetic value features hv [B][96] (columns 90..95 NaN: never read) and b2, chosen so that the pre-tanh z of the batch spans
    tanh's saturation (|z| ~ 20), its linear range and z ~ 0 (row 0 by construction of b2), with hidden units on both sides of 0."""
    rng = np.random.RandomState(seed)
    base = rng.uniform(0.0, 1.0, (B, 90))
    base[:, rng.rand(90) < 0.2] = 0.0
    base[:, 89] = rng.uniform(0.5, 1.5, B)                                   # the last feature always counts
    scale = np.array([1.0, 40.0, -1.0, 0.3, 3.0, 0.01, 1.0, 8.0])[np.arange(B) % 8]
    base = base * np.abs(scale)[:, None]
    _, z0, _ = S.value_mlp(base, w1t, b1, w2, 0.0)
    b2 = np.float32(-z0[0])
    hv = np.full((B, 96), np.nan)
    hv[:, :90] = base
    return hv.astype(np.float32), float(b2)


@pytest.mark.parametrize("B", [1, 7, 8, 9, 15, 16, 17, 203])
def test_value_mlp_against_fp64(B):
    """k_value_mlp through cz_net_heads_fc with synthetic features: the 8-position tails, NaN in columns 90..95 ignored, pre-tanh
    values from 0 (accurate only relative to the sum of |terms|) through saturation, against fp64 within the accumulation bound.
    Dropping one of the 90 features moves z by ~1 % of its terms' size."""
    from cchess_zero_b200.net import NativePlan
    plan = NativePlan(_net(1, seed=30), 8)
    wp, bp, w1t, b1, w2, _ = _plan_fc(plan)
    hv, b2 = _value_inputs(B, w1t, b1, w2, seed=B)
    plan.b2t.fill_(b2)
    hp = _trunk_out(B, seed=B).reshape(B, -1)[:, :192].contiguous()
    hp[:, 180:] = 0
    lo_k, v_k = _heads_fc(plan, hp, torch.from_numpy(hv).cuda())
    v, z, bv = _value_bound(hv.astype(np.float64), w1t, b1, w2, b2)
    _, _, h = S.value_mlp(hv.astype(np.float64), w1t, b1, w2, b2)
    if B >= 8:
        assert (h < 0).any() and (h > 0).any() and np.abs(z).max() > 15 and np.abs(z).min() < 1e-3
    print("value MLP B=%d: z in [%.3g, %.3g], min |z| %.3g" % (B, z.min(), z.max(), np.abs(z).min()))
    assert np.isfinite(_np(v_k)).all()
    assert _report("value MLP B=%d" % B, np.abs(_np(v_k) - v), bv) <= 1
    hpn = hp.cpu().double().numpy()
    assert _report("policy FC (mma.sync) B=%d" % B, np.abs(_np(lo_k) - S.policy_fc(hpn, wp, bp)), _fc_bound(hpn, wp, bp)) <= 1


# ---------------------------------------------------------------------------------------------------------------------------------
# batch invariance: a row's outputs do not depend on the rows beside it or on its place in the launch
# ---------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["first_conv", "heads", "heads_tc", "heads_fc"])
def test_rows_do_not_depend_on_the_batch(path):
    """A shuffled batch gives each row the bits it gets in the original order and alone at B = 1, in the same code path (the tc path
    is called at B = 1 too)."""
    from cchess_zero_b200.net import NativePlan
    B = 200 if path == "heads_tc" else 77
    plan = NativePlan(_net(1, seed=40), B)
    perm = np.random.RandomState(1).permutation(B)
    pick = [0, 5, 63, 64, B - 1]
    if path == "first_conv":
        boards = _boards(B, seed=40)
        run = lambda idx: [_first_conv(np.ascontiguousarray(boards[idx]), plan.w1, plan.b1).cpu()]      # noqa: E731
    elif path in ("heads", "heads_tc"):
        x = _trunk_out(B, seed=40)
        wh, bh = _head_weights(seed=40)
        run = lambda idx: [torch.from_numpy(a) for a in _heads(plan, x[torch.from_numpy(idx).cuda()].contiguous(), wh, bh, path == "heads_tc")]   # noqa: E731
    else:
        hv = torch.from_numpy(_value_inputs(B, *_plan_fc(plan)[2:5], seed=40)[0]).cuda()
        hp = _trunk_out(B, seed=41).reshape(B, -1)[:, :192].contiguous()
        hp[:, 180:] = 0
        run = lambda idx: [t.cpu() for t in _heads_fc(plan, hp[torch.from_numpy(idx).cuda()].contiguous(), hv[torch.from_numpy(idx).cuda()].contiguous())]   # noqa: E731
    full = run(np.arange(B))
    shuf = run(perm)
    for a, b in zip(full, shuf):
        assert torch.equal(a[torch.from_numpy(perm)].contiguous().view(-1).view(torch.int8), b.contiguous().view(-1).view(torch.int8))
    for i in pick:
        one = run(np.array([i]))
        for a, b in zip(full, one):
            assert torch.equal(a[i:i + 1].contiguous().view(-1).view(torch.int8), b.contiguous().view(-1).view(torch.int8)), (path, i)


# ---------------------------------------------------------------------------------------------------------------------------------
# NaN through the ReLUs
# ---------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("tc", [False, True])
def test_nan_trunk_output_makes_that_position_nan(tc):
    """A NaN in one position's trunk output (an overflowed fp16 trunk) makes that position's logits and value NaN, as torch.relu /
    tf.nn.relu would; every other position is bit-identical.  A ReLU that clips NaN to 0 gives bias-valued logits and a finite value."""
    from cchess_zero_b200.net import NativePlan
    B = 130 if tc else 9
    plan = NativePlan(_net(1, seed=50), B)
    x = _trunk_out(B, seed=50).abs()
    wh, bh = _head_weights(seed=50)
    clean = _heads(plan, x, wh, bh, tc)
    x[3, 17, 40] = float("nan")
    got = _heads(plan, x, wh, bh, tc)
    assert np.isnan(got[2][3]).all() and np.isnan(got[3][3])
    others = np.arange(B) != 3
    for a, b in zip(clean, got):
        assert np.array_equal(a[others], b[others], equal_nan=True)         # hv columns 90..95 hold the (NaN) sentinel


def test_nan_features_reach_only_their_own_outputs():
    """cz_net_heads_fc: a NaN value feature makes that position's value NaN (logits unchanged); a NaN policy feature makes its logits
    NaN (value unchanged); every other position is bit-identical."""
    from cchess_zero_b200.net import NativePlan
    B = 12
    plan = NativePlan(_net(1, seed=51), B)
    hv = torch.from_numpy(_value_inputs(B, *_plan_fc(plan)[2:5], seed=51)[0]).cuda()
    hp = _trunk_out(B, seed=51).abs().reshape(B, -1)[:, :192].contiguous()
    hp[:, 180:] = 0
    lo0, v0 = [t.cpu() for t in _heads_fc(plan, hp, hv)]
    hv[4, 30] = float("nan")
    hp[7, 101] = float("nan")
    lo, v = [t.cpu() for t in _heads_fc(plan, hp, hv)]
    assert torch.isnan(v[4]) and not torch.isnan(v[7]) and torch.equal(lo[4], lo0[4])
    assert torch.isnan(lo[7]).all() and torch.equal(v[7], v0[7])
    rest = torch.from_numpy(~np.isin(np.arange(B), [4, 7]))
    assert torch.equal(lo[rest], lo0[rest]) and torch.equal(v[rest], v0[rest])


# ---------------------------------------------------------------------------------------------------------------------------------
# k_tower_small
# ---------------------------------------------------------------------------------------------------------------------------------

def _tower(plan, boards, w1=None, wh=None, bh=None):
    """cz_net_tower_small on canary buffers with the plan's weights (w1 / wh / bh may be replaced) -> (hp fp16 [n][192], hv [n][96])."""
    n = len(boards)
    hp, hv = _canary(n, 192, dtype=torch.float16), _canary(n, 96)
    assert _lib().cz_net_tower_small(torch.from_numpy(boards).cuda().data_ptr(), n, plan.n_conv, (plan.w1 if w1 is None else w1).data_ptr(),
                                     plan.blob.data_ptr(), plan.bias.data_ptr(), (plan.wh if wh is None else wh).data_ptr(),
                                     (plan.bh if bh is None else bh).data_ptr(), hp.data_ptr(), hv.data_ptr(), _st()) == 0
    torch.cuda.synchronize()
    assert _untouched(hp, n) and _untouched(hv, n)
    return hp[:n], hv[:n]


def _tower_boards(n, seed):
    """Random-play positions (side-to-move canonical), with a kings-only board first: a near-empty image beside crowded ones."""
    from oracle import oracle as O
    rng = np.random.RandomState(seed)
    out, b, side = [], O.from_state(O.START), 0
    while len(out) < n:
        c = np.zeros(96, np.uint8)
        c[:90] = O.flip_board(b) if side == 1 else b
        out.append(c)
        mv = O.legal_moves(b, side)
        b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
        if cap in (1, 8):
            b, side = O.from_state(O.START), 0
        for _ in range(rng.randint(0, 6)):
            mv = O.legal_moves(b, side)
            b, cap = O.apply_move(b, mv[rng.randint(len(mv))]); side ^= 1
            if cap in (1, 8):
                b, side = O.from_state(O.START), 0
    out = np.stack(out)
    kings = np.where(np.isin(out[0, :90], (1, 8)), out[0, :90], 0)          # the two generals (codes 1 / 8) only
    assert (kings > 0).sum() == 2
    out[0, :90] = kings
    return out


def _plan_trunk(plan):
    """The plan's trunk operands as plain float64 tensors: w1 [9][14][128], convs [n_conv][3][3][128][128] (un-laid-out blob), biases."""
    convs = S.unlayout_tower_blob(_np(plan.blob))
    base = [c for blk in plan._base.blocks for c in blk]
    for L, (w, _) in enumerate(base):                                        # the blob is the folded base plan, conv by conv
        assert np.array_equal(convs[L], _np(w.permute(2, 3, 1, 0)))
    return _np(plan.w1), convs, _np(plan.bias)


def _shift_net(blocks, seed):
    """A network whose trunk is exact in f32: every 3x3 convolution has ONE nonzero weight per output channel (source channel
    perm_L[c], tap t_L[c], value s_L, both drawn per layer), w1 and all biases are multiples of 2^-8.  Activations stay multiples
    of 2^-8 below 2^8, so every f32 sum in the kernel is exact and the kernel's trunk equals tower(round16=True) bit for bit; a
    layer reading another layer's taps, channels or scale, or a lost skip, changes the image by whole values."""
    net = _net(blocks, seed, exact_bn=True)
    rng = np.random.RandomState(seed)
    with torch.no_grad():
        net.conv_in.weight.copy_(torch.from_numpy(rng.randint(-256, 257, (128, 14, 3, 3)) / 256.0))
        net.conv_in.bias.copy_(torch.from_numpy(rng.randint(-128, 129, 128) / 256.0))
        for blk in net.blocks:
            for conv, sign, lo, hi in ((blk.c1, -1.0, 0, 512), (blk.c2, 1.0, -256, 257)):
                w = np.zeros((128, 128, 3, 3))
                tap = rng.randint(0, 9, 128)
                w[np.arange(128), rng.permutation(128), tap // 3, tap % 3] = sign * rng.choice([1.0, 2.0])
                conv.weight.copy_(torch.from_numpy(w))
                conv.bias.copy_(torch.from_numpy(rng.randint(lo, hi, 128) / 256.0))
    return net


def _tower_head_bounds(x, wh, bh):
    """The tower's head on the CUDA cores: per term an f32 product, then a pair sum and a running sum over 64 pairs plus the bias
    (<= 67 roundings; c = 2, n = 67 ... taken as n = 129 to cover any order), then the fp16 store of hp."""
    hp, hv = S.head_conv(x, wh, bh)
    t = np.abs(x) @ np.abs(wh).T + np.abs(bh)
    acc = 2 * 129 * U * t
    bhp = np.zeros_like(hp)
    bhp[:, :180] = acc[..., :2].reshape(len(x), 180)
    return hp, hv, bhp + S.ulp16(hp), acc[..., 2]


@pytest.mark.parametrize("blocks,n_pos", [(1, 1), (2, 2), (3, 5), (7, 16), (19, 5)])
def test_tower_exact_trunk_and_heads_against_fp64(blocks, n_pos):
    """k_tower_small on an exact trunk (_shift_net): the 16-stage weight ring wraps at a different tap for 1 / 2 / 3 / 7 / 19 blocks,
    and each layer reads its own taps.  hv against the fp64 head of the exact final image with f32 head weights whose fp16 residue
    is ~4.2e-4 (a head convolution that rounds wh to fp16 misses the bound by ~25x), hp within one fp16 ulp, K padding zero."""
    from cchess_zero_b200.net import SmallTowerPlan
    plan = SmallTowerPlan(_shift_net(blocks, seed=blocks), 16)
    boards = _tower_boards(n_pos, seed=60 + blocks)
    w1, convs, biases = _plan_trunk(plan)
    assert ((convs != 0).sum(axis=(1, 2, 3)) == 1).all()
    wh, bh = _head_weights(seed=blocks)
    hp_k, hv_k = _tower(plan, boards, wh=wh, bh=bh)
    hp, hv, x = S.tower(boards, w1, convs, biases, _np(wh), _np(bh), round16=True)
    assert np.abs(x).max() < 256 and (x > 0).mean() > 0.2
    _, _, bhp, bhv = _tower_head_bounds(x, _np(wh), _np(bh))
    hp_k, hv_k = hp_k.cpu().double().numpy(), _np(hv_k)
    assert not hp_k[:, 180:].any()
    assert _report("tower(exact) %d blocks n=%d hv" % (blocks, n_pos), np.abs(hv_k[:, :90] - hv), bhv) <= 1
    assert _report("tower(exact) %d blocks n=%d hp" % (blocks, n_pos), np.abs(hp_k - hp), bhp) <= 1


@pytest.mark.parametrize("blocks,n_pos", [(1, 16), (2, 1), (3, 2), (7, 5), (19, 16)])
def test_tower_against_fp64_rounding_where_the_kernel_rounds(blocks, n_pos):
    """k_tower_small with random weights (each layer scaled differently) against tower(round16=True), the fp64 trunk that rounds to
    fp16 where the kernel does, and tower(round16=False), plain fp64; the errors against both are printed.  f32 and fp64 sums differ
    by a few units of 2^-24, which flips an fp16 rounding only now and then, but of the 11 520 roundings per layer some do flip, and
    each flip moves the next layer's sums by about one fp16 ulp of one term, which flips others: over the layers the kernel drifts
    from the rounded reference by as much as the rounded reference drifts from fp64.  Measured on an H100 (80 GB HBM3, 700 W):
    kernel-vs-round16 / round16-vs-fp64 = 0.37, 0.57, 0.90, 1.18, 1.49 at 1 / 2 / 3 / 7 / 19 blocks.  So this test bounds the kernel at
    2x the fp16 trunk's own rounding noise (a wrong tap, channel or layer is O(1) of the head); the arithmetic of every layer is
    held bit for bit by test_tower_exact_trunk_and_heads_against_fp64."""
    from cchess_zero_b200.net import SmallTowerPlan
    net = _net(blocks, seed=70 + blocks)
    rng = np.random.RandomState(blocks)
    with torch.no_grad():
        for blk in net.blocks:
            for conv in (blk.c1, blk.c2):
                conv.weight.mul_(float(rng.uniform(0.6, 1.6)))
    plan = SmallTowerPlan(net, 16)
    boards = _tower_boards(n_pos, seed=80 + blocks)
    w1, convs, biases = _plan_trunk(plan)
    wh, bh = _np(plan.wh), _np(plan.bh)
    hp_k, hv_k = _tower(plan, boards)
    hp_k, hv_k = hp_k.cpu().double().numpy(), _np(hv_k)[:, :90]
    hp16, hv16, _ = S.tower(boards, w1, convs, biases, wh, bh, round16=True)
    hp64, hv64, _ = S.tower(boards, w1, convs, biases, wh, bh, round16=False)
    scale = max(np.abs(hp64).max(), np.abs(hv64).max())
    e_k16 = max(np.abs(hp_k - hp16).max(), np.abs(hv_k - hv16).max()) / scale
    e_k64 = max(np.abs(hp_k - hp64).max(), np.abs(hv_k - hv64).max()) / scale
    e_1664 = max(np.abs(hp16 - hp64).max(), np.abs(hv16 - hv64).max()) / scale
    print("tower %d blocks n=%d, relative to max|head| %.3g: kernel vs round16 %.3e, kernel vs fp64 %.3e, round16 vs fp64 %.3e (ratio %.3f)"
          % (blocks, n_pos, scale, e_k16, e_k64, e_1664, e_k16 / e_1664))
    assert e_1664 > 0 and e_k16 < 2.0 * e_1664


def test_tower_rows_do_not_depend_on_the_batch_and_nan_weight_row():
    """Each cluster's outputs are bit-identical shuffled and alone; a NaN row of w1 for piece code 12 makes NaN only the positions that
    hold that piece (through every layer), the others bit-identical."""
    from cchess_zero_b200.net import SmallTowerPlan
    plan = SmallTowerPlan(_net(2, seed=90), 16)
    boards = _tower_boards(16, seed=90)
    hp, hv = [t.cpu() for t in _tower(plan, boards)]
    perm = np.random.RandomState(2).permutation(16)
    hp2, hv2 = [t.cpu() for t in _tower(plan, np.ascontiguousarray(boards[perm]))]
    assert torch.equal(hp[perm].view(torch.int16), hp2.view(torch.int16)) and torch.equal(hv[perm].view(torch.int32), hv2.view(torch.int32))
    for i in (0, 7, 15):
        a, b = [t.cpu() for t in _tower(plan, boards[i:i + 1].copy())]
        assert torch.equal(a.view(torch.int16), hp[i:i + 1].view(torch.int16)) and torch.equal(b.view(torch.int32), hv[i:i + 1].view(torch.int32))
    has = (boards[:, :82] == 12).any(axis=1)
    assert has.any() and not has.all()
    w1 = plan.w1.clone()
    w1[:, 11, :] = float("nan")
    hpn, hvn = [t.cpu() for t in _tower(plan, boards, w1=w1)]
    nan = torch.isnan(hvn[:, :90]).any(1) | torch.isnan(hpn[:, :180].float()).any(1)
    assert np.array_equal(nan.numpy(), has)
    keep = torch.from_numpy(~has)
    assert torch.equal(hpn[keep].view(torch.int16), hp[keep].view(torch.int16)) and torch.equal(hvn[keep].view(torch.int32), hv[keep].view(torch.int32))
