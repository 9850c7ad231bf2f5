"""TEST INFRASTRUCTURE ONLY.  float64 statements of the hand-written network kernels (csrc/cz_net.cu, csrc/cz_tower.cu), one
function per kernel stage, taking its operands rounded exactly as the kernel receives them (fp16 weights as fp16 values, f32 as f32),
so that a kernel's output can be held to a bound derived from its own arithmetic rather than to the end-to-end network.

Shapes and layouts follow include/cchess_b200.h and the kernels' headers:
  canonical boards  u8 [B][96]: image cell (r, f) of the [9][10] image reads byte r*9 + f (the reference's quirk, main.py:550-555);
                    bytes 82..95 are never read.  Code c in 1..14 sets plane c - 1.
  w1                fp16 [9 taps][14 pieces][128]: tap = kh*3 + kw, i.e. the TF kernel [3][3][14][128] flattened.
  activations       [B][90][128], cell = r*10 + f (NHWC).
  hp                fp16 [B][192]: policy features in tf.reshape order cell*2 + c, zero K padding 180..191.
  hv                f32 [B][96]: value features, 90..95 unused.
Kernel-layout tensors are turned back into plain ones by the `unlayout_*` helpers.  ReLU is np.maximum, which propagates NaN."""
import numpy as np

from oracle.net_numpy import conv2d_same, relu

NLABEL = 2086


def f64(a):
    return np.asarray(a, dtype=np.float64)


def r16(a):
    """fp16 rounding of a float64 array (round to nearest even, straight from float64), back as float64."""
    return f64(a).astype(np.float16).astype(np.float64)


def ulp16(a):
    """Spacing of fp16 at |a| (2^-24 at zero): one fp16 ulp of the value."""
    return np.spacing(np.abs(f64(a)).astype(np.float16)).astype(np.float64)


def image(canon_boards):
    """u8 [B][96] canonical boards -> one-hot float64 [B][9][10][14]: cell (r, f) <- byte r*9 + f."""
    b = np.asarray(canon_boards, dtype=np.uint8)
    r, f = np.meshgrid(np.arange(9), np.arange(10), indexing="ij")
    codes = b[:, (r * 9 + f)].astype(np.int64)                              # [B][9][10]
    x = np.zeros(codes.shape + (15,), dtype=np.float64)
    np.put_along_axis(x, codes[..., None], 1.0, axis=-1)
    return x[..., 1:]


def first_conv(canon_boards, w1, b1):
    """k_first_conv: relu(conv3x3(image, w1) + b1).  -> (float64 value before the fp16 store [B][90][128], its fp16 rounding)."""
    v = relu(conv2d_same(image(canon_boards), f64(w1).reshape(3, 3, 14, 128), f64(b1)))
    v = v.reshape(len(v), 90, 128)
    return v, r16(v)


def conv3x3(x, k, b):
    """One 3x3 128 -> 128 convolution of [B][90][128] activations with a TF kernel [3][3][128][128]."""
    return conv2d_same(f64(x).reshape(-1, 9, 10, 128), f64(k), f64(b)).reshape(-1, 90, 128)


def head_conv(x, wh, bh):
    """k_head_conv_mma (and the tower's head): relu(x . wh^T + bh) per cell.  x [B][90][128], wh [3][128] (policy 2 + value 1),
    bh [3].  -> (hp float64 [B][192] in flatten order cell*2 + c with zero padding 180..191, hv float64 [B][90])."""
    s = relu(f64(x) @ f64(wh).T + f64(bh))                                     # [B][90][3]
    hp = np.zeros((len(s), 192), dtype=np.float64)
    hp[:, :180] = s[..., :2].reshape(len(s), 180)
    return hp, s[..., 2]


def value_mlp(hv, w1t, b1, w2, b2):
    """k_value_mlp: tanh(relu(hv[:, :90] . w1t + b1) . w2 + b2).  -> (value [B], pre-tanh z [B], hidden pre-activations [B][256])."""
    h = f64(hv)[:, :90] @ f64(w1t) + f64(b1)
    z = relu(h) @ f64(w2).reshape(256) + f64(b2).reshape(())
    return np.tanh(z), z, h


def policy_fc(hp, wp, bp):
    """k_policy_fc / k_policy_fc_tc: hp[:, :180] . wp[:2086, :180]^T + bp[:2086].  wp is label-major (the kernels' [2112][192])."""
    return f64(hp)[:, :180] @ f64(wp)[:NLABEL, :180].T + f64(bp)[:NLABEL]


def tower(canon_boards, w1, convs, biases, wh, bh, round16=True):
    """k_tower_small: first conv, len(convs) / 2 residual blocks [conv -> ReLU -> conv -> +skip -> ReLU], the head convolutions.
    convs [n_conv][3][3][128][128] TF kernels (fp16 values), biases [1 + n_conv][128] (layer 0 = first conv).  With round16 every
    layer's output (after bias, skip and ReLU) is rounded to fp16, as the kernel stores it; without, the trunk is plain float64.
    -> (hp [B][192], hv [B][90], final trunk image [B][90][128]), head outputs before the fp16 store of hp."""
    rd = r16 if round16 else f64
    v, _ = first_conv(canon_boards, w1, biases[0])
    x = rd(v)
    for L in range(0, len(convs), 2):
        y = rd(relu(conv3x3(x, convs[L], biases[L + 1])))
        x = rd(relu(conv3x3(y, convs[L + 1], biases[L + 2]) + x))
    hp, hv = head_conv(x, wh, bh)
    return hp, hv, x


# ---- kernel layouts -> plain tensors ----------------------------------------------------------------------------------------------

def unlayout_wp_tiled(wp_tiled):
    """wgmma policy-FC weights [17 label tiles][24 k-chunks][128 labels][8] -> label-major [2176][192]."""
    a = np.asarray(wp_tiled)
    return a.reshape(17, 24, 128, 8).transpose(0, 2, 1, 3).reshape(17 * 128, 192)


def unlayout_hp_tiled(hp_tiled):
    """k_head_conv_mma<true> output [position tiles][24 k-chunks][128 positions][8] -> row-major [tiles * 128][192]."""
    a = np.asarray(hp_tiled)
    t = a.size // (24 * 128 * 8)
    return a.reshape(t, 24, 128, 8).transpose(0, 2, 1, 3).reshape(t * 128, 192)


def unlayout_tower_blob(blob, cl=4):
    """cz_net_tower_small weight blob [conv][tap][rank][k-chunk 16][out channel 128/cl][8 in channels] (out = rank*NC + o,
    in = k-chunk*8 + e) -> TF kernels [conv][3][3][128 in][128 out]."""
    nc = 128 // cl
    a = np.asarray(blob)
    n = a.size // (9 * 128 * 128)
    return a.reshape(n, 9, cl, 16, nc, 8).transpose(0, 1, 3, 5, 2, 4).reshape(n, 3, 3, 128, 128)
