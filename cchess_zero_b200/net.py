"""The policy-value ResNet of the reference (policy_value_network.py:9-214), re-implemented in PyTorch.

Architecture (policy_value_network.py:45-74, 151-162), NHWC input [B,9,10,14]:
  conv3x3(14->128)+bias -> BN(no gamma/beta, eps 1e-5) -> ReLU
  res_block_nums x [conv3x3 -> BN -> ReLU -> conv3x3 -> BN -> +skip -> ReLU]
  policy: conv1x1(128->2) -> BN -> ReLU -> flatten (h, w, c) 180 -> FC 2086   (raw LOGITS, no softmax: line 64/210)
  value : conv1x1(128->1) -> BN -> ReLU -> flatten 90 -> FC 256 ReLU -> FC 1 tanh
Reference quirk kept by default: the TF1 graph never runs the batch-norm UPDATE_OPS
(policy_value_network.py:104-106), so inference statistics stay at (mean 0, var 1) forever;
`update_moving_stats=True` gives conventional behaviour.

The tensor-core work (residual convolutions) goes through cuDNN/cuBLAS; this module is plumbing for the
engine, which hands it a device-resident [B,9,10,14] batch and reads back logits/value on the device."""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

NLABEL = 2086


class RefBatchNorm(nn.Module):
    """tf.contrib.layers.batch_norm(center=False, scale=False, epsilon=1e-5, decay=0.999)."""

    def __init__(self, ch, eps=1e-5, decay=0.999, update_moving_stats=False):
        super().__init__()
        self.eps, self.decay, self.update = eps, decay, update_moving_stats
        self.register_buffer("running_mean", torch.zeros(ch))
        self.register_buffer("running_var", torch.ones(ch))

    def forward(self, x):
        if self.training:
            mean = x.mean(dim=(0, 2, 3))
            var = x.var(dim=(0, 2, 3), unbiased=False)
            if self.update:
                n = x.numel() / x.shape[1]
                with torch.no_grad():
                    self.running_mean.mul_(self.decay).add_(mean.detach() * (1 - self.decay))
                    self.running_var.mul_(self.decay).add_(var.detach() * (n / max(n - 1, 1)) * (1 - self.decay))
        else:
            mean, var = self.running_mean, self.running_var
        return (x - mean[None, :, None, None]) * torch.rsqrt(var[None, :, None, None] + self.eps)


class ResBlock(nn.Module):
    def __init__(self, ch, **bn):
        super().__init__()
        self.c1 = nn.Conv2d(ch, ch, 3, padding=1)
        self.b1 = RefBatchNorm(ch, **bn)
        self.c2 = nn.Conv2d(ch, ch, 3, padding=1)
        self.b2 = RefBatchNorm(ch, **bn)

    def forward(self, x):
        y = F.relu(self.b1(self.c1(x)))
        y = self.b2(self.c2(y))
        return F.relu(x + y)


class PolicyValueNet(nn.Module):
    def __init__(self, res_block_nums=7, filters=128, update_moving_stats=False):
        super().__init__()
        bn = dict(update_moving_stats=update_moving_stats)
        self.conv_in = nn.Conv2d(14, filters, 3, padding=1)
        self.bn_in = RefBatchNorm(filters, **bn)
        self.blocks = nn.ModuleList([ResBlock(filters, **bn) for _ in range(res_block_nums)])
        self.p_conv = nn.Conv2d(filters, 2, 1)
        self.p_bn = RefBatchNorm(2, **bn)
        self.p_fc = nn.Linear(180, NLABEL)
        self.v_conv = nn.Conv2d(filters, 1, 1)
        self.v_bn = RefBatchNorm(1, **bn)
        self.v_fc1 = nn.Linear(90, 256)
        self.v_fc2 = nn.Linear(256, 1)
        for m in self.modules():  # tf.layers / contrib defaults: glorot-uniform kernels, zero biases
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)

    def forward(self, x_nhwc):
        """x_nhwc: [B,9,10,14] -> (logits [B,2086], value [B,1])"""
        x = x_nhwc.permute(0, 3, 1, 2)
        x = F.relu(self.bn_in(self.conv_in(x)))
        for b in self.blocks:
            x = b(x)
        p = F.relu(self.p_bn(self.p_conv(x))).permute(0, 2, 3, 1).reshape(x.shape[0], 180)
        v = F.relu(self.v_bn(self.v_conv(x))).permute(0, 2, 3, 1).reshape(x.shape[0], 90)
        logits = self.p_fc(p)
        value = torch.tanh(self.v_fc2(F.relu(self.v_fc1(v))))
        return logits, value


_DT = {"fp32": torch.float32, "tf32": torch.float32, "tf32x3": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def make_plan(net, precision, owner=None):
    """The inference plan of a precision name: "tf32x3" (fp32-accurate on the TF32 tensor cores) has its own class."""
    return SplitTf32Plan(net, owner=owner) if precision == "tf32x3" else InferencePlan(net, precision, owner=owner)


class _VersionedPlan:
    """A plan that holds folded COPIES of its owner's weights.  policy_value_network.weights_version is bumped whenever the weights
    change; refresh_if_stale re-derives the copies in place (`refresh`) when the plan's version is behind."""

    def refresh_if_stale(self):
        if self.owner is not None and self.owner.weights_version != self.version:
            self.refresh()
            return True
        return False


class InferencePlan(_VersionedPlan):
    """Eval-mode forward with batch norm folded into the convolutions, channels-last, in one of
    fp32 / tf32 / bf16 / fp16.  Takes the engine's NHWC batch as-is (its NCHW view is already
    channels_last) and returns float32 logits / value on the device."""

    def __init__(self, net, precision="fp32", fused=True, owner=None):
        assert precision in _DT
        self.precision = precision
        self.dtype = _DT[precision]
        self.net = net
        self.owner = owner                      # policy_value_network whose weights_version tells when the folded copies are stale
        self.version = getattr(owner, "weights_version", 0)
        self._assign(self._fold_all(net))
        self.fused = bool(fused) and self._probe_fused()
        if os.environ.get("CCHESS_CUDNN_BENCHMARK", "0") == "1":
            torch.backends.cudnn.benchmark = True     # let cuDNN time its engines for the (fixed) tower shapes

    def _fold_all(self, net):
        """Folded copies of the weights (BN into the convolutions), in this plan's dtype / memory format."""
        dt = self.dtype

        def fold(conv, bn):
            s = torch.rsqrt(bn.running_var + bn.eps)
            w = (conv.weight * s[:, None, None, None]).detach()
            b = ((conv.bias - bn.running_mean) * s).detach()
            return w.to(dt).contiguous(memory_format=torch.channels_last), b.to(dt).contiguous()

        with torch.no_grad():
            wp, bp = fold(net.p_conv, net.p_bn)
            wv, bv = fold(net.v_conv, net.v_bn)
            return dict(
                w_in=fold(net.conv_in, net.bn_in),
                blocks=[(fold(b.c1, b.b1), fold(b.c2, b.b2)) for b in net.blocks],
                w_head=(torch.cat([wp, wv], 0).contiguous(memory_format=torch.channels_last), torch.cat([bp, bv], 0).contiguous()),
                p_fc=(net.p_fc.weight.detach().to(dt).contiguous(), net.p_fc.bias.detach().to(dt).contiguous()),
                v_fc1=(net.v_fc1.weight.detach().float().contiguous(), net.v_fc1.bias.detach().float().contiguous()),
                v_fc2=(net.v_fc2.weight.detach().float().contiguous(), net.v_fc2.bias.detach().float().contiguous()))

    def _assign(self, d):
        self.w_in, self.blocks, self.w_head, self.p_fc, self.v_fc1, self.v_fc2 = d["w_in"], d["blocks"], d["w_head"], d["p_fc"], d["v_fc1"], d["v_fc2"]

    def refresh(self):
        """Re-fold the (trained / restored) weights INTO the existing tensors, so that CUDA graphs that captured this
        plan keep evaluating with the current weights (MCTS_tree and SelfPlay hold such graphs across train_step)."""
        d = self._fold_all(self.net)
        with torch.no_grad():
            for name in ("w_in", "w_head", "p_fc", "v_fc1", "v_fc2"):
                for dst, src in zip(getattr(self, name), d[name]):
                    dst.copy_(src)
            for (c1, c2), (n1, n2) in zip(self.blocks, d["blocks"]):
                for dst, src in zip(c1 + c2, n1 + n2):
                    dst.copy_(src)
        self.version = getattr(self.owner, "weights_version", self.version)

    def _probe_fused(self):
        try:
            x = torch.randn(4, 128, 9, 10, device=self.w_in[0].device, dtype=self.dtype).contiguous(memory_format=torch.channels_last)
            (w, b) = self.blocks[0][0] if self.blocks else self.w_in
            if w.shape[1] != 128:
                return False
            with self._ctx():
                a = torch.cudnn_convolution_relu(x, w, b, (1, 1), (1, 1), (1, 1), 1)
                r = F.relu(F.conv2d(x, w, b, padding=1))
                a2 = torch.cudnn_convolution_add_relu(x, w, x, 1.0, b, (1, 1), (1, 1), (1, 1), 1)
                r2 = F.relu(F.conv2d(x, w, b, padding=1) + x)
            tol = 1e-4 if self.dtype == torch.float32 else 5e-2
            return bool(torch.allclose(a.float(), r.float(), atol=tol, rtol=tol) and torch.allclose(a2.float(), r2.float(), atol=tol, rtol=tol))
        except Exception:
            return False

    def _ctx(self):
        return _Tf32(self.precision in ("tf32", "tf32x3"))

    def make_input(self, B):
        return torch.zeros((B, 9, 10, 14), dtype=self.dtype, device=self.w_in[0].device)

    def _conv_relu(self, x, wb, pad):
        w, b = wb
        if self.fused and pad == 1:
            return torch.cudnn_convolution_relu(x, w, b, (1, 1), (pad, pad), (1, 1), 1)
        return F.relu_(F.conv2d(x, w, b, padding=pad))

    def _conv_add_relu(self, x, wb, skip):
        w, b = wb
        if self.fused:
            return torch.cudnn_convolution_add_relu(x, w, skip, 1.0, b, (1, 1), (1, 1), (1, 1), 1)
        return F.relu_(F.conv2d(x, w, b, padding=1).add_(skip))

    @torch.no_grad()
    def __call__(self, nn_in, logits_out=None, value_out=None):
        """nn_in: [B,9,10,14] of self.dtype on the device."""
        B = nn_in.shape[0]
        with self._ctx():
            x = nn_in.permute(0, 3, 1, 2)
            if x.dtype != self.dtype:
                x = x.to(self.dtype)
            x = self._conv_relu(x, self.w_in, 1)
            for c1, c2 in self.blocks:
                y = self._conv_relu(x, c1, 1)
                x = self._conv_add_relu(y, c2, x)
            h = F.relu_(F.conv2d(x, self.w_head[0], self.w_head[1]))      # [B,3,9,10] channels_last
            h = h.permute(0, 2, 3, 1)                                      # [B,9,10,3]
            p = h[..., :2].reshape(B, 180)
            v = h[..., 2].reshape(B, 90).float()
            logits = F.linear(p, self.p_fc[0], self.p_fc[1]).float()
            value = torch.tanh(F.linear(F.relu_(F.linear(v, self.v_fc1[0], self.v_fc1[1])), self.v_fc2[0], self.v_fc2[1]))
        if logits_out is not None:
            logits_out.copy_(logits)
            value_out.copy_(value.reshape(value_out.shape))
            return None
        return logits, value


def tf32_hi(t):
    """Round an f32 tensor to the 10-bit TF32 mantissa (nearest, ties away from zero): the low 13 bits of the result are zero, so the
    tensor-core kernels' own f32 -> tf32 conversion leaves it unchanged.  Same operation as csrc/cz_net.cu: tf32_hi."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32).reshape(t.shape)


SPLIT_SCALE = 2048.0      # 2^11: the lo halves travel scaled into fp16's normal range (csrc/cz_net.cu: SPLIT_SCALE)


def split_weights(w):
    """[O, C, kh, kw] f32 -> (hi(w) f32 [O, C, kh, kw], { hi(w) | (w - hi(w)) * 2^11 } fp16 [O, 2C, kh, kw]): the weight side of
    the three-product convolution.  Both fp16 halves have <= 11 significant bits: exact in fp16 up to its range."""
    h = tf32_hi(w)
    return h, torch.cat([h, (w - h) * SPLIT_SCALE], 1).to(torch.float16)


def split_acts(x):
    """[B, C, H, W] f32 -> (hi(x) f32 [B, C, H, W], { (x - hi(x)) * 2^11 | hi(x) } fp16 [B, 2C, H, W]): torch statement of
    the split in csrc/cz_net.cu: k_epilogue_split."""
    h = tf32_hi(x)
    return h, torch.cat([(x - h) * SPLIT_SCALE, h], 1).to(torch.float16)


class SplitTf32Plan(InferencePlan):
    """precision="tf32x3": the reference's fp32 arithmetic (policy_value_network.py:202-214) reproduced to ~1e-5 of max |logit| ON
    the tensor cores, for the contract "NN outputs match within 1e-3 fp32" at trained-network magnitudes (fp16 / tf32 carry 10-11-bit
    mantissas through 15-39 convolutions and miss an absolute 1e-3 on logits of size 8, DESIGN.md section 4), at a tenth of the
    cost of cuDNN's fp32 convolutions (which do not use the tensor cores: 57x slower than fp16).

    Every activation x and weight w is split into hi = tf32(x) (10-bit mantissa) and lo = x - hi; per convolution
        s   = conv_fp16({ lo(x) 2^11 | hi(x) }, { hi(w) | lo(w) 2^11 })        the two small cross terms, K = 2 x 1152; the operands
                                                                              have <= 11 significant bits, i.e. are exact in fp16
        out = relu(conv_tf32(hi(x), hi(w)) + 2^-11 s [+ skip] + bias)         the full-size term; the f32 epilogue AND the hi / lo split
                                                                              of `out` for the next convolution are one streaming
                                                                              pass of this package (csrc/cz_net.cu: k_epilogue_split)
    What is dropped (lo*lo, the 11-bit rounding of the two lo operands and of s) is O(2^-22) relative.  The two terms are accumulated
    SEPARATELY because the tensor cores' f32 accumulator truncates (tools/tf32x3_probe.py: -6.6e-9 relative per accumulated term,
    linear in K): one TF32 convolution over { hi | lo | hi } x { hi | hi | lo } (K = 3456) measured 9.6e-6 relative per layer,
    hi*hi apart from the cross terms 3.4e-6 (hi*hi in two / four input-channel groups: 1.6e-6 / 7.7e-7 for +35 % / +90 % time).
    The first
    convolution takes the one-hot planes (exact in any precision) against { hi(w) | lo(w) } with 2 x 14 channels in TF32; the heads
    (3 of 128 channels, 180 -> 2086, 90 -> 256 -> 1) run in true fp32."""

    def __init__(self, net, owner=None):
        import ctypes as C
        from ._lib import lib
        self._C, self._lib = C, lib()
        self._bufs = {}
        super().__init__(net, "tf32x3", owner=owner)

    def _fold_all(self, net):
        d = super()._fold_all(net)                                   # f32 folded weights, channels_last
        cl = lambda t: t.contiguous(memory_format=torch.channels_last)  # noqa: E731
        with torch.no_grad():
            w, b = d["w_in"]
            h = tf32_hi(w)
            d["w_in"] = (cl(torch.cat([h, w - h], 1)), b)                # [128, 28, 3, 3]: { hi | lo } against the planes twice

            def ws(wb):
                h, w2 = split_weights(wb[0])
                return cl(h), cl(w2), wb[1]                             # f32 [128,128,3,3], fp16 [128,256,3,3], bias
            d["blocks"] = [(ws(c1), ws(c2)) for c1, c2 in d["blocks"]]
        return d

    def _probe_fused(self):
        return False          # the epilogue is this package's own kernel (k_epilogue_split); the library convolutions run bare

    def _buffers(self, B, dev):
        """x f32 [B,9,10,128] (block input / skip / heads' input), hi f32 [B,9,10,128], x2 fp16 [B,9,10,256]: one set per batch size,
        allocated on the first (eager, warm-up) call; every consumer is issued on the same stream before the next producer."""
        bufs = self._bufs.get(B)
        if bufs is None:
            bufs = self._bufs[B] = (torch.empty((B, 9, 10, 128), dtype=torch.float32, device=dev),
                                    torch.empty((B, 9, 10, 128), dtype=torch.float32, device=dev),
                                    torch.empty((B, 9, 10, 256), dtype=torch.float16, device=dev))
        return bufs

    def _epilogue(self, t, s, bias, skip, x, hi, x2, n_pix):
        """v = relu(t + 2^-11 s + bias [+ skip]) -> x (optional) and the split (hi, x2) of v (optional): csrc/cz_net.cu: k_epilogue_split."""
        cl = torch.channels_last
        t = t.contiguous(memory_format=cl)                    # (the library already returns channels_last: no copy)
        s = None if s is None else s.contiguous(memory_format=cl)
        p = lambda z: None if z is None else z.data_ptr()  # noqa: E731
        rc = self._lib.cz_net_epilogue_split(t.data_ptr(), p(s), bias.data_ptr(), p(skip), p(x), p(hi), p(x2), n_pix,
                                             self._C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc:
            raise RuntimeError("cz_net_epilogue_split failed (%d)" % rc)

    @torch.no_grad()
    def __call__(self, nn_in, logits_out=None, value_out=None):
        """nn_in: [B,9,10,14] one-hot planes (any float dtype) on the device."""
        B = nn_in.shape[0]
        X, HI, X2 = self._buffers(B, nn_in.device)
        hi_v, x2_v = HI.permute(0, 3, 1, 2), X2.permute(0, 3, 1, 2)          # NCHW views of NHWC memory = channels_last
        n_pix, nb = B * 90, len(self.blocks)
        x = nn_in.permute(0, 3, 1, 2).float()
        with self._ctx():
            t = F.conv2d(torch.cat([x, x], 1).contiguous(memory_format=torch.channels_last), self.w_in[0], None, padding=1)
            self._epilogue(t, None, self.w_in[1], None, X, HI if nb else None, X2 if nb else None, n_pix)
            for i, ((wh1, ws1, b1), (wh2, ws2, b2)) in enumerate(self.blocks):
                t, s = F.conv2d(hi_v, wh1, None, padding=1), F.conv2d(x2_v, ws1, None, padding=1)
                self._epilogue(t, s, b1, None, None, HI, X2, n_pix)             # y = relu(conv1(x)): only its split is needed
                t, s = F.conv2d(hi_v, wh2, None, padding=1), F.conv2d(x2_v, ws2, None, padding=1)
                last = i == nb - 1
                self._epilogue(t, s, b2, X, X, None if last else HI, None if last else X2, n_pix)   # x = relu(conv2(y) + x)
        with _Tf32(False):
            h = F.relu_(F.conv2d(X.permute(0, 3, 1, 2), self.w_head[0], self.w_head[1])).permute(0, 2, 3, 1)
            p = h[..., :2].reshape(B, 180)
            v = h[..., 2].reshape(B, 90)
            logits = F.linear(p, self.p_fc[0], self.p_fc[1])
            value = torch.tanh(F.linear(F.relu_(F.linear(v, self.v_fc1[0], self.v_fc1[1])), self.v_fc2[0], self.v_fc2[1]))
        if logits_out is not None:
            logits_out.copy_(logits)
            value_out.copy_(value.reshape(value_out.shape))
            return None
        return logits, value


def _ends_weights(net, base):
    """Kernel-layout copies of the weights both native plans share, derived from the folded fp16 base plan: the first convolution
    (w1, fp16 [9 taps][14 pieces][128]), the 1x1 head convolutions (wh, bh), the value MLP (w1t, bv1, w2, b2t) and the zero-padded
    policy FC (wp fp16 [2112][192], bp f32 [2112])."""
    dev = base.w_in[0].device
    with torch.no_grad():
        w, _ = base.w_in                                                    # folded conv_in: [128,14,3,3] fp16
        wh, bh = base.w_head                                                # [3,128,1,1]
        wp = torch.zeros((2112, 192), dtype=torch.float16, device=dev)
        wp[:NLABEL, :180] = net.p_fc.weight.detach().to(torch.float16)
        bp = torch.zeros((2112,), dtype=torch.float32, device=dev)
        bp[:NLABEL] = net.p_fc.bias.detach().float()
        return dict(w1=w.float().permute(2, 3, 1, 0).reshape(9, 14, 128).to(torch.float16).contiguous(),
                    wh=wh.float().reshape(3, 128).contiguous(), bh=bh.float().contiguous(),
                    w1t=net.v_fc1.weight.detach().float().t().contiguous(),        # [90,256]
                    bv1=net.v_fc1.bias.detach().float().contiguous(),
                    w2=net.v_fc2.weight.detach().float().reshape(256).contiguous(),
                    b2t=net.v_fc2.bias.detach().float().reshape(1).contiguous(), wp=wp, bp=bp)


class _NativeEnds(_VersionedPlan):
    """What the two fp16 plans with hand-written kernels share: the folded base plan, the kernel-layout weights (`_derive`, refreshed
    into the SAME device tensors so that captured CUDA graphs stay valid) and the input contract: uint8 [B,96] canonical boards in,
    float32 logits / value written in place."""

    precision = "fp16"
    dtype = torch.uint8

    def __init__(self, net, max_batch, owner):
        import ctypes as C
        from ._lib import lib
        self._C, self._lib = C, lib()
        self._base = InferencePlan(net, "fp16", owner=owner)
        self.net, self.owner, self.version, self.max_batch = net, owner, self._base.version, max_batch
        for k, v in self._derive().items():
            setattr(self, k, v)
        dev = self._base.w_in[0].device
        self.hp = torch.zeros((max_batch, 192), dtype=torch.float16, device=dev)
        self.hv = torch.zeros((max_batch, 96), dtype=torch.float32, device=dev)

    def refresh(self):
        """New weights into the SAME device tensors; see InferencePlan.refresh."""
        self._base.refresh()
        with torch.no_grad():
            for k, v in self._derive().items():
                getattr(self, k).copy_(v)
        self.version = self._base.version

    def make_input(self, B):
        return torch.zeros((B, 96), dtype=torch.uint8, device=self.hp.device)


class NativePlan(_NativeEnds):
    """fp16 inference plan whose ends are the hand-written kernels of csrc/cz_net.cu:
         board bytes --cz_net_first_conv--> [B,90,128] --library cuDNN convs (residual tower)--> --cz_net_heads--> logits, value
    Input is the engine's CZ_BOARD output (uint8 [B,96], the side-to-move-canonical board); the one-hot
    [9,10,14] tensor is never built.  Outputs are written straight into the float32 buffers the engine reads.  Batches of 128 rows
    or more take the wgmma policy FC (cz_net_heads_tc), smaller ones the mma.sync kernels (cz_net_heads)."""

    first_conv = "gather"        # the first convolution is a gather-add of weight rows (k_first_conv)

    def __init__(self, net, max_batch, owner=None):
        super().__init__(net, max_batch, owner)
        self.blocks, self.fused = self._base.blocks, self._base.fused
        dev = self.hp.device
        self.x1 = torch.empty((max_batch, 9, 10, 128), dtype=torch.float16, device=dev)
        # policy features in the tiled operand layout of the wgmma policy FC (rows beyond the batch stay zero)
        self.hp_tiled = torch.zeros(((max_batch + 127) // 128, 24, 128, 8), dtype=torch.float16, device=dev)

    def _derive(self):
        d = _ends_weights(self.net, self._base)
        with torch.no_grad():
            d["b1"] = self._base.w_in[1].float().contiguous()
            # policy FC weights as wgmma operand tiles: [17 label tiles][24 k-chunks][128 labels][8 features]
            wp_pad = torch.zeros((2176, 192), dtype=torch.float16, device=d["wp"].device)
            wp_pad[:2112] = d["wp"]
            d["bp_pad"] = torch.zeros((2176,), dtype=torch.float32, device=d["bp"].device)
            d["bp_pad"][:2112] = d["bp"]
            d["wp_tiled"] = wp_pad.reshape(17, 128, 24, 8).permute(0, 2, 1, 3).contiguous()
        return d

    @torch.no_grad()
    def __call__(self, boards, logits_out, value_out):
        B = boards.shape[0]
        assert B <= self.max_batch and boards.dtype == torch.uint8 and logits_out.dtype == torch.float32
        st = self._C.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self._lib.cz_net_first_conv(boards.data_ptr(), B, self.w1.data_ptr(), self.b1.data_ptr(), self.x1.data_ptr(), st)
        if rc:
            raise RuntimeError("cz_net_first_conv failed (%d)" % rc)
        x = self.x1[:B].permute(0, 3, 1, 2)                                     # NCHW view of NHWC memory = channels_last
        for c1, c2 in self.blocks:
            y = self._base._conv_relu(x, c1, 1)
            x = self._base._conv_add_relu(y, c2, x)
        if not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        if B >= 128:
            rc = self._lib.cz_net_heads_tc(x.data_ptr(), B, self.wh.data_ptr(), self.bh.data_ptr(), self.w1t.data_ptr(), self.bv1.data_ptr(),
                                           self.w2.data_ptr(), self.b2t.data_ptr(), self.wp_tiled.data_ptr(), self.bp_pad.data_ptr(),
                                           self.hp_tiled.data_ptr(), self.hv.data_ptr(), logits_out.data_ptr(), value_out.data_ptr(), st)
        else:
            rc = self._lib.cz_net_heads(x.data_ptr(), B, self.wh.data_ptr(), self.bh.data_ptr(), self.w1t.data_ptr(), self.bv1.data_ptr(),
                                        self.w2.data_ptr(), self.b2t.data_ptr(), self.wp.data_ptr(), self.bp.data_ptr(), self.hp.data_ptr(), self.hv.data_ptr(),
                                        logits_out.data_ptr(), value_out.data_ptr(), st)
        if rc:
            raise RuntimeError("cz_net_heads failed (%d)" % rc)
        self._keep = x
        return None


class SmallTowerPlan(_NativeEnds):
    """fp16 plan for a FEW positions (play mode, single-tree search; BASELINE config 5): the whole convolutional trunk runs in
    ONE launch of csrc/cz_tower.cu (a thread-block cluster of 4 CTAs per position, activations resident in shared memory, weights
    streamed by TMA, wgmma accumulating in registers), followed by the value MLP || policy FC kernels of csrc/cz_net.cu:
        board bytes --cz_net_tower_small--> head features --cz_net_heads_fc--> logits, value            (3 kernels per evaluation)
    Same input / output contract as NativePlan."""

    first_conv = "tower"
    CL = 4                       # CTAs per cluster in csrc/cz_tower.cu: CTA r computes output channels [32 r, 32 r + 32)

    def __init__(self, net, max_batch, owner=None):
        super().__init__(net, max_batch, owner)
        self.fused = True
        self.n_conv = 2 * len(self._base.blocks)

    def _derive(self):
        base, CL = self._base, self.CL
        NC = 128 // CL
        d = _ends_weights(self.net, base)
        with torch.no_grad():
            convs = [c for blk in base.blocks for c in blk]                       # (w [128,128,3,3] fp16, b [128]) in execution order
            d["bias"] = torch.stack([base.w_in[1].float()] + [cb.float() for _, cb in convs]).contiguous()
            # [conv][tap][rank][k-chunk 16][out channel NC][8 in channels]: the shared-memory image of one TMA stage, see cz_tower.cu
            d["blob"] = torch.stack([cw.permute(2, 3, 0, 1).reshape(9, CL, NC, 16, 8).permute(0, 1, 3, 2, 4) for cw, _ in convs]).to(torch.float16).contiguous()
        return d

    @torch.no_grad()
    def __call__(self, boards, logits_out, value_out):
        B = boards.shape[0]
        assert B <= self.max_batch and boards.dtype == torch.uint8 and logits_out.dtype == torch.float32
        assert self.blob.numel() * 2 == self._lib.cz_net_tower_blob_bytes(self.n_conv)
        st = self._C.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self._lib.cz_net_tower_small(boards.data_ptr(), B, self.n_conv, self.w1.data_ptr(), self.blob.data_ptr(), self.bias.data_ptr(),
                                          self.wh.data_ptr(), self.bh.data_ptr(), self.hp.data_ptr(), self.hv.data_ptr(), st)
        if rc:
            raise RuntimeError("cz_net_tower_small failed (%d)" % rc)
        rc = self._lib.cz_net_heads_fc(self.hp.data_ptr(), self.hv.data_ptr(), B, self.w1t.data_ptr(), self.bv1.data_ptr(), self.w2.data_ptr(),
                                       self.b2t.data_ptr(), self.wp.data_ptr(), self.bp.data_ptr(), logits_out.data_ptr(), value_out.data_ptr(), st)
        if rc:
            raise RuntimeError("cz_net_heads_fc failed (%d)" % rc)
        return None


class _Tf32:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = self.on
        torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.prev


def train_step_module(net, opt, x, pi, z, learning_rate, c_l2=1e-4, global_norm=100, group=None):
    """One optimiser step with the reference's loss and update rule (policy_value_network.py:76-126):
    softmax cross-entropy(pi, logits) + MSE(z, value) + 1e-4 * sum(w^2)/2 over ALL trainables, Nesterov momentum,
    clip_by_global_norm(100), NaN check.  When torch.distributed is initialised with more than one rank the
    gradients are averaged with one all_reduce per step before clipping -- the data-parallel replacement of
    policy_value_network_gpus.average_gradients (policy_value_network_gpus.py:216-250): each rank's mini-batch is
    one 'tower', batch-norm statistics stay per tower exactly as in the reference's tower_loss."""
    import torch.distributed as dist
    net.train()
    for gp in opt.param_groups:
        gp["lr"] = float(learning_rate)
    logits, value = net(x)
    policy_loss = (-(pi * F.log_softmax(logits, dim=1)).sum(dim=1)).mean()
    value_loss = F.mse_loss(value, z)
    l2 = sum((p * p).sum() for p in net.parameters()) * (0.5 * c_l2)
    loss = value_loss + policy_loss + l2
    opt.zero_grad(set_to_none=True)
    loss.backward()
    params = [p for p in net.parameters() if p.grad is not None]
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        flat = torch.cat([p.grad.reshape(-1) for p in params])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat /= dist.get_world_size(group)
        o = 0
        for p in params:
            k = p.grad.numel()
            p.grad.copy_(flat[o:o + k].view_as(p.grad))
            o += k
    torch.nn.utils.clip_grad_norm_(params, global_norm)
    if not all(torch.isfinite(p.grad).all() for p in params):
        raise FloatingPointError("NaN Found!")   # tf.check_numerics, policy_value_network.py:122
    opt.step()
    accuracy = (logits.argmax(1) == pi.argmax(1)).float().mean().item()
    return accuracy, loss.item()


class policy_value_network(object):
    """Drop-in for the reference class of the same name (policy_value_network.py:8-214):
    forward(positions) -> (logits np [B,2086] f32, value np [B,1] f32); train_step; save; restore."""

    save_dir = "./models"        # policy_value_network.py:12; the gpus variant overrides it BEFORE train_restore() runs

    def __init__(self, res_block_nums=7, precision=None, device=None, seed=0, update_moving_stats=False, save_dir=None):
        if not torch.cuda.is_available():
            raise RuntimeError("policy_value_network needs a CUDA device")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.save_dir = save_dir or type(self).save_dir
        self.filters_size = 128
        self.prob_size = NLABEL
        self.c_l2 = 0.0001
        self.momentum = 0.9
        self.global_norm = 100
        self.global_step = 0
        self.precision = precision or os.environ.get("CCHESS_NN_PRECISION", "fp16")
        if seed is not None:
            torch.manual_seed(seed)
        self.net = PolicyValueNet(res_block_nums, self.filters_size, update_moving_stats).to(self.device)
        self.net = self.net.to(memory_format=torch.channels_last)
        self.opt = torch.optim.SGD(self.net.parameters(), lr=1e-3, momentum=self.momentum, nesterov=True)
        self._plan = None
        # bumped whenever the weights change (train_step / restore): every plan handed out (and every CUDA graph that captured
        # one: MCTS_tree, SelfPlay) re-folds its weight copies in place before its next search -- see InferencePlan.refresh
        self.weights_version = 0
        self.train_restore()

    # -- inference -------------------------------------------------------------------------------
    def plan(self):
        if self._plan is None:
            self.net.eval()
            self._plan = make_plan(self.net, self.precision, owner=self)
        self._plan.refresh_if_stale()
        return self._plan

    def native_plan(self, max_batch, first_conv=None):
        """fp16 plan with the hand-written first-conv / head kernels (engine path); see NativePlan.  first_conv names the first-layer
        kernel: None or "gather" (the gather-add, the only one there is)."""
        if first_conv not in (None, "gather"):
            raise ValueError("first_conv=%r: the 'tc' and 'mma' first-convolution variants were removed; only 'gather' remains" % (first_conv,))
        self.net.eval()
        return NativePlan(self.net, max_batch, owner=self)

    def small_plan(self, max_batch):
        """fp16 plan for <= 16 positions per call: the whole trunk in one cluster kernel (csrc/cz_tower.cu); see SmallTowerPlan."""
        self.net.eval()
        return SmallTowerPlan(self.net, max_batch, owner=self)

    @property
    def nn_dtype(self):
        return _DT[self.precision]

    def forward_device(self, nn_in, logits_out=None, value_out=None):
        return self.plan()(nn_in, logits_out, value_out)

    def forward(self, positions):
        """policy_value_network.py:202-214: host arrays in, host arrays out."""
        x = torch.as_tensor(np.asarray(positions, dtype=np.float32)).reshape(-1, 9, 10, 14)
        x = x.to(self.device, non_blocking=True).to(self.nn_dtype)
        logits, value = self.plan()(x)
        return logits.cpu().numpy(), value.reshape(-1, 1).cpu().numpy()

    # -- training (policy_value_network.py:76-126, 186-199) ---------------------------------------
    def train_step(self, positions, probs, winners, learning_rate):
        x = torch.as_tensor(np.asarray(positions, dtype=np.float32)).reshape(-1, 9, 10, 14).to(self.device)
        pi = torch.as_tensor(np.asarray(probs, dtype=np.float32)).to(self.device)
        z = torch.as_tensor(np.asarray(winners, dtype=np.float32)).reshape(-1, 1).to(self.device)
        return self.train_step_device(x, pi, z, learning_rate)

    def train_step_device(self, x, pi, z, learning_rate):
        """train_step on a mini-batch that is already on the device: x f32 [B,9,10,14], pi f32 [B,2086], z f32 [B,1]."""
        accuracy, loss = train_step_module(self.net, self.opt, x, pi, z, learning_rate, self.c_l2, self.global_norm)
        self.net.eval()
        self.weights_version += 1
        self.global_step += 1
        return accuracy, loss, self.global_step

    # -- checkpoints (policy_value_network.py:164-184) -------------------------------------------
    def save(self, in_global_step):
        """Same call shape and file naming as tf.train.Saver in the reference (best_model.ckpt-<step> + a `checkpoint` index);
        the payload is a torch state_dict -- the reference's TensorFlow checkpoints cannot be read (no TF in this stack, and no
        reference weights ship with the repo).  Both files are written to a temporary name and renamed: a crash never leaves
        the index pointing at a half-written checkpoint."""
        os.makedirs(self.save_dir, exist_ok=True)
        path = os.path.join(self.save_dir, "best_model.ckpt-%d" % int(in_global_step))
        tmp = path + ".tmp.%d" % os.getpid()
        torch.save(dict(model=self.net.state_dict(), opt=self.opt.state_dict(), global_step=int(in_global_step)), tmp)
        os.replace(tmp, path)
        idx = os.path.join(self.save_dir, "checkpoint")
        with open(idx + ".tmp", "w") as f:
            f.write(os.path.basename(path) + "\n")
        os.replace(idx + ".tmp", idx)
        print("Model saved in file: {}".format(path))
        return path

    def restore(self, file):
        print("Restoring from {0}".format(file))
        ck = torch.load(file, map_location=self.device, weights_only=True)   # tensors / numbers only: no arbitrary unpickling
        self.net.load_state_dict(ck["model"])
        self.opt.load_state_dict(ck["opt"])
        self.global_step = ck.get("global_step", 0)
        self.weights_version += 1

    def train_restore(self):
        idx = os.path.join(self.save_dir, "checkpoint")
        if os.path.isfile(idx):
            name = open(idx).read().strip()
            if name and os.path.isfile(os.path.join(self.save_dir, name)):
                self.restore(os.path.join(self.save_dir, name))
                print("Successfully loaded:", name)
                return
        print("Could not find old network weights")


class policy_value_network_gpus(policy_value_network):
    """policy_value_network_gpus.py:9-379 replaced the batch split over in-graph towers; here every rank
    owns one replica (one process per GPU), so the multi-GPU class is the single-GPU one per rank.
    save_dir is './gpu_models' from the start (policy_value_network_gpus.py:14), so a resumed run restores from it."""

    save_dir = "./gpu_models"

    def __init__(self, num_gpus=1, res_block_nums=7, **kw):
        super().__init__(res_block_nums, **kw)
        self.num_gpus = num_gpus
