"""Layers with explicit forward / backward shared by the native trainers, and the plumbing of a trainer whose
parameters live in one ``flat_params.ParamSpace``.

A layer keeps the tensors its backward needs on its own stack (``saved``): ``fwd`` pushes, ``bwd`` pops, so a layer
may run forward several times before its backward passes run in reverse order.  It finds its conv weights,
gradients and gradient buckets through the trainer (``space_of`` / ``space_of_param``).
"""
import math

import torch

from . import conv_grad as G
from . import ops
from .dist import world_size
from .flat_params import drop_packed_caches, load_checkpoint, save_checkpoint


class Grad:
    """gradient wrt an activation: fp32 NHWC + (optionally) its fp16 planes and its column sums (what the producing
    norm-backward kernel accumulated on the side: the bias gradient of the conv this activation came out of)"""
    __slots__ = ("g", "p", "colsum")

    def __init__(self, g, p=None, colsum=None):
        self.g, self.p, self.colsum = g, p, colsum

    def planes(self):
        if self.p is None:
            self.p = ops.f32_to_planes(self.g, ops.CVT_PLAIN)
        return self.p


class Layer:
    def __init__(self, tr):
        self.tr = tr
        self.saved = []

    def cp(self, mod):
        return self.tr.space_of(mod).convs[mod]

    def gof(self, p):
        return self.tr.space_of_param(p).g(p)

    def done(self, mod):
        self.tr.space_of(mod).done(mod)

    def bias_grad(self, cp, g):
        """cp.gb += column sums of the output gradient ``g`` (a Grad, or a bare fp32 NHWC tensor)"""
        if cp.gb is None:
            return
        t = g.g if isinstance(g, Grad) else g
        Cc = t.shape[-1]
        if isinstance(g, Grad) and g.colsum is not None:
            ops.add_inplace(cp.gb[:Cc], g.colsum)
        else:
            ops.colsum_(cp.gb[:Cc], t.reshape(-1, Cc))


class ConvModuleL(Layer):
    """conv (no bias) -> BatchNorm2d in training mode -> ReLU or LeakyReLU(0.2) (``act`` "relu" / "lrelu"): mmcv's
    ConvModule, the Discriminator's middle layers, and the index heads' 3x3 ConvModules run as one conv (a
    ``ConvStack``) with one BatchNorm per member over its own channels.  BatchNorm normalises with the batch
    statistics (biased variance) and updates the running statistics with its momentum and the unbiased variance.

    ``fwd`` takes the conv's operand planes (space-to-depth planes for "k4s2"); ``bwd`` the fp32 NHWC gradient of the
    output and returns the operand's fp32 gradient (None without ``need_dx``), or with ``split`` the gradients of its
    first ``split`` channels and of the rest, one data-gradient launch each.  ``bwd(..., want_params=False)``
    computes the data gradient alone: no parameter gradient, nothing reported ``done``."""

    def __init__(self, tr, conv, bns, kind, act, need_dx=True):
        super().__init__(tr)
        self.conv, self.bns, self.kind, self.act, self.need_dx = conv, tuple(bns), kind, act, need_dx
        bn0 = self.bns[0]
        assert getattr(conv, "bias", None) is None
        assert all(bn.eps == bn0.eps and bn.momentum == bn0.momentum and bn.momentum is not None
                   and bn.track_running_stats for bn in self.bns)
        self.eps, self.momentum = bn0.eps, bn0.momentum
        if len(self.bns) == 1:
            self.gamma = None           # the module's own parameters, looked up per call (the flat store rebinds them)
            self.rmean, self.rvar, self.nbt = bn0.running_mean, bn0.running_var, bn0.num_batches_tracked
            return
        sp = tr.space_of(bn0)
        self.gamma, self.dgamma = sp.joint([bn.weight for bn in self.bns])
        self.beta, self.dbeta = sp.joint([bn.bias for bn in self.bns])
        # running statistics and step counters: views into one buffer each, so that one bn_update_running launch
        # (and one increment) serves every BatchNorm; state_dict / load_state_dict see the same tensors as before
        C = bn0.num_features
        with torch.no_grad():
            self.rmean = torch.cat([bn.running_mean.float() for bn in self.bns]).contiguous()
            self.rvar = torch.cat([bn.running_var.float() for bn in self.bns]).contiguous()
            self.nbt = torch.stack([bn.num_batches_tracked for bn in self.bns]).contiguous()
        for k, bn in enumerate(self.bns):
            bn.running_mean = self.rmean[k * C:(k + 1) * C]
            bn.running_var = self.rvar[k * C:(k + 1) * C]
            bn.num_batches_tracked = self.nbt[k]

    def _affine(self):
        if self.gamma is not None:
            return self.gamma, self.beta
        bn = self.bns[0]
        return bn.weight.detach(), bn.bias.detach()

    def fwd(self, a, out="planes", drop=None):
        """a planes [T,N,H,W,Cin] (or [T,4,N,H/2,W/2,Cin]) -> act(BN(conv(a))) [* drop[image, channel]] as planes
        or fp32 NHWC (``out``)"""
        if a.dim() == 6:
            N, H, W = a.shape[2], 2 * a.shape[3], 2 * a.shape[4]
        else:
            _, N, H, W, _ = a.shape
        cp = self.cp(self.conv)
        assert cp.co == cp.co_p, "BatchNorm'd conv widths are multiples of 8"
        pre = G.forward(self.kind, a, cp.wn, None, n=N, in_hw=(H, W))
        C = cp.co
        gamma, beta = self._affine()
        st = ops.norm_stats(pre, C, n=1)
        ops.bn_update_running(st, self.rmean, self.rvar, pre.numel() // C, self.momentum)
        self.nbt += 1
        if out == "planes" and drop is None:
            y = ops.norm_apply(pre, st, gamma, beta, act=self.act, groups=C, eps=self.eps, n=1)
        else:
            f, p = ops.norm_apply_ex(pre, st, gamma, beta, act=self.act, groups=C, eps=self.eps, n=1, drop=drop,
                                     want_f32=(out == "f32"), want_planes=(out == "planes"))
            y = f if out == "f32" else p
        self.saved.append((a, pre, st, drop, H, W))
        return y

    def bwd(self, dy, split=None, want_params=True):
        a, pre, st, drop, H, W = self.saved.pop()
        N = pre.shape[0]
        cp = self.cp(self.conv)
        gamma, beta = self._affine()
        dgamma = dbeta = None
        if want_params:
            if self.gamma is not None:
                dgamma, dbeta = self.dgamma, self.dbeta
            else:
                dgamma, dbeta = self.gof(self.bns[0].weight), self.gof(self.bns[0].bias)
        _, dpre = ops.norm_bwd(pre, st, gamma, beta, dy, act=self.act, groups=cp.co, eps=self.eps, dgamma=dgamma,
                               dbeta=dbeta, want_planes=True, want_dx=False, n=1, dy_scale=drop)
        if want_params:
            for bn in self.bns:
                self.done(bn)
            G.wgrad(self.kind, dpre, a, cp.gw, n=N)
            self.done(self.conv)
        if not self.need_dx:
            return None
        if split is None:
            return G.dgrad(self.kind, dpre, cp.wt, n=N, in_hw=(H, W))
        taps = tuple((-ty, -tx, 0) for ty, tx, _ in G.fwd_taps(self.kind, N))
        # each half of the transposed weight planes as its own (small) contiguous operand
        return tuple(ops.tap_conv(dpre, wt.contiguous(), None, taps, n=N, out_hw=(H, W))
                     for wt in (cp.wt[:, :, :split], cp.wt[:, :, split:]))


def conv_module(tr, cm, need_dx=True):
    """the ConvModuleL of an mmcv ConvModule (conv 3x3 or 1x1 -> BatchNorm2d -> ReLU)"""
    return ConvModuleL(tr, cm.conv, (cm.bn,), "k3" if cm.conv.kernel_size[0] == 3 else "k1", "relu", need_dx)


class BasicConvBlockL:
    """BasicConvBlock (unet_arch.py:113-181): ConvModules in sequence; the last one's output is fp32 NHWC (it feeds a
    pooling / upsampling conversion or a skip connection).  ``need_dx=False``: the block's input is constant (a
    frozen feature map), so its first conv computes no data gradient and ``bwd`` returns None."""

    def __init__(self, tr, blk, need_dx=True):
        self.convs = [conv_module(tr, c, need_dx=need_dx or i > 0) for i, c in enumerate(blk.convs)]

    def fwd(self, a):
        n = len(self.convs)
        for i, c in enumerate(self.convs):
            a = c.fwd(a, out="f32" if i == n - 1 else "planes")
        return a

    def bwd(self, d, split=None):
        for i in reversed(range(len(self.convs))):
            d = self.convs[i].bwd(d, split=split if i == 0 else None)
        return d


class UpConvBlockL:
    """UpConvBlock (unet_arch.py:12-110) with InterpConv upsampling: bilinear x2 -> 1x1 ConvModule, cat([skip, up]),
    conv block.  ``bwd`` -> (gradient of the skip map, gradient of the coarse input), both fp32 NHWC"""

    def __init__(self, tr, ucb):
        self.up = conv_module(tr, ucb.upsample.interp_upsample[1])
        self.block = BasicConvBlockL(tr, ucb.conv_block)
        self.saved = []

    def fwd(self, skip, x):
        up = self.up.fwd(ops.f32_to_planes(x, ops.CVT_BILINEAR2X))
        self.saved.append(skip.shape[-1])
        return self.block.fwd(torch.cat((ops.f32_to_planes(skip), up), dim=-1))    # torch.cat([skip, x], 1) :107

    def bwd(self, d):
        cs = self.saved.pop()
        d_skip, d_up = self.block.bwd(d, split=cs)
        return d_skip, ops.bilinear2x_bwd(self.up.bwd(d_up))


class UNetL:
    """The encoder stages and decoder blocks of a UNet (unet_arch.py:460-471) or ShapeUNet (:657-672).  Stage i > 0
    reads MaxPool2d(2) of the previous stage's output, whose backward routes to each window's first maximum, added
    into the skip connection's gradient.  ShapeUNet appends an embedding broadcast over H, W to every stage's operand
    (``e``); its gradient is summed per image, in a fixed order.  ``need_dx=False``: the input is constant and there
    is no embedding, so stage 0 computes no data gradient."""

    def __init__(self, tr, unet, need_dx=True):
        self.stages = [BasicConvBlockL(tr, s[-1], need_dx=need_dx or i > 0) for i, s in enumerate(unet.encoder)]
        self.dec = [UpConvBlockL(tr, d) for d in unet.decoder]
        self.saved = []

    def order(self):
        """the ConvModules' (bn, conv) in the order the backward pass finishes them: decoder blocks from the finest,
        then encoder stages from the coarsest"""
        cms = []
        for d in self.dec:
            cms += reversed([d.up] + d.block.convs)
        for stage in reversed(self.stages):
            cms += reversed(stage.convs)
        return [m for cm in cms for m in (cm.bns[0], cm.conv)]

    def fwd(self, x, e=None):
        """x fp32 NHWC [N,H,W,C], e fp32 [N,Ce] or None -> the full-resolution decoder output, fp32 NHWC"""
        enc = []
        for i, stage in enumerate(self.stages):
            src, mode = (x, ops.CVT_PLAIN) if i == 0 else (enc[-1], ops.CVT_MAXPOOL2)
            a = ops.f32_to_planes(src, mode) if e is None else ops.f32_to_planes_bcast(src, e, mode)
            enc.append(stage.fwd(a))
        self.saved.append((x.shape[-1], enc))
        y = enc[-1]
        for i in reversed(range(len(self.dec))):
            y = self.dec[i].fwd(enc[i], y)
        return y

    def bwd(self, d, de=None):
        """d fp32 NHWC gradient of the output; the embedding's gradient is added into ``de`` fp32 [N,Ce] (when
        ``fwd`` was given ``e``)"""
        c0, enc = self.saved.pop()
        c_e = 0 if de is None else de.shape[1]
        d_skip = []
        for blk in self.dec:
            s, d = blk.bwd(d)
            d_skip.append(s)
        for i in reversed(range(len(self.stages))):
            da = self.stages[i].bwd(d)
            if i > 0:
                x, d = enc[i - 1], d_skip[i - 1]
                ops.maxpool2_bcast_bwd(da, x.shape[-1], c_e, x=x, dx=d, de=de, pool=True, in_hw=x.shape[1:3],
                                       accumulate=True)
            elif de is not None:
                ops.maxpool2_bcast_bwd(da, c0, c_e, de=de, pool=False, accumulate=True)


class SingleSpaceTrainer:
    """Plumbing of a trainer whose parameters, gradients and Adam moments live in one ParamSpace.  A subclass sets
    ``space``, ``device``, ``lr``, ``betas`` and ``eps`` and defines ``_nets()``, the checkpoint's
    {name: module}."""

    # ---- used by the layers
    def space_of(self, mod):
        return self.space

    def space_of_param(self, p):
        return self.space

    def _sync_from_rank0(self):
        self.space.sync_from_rank0()
        drop_packed_caches(*self._nets().values())

    def _begin_step(self, n):
        """-> the step's static loss scale 2^floor(log2 n), a power of two undone inside Adam (d loss / d output ~
        1/n of a mean over n elements is below fp16 resolution); zeroes the gradients and makes the weight planes"""
        S = self.loss_scale = 2.0 ** math.floor(math.log2(n))
        self.space.flat_g.zero_()
        self.space.prepare(ops.get_terms())
        return S

    def adam_step(self):
        self.space.wait()
        self.space.adam(self.lr, self.betas, self.eps, 1.0 / (world_size() * self.loss_scale))
        drop_packed_caches(*self._nets().values())

    # ---- checkpoint / resume: the reference layout of ``_nets()`` plus the optimiser state
    def save(self, path):
        save_checkpoint(path, self._nets(), self.space.state())

    def load(self, path):
        opt = load_checkpoint(path, self._nets(), self.device)
        if opt is not None:
            self.space.load_state(opt)
        self._sync_from_rank0()
