"""Training step of the top-level VQGAN on the H100 kernels: forward with saved activations, hand-written backward,
GAN losses, two flat-buffer Adam optimisers and the data-parallel gradient all-reduce.

Mirrors ``VQImageSegmTextureModel.training_step`` / ``optimize_parameters`` (models/vqgan_model.py:444-488, :329-344)
with ``models/losses/vqgan_loss.py`` (adaptive weight :5-12, hinge :21-26, DiffAugment 'color,translation' :29-80),
``Discriminator`` (models/archs/vqgan_arch.py:1155-1203, BatchNorm in training mode) and the straight-through /
legacy-beta codebook loss of ``VectorQuantizerTexture.forward`` (:270-281); ``loss.backward()`` is replaced by the
explicit backward below.  The perceptual term ``perceptual_weight * LPIPS(x, xrec)`` (vqgan_model.py:450-451) runs when
an ``lpips.LPIPS`` module is passed as ``perceptual=``; without one it is zero (BASELINE config 5, where the lpips
package and its VGG weights are not available).

Every dense contraction runs on the wgmma tap-GEMM: forward convs, data gradients (the forward kernel on transposed
weight planes with negated taps; four parity launches for the strided convs), weight gradients (``t2h_conv_wgrad``:
MN-major operands, pixel-patch contraction, split over the SMs with TMA reduce-add), and the AttnBlock products.
The HBM-bound pieces are the kernels of csrc/gan.cu.

Storage: generator and discriminator each have a ``flat_params.ParamSpace``: parameters, gradients and Adam moments
in flat fp32 buffers (conv weights tap-major, the ``nn.Parameter`` objects OIHW views of them), gradient buckets
all-reduced while the rest of the backward pass runs (the layers report each finished module with ``done``), one
Adam launch per optimiser.

A micro-batch behaves exactly like one DDP rank of the reference: its own BatchNorm batch statistics in the
discriminator, its own adaptive weight, its own DiffAugment draws; gradients of micro-batches and ranks are averaged.
"""
import math

import torch

from . import conv_grad as G
from . import ops
from .dist import world_size
from .flat_params import ParamSpace, drop_packed_caches, load_checkpoint, save_checkpoint
from .ops import CVT_PLAIN, CVT_S2D, CVT_UP2X
from .train_layers import ConvModuleL, Grad, Layer
from .vqgan_arch import AttnBlock, Decoder, Discriminator, Downsample, Encoder, ResnetBlock, Upsample

NETS = ("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv")    # the generator's nets, as checkpointed
DS = 256.0      # extra scale of the (small) attention-score gradients inside AttnBlock, undone by the consumer's alpha


# ----------------------------------------------------------------------------
# layers with explicit forward / backward (saved tensors on a per-layer stack)
# ----------------------------------------------------------------------------
class Act:
    """fp32 NHWC activation + the GroupNorm(32) statistics its producer accumulated (or None)"""
    __slots__ = ("x", "stats")

    def __init__(self, x, stats=None):
        self.x, self.stats = x, stats


def _stats(act, groups=32):
    return act.stats if act.stats is not None else ops.norm_stats(act.x, groups)


class ConvL(Layer):
    """conv (k3 / down / up2x+k3 / k1) on an fp32 NHWC activation, GroupNorm statistics of the output fused"""

    def __init__(self, tr, conv, kind, pre="plain", need_dx=True):
        super().__init__(tr)
        self.conv, self.kind, self.pre, self.need_dx = conv, kind, pre, need_dx

    def fwd(self, act):
        x = act.x
        N, H, W, _ = x.shape
        if self.pre == "s2d":
            a = ops.f32_to_planes(x, CVT_S2D)
        elif self.pre == "up2x":
            a = ops.f32_to_planes(x, CVT_UP2X)
            H, W = 2 * H, 2 * W
        else:
            a = ops.f32_to_planes(x, CVT_PLAIN)
        cp = self.cp(self.conv)
        y, st = G.forward(self.kind, a, cp.wn, cp.b, n=N, in_hw=(H, W), want_stats=True)
        self.saved.append((a, N, H, W))
        return Act(y, st)

    def bwd(self, grad):
        a, N, H, W = self.saved.pop()
        cp = self.cp(self.conv)
        dyp = grad.planes()
        self.bias_grad(cp, grad)
        G.wgrad(self.kind, dyp, a, cp.gw, n=N)
        self.done(self.conv)
        if not self.need_dx:
            return None
        dx = G.dgrad(self.kind, dyp, cp.wt, n=N, in_hw=(H, W))
        if self.pre == "up2x":
            dx = ops.sumpool2(dx)
        return Grad(dx)


class ConvInImageL(Layer):
    """network-entry conv on an fp32 NCHW image (3 -> ch): no data gradient"""

    def __init__(self, tr, conv):
        super().__init__(tr)
        self.conv = conv

    def fwd(self, x_nchw):
        N, _, H, W = x_nchw.shape
        a = ops.nchw_to_planes(x_nchw)
        cp = self.cp(self.conv)
        y, st = G.forward("k3", a, cp.wn, cp.b, n=N, in_hw=(H, W), want_stats=True)
        self.saved.append((a, N))
        return Act(y, st)

    def bwd(self, grad):
        a, N = self.saved.pop()
        cp = self.cp(self.conv)
        self.bias_grad(cp, grad)
        G.wgrad("k3", grad.planes(), a, cp.gw, n=N)
        self.done(self.conv)
        return None


class NormConvOutL(Layer):
    """GroupNorm -> swish -> 3x3 conv at the end of Encoder / Decoder (vqgan_arch.py:916-918, :1030-1032);
    ``nchw``: the decoder's image output [N,3,H,W]"""

    def __init__(self, tr, norm, conv, nchw):
        super().__init__(tr)
        self.norm, self.conv, self.nchw = norm, conv, nchw

    def fwd(self, act):
        st = _stats(act)
        a = ops.group_norm(act.x, self.norm.weight.detach(), self.norm.bias.detach(), swish=True, eps=self.norm.eps,
                           stats=st)
        N, H, W, _ = act.x.shape
        cp = self.cp(self.conv)
        wn = cp.wn[:, :, :cp.co] if cp.co != cp.co_p else cp.wn
        b = cp.b[:cp.co]
        y = G.forward("k3", a, wn, b, n=N, in_hw=(H, W), nchw_out=self.nchw)
        self.saved.append((act.x, st, a, N, H, W))
        return y

    def wgrad_only(self, dy_nchw_or_nhwc, gw):
        """weight gradient of the conv alone into ``gw`` (the adaptive weight's two autograd.grad calls,
        vqgan_loss.py:6-8), saved tensors left in place"""
        x, st, a, N, H, W = self.saved[-1]
        G.wgrad("k3", self._dy_planes(dy_nchw_or_nhwc), a, gw, n=N)

    def wgrad_pair(self, dy1, dy2):
        """the conv's weight gradients for two output gradients in ONE launch (NCHW path, Cout <= 8: the two are
        stacked along the output channels, 8 apart) -> (gw1, gw2), each shaped like the conv's gradient buffer"""
        x, st, a, N, H, W = self.saved[-1]
        cp = self.cp(self.conv)
        taps, co_p, ci_p = cp.gw.shape
        if not self.nchw or co_p != 8:
            g1, g2 = torch.zeros_like(cp.gw), torch.zeros_like(cp.gw)
            self.wgrad_only(dy1, g1)
            self.wgrad_only(dy2, g2)
            return g1, g2
        Cc = dy1.shape[1]
        both = torch.zeros((N, 16, H, W), dtype=torch.float32, device=dy1.device)
        both[:, :Cc] = dy1
        both[:, 8:8 + Cc] = dy2
        gw2 = torch.zeros((taps, 16, ci_p), dtype=torch.float32, device=dy1.device)
        G.wgrad("k3", ops.nchw_to_planes(both, c_pad=16), a, gw2, n=N)
        return gw2[:, :8].contiguous(), gw2[:, 8:].contiguous()

    def _dy_planes(self, dy):
        return ops.nchw_to_planes(dy) if self.nchw else ops.f32_to_planes(dy, CVT_PLAIN)

    def bwd(self, dy, gw_known=None):
        """``gw_known``: the conv's weight gradient for ``dy`` when the caller already has it (the trainer: by
        linearity from the adaptive weight's two gradients) -- it is added instead of being recomputed.  ``dy`` may
        be a Grad that already holds the planes and column sums (the segm tokenizer's fused BCE loss kernel)."""
        x, st, a, N, H, W = self.saved.pop()
        cp = self.cp(self.conv)
        if isinstance(dy, Grad):
            dyp = dy.p
            if cp.gb is not None:
                ops.add_inplace(cp.gb[:cp.co], dy.colsum)
        else:
            dyp = self._dy_planes(dy)
            if cp.gb is not None:
                g2 = ops.nchw_to_nhwc(dy) if self.nchw else dy
                ops.colsum_(cp.gb[:cp.co], g2.reshape(-1, cp.co))
        if gw_known is not None:
            cp.gw.add_(gw_known)
        else:
            G.wgrad("k3", dyp, a, cp.gw, n=N)
        self.done(self.conv)
        # pass 1 of the norm backward (sum du, sum du*xhat) rides in the data-gradient conv's epilogue where it can
        nb = ops.nb_context(x, st, self.norm.weight.detach(), self.norm.bias.detach(), act="swish", groups=32,
                            eps=self.norm.eps)
        da = G.dgrad("k3", dyp, cp.wt, n=N, in_hw=(H, W), nb=nb)
        cs = torch.zeros(x.shape[-1], dtype=torch.float32, device=x.device)
        dx, dxp = ops.norm_bwd(x, st, self.norm.weight.detach(), self.norm.bias.detach(), da, act="swish", groups=32,
                               eps=self.norm.eps, dgamma=self.gof(self.norm.weight), dbeta=self.gof(self.norm.bias),
                               want_planes=True, colsum_out=cs, sums=nb["sums"] if nb else None)
        self.done(self.norm)
        return Grad(dx, dxp, cs)


class ResL(Layer):
    """ResnetBlock (vqgan_arch.py:597-617; temb None, dropout 0)"""

    def __init__(self, tr, blk):
        super().__init__(tr)
        self.b = blk
        assert not blk.use_conv_shortcut

    def fwd(self, act):
        b = self.b
        x = act.x
        N, H, W, _ = x.shape
        st1 = _stats(act)
        a1 = ops.group_norm(x, b.norm1.weight.detach(), b.norm1.bias.detach(), swish=True, eps=b.norm1.eps, stats=st1)
        c1, c2 = self.cp(b.conv1), self.cp(b.conv2)
        h1, st2 = G.forward("k3", a1, c1.wn, c1.b, n=N, in_hw=(H, W), want_stats=True)
        if st2 is None:      # fewer than 2 channels per group: the statistics cannot ride in the conv epilogue
            st2 = ops.norm_stats(h1, 32)
        a2 = ops.group_norm(h1, b.norm2.weight.detach(), b.norm2.bias.detach(), swish=True, eps=b.norm2.eps, stats=st2)
        xp = None
        sc = x
        if b.in_channels != b.out_channels:
            cs = self.cp(b.nin_shortcut)
            xp = ops.f32_to_planes(x, CVT_PLAIN)
            sc = G.forward("k1", xp, cs.wn, cs.b, n=N, in_hw=(H, W))
        y, st = G.forward("k3", a2, c2.wn, c2.b, n=N, in_hw=(H, W), residual=sc, want_stats=True)
        self.saved.append((x, st1, a1, h1, st2, a2, xp, N, H, W))
        return Act(y, st)

    def bwd(self, grad):
        b = self.b
        x, st1, a1, h1, st2, a2, xp, N, H, W = self.saved.pop()
        c1, c2 = self.cp(b.conv1), self.cp(b.conv2)
        dop = grad.planes()
        self.bias_grad(c2, grad)
        G.wgrad("k3", dop, a2, c2.gw, n=N)
        self.done(b.conv2)
        nb2 = ops.nb_context(h1, st2, b.norm2.weight.detach(), b.norm2.bias.detach(), act="swish", groups=32,
                             eps=b.norm2.eps)
        d_a2 = G.dgrad("k3", dop, c2.wt, n=N, in_hw=(H, W), nb=nb2)
        d_h1, d_h1p = ops.norm_bwd(h1, st2, b.norm2.weight.detach(), b.norm2.bias.detach(), d_a2, act="swish",
                                   groups=32, eps=b.norm2.eps, dgamma=self.gof(b.norm2.weight),
                                   dbeta=self.gof(b.norm2.bias), want_planes=True, want_dx=False,
                                   colsum_out=c1.gb[:h1.shape[-1]] if c1.gb is not None else None,   # conv1's bias gradient
                                   sums=nb2["sums"] if nb2 else None)
        self.done(b.norm2)
        del d_a2, a2, h1
        G.wgrad("k3", d_h1p, a1, c1.gw, n=N)
        self.done(b.conv1)
        nb1 = ops.nb_context(x, st1, b.norm1.weight.detach(), b.norm1.bias.detach(), act="swish", groups=32,
                             eps=b.norm1.eps)
        d_a1 = G.dgrad("k3", d_h1p, c1.wt, n=N, in_hw=(H, W), nb=nb1)
        del d_h1, d_h1p, a1
        d_sc = grad.g
        if xp is not None:
            cs = self.cp(b.nin_shortcut)
            self.bias_grad(cs, grad)
            G.wgrad("k1", dop, xp, cs.gw, n=N)
            self.done(b.nin_shortcut)
            d_sc = G.dgrad("k1", dop, cs.wt, n=N, in_hw=(H, W))
        csum = torch.zeros(x.shape[-1], dtype=torch.float32, device=x.device)
        dx, dxp = ops.norm_bwd(x, st1, b.norm1.weight.detach(), b.norm1.bias.detach(), d_a1, act="swish", groups=32,
                               eps=b.norm1.eps, dgamma=self.gof(b.norm1.weight), dbeta=self.gof(b.norm1.bias),
                               add=d_sc, want_planes=True, colsum_out=csum, sums=nb1["sums"] if nb1 else None)
        self.done(b.norm1)
        return Grad(dx, dxp, csum)


class AttnL(Layer):
    """AttnBlock (vqgan_arch.py:636-661): single-head attention over the H*W tokens of each image; q | k | v as one
    projection, v and the transposed products read MN-major (no transposed copies), as the transformer's attention"""

    def __init__(self, tr, blk):
        super().__init__(tr)
        self.b = blk

    def _qkv(self):
        """-> (W [3C, C], dW, b [3C], db): q | k | v as one projection.  In the trainer's flat space the three
        weights (and biases) are adjacent, so these are views; a space with separate per-conv buffers gets one
        concatenated copy whose slices REPLACE the per-conv buffers (gradients then land where grad_of looks)."""
        mods = (self.b.q, self.b.k, self.b.v)
        q, k, v = (self.cp(m) for m in mods)
        Cc = q.co
        sp = self.tr.space_of(self.b.q)
        if isinstance(sp, ParamSpace):
            w, gw = sp.joint([m.weight for m in mods], Cc)
            b, gb = sp.joint([m.bias for m in mods])
            return w, gw, b, gb
        hit = getattr(self, "_qkv_cat", None)
        if hit is None:
            w = torch.cat([c_.w[0] for c_ in (q, k, v)], 0).contiguous()
            b = torch.cat([c_.b for c_ in (q, k, v)], 0).contiguous()
            gw, gb = torch.zeros_like(w), torch.zeros_like(b)
            for i, c_ in enumerate((q, k, v)):
                c_.w, c_.b = w[i * Cc:(i + 1) * Cc].view(1, Cc, Cc), b[i * Cc:(i + 1) * Cc]
                if c_.gw is not None:
                    c_.gw, c_.gb = gw[i * Cc:(i + 1) * Cc].view(1, Cc, Cc), gb[i * Cc:(i + 1) * Cc]
            hit = self._qkv_cat = (w, gw, b, gb)
        return hit

    def fwd(self, act):
        b = self.b
        x = act.x
        N, H, W, Cc = x.shape
        HW = H * W
        st = _stats(act)
        hn = ops.group_norm(x, b.norm.weight.detach(), b.norm.bias.detach(), swish=False, eps=b.norm.eps, stats=st)
        T = hn.shape[0]
        wqkv, _, bqkv, _ = self._qkv()
        wp = ops.f32_to_planes_rows(wqkv).unsqueeze(1)                                  # [T,1,3C,C]
        qkv = ops.linear(hn.view(T, N * HW, Cc), wp, bqkv, planes_out=True)             # [T, M, 3C]
        s = ops.mha_scores(qkv[:, :, :Cc], N, HW, 1, k=qkv[:, :, Cc:2 * Cc])            # fp32 [N,1,HW,HW]
        p = ops.softmax_rows(s, scale=float(int(Cc) ** (-0.5)))
        o = ops.mha_pv(p, qkv[:, :, 2 * Cc:], N, HW, 1, v_tok=True)                     # planes [T, M, C]
        cpo = self.cp(b.proj_out)
        y, sto = G.forward("k1", o.view(T, N, H, W, Cc), cpo.wn, cpo.b, n=N, in_hw=(H, W), residual=x, want_stats=True)
        self.saved.append((x, st, hn, wp, qkv, p, o, N, H, W))
        return Act(y, sto)

    def bwd(self, grad):
        b = self.b
        x, st, hn, wp, qkv, p, o, N, H, W = self.saved.pop()
        Cc = x.shape[-1]
        HW, M = H * W, N * H * W
        T = hn.shape[0]
        scale = float(int(Cc) ** (-0.5))
        cpo = self.cp(b.proj_out)
        dop = grad.planes().view(T, M, Cc)
        self.bias_grad(cpo, grad)
        ops.wgrad(dop, o, cpo.gw[0], k_split=ops.wgrad_k_split(Cc, Cc, M), accumulate=True)
        self.done(b.proj_out)
        d_o = ops.linear(dop, cpo.wn, w_kn=True, planes_out=True)                       # planes [T,M,C] = dY Wp
        q, k, v = qkv[:, :, :Cc], qkv[:, :, Cc:2 * Cc], qkv[:, :, 2 * Cc:]
        d_qkv = torch.empty((M, 3 * Cc), dtype=torch.float32, device=x.device)
        ops.mha_pv(p, d_o, N, HW, 1, planes_out=False, out=d_qkv[:, 2 * Cc:], p_mn=True, v_tok=True)       # dV
        dp = ops.mha_scores(d_o, N, HW, 1, k=v)                                                             # dP
        dsp = ops.softmax_bwd_planes(p, dp, scale, out_scale=DS)
        ops.mha_pv(dsp, k, N, HW, 1, planes_out=False, out=d_qkv[:, :Cc], alpha=1.0 / DS, v_tok=True)       # dQ
        ops.mha_pv(dsp, q, N, HW, 1, planes_out=False, out=d_qkv[:, Cc:2 * Cc], alpha=1.0 / DS, p_mn=True,
                   v_tok=True)                                                                              # dK
        _, gwqkv, _, gbqkv = self._qkv()
        dqkvp = ops.f32_to_planes_rows(d_qkv)
        ops.colsum_(gbqkv, d_qkv)
        ops.wgrad(dqkvp, hn.view(T, M, Cc), gwqkv, k_split=ops.wgrad_k_split(3 * Cc, Cc, M), accumulate=True)
        for m_ in (b.q, b.k, b.v):
            self.done(m_)
        d_hn = ops.linear(dqkvp, wp, w_kn=True)                                         # [M, C]
        csum = torch.zeros(Cc, dtype=torch.float32, device=x.device)
        dx, dxp = ops.norm_bwd(x, st, b.norm.weight.detach(), b.norm.bias.detach(), d_hn.view(N, H, W, Cc), act=None,
                               groups=32, eps=b.norm.eps, dgamma=self.gof(b.norm.weight),
                               dbeta=self.gof(b.norm.bias), add=grad.g, want_planes=True, colsum_out=csum)
        self.done(b.norm)
        return Grad(dx, dxp, csum)


class Lin1x1L(Layer):
    """quant_conv / post_quant_conv (vqgan_model.py:418-422): 1x1 conv on an fp32 NHWC tensor"""

    def __init__(self, tr, conv):
        super().__init__(tr)
        self.conv = conv

    def fwd(self, x, want_stats=False):
        N, H, W, _ = x.shape
        a = ops.f32_to_planes(x, CVT_PLAIN)
        cp = self.cp(self.conv)
        out = G.forward("k1", a, cp.wn, cp.b, n=N, in_hw=(H, W), want_stats=want_stats)
        self.saved.append((a, N, H, W))
        return out

    def bwd(self, grad):
        a, N, H, W = self.saved.pop()
        cp = self.cp(self.conv)
        dyp = grad.planes()
        self.bias_grad(cp, grad)
        G.wgrad("k1", dyp, a, cp.gw, n=N)
        self.done(self.conv)
        return Grad(G.dgrad("k1", dyp, cp.wt, n=N, in_hw=(H, W)))


class Seq:
    def __init__(self, layers):
        self.layers = layers

    def fwd(self, h):
        for layer in self.layers:
            h = layer.fwd(h)
        return h

    def bwd(self, g):
        for layer in reversed(self.layers):
            g = layer.bwd(g)
        return g


def encoder_layers(tr, enc):
    body = []
    for i_level in range(enc.num_resolutions):
        lvl = enc.down[i_level]
        for i_block in range(enc.num_res_blocks):
            body.append(ResL(tr, lvl.block[i_block]))
            if len(lvl.attn) > 0:
                body.append(AttnL(tr, lvl.attn[i_block]))
        if i_level != enc.num_resolutions - 1:
            body.append(ConvL(tr, lvl.downsample.conv, "down", pre="s2d"))
    body += mid_layers(tr, enc.mid)
    return ConvInImageL(tr, enc.conv_in), Seq(body), NormConvOutL(tr, enc.norm_out, enc.conv_out, nchw=False)


def mid_layers(tr, mid):
    """the middle block (ResnetBlock, AttnBlock, ResnetBlock) of an Encoder, Decoder or DecoderRes"""
    return [ResL(tr, mid.block_1), AttnL(tr, mid.attn_1), ResL(tr, mid.block_2)]


def decoder_up_layers(tr, dec, top_level, bottom_level=0):
    """the decoder's levels ``top_level`` down to ``bottom_level`` (blocks, attention, the upsample of every level but
    0), in forward order"""
    body = []
    for i_level in reversed(range(bottom_level, top_level + 1)):
        lvl = dec.up[i_level]
        for i_block in range(dec.num_res_blocks + 1):
            body.append(ResL(tr, lvl.block[i_block]))
            if len(lvl.attn) > 0:
                body.append(AttnL(tr, lvl.attn[i_block]))
        if i_level != 0:
            body.append(ConvL(tr, lvl.upsample.conv, "k3", pre="up2x"))
    return body


def decoder_layers(tr, dec):
    body = mid_layers(tr, dec.mid) + decoder_up_layers(tr, dec, dec.num_resolutions - 1)
    return ConvL(tr, dec.conv_in, "k3"), Seq(body), NormConvOutL(tr, dec.norm_out, dec.conv_out, nchw=True)


def _res_order(b):
    out = [b.conv2, b.norm2, b.conv1]
    if b.in_channels != b.out_channels:
        out.append(b.nin_shortcut)
    return out + [b.norm1]


def _attn_order(a):
    return [a.proj_out, (a.q, a.k, a.v), a.norm]


def mid_order(mid):
    """the middle block's leaf modules in backward-completion order"""
    return _res_order(mid.block_2) + _attn_order(mid.attn_1) + _res_order(mid.block_1)


def decoder_up_order(dec, top_level):
    """leaf modules of the decoder's levels 0..``top_level`` in backward-completion order (norm_out / conv_out
    excluded)"""
    order = []
    for i_level in range(top_level + 1):
        lvl = dec.up[i_level]
        if i_level != 0:
            order.append(lvl.upsample.conv)
        for i_block in reversed(range(dec.num_res_blocks + 1)):
            if len(lvl.attn) > 0:
                order += _attn_order(lvl.attn[i_block])
            order += _res_order(lvl.block[i_block])
    return order


def encoder_order(enc):
    """leaf modules of an Encoder in backward-completion order"""
    order = [enc.conv_out, enc.norm_out] + mid_order(enc.mid)
    for i_level in reversed(range(enc.num_resolutions)):
        lvl = enc.down[i_level]
        if i_level != enc.num_resolutions - 1:
            order.append(lvl.downsample.conv)
        for i_block in reversed(range(enc.num_res_blocks)):
            if len(lvl.attn) > 0:
                order += _attn_order(lvl.attn[i_block])
            order += _res_order(lvl.block[i_block])
    order.append(enc.conv_in)
    return order


def backward_order(model, disc=None):
    """leaf modules of the generator in the order the backward pass finishes their gradients"""
    dec = model.decoder
    order = [dec.conv_out, dec.norm_out] + decoder_up_order(dec, dec.num_resolutions - 1)
    order += mid_order(dec.mid) + [dec.conv_in]
    q = model.quantize
    books = list(q.embedding_list) if hasattr(q, "embedding_list") else [q.embedding]   # texture | plain quantizer
    order += [model.post_quant_conv] + books + [model.quant_conv]
    return order + encoder_order(model.encoder)


# ----------------------------------------------------------------------------
# Discriminator (vqgan_arch.py:1155-1203) forward / backward
# ----------------------------------------------------------------------------
class DiscNet(Layer):
    """conv4x4 s2 + LeakyReLU | (n_layers-1) x [conv4x4 s2, BN, LeakyReLU] | conv4x4 s1, BN, LeakyReLU | conv4x4 s1 -> 1.
    BatchNorm uses batch statistics (training mode) and updates its running statistics, as the reference's disc
    (always .train(), vqgan_model.py:412)."""

    def __init__(self, tr, disc):
        super().__init__(tr)
        mods = list(disc.main)
        self.first, self.last = mods[0], mods[-1]
        self.mid = [ConvModuleL(tr, conv, (bn,), "k4s2" if conv.stride[0] == 2 else "k4s1", "lrelu")
                    for conv, bn in zip(mods[2:-1:3], mods[3:-1:3])]

    def order(self):
        return [self.last] + [m for cm in reversed(self.mid) for m in (cm.bns[0], cm.conv)] + [self.first]

    def fwd(self, x_nchw):
        """fp32 NCHW image batch -> logits fp32 [N,h,w,1]"""
        N, _, H, W = x_nchw.shape
        c0 = self.cp(self.first)
        a0 = ops.planes_s2d(ops.nchw_to_planes(x_nchw))
        y0 = G.forward("k4s2", a0, c0.wn, c0.b, n=N, in_hw=(H, W), planes_out=True, act=ops.ACT_LRELU)
        h = y0
        for m in self.mid:
            self.cp(m.conv)     # a StandaloneSpace packs a conv's weights at its first lookup, ahead of the operand
            h = m.fwd(ops.planes_s2d(h) if m.kind == "k4s2" else h)
        cl = self.cp(self.last)
        logits = G.forward("k4s1", h, cl.wn[:, :, :1], cl.b[:1], n=N, in_hw=h.shape[2:4])
        self.saved.append((a0, y0, H, W, h))
        return logits

    def bwd(self, dlogits, want_params, want_input, dx_out=None):
        """dlogits fp32 [N,h,w,1]; parameter gradients are accumulated when ``want_params``; with ``want_input`` the
        image gradient is written to ``dx_out`` fp32 NCHW [N,3,H,W]"""
        a0, y0, H, W, h = self.saved.pop()
        _, N, hh, ww, _ = h.shape
        cl = self.cp(self.last)
        ho, wo = dlogits.shape[1:3]
        dlp = ops.nchw_to_planes(dlogits.view(N, 1, ho, wo))                 # [T,N,ho,wo,8]
        if want_params:
            ops.colsum_(cl.gb[:1], dlogits.reshape(-1, 1))
            G.wgrad("k4s1", dlp, h, cl.gw, n=N)
            self.done(self.last)
        g = G.dgrad("k4s1", dlp, cl.wt, n=N, in_hw=(hh, ww))
        for m in reversed(self.mid):
            g = m.bwd(g, want_params=want_params)
        c0 = self.cp(self.first)
        dpre, dprep = ops.lrelu_bwd(y0, g)
        if want_params:
            self.bias_grad(c0, dpre)
            G.wgrad("k4s2", dprep, a0, c0.gw, n=N)
            self.done(self.first)
        if want_input:
            G.dgrad("k4s2", dprep, c0.wt, n=N, in_hw=(H, W), cin=3, out=dx_out, d_strides=(3 * H * W, W, 1, H * W))
        return dx_out


# ----------------------------------------------------------------------------
# the trainer
# ----------------------------------------------------------------------------
class VQGANTrainer:
    """Owns a ``pipeline.VQImageSegmTextureModel`` (encoder, decoder, quantize, quant_conv, post_quant_conv) and a
    ``Discriminator``; ``optimize_parameters(data, step)`` is one reference training step."""
    fixed = None

    def __init__(self, model, disc, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, disc_start_step=0, disc_weight_max=1.0,
                 perceptual_weight=1.0, diff_aug=True, beta=0.25, micro_batch=None, bucket_bytes=48 << 20,
                 perceptual=None):
        """``perceptual``: a ``text2human_b200.lpips.LPIPS`` (frozen) adding ``perceptual_weight`` x LPIPS(x, xrec) to
        nll_loss, as the reference does; None: the perceptual term is zero"""
        self.model, self.disc = model, disc
        self.perceptual, self.perceptual_weight = perceptual, perceptual_weight
        self.lr, self.betas, self.eps = lr, betas, eps
        self.disc_start_step, self.disc_weight_max = disc_start_step, disc_weight_max
        self.diff_aug, self.beta = diff_aug, beta
        self.micro_batch = micro_batch
        self.device = next(model.parameters()).device
        dev = self.device
        order, self.quantizer = self._build(model, bucket_bytes)
        self.dnet = DiscNet(self, disc)
        self.gen = ParamSpace(order, dev, bucket_bytes)
        self.dsc = ParamSpace(self.dnet.order(), dev, bucket_bytes)
        self.spaces = [sp for sp in (self.gen, self.dsc, self.fixed) if sp is not None]
        self._space = {}
        for sp in self.spaces:
            for mod, _, _ in sp.mod_span:
                self._space[mod] = sp
        self._pspace = {}
        for sp in self.spaces:
            for p, _, _ in sp.slots:
                self._pspace[id(p)] = sp
        ws = [e.weight for e in self.quantizer.embedding_list]
        n_e, D = ws[0].shape
        cb, gcb = self.gen.joint(ws, D)
        self.codebook, self.g_codebook = cb.view(18, n_e, D), gcb.view(18, n_e, D)
        self.force_no_reduce = False    # True: no gradient all-reduce even with several ranks
        self.aug_draw_fn = None     # tests inject the reference's recorded DiffAugment draws here
        self.log = {}
        self._sync_from_rank0()

    def _build(self, model, bucket_bytes):
        """the generator's layers -> (its stepped modules in backward-completion order, its texture quantizer); a
        subclass may also set ``fixed``, a ParamSpace of modules whose gradients are computed but never stepped"""
        self.enc_in, self.enc_body, self.enc_out = encoder_layers(self, model.encoder)
        self.dec_in, self.dec_body, self.dec_out = decoder_layers(self, model.decoder)
        self.qconv, self.pqconv = Lin1x1L(self, model.quant_conv), Lin1x1L(self, model.post_quant_conv)
        return backward_order(model), model.quantize

    # ---- plumbing used by the layers
    def space_of(self, mod):
        return self._space[mod]

    def space_of_param(self, p):
        return self._pspace[id(p)]

    def wait_reduced(self):
        self.gen.wait()
        self.dsc.wait()

    def _sync_from_rank0(self):
        self.gen.sync_from_rank0()
        self.dsc.sync_from_rank0()
        drop_packed_caches(self.model, self.disc)

    # ---- random draws of DiffAugment, in the reference's order (vqgan_loss.py:47-79)
    def _aug_draws(self, B, H, W, device, generator=None):
        if self.aug_draw_fn is not None:
            return self.aug_draw_fn(B, H, W, device)
        return self.default_aug_draws(B, H, W, device, generator)

    @staticmethod
    def default_aug_draws(B, H, W, device, generator=None):
        r = torch.cat([torch.rand(B, 1, 1, 1, device=device, generator=generator).view(B, 1) for _ in range(3)], 1)
        sx, sy = int(H * 0.125 + 0.5), int(W * 0.125 + 0.5)
        tx = torch.randint(-sx, sx + 1, size=[B, 1, 1], device=device, generator=generator).view(B, 1)
        ty = torch.randint(-sy, sy + 1, size=[B, 1, 1], device=device, generator=generator).view(B, 1)
        return r.contiguous(), torch.cat([tx, ty], 1).int().contiguous()

    # ---- generator forward / backward
    def gen_forward(self, x, mask):
        m = self.model
        h = self.enc_out.fwd(self.enc_body.fwd(self.enc_in.fwd(x)))          # fp32 NHWC latent
        z = self.qconv.fwd(h)
        B, Hz, Wz, D = z.shape
        ids = ops.mask_to_ids(mask, Hz, Wz)
        r = ops.vq_search(z, self.codebook, ids, cont_stride=1024, want_list=False, want_nchw=False)
        self._vq = (z, r["idx"], ids)
        q, stq = self.pqconv.fwd(r["zq_nhwc"], want_stats=True)
        xrec = self.dec_out.fwd(self.dec_body.fwd(self.dec_in.fwd(Act(q, stq))))
        return xrec, r["sqerr"], z.numel()

    def gen_backward(self, dxrec, cb_scale, conv_out_gw=None):
        """dxrec fp32 NCHW (already multiplied by the loss scale); cb_scale = loss scale x d(loss)/d(codebook_loss);
        conv_out_gw: decoder.conv_out's weight gradient for dxrec if already known"""
        g = self.dec_in.bwd(self.dec_body.bwd(self.dec_out.bwd(dxrec, gw_known=conv_out_gw)))
        g = self.pqconv.bwd(g)
        z, idx, ids = self._vq
        nel = z.numel()
        dz = ops.vq_bwd(z, self.codebook, idx, ids, g.g, self.g_codebook, 2.0 * cb_scale / nel,
                        2.0 * self.beta * cb_scale / nel)
        for e in self.quantizer.embedding_list:
            self.gen.done(e)
        g = self.qconv.bwd(Grad(dz))
        self.enc_in.bwd(self.enc_body.bwd(self.enc_out.bwd(g.g)))
        self._vq = None

    # ---- one micro-batch
    def _micro_step(self, x, mask, step, n_micro, last, generator):
        B, _, H, W = x.shape
        dev = x.device
        S = self.loss_scale
        reduce = last and not self.force_no_reduce      # buckets fire during the LAST micro-batch's backward only
        # l1 sum, fake-logit sum, -, hinge real, hinge fake, -, -, -, then B perceptual values
        acc = torch.zeros(8 + B, dtype=torch.float64, device=dev)
        dw = torch.zeros(1, dtype=torch.float32, device=dev)
        xrec, sqerr, z_numel = self.gen_forward(x, mask)
        nel = xrec.numel()
        g_nll = ops.l1_loss(x, xrec, acc[0:1], gscale=S / nel)
        if self.perceptual is not None:
            # nll = mean(|x - xrec| + w * p_loss[b]) over [B,3,H,W]: d nll / d p_loss[b] = w / B; the trunk's
            # activations are freed here, before the discriminator's exist
            acc[8:] = self.perceptual.run(x, xrec, g=g_nll, alpha=self.perceptual_weight * S / B)
        if self.diff_aug:
            r, t = self._aug_draws(B, H, W, dev, generator)
            xr = ops.diffaug_fwd(xrec, r, t)
        else:
            xr = xrec
        logits_fake = self.dnet.fwd(xr)
        d_lf = ops.hinge_loss(logits_fake, acc[1:2], 0.0, gscale=-S / logits_fake.numel())     # g_loss = -mean
        d_xr = torch.empty_like(xrec)
        self.dnet.bwd(d_lf, want_params=False, want_input=True, dx_out=d_xr)
        g_g = ops.diffaug_bwd(d_xr, r, t) if self.diff_aug else d_xr
        # adaptive weight from the two gradients wrt decoder.conv_out.weight (vqgan_loss.py:5-12)
        rg, gg = self.dec_out.wgrad_pair(g_nll, g_g)
        ops.adaptive_weight(rg, gg, dw, 1.0 / S, self.disc_weight_max, 1.0 if step >= self.disc_start_step else 0.0)
        dxrec = ops.axpy_dev(g_nll, g_g, dw)                 # loss = nll + d_weight * g_loss + codebook_loss
        self.gen.arm(reduce)
        # conv_out's weight gradient is linear in dxrec: rg + d_weight * gg, no third weight-gradient launch
        self.gen_backward(dxrec, S, conv_out_gw=ops.axpy_dev(rg, gg, dw))
        out = dict(acc=acc, dw=dw, nel=nel, n_logit=logits_fake.numel(), sqerr=sqerr, z_numel=z_numel)
        # ---- discriminator update (step > disc_start_step, vqgan_model.py:475-486)
        if step > self.disc_start_step:
            Sd = self.disc_scale
            if self.diff_aug:
                r2, t2 = self._aug_draws(B, H, W, dev, generator)
                real_in = ops.diffaug_fwd(x, r2, t2)
            else:
                real_in = x
            lr_ = self.dnet.fwd(real_in)
            lf_ = self.dnet.fwd(xr)
            d_lr = ops.hinge_loss(lr_, acc[3:4], 1.0, gscale=0.5 * Sd / lr_.numel())
            d_lf2 = ops.hinge_loss(lf_, acc[4:5], -1.0, gscale=0.5 * Sd / lf_.numel())
            self.dsc.arm(False)
            self.dnet.bwd(d_lf2, want_params=True, want_input=False)
            self.dsc.arm(reduce)
            self.dnet.bwd(d_lr, want_params=True, want_input=False)
            out["n_dlogit"] = lr_.numel()
        return out

    def training_step(self, data, step, generator=None):
        """forward, losses, backward of generator and discriminator over all micro-batches; gradients are left in
        the flat buffers (scaled by ``loss_scale`` / ``disc_scale`` x number of micro-batches, summed over ranks)."""
        x = data['image'].float().to(self.device).contiguous()
        mask = data['texture_mask'].float().to(self.device).contiguous()
        B = x.shape[0]
        mb = self.micro_batch or B
        assert B % mb == 0
        n_micro = B // mb
        terms = ops.get_terms()
        # static loss scales (powers of two, undone inside Adam): d nll / d xrec = sign/numel would be ~1e-8
        nel = mb * x.shape[1] * x.shape[2] * x.shape[3]
        self.loss_scale = 2.0 ** math.floor(math.log2(nel))
        self.disc_scale = 2.0 ** 14
        self.n_micro = n_micro
        for sp in self.spaces:
            sp.flat_g.zero_()
            sp.prepare(terms)
        outs = []
        for i in range(n_micro):
            outs.append(self._micro_step(x[i * mb:(i + 1) * mb], mask[i * mb:(i + 1) * mb], step, n_micro,
                                         i == n_micro - 1, generator))
        for sp in self.spaces:
            sp.release()
        self._outs = outs
        self._did_disc = step > self.disc_start_step
        return outs

    def losses(self):
        """the reference's logged scalars (one device->host read; means over the micro-batches)"""
        o = self._outs
        n = len(o)
        l1 = sum(float(r["acc"][0]) / r["nel"] for r in o) / n
        p = sum(float(r["acc"][8:].mean()) for r in o) / n
        nll = l1 + self.perceptual_weight * p
        g_loss = -sum(float(r["acc"][1]) / r["n_logit"] for r in o) / n
        cb = sum((1.0 + self.beta) * float(r["sqerr"][0]) / r["z_numel"] for r in o) / n
        dw = sum(float(r["dw"][0]) for r in o) / n
        out = dict(nll_loss=nll, g_loss=g_loss, codebook_loss=cb, d_weight=dw, loss=nll + dw * g_loss + cb, l1=l1,
                   perceptual=p)
        if self._did_disc:
            out["d_loss"] = sum(0.5 * (float(r["acc"][3]) + float(r["acc"][4])) / r["n_dlogit"] for r in o) / n
        return out

    def adam_step(self):
        world = world_size()
        self.wait_reduced()
        self.gen.adam(self.lr, self.betas, self.eps, 1.0 / (world * self.n_micro * self.loss_scale))
        if self._did_disc:
            self.dsc.adam(self.lr, self.betas, self.eps, 1.0 / (world * self.n_micro * self.disc_scale))
        drop_packed_caches(self.model, self.disc)

    def optimize_parameters(self, data, step, generator=None):
        self.training_step(data, step, generator)
        self.adam_step()

    # ---- checkpoint / resume incl. optimiser state (the reference saves only the networks, vqgan_model.py:59-84)
    def _nets(self):
        return dict({k: getattr(self.model, k) for k in NETS}, discriminator=self.disc)

    def save(self, path):
        save_checkpoint(path, self._nets(), dict(gen=self.gen.state(), disc=self.dsc.state()))

    def load(self, path):
        opt = load_checkpoint(path, self._nets(), self.device)
        if opt is not None:
            self.gen.load_state(opt["gen"])
            self.dsc.load_state(opt["disc"])
        self._sync_from_rank0()
