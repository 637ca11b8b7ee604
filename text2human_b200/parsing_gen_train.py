"""Training step of the parsing generator (``ParsingGenModel.optimize_parameters``, models/parsing_gen_model.py:80-95;
trained by train_parsing_gen.py with configs/parsing_gen.yml) on the H100 kernels.

The nets are ShapeAttrEmbedding, ShapeUNet and FCNHead (the ``parsing_gen_arch`` mirrors) in training mode:

  * every mmcv ConvModule is conv (no bias) -> BatchNorm2d with batch statistics (biased variance, eps 1e-5; running
    statistics updated with momentum 0.1 and the unbiased variance) -> ReLU: a wgmma tap-GEMM, ``norm_stats`` over
    the whole batch, and the norm apply / backward kernels with the ReLU code;
  * every ShapeUNet encoder stage reads [MaxPool2d(2) of] cat([x, embedding broadcast over H, W]) as one conversion
    (``f32_to_planes_bcast``); its backward (``maxpool2_bcast_bwd``) routes the x part to each window's first
    maximum, added to the skip connection's gradient, and sums the broadcast channels per image, in a fixed order,
    into the embedding's gradient;
  * the decoder is UNet's (bilinear x2, a 1x1 ConvModule, cat([skip, up]), two 3x3 ConvModules); the bilinear
    upsample's backward is its exact adjoint as a gather (``bilinear2x_bwd``), and the concatenation's gradient is
    split by running the first conv's data gradient once per half of its input channels;
  * FCNHead: a 3x3 ConvModule, Dropout2d (one Bernoulli per image and channel, kept channels scaled by 1/(1-p),
    applied in the norm apply before the plane split and to the gradient inside the norm backward), the 1x1
    ``conv_seg`` with bias;
  * loss: CrossEntropyLoss (F.cross_entropy with ignore_index=-100, then the mean over all B*H*W pixels, ignored ones
    included) in one fused kernel (``ce_logits``) that writes the loss sum, conv_seg's output gradient as fp16
    planes and its bias gradient;
  * the embedding's backward (``shape_attr_embed_bwd``) recomputes the tiny forward and accumulates every parameter
    gradient in fp32, in a fixed order;
  * Adam (weight_decay 0, default betas / eps) on one ``flat_params.ParamSpace``, gradient buckets all-reduced over
    the default process group while the backward pass runs, as in the other native trainers.

The layers below (``ConvModuleL``, ``BasicConvBlockL``, ``UpConvBlockL``) are those of any mmcv-style UNet; the
trainer composes them for ShapeUNet + FCNHead.
"""
import math

import torch
import torch.nn as nn

from . import conv_grad as G
from . import ops
from .dist import world_size
from .flat_params import ParamSpace, drop_packed_caches, load_checkpoint, save_checkpoint
from .parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
from .vqgan_train import Layer

NETS = ("embedder", "encoder", "decoder")      # parsing_gen.pth (parsing_gen_model.py:185-194)


class ParsingGenNets(nn.Module):
    """attr_embedder / parsing_encoder / parsing_decoder built as ParsingGenModel.__init__ does
    (parsing_gen_model.py:23-42; ``opt`` holds the keys of configs/parsing_gen.yml)"""

    def __init__(self, opt):
        super().__init__()
        self.attr_embedder = ShapeAttrEmbedding(dim=opt['embedder_dim'], out_dim=opt['embedder_out_dim'],
                                                cls_num_list=opt['attr_class_num'])
        self.parsing_encoder = ShapeUNet(in_channels=opt['encoder_in_channels'])
        self.parsing_decoder = FCNHead(in_channels=opt['fc_in_channels'], in_index=opt['fc_in_index'],
                                       channels=opt['fc_channels'], num_convs=opt['fc_num_convs'],
                                       concat_input=opt['fc_concat_input'], dropout_ratio=opt['fc_dropout_ratio'],
                                       num_classes=opt['fc_num_classes'], align_corners=opt['fc_align_corners'])


# ----------------------------------------------------------------------------
# layers with explicit forward / backward (saved tensors on a per-layer stack)
# ----------------------------------------------------------------------------
class ConvModuleL(Layer):
    """mmcv ConvModule (conv without bias -> BatchNorm2d -> ReLU) in training mode; ``fwd`` takes the conv's input
    planes, ``bwd`` the fp32 NHWC gradient of the output and returns the input operand's fp32 gradient (or, with
    ``split``, the gradients of its first ``split`` channels and of the rest, one data-gradient launch each)"""

    def __init__(self, tr, cm, need_dx=True):
        super().__init__(tr)
        self.cm, self.need_dx = cm, need_dx
        self.kind = "k3" if cm.conv.kernel_size[0] == 3 else "k1"
        bn = cm.bn
        assert bn.momentum is not None and bn.track_running_stats and cm.conv.bias is None

    def fwd(self, a, out="planes", drop=None):
        """a planes [T,N,H,W,Cin_p] -> ReLU(BN(conv(a))) [* drop[image, channel]] as planes or fp32 NHWC (``out``)"""
        _, N, H, W, _ = a.shape
        cp = self.cp(self.cm.conv)
        assert cp.co == cp.co_p, "ConvModule widths are multiples of 8"
        pre = G.forward(self.kind, a, cp.wn, None, n=N, in_hw=(H, W))
        bn = self.cm.bn
        C = cp.co
        st = ops.norm_stats(pre, C, n=1)
        ops.bn_update_running(st, bn.running_mean, bn.running_var, N * H * W, bn.momentum)
        bn.num_batches_tracked += 1
        w, b = bn.weight.detach(), bn.bias.detach()
        if out == "planes" and drop is None:
            y = ops.norm_apply(pre, st, w, b, act="relu", groups=C, eps=bn.eps, n=1)
        else:
            f, p = ops.norm_apply_ex(pre, st, w, b, act="relu", groups=C, eps=bn.eps, n=1, drop=drop,
                                     want_f32=(out == "f32"), want_planes=(out == "planes"))
            y = f if out == "f32" else p
        self.saved.append((a, pre, st, drop))
        return y

    def bwd(self, dy, split=None):
        a, pre, st, drop = self.saved.pop()
        N, H, W, _ = pre.shape
        cp = self.cp(self.cm.conv)
        bn = self.cm.bn
        _, dpre = ops.norm_bwd(pre, st, bn.weight.detach(), bn.bias.detach(), dy, act="relu", groups=cp.co,
                               eps=bn.eps, dgamma=self.gof(bn.weight), dbeta=self.gof(bn.bias), want_planes=True,
                               want_dx=False, n=1, dy_scale=drop)
        self.done(bn)
        G.wgrad(self.kind, dpre, a, cp.gw, n=N)
        self.done(self.cm.conv)
        if not self.need_dx:
            return None
        if split is None:
            return G.dgrad(self.kind, dpre, cp.wt, n=N, in_hw=(H, W))
        taps = tuple((-ty, -tx, 0) for ty, tx, _ in G.fwd_taps(self.kind, N))
        # each half of the transposed weight planes as its own (small) contiguous operand
        return tuple(ops.tap_conv(dpre, wt.contiguous(), None, taps, n=N, out_hw=(H, W))
                     for wt in (cp.wt[:, :, :split], cp.wt[:, :, split:]))


class BasicConvBlockL:
    """BasicConvBlock (unet_arch.py:113-181): ConvModules in sequence; the last one's output is fp32 NHWC (it feeds a
    pooling / upsampling conversion or a skip connection).  ``need_dx=False``: the block's input is constant (a
    frozen feature map), so its first conv computes no data gradient and ``bwd`` returns None."""

    def __init__(self, tr, blk, need_dx=True):
        self.convs = [ConvModuleL(tr, c, need_dx=need_dx or i > 0) for i, c in enumerate(blk.convs)]

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
        self.up = ConvModuleL(tr, ucb.upsample.interp_upsample[1])
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


def unet_decode_layers(tr, decoder):
    return [UpConvBlockL(tr, d) for d in decoder]


def backward_order(embedder, unet, head):
    """the parameter-holding modules in the order the backward pass finishes their gradients"""
    return [head.conv_seg, head.convs[0].bn, head.convs[0].conv] + unet_backward_order(unet) + \
        embedder_linears(embedder)


def unet_backward_order(unet):
    """a UNet's ConvModules (bn, conv) in the order the backward pass finishes them: decoder blocks from the finest,
    then encoder stages from the coarsest"""
    def cm(c):
        return [c.bn, c.conv]
    order = []
    for d in unet.decoder:
        for c in reversed(d.conv_block.convs):
            order += cm(c)
        order += cm(d.upsample.interp_upsample[1])
    for stage in reversed(unet.encoder):
        for c in reversed(stage[-1].convs):
            order += cm(c)
    return order


def embedder_linears(emb):
    """per attribute (Linear(cls_i, dim), Linear(dim, dim)), then the fusion's two Linears"""
    out = []
    for i in range(emb.attr_num):
        m = getattr(emb, f"attr_{i}")
        out += [m[0], m[2]]
    return out + [emb.fusion[0], emb.fusion[2]]


# ----------------------------------------------------------------------------
# the trainer
# ----------------------------------------------------------------------------
class ParsingGenTrainer:
    """Owns the three mirror nets (``embedder`` ShapeAttrEmbedding, ``unet`` ShapeUNet, ``head`` FCNHead);
    ``optimize_parameters(data)`` is one reference training step on the batch dict of DeepFashionAttrPoseDataset
    (``densepose`` [B,1,H,W], ``attr`` [B,n_attr], ``segm`` [B,H,W] or [B,1,H,W] class ids, -100 = ignored).
    ``lr`` may be changed between steps (update_learning_rate runs on the host).  The mirrors keep their eval-mode
    inference path: after each Adam step their packed (BatchNorm-folded) weights are rebuilt from the trained
    parameters and running statistics."""

    def __init__(self, embedder, unet, head, lr=1e-4, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8,
                 bucket_bytes=48 << 20):
        if weight_decay != 0:
            raise NotImplementedError("ParsingGenTrainer: weight_decay must be 0 (every parsing_gen config uses 0)")
        self.embedder, self.unet, self.head = embedder, unet, head
        self.lr, self.betas, self.eps = lr, betas, eps
        self.device = embedder.fusion[0].weight.device
        self.n_classes = head.num_classes
        self.p_drop = head.dropout.p if head.dropout is not None else 0.0
        # (stage 0's operand gradient is computed for its embedding channels; the pose's channel is not used)
        self.stages = [BasicConvBlockL(self, s[-1]) for s in unet.encoder]
        self.dec = unet_decode_layers(self, unet.decoder)
        self.head_conv = ConvModuleL(self, head.convs[0])
        self.space = ParamSpace(backward_order(embedder, unet, head), self.device, bucket_bytes)
        offs = []
        for m in embedder_linears(embedder):
            offs += [self.space.g(m.weight).storage_offset(), self.space.g(m.bias).storage_offset()]
        self.goff = torch.tensor(offs, dtype=torch.int64, device=self.device)
        self._out = None
        self._sync_from_rank0()

    # ---- plumbing used by the layers
    def space_of(self, mod):
        return self.space

    def space_of_param(self, p):
        return self.space

    def _nets(self):
        return dict(embedder=self.embedder, encoder=self.unet, decoder=self.head)

    def _sync_from_rank0(self):
        self.space.sync_from_rank0()
        drop_packed_caches(*self._nets().values())

    def draw_dropout_mask(self, B, generator=None):
        """nn.Dropout2d's draw: one Bernoulli(1-p) per image and channel of the head's ConvModule output"""
        return torch.empty((B, self.head.channels), device=self.device).bernoulli_(1.0 - self.p_drop,
                                                                                   generator=generator)

    # ---- one step
    def training_step(self, data, dropout_mask=None):
        """forward, loss and backward on this rank's batch; gradients are left in the flat buffer, multiplied by
        ``loss_scale`` and summed over ranks.  ``dropout_mask`` [B, head.channels] (0/1): the Dropout2d draw to use
        (default: drawn on the device as nn.Dropout2d does)."""
        dev = self.device
        pose = data['densepose'].to(dev).float().contiguous()
        attr = data['attr'].to(dev)
        segm = data['segm'].to(dev)
        B, Cp, H, W = pose.shape
        if segm.dim() == 4:
            segm = segm.squeeze(1)
        if tuple(segm.shape) != (B, H, W):
            raise ValueError(f"segm must be [B, H, W] = {(B, H, W)}, got {tuple(segm.shape)}")
        # both inputs are validated before any launch of the step (F.one_hot and F.cross_entropy reject them too)
        self.embedder.check_attributes(attr)
        ops.check_labels(segm, self.n_classes)
        attr = attr.to(torch.int64).contiguous()
        segm = segm.to(torch.int64).contiguous()
        drop = None
        if self.p_drop > 0:
            mask = dropout_mask.to(dev) if dropout_mask is not None else self.draw_dropout_mask(B)
            if tuple(mask.shape) != (B, self.head.channels):
                raise ValueError(f"dropout_mask must be [B, {self.head.channels}], got {tuple(mask.shape)}")
            drop = mask.float().div(1.0 - self.p_drop).contiguous()
        npix = B * H * W
        # static loss scale (a power of two, undone inside Adam): d loss / d logit ~ 1/npix is below fp16 resolution
        S = self.loss_scale = 2.0 ** math.floor(math.log2(npix))
        sp = self.space
        sp.flat_g.zero_()
        sp.prepare(ops.get_terms())
        packed = self.embedder._packed()
        e = ops.shape_attr_embed(attr, packed)
        Ce = e.shape[1]
        # ---- ShapeUNet encoder (unet_arch.py:657-668)
        x = pose.reshape(B, H, W, 1) if Cp == 1 else ops.nchw_to_nhwc(pose)
        enc, ins = [], []
        for i, stage in enumerate(self.stages):
            ins.append(x)
            x = stage.fwd(ops.f32_to_planes_bcast(x, e, ops.CVT_PLAIN if i == 0 else ops.CVT_MAXPOOL2))
            enc.append(x)
        # ---- decoder (unet_arch.py:669-672) and head
        x = enc[-1]
        for i in reversed(range(len(self.dec))):
            x = self.dec[i].fwd(enc[i], x)
        assert self.head.in_index in (-1, len(enc) - 1), "FCNHead reads the full-resolution decoder output"
        y = self.head_conv.fwd(ops.f32_to_planes(x), out="planes", drop=drop)
        cps = sp.convs[self.head.conv_seg]
        C = self.n_classes
        wn = cps.wn[:, :, :C] if cps.co != cps.co_p else cps.wn
        logits = G.forward("k1", y, wn, cps.b[:C], n=B, in_hw=(H, W))
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        cs = torch.zeros(C, dtype=torch.float32, device=dev)
        dlp = ops.ce_logits(logits, segm, loss, gscale=S / npix, colsum_out=cs, checked=True)
        del logits
        # ---- backward
        sp.arm(True)
        ops.add_inplace(cps.gb[:C], cs)
        G.wgrad("k1", dlp, y, cps.gw, n=B)
        sp.done(self.head.conv_seg)
        d = self.head_conv.bwd(G.dgrad("k1", dlp, cps.wt, n=B, in_hw=(H, W)))
        del dlp, y
        d_skip = [None] * len(self.dec)
        for i in range(len(self.dec)):
            d_skip[i], d = self.dec[i].bwd(d)
        de = torch.zeros((B, Ce), dtype=torch.float32, device=dev)
        for i in reversed(range(len(self.stages))):
            da = self.stages[i].bwd(d)
            if i > 0:
                d = d_skip[i - 1]
                ops.maxpool2_bcast_bwd(da, ins[i].shape[-1], Ce, x=ins[i], dx=d, de=de, pool=True,
                                       in_hw=ins[i].shape[1:3], accumulate=True)
            else:
                ops.maxpool2_bcast_bwd(da, ins[0].shape[-1], Ce, de=de, pool=False, accumulate=True)
        ops.shape_attr_embed_bwd(attr, packed, de, sp.flat_g, self.goff)
        for m in embedder_linears(self.embedder):
            sp.done(m)
        sp.release()
        self._out = dict(loss=loss, npix=npix)
        return self._out

    def losses(self):
        """the reference's log_dict (parsing_gen_model.py:95); one device->host read"""
        o = self._out
        return dict(loss_total=float(o["loss"][0]) / o["npix"])

    def adam_step(self):
        self.space.wait()
        self.space.adam(self.lr, self.betas, self.eps, 1.0 / (world_size() * self.loss_scale))
        drop_packed_caches(*self._nets().values())

    def optimize_parameters(self, data, dropout_mask=None):
        self.training_step(data, dropout_mask)
        self.adam_step()

    # ---- checkpoint / resume: the reference layout (parsing_gen_model.py:185-194) plus the optimiser state
    def save(self, path):
        save_checkpoint(path, self._nets(), self.space.state())

    def load(self, path):
        opt = load_checkpoint(path, self._nets(), self.device)
        if opt is not None:
            self.space.load_state(opt)
        self._sync_from_rank0()
