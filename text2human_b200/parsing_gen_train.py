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

The layers (``ConvModuleL``, ``UNetL``) and the step's plumbing (``SingleSpaceTrainer``) come from
``train_layers``; the trainer composes them for ShapeUNet + FCNHead.
"""
import torch
import torch.nn as nn

from . import conv_grad as G
from . import ops
from .flat_params import ParamSpace
from .parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
from .train_layers import SingleSpaceTrainer, UNetL, conv_module

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


def backward_order(embedder, unet_layers, head):
    """the parameter-holding modules in the order the backward pass finishes their gradients"""
    return [head.conv_seg, head.convs[0].bn, head.convs[0].conv] + unet_layers.order() + embedder_linears(embedder)


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
class ParsingGenTrainer(SingleSpaceTrainer):
    """Owns the three mirror nets (``embedder`` ShapeAttrEmbedding, ``unet`` ShapeUNet, ``head`` FCNHead);
    ``optimize_parameters(data)`` is one reference training step on the batch dict of DeepFashionAttrPoseDataset
    (``densepose`` [B,1,H,W], ``attr`` [B,n_attr], ``segm`` [B,H,W] or [B,1,H,W] class ids, -100 = ignored).
    ``lr`` may be changed between steps (update_learning_rate runs on the host).  The mirrors keep their eval-mode
    inference path: after each Adam step their packed (BatchNorm-folded) weights are rebuilt from the trained
    parameters and running statistics.  Checkpoints have the reference layout (parsing_gen_model.py:185-194) plus
    the optimiser state."""

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
        self.unet_l = UNetL(self, unet)
        self.head_conv = conv_module(self, head.convs[0])
        self.space = ParamSpace(backward_order(embedder, self.unet_l, head), self.device, bucket_bytes)
        offs = []
        for m in embedder_linears(embedder):
            offs += [self.space.g(m.weight).storage_offset(), self.space.g(m.bias).storage_offset()]
        self.goff = torch.tensor(offs, dtype=torch.int64, device=self.device)
        self._out = None
        self._sync_from_rank0()

    def _nets(self):
        return dict(embedder=self.embedder, encoder=self.unet, decoder=self.head)

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
        S = self._begin_step(npix)
        sp = self.space
        packed = self.embedder._packed()
        e = ops.shape_attr_embed(attr, packed)
        # ---- ShapeUNet (unet_arch.py:657-672) and head
        x = self.unet_l.fwd(pose.reshape(B, H, W, 1) if Cp == 1 else ops.nchw_to_nhwc(pose), e)
        assert self.head.in_index in (-1, len(self.unet_l.stages) - 1), \
            "FCNHead reads the full-resolution decoder output"
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
        de = torch.zeros_like(e)
        self.unet_l.bwd(d, de)
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

    def optimize_parameters(self, data, dropout_mask=None):
        self.training_step(data, dropout_mask)
        self.adam_step()
