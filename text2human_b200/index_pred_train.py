"""Training step of the index-prediction nets (``VQGANTextureAwareSpatialHierarchyInferenceModel.feed_data`` /
``optimize_parameters``, models/hierarchy_inference_model.py:178-245; trained by train_index_prediction.py with
configs/index_pred_net.yml) on the H100 kernels.

  * ground truth from the frozen hierarchy (``feed_data``): ``feature_t`` = the top level's post-quant-conv feature
    (``top_encode_nhwc``, kept NHWC for the UNet) and, per latent position, the bottom quantizer's own-codebook index
    and texture id (bot_encoder -> bot_quant_conv -> the 2x2-patch ``vq_search``); ``bot_decoder_res`` is not run;
  * the UNet guidance encoder (the ``index_pred_arch`` mirror) in training mode through the parsing generator's
    layers (``BasicConvBlockL`` / ``UpConvBlockL``: conv -> BatchNorm2d on batch statistics -> ReLU); stage i > 0
    reads MaxPool2d(2) of the previous stage, whose backward routes to each window's first maximum, added into that
    stage's skip gradient; stage 0's input is the frozen feature, so its first conv computes no data gradient;
  * the 18 heads of MultiHeadFCNHead: their 3x3 ConvModules run as ONE conv of 18*64 output channels (a
    ``ConvStack`` in the parameter store), one BatchNorm over 1152 channels (the 18 BatchNorms' parameters and
    running statistics are views of shared buffers), and the 18 Dropout2d draws as one head-major [B, 1152] factor;
  * loss: the sum over heads of CrossEntropyLoss(ignore_index=-1), i.e. each position's cross-entropy in its own
    texture's head (every other head ignores it), summed and divided by B*h*w, in one routed kernel
    (``routed_head_ce``) that scores each position with its own head only and writes the conv_seg gradients straight
    into the flat gradient store;
  * Adam (weight_decay 0) on one ``flat_params.ParamSpace``, gradient buckets all-reduced over the default process
    group while the backward pass runs, as in the other native trainers.
"""
import math

import torch
import torch.nn as nn

from . import conv_grad as G
from . import ops
from .dist import world_size
from .flat_params import ConvStack, ParamSpace, drop_packed_caches, load_checkpoint, save_checkpoint
from .index_pred_arch import MultiHeadFCNHead, UNet
from .parsing_gen_train import BasicConvBlockL, unet_backward_order, unet_decode_layers
from .vqgan_arch import conv1x1_nhwc
from .vqgan_train import Layer

NETS = ("guidance_encoder", "index_decoder")    # index_pred_net.pth (hierarchy_inference_model.py:310-323)
IGNORE = -1                                     # the reference's ignore_index


class IndexPredNets(nn.Module):
    """guidance_encoder / index_decoder built as the reference's __init__ does (hierarchy_inference_model.py:89-103;
    ``opt`` holds the keys of configs/index_pred_net.yml)"""

    def __init__(self, opt):
        super().__init__()
        self.guidance_encoder = UNet(in_channels=opt['encoder_in_channels'])
        self.index_decoder = MultiHeadFCNHead(
            in_channels=opt['fc_in_channels'], in_index=opt['fc_in_index'], channels=opt['fc_channels'],
            num_convs=opt['fc_num_convs'], concat_input=opt['fc_concat_input'],
            dropout_ratio=opt['fc_dropout_ratio'], num_classes=opt['fc_num_classes'],
            align_corners=opt['fc_align_corners'], num_head=18)


class HeadConvsL(Layer):
    """The heads' 3x3 ConvModules as one stacked ConvModule in training mode: conv (64 -> 18*64), BatchNorm2d over
    the 1152 stacked channels (each channel's statistics are its own head's), ReLU, Dropout2d factor; ``fwd`` -> the
    fp32 NHWC [B,h,w,18*64] that conv_seg reads, ``bwd`` -> the fp32 gradient of the input feature map."""

    def __init__(self, tr, fcn, stack):
        super().__init__(tr)
        self.stack = stack
        self.bns = tuple(seq[0].bn for seq in fcn.convs_list)
        bn0 = self.bns[0]
        assert all(bn.eps == bn0.eps and bn.momentum == bn0.momentum and bn.track_running_stats for bn in self.bns)
        self.eps, self.momentum = bn0.eps, bn0.momentum
        sp = tr.space
        self.gamma, self.dgamma = sp.joint([bn.weight for bn in self.bns])
        self.beta, self.dbeta = sp.joint([bn.bias for bn in self.bns])
        # running statistics and step counters: views into one buffer each, so that one bn_update_running launch
        # (and one increment) serves the 18 BatchNorms; state_dict / load_state_dict see the same tensors as before
        C = fcn.channels
        with torch.no_grad():
            self.rmean = torch.cat([bn.running_mean.float() for bn in self.bns]).contiguous()
            self.rvar = torch.cat([bn.running_var.float() for bn in self.bns]).contiguous()
            self.nbt = torch.stack([bn.num_batches_tracked for bn in self.bns]).contiguous()
        for k, bn in enumerate(self.bns):
            bn.running_mean = self.rmean[k * C:(k + 1) * C]
            bn.running_var = self.rvar[k * C:(k + 1) * C]
            bn.num_batches_tracked = self.nbt[k]

    def fwd(self, a, drop):
        """a planes [T,B,h,w,Cin] -> ReLU(BN(conv(a))) [* drop[image, channel]] fp32 NHWC"""
        _, N, H, W, _ = a.shape
        cp = self.cp(self.stack)
        pre = G.forward("k3", a, cp.wn, None, n=N, in_hw=(H, W))
        st = ops.norm_stats(pre, cp.co, n=1)
        ops.bn_update_running(st, self.rmean, self.rvar, N * H * W, self.momentum)
        self.nbt += 1
        y, _ = ops.norm_apply_ex(pre, st, self.gamma, self.beta, act="relu", groups=cp.co, eps=self.eps, n=1,
                                 drop=drop, want_f32=True)
        self.saved.append((a, pre, st, drop))
        return y

    def bwd(self, dy):
        a, pre, st, drop = self.saved.pop()
        N, H, W, _ = pre.shape
        cp = self.cp(self.stack)
        _, dpre = ops.norm_bwd(pre, st, self.gamma, self.beta, dy, act="relu", groups=cp.co, eps=self.eps,
                               dgamma=self.dgamma, dbeta=self.dbeta, want_planes=True, want_dx=False, n=1,
                               dy_scale=drop)
        for bn in self.bns:
            self.done(bn)
        G.wgrad("k3", dpre, a, cp.gw, n=N)
        self.done(self.stack)
        return G.dgrad("k3", dpre, cp.wt, n=N, in_hw=(H, W))


class IndexPredTrainer:
    """Owns the two mirror nets (``unet`` index_pred_arch.UNet, ``fcn`` MultiHeadFCNHead) and, for ``feed_data``,
    the frozen ``hierarchy`` (a pipeline.HierarchyVQSpatialTextureAwareModel loaded from vqvae_top.pth /
    vqvae_bottom.pth; may be None when the caller supplies the ground truth).  ``optimize_parameters`` is one
    reference training step; ``lr`` may be changed between steps.  The nets stay in eval mode: their inference path
    (``UNet.forward_nhwc``, ``MultiHeadFCNHead.forward_logits``, ``bot_index_prediction``) sees the trained
    parameters and running statistics after every Adam step and every load."""

    def __init__(self, unet, fcn, hierarchy=None, lr=1e-4, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8,
                 bucket_bytes=48 << 20):
        if weight_decay != 0:
            raise NotImplementedError("IndexPredTrainer: weight_decay must be 0 (configs/index_pred_net.yml uses 0)")
        if fcn.in_index not in (-1, unet.num_stages - 1):
            raise NotImplementedError("MultiHeadFCNHead must read the UNet's full-resolution output (fc_in_index 4)")
        self.unet, self.fcn, self.hierarchy = unet.eval(), fcn.eval(), hierarchy
        self.lr, self.betas, self.eps = lr, betas, eps
        self.device = fcn.conv_seg_head_list[0].weight.device
        self.n_head, self.n_classes, self.channels = fcn.num_head, fcn.num_classes, fcn.channels
        self.p_drop = fcn.dropout.p if fcn.dropout is not None else 0.0
        self.stack = ConvStack(seq[0].conv for seq in fcn.convs_list)
        self.segs = tuple(fcn.conv_seg_head_list)
        bns = tuple(seq[0].bn for seq in fcn.convs_list)
        self.space = ParamSpace([self.segs, bns, self.stack] + unet_backward_order(unet), self.device, bucket_bytes)
        G_, K, C = self.n_head, self.n_classes, self.channels
        w, gw = self.space.joint([c.weight for c in self.segs], C)
        b, gb = self.space.joint([c.bias for c in self.segs])
        self.w_seg, self.gw_seg = w.view(G_, K, C), gw.view(G_, K, C)
        self.b_seg, self.gb_seg = b.view(G_, K), gb.view(G_, K)
        self.stages = [BasicConvBlockL(self, s[-1], need_dx=i > 0) for i, s in enumerate(unet.encoder)]
        self.dec = unet_decode_layers(self, unet.decoder)
        self.head = HeadConvsL(self, fcn, self.stack)
        self._gt = None
        self._out = None
        self._sync_from_rank0()

    # ---- plumbing used by the layers
    def space_of(self, mod):
        return self.space

    def space_of_param(self, p):
        return self.space

    def _nets(self):
        return dict(guidance_encoder=self.unet, index_decoder=self.fcn)

    def _sync_from_rank0(self):
        self.space.sync_from_rank0()
        drop_packed_caches(*self._nets().values())

    def draw_dropout_mask(self, B, generator=None):
        """the 18 nn.Dropout2d draws of one step, in head order: [num_head, B, channels] Bernoulli(1-p)"""
        return torch.empty((self.n_head, B, self.channels), device=self.device).bernoulli_(1.0 - self.p_drop,
                                                                                          generator=generator)

    # ---- inputs
    def _check_images(self, data):
        if not isinstance(data, dict) or 'image' not in data or 'texture_mask' not in data:
            raise ValueError("a batch is a dict with 'image' [B,3,H,W] and 'texture_mask' [B,1,H,W]")
        image, mask = data['image'], data['texture_mask']
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be [B, 3, H, W], got {tuple(image.shape)}")
        B, _, H, W = image.shape
        if H % 256 or W % 256:
            raise ValueError(f"image H, W must be multiples of 256 (the 1/16 latent feeds a UNet that pools 4 times), "
                             f"got {H}x{W}")
        if tuple(mask.shape) != (B, 1, H, W):
            raise ValueError(f"texture_mask must be [B, 1, H, W] = {(B, 1, H, W)}, got {tuple(mask.shape)}")
        if self.hierarchy is None:
            raise ValueError("feed_data needs the frozen hierarchy (IndexPredTrainer(..., hierarchy=...))")

    @torch.no_grad()
    def feed_data(self, data):
        """the reference's feed_data on a batch dict (image [B,3,H,W] in [-1,1], texture_mask [B,1,H,W] texture ids):
        -> dict(feature_t fp32 NHWC [B,h,w,256], own int64 [B,h,w] own-codebook index, tex int64 [B,h,w] texture
        id), kept for the next training_step"""
        self._check_images(data)
        dev = self.device
        image = data['image'].to(dev).float().contiguous()
        mask = data['texture_mask'].to(dev).float()
        hier = self.hierarchy
        feature_t, _ = hier.top_encode_nhwc(image, mask)
        z = conv1x1_nhwc(hier.bot_encoder.forward_nhwc(image), hier.bot_quant_conv)
        q = hier.bot_quantize
        ps = q.spatial_size
        ids = ops.mask_to_ids(mask, z.shape[1] // ps, z.shape[2] // ps)
        r = ops.vq_search(z, q._codebook(), ids, ps=ps, cont_stride=q.n_e, want_list=False, want_nchw=False,
                          want_nhwc=False, want_err=False)
        self._gt = dict(feature_t=feature_t, own=r["idx"], tex=ids.long())
        return self._gt

    def _batch(self, data, feature_t, targets):
        """-> (feature fp32 NHWC, own, tex), every caller-supplied input checked before any launch"""
        if feature_t is None:
            if targets is not None:
                raise ValueError("targets come with feature_t")
            if data is not None:
                self.feed_data(data)
            if self._gt is None:
                raise ValueError("no batch: pass data (or call feed_data), or feature_t and targets")
            return self._gt["feature_t"], self._gt["own"], self._gt["tex"]
        if targets is None or len(targets) != 2:
            raise ValueError("feature_t needs targets = (own-codebook index [B,h,w], texture id [B,h,w])")
        if feature_t.dim() != 4 or feature_t.shape[1] != self.unet.encoder[0][-1].convs[0].conv.in_channels:
            raise ValueError(f"feature_t must be [B, {self.unet.encoder[0][-1].convs[0].conv.in_channels}, h, w], "
                             f"got {tuple(feature_t.shape)}")
        B, _, h, w = feature_t.shape
        f = 2 ** (self.unet.num_stages - 1)
        if h % f or w % f:
            raise ValueError(f"feature_t h, w must be multiples of {f} (the UNet pools {self.unet.num_stages - 1} "
                             f"times), got {h}x{w}")
        own, tex = targets
        for name, t in (("own", own), ("tex", tex)):
            if tuple(t.shape) != (B, h, w):
                raise ValueError(f"{name} must be [B, h, w] = {(B, h, w)}, got {tuple(t.shape)}")
        own, tex = own.to(self.device), tex.to(self.device)
        ops.check_routed_targets(tex, own, self.n_head, self.n_classes, IGNORE)
        x = ops.nchw_to_nhwc(feature_t.to(self.device).float().contiguous())
        return x, own.to(torch.int64), tex.to(torch.int64)

    def _drop_factor(self, dropout_mask, B):
        if self.p_drop <= 0:
            if dropout_mask is not None:
                raise ValueError("dropout_mask given, but the heads have no Dropout2d (dropout_ratio 0)")
            return None
        mask = dropout_mask.to(self.device) if dropout_mask is not None else self.draw_dropout_mask(B)
        if tuple(mask.shape) != (self.n_head, B, self.channels):
            raise ValueError(f"dropout_mask must be [{self.n_head}, {B}, {self.channels}], got {tuple(mask.shape)}")
        return mask.float().div(1.0 - self.p_drop).permute(1, 0, 2).reshape(B, -1).contiguous()

    # ---- one step
    def training_step(self, data=None, dropout_mask=None, *, feature_t=None, targets=None):
        """forward, loss and backward on this rank's batch; gradients are left in the flat buffer, multiplied by
        ``loss_scale`` and summed over ranks.  The batch is ``data`` (run through the frozen hierarchy), else the
        ground truth of the last feed_data, else ``feature_t`` (fp32 NCHW [B,256,h,w]) with ``targets`` = (own
        index, texture id), each int [B,h,w]: a position whose texture id lies outside [0, 18) or whose target is
        -1 is ignored.  ``dropout_mask`` [18, B, channels] (0/1): the heads' Dropout2d draws in head order (default:
        drawn on the device)."""
        if feature_t is not None:
            B = feature_t.shape[0]
        elif data is not None:
            self._check_images(data)
            B = data['image'].shape[0]
        else:
            B = self._gt["feature_t"].shape[0] if self._gt is not None else 0
        drop = self._drop_factor(dropout_mask, B)       # checked before feed_data launches anything
        x, own, tex = self._batch(data, feature_t, targets)
        B, h, w, _ = x.shape
        M = B * h * w
        # static loss scale (a power of two, undone inside Adam): d loss / d logit ~ 1/M is below fp16 resolution
        S = self.loss_scale = 2.0 ** math.floor(math.log2(M))
        sp = self.space
        sp.flat_g.zero_()
        sp.prepare(ops.get_terms())
        # ---- UNet encoder / decoder (unet_arch.py:460-471)
        a = ops.f32_to_planes(x)
        enc = []
        for i, stage in enumerate(self.stages):
            if i > 0:
                a = ops.f32_to_planes(enc[-1], ops.CVT_MAXPOOL2)
            enc.append(stage.fwd(a))
        x = enc[-1]
        for i in reversed(range(len(self.dec))):
            x = self.dec[i].fwd(enc[i], x)
        # ---- heads and the routed loss
        y = self.head.fwd(ops.f32_to_planes(x), drop)
        loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        sp.arm(True)
        dy = ops.routed_head_ce(y.view(M, -1), tex, own, self.w_seg, self.b_seg, loss, self.gw_seg, self.gb_seg,
                                gscale=S / M)
        del y
        for c in self.segs:
            sp.done(c)
        # ---- backward
        d = self.head.bwd(dy.view(B, h, w, -1))
        del dy
        d_skip = [None] * len(self.dec)
        for i in range(len(self.dec)):
            d_skip[i], d = self.dec[i].bwd(d)
        for i in reversed(range(len(self.stages))):
            da = self.stages[i].bwd(d)
            if i > 0:
                d = d_skip[i - 1]
                ops.maxpool2_bcast_bwd(da, enc[i - 1].shape[-1], 0, x=enc[i - 1], dx=d, pool=True,
                                       in_hw=enc[i - 1].shape[1:3], accumulate=True)
        sp.release()
        self._out = dict(loss=loss, npix=M)
        return self._out

    def losses(self):
        """the reference's log_dict (hierarchy_inference_model.py:245); one device->host read"""
        o = self._out
        return dict(loss_total=float(o["loss"][0]) / o["npix"])

    def adam_step(self):
        self.space.wait()
        self.space.adam(self.lr, self.betas, self.eps, 1.0 / (world_size() * self.loss_scale))
        drop_packed_caches(*self._nets().values())

    def optimize_parameters(self, data=None, dropout_mask=None, *, feature_t=None, targets=None):
        self.training_step(data, dropout_mask, feature_t=feature_t, targets=targets)
        self.adam_step()

    # ---- the reference's validation metric (hierarchy_inference_model.py:247-298, without the image dumps)
    @torch.no_grad()
    def accuracy(self, data=None, *, feature_t=None, targets=None):
        """share of latent positions (ignored ones count in the denominator, as in the reference) whose own head's
        argmax equals the ground-truth index, eval-mode nets; ``data`` is a batch dict or an iterable of them"""
        if feature_t is not None:
            batches = [(None, feature_t, targets)]
        else:
            batches = ((d, None, None) for d in ([data] if isinstance(data, dict) else data))
        acc, num = 0.0, 0
        for batch in batches:           # one batch's ground truth alive at a time
            x, own, tex = self._batch(*batch)
            B, h, w, _ = x.shape
            feat = self.unet.forward_nhwc(x, nhwc_in=True)[self.fcn.in_index]
            tex = tex.reshape(-1)
            pred = ops.argmax_heads(self.fcn.forward_logits(feat), tex)
            live = (tex >= 0) & (tex < self.n_head)
            acc += float(((pred == own.reshape(-1)) & live).sum()) / (h * w)
            num += B
        return acc / num

    # ---- checkpoint / resume: the reference layout (hierarchy_inference_model.py:310-323) plus the optimiser state
    def save(self, path):
        save_checkpoint(path, self._nets(), self.space.state())

    def load(self, path):
        opt = load_checkpoint(path, self._nets(), self.device)
        if opt is not None:
            self.space.load_state(opt)
        self._sync_from_rank0()
