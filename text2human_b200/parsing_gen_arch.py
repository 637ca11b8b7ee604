"""H100-native mirror of the parsing generator of ``SampleFromPoseModel`` (pose + shape attributes -> parsing map,
``generate_parsing_map``, reference models/sample_model.py:431-437): ShapeAttrEmbedding
(models/archs/shape_attr_embedding_arch.py), ShapeUNet (models/archs/unet_arch.py:503-674) and FCNHead
(models/archs/fcn_arch.py:159-225), inference only (eval-mode BatchNorm, Dropout2d is the identity).

Same constructor arguments, ``forward`` return structures and ``state_dict`` keys as the reference classes, so
``parsing_gen.pth`` (``embedder`` / ``encoder`` / ``decoder``) loads with ``strict=True``.  Arithmetic runs in libt2h:

* the embedding (15 one-hot Linears, which are column gathers, + 17 small Linears) is one fp32 launch per batch;
* every ShapeUNet encoder stage reads cat([x, embedding broadcast over H, W]) (with MaxPool2d(2) first for stages
  1..4) as one fp32 -> fp16-plane conversion that writes the broadcast channels itself -- the concatenation is kept
  (same arithmetic as the reference), only the expanded tensor is never materialised;
* the convolutions are index_pred_arch's ConvModule tap-GEMMs (BatchNorm folded), the decoder is UNet's;
* the parsing map is ``t2h_argmax_heads`` with one head (lowest index on ties, as torch.argmax).
"""
import torch
import torch.nn as nn

from . import ops
from .index_pred_arch import ConvModule, build_unet_stages, unet_decode
from .vqgan_arch import _cached


class ShapeAttrEmbedding(nn.Module):
    """per attribute i: Linear(cls_num_i, dim) on the one-hot code -> LeakyReLU -> Linear(dim, dim); the n_attr
    results concatenated -> Linear -> LeakyReLU -> Linear(out_dim, out_dim).  forward(attr int [B, n_attr]) ->
    fp32 [B, out_dim]."""

    def __init__(self, dim, out_dim, cls_num_list):
        super().__init__()
        for idx, cls_num in enumerate(cls_num_list):
            setattr(self, f'attr_{idx}', nn.Sequential(nn.Linear(cls_num, dim), nn.LeakyReLU(), nn.Linear(dim, dim)))
        self.cls_num_list = cls_num_list
        self.attr_num = len(cls_num_list)
        self.fusion = nn.Sequential(nn.Linear(dim * self.attr_num, out_dim), nn.LeakyReLU(),
                                    nn.Linear(out_dim, out_dim))

    def _packed(self):
        mods = [getattr(self, f'attr_{i}') for i in range(self.attr_num)]
        srcs = tuple(p for m in mods + [self.fusion] for p in (m[0].weight, m[0].bias, m[2].weight, m[2].bias))

        def build():
            f = lambda t: t.detach().float().contiguous()   # noqa: E731
            off = [0]
            for c in self.cls_num_list:
                off.append(off[-1] + c)
            dev = self.fusion[0].weight.device
            return dict(cls_off=torch.tensor(off, dtype=torch.int32, device=dev),
                        w1t=f(torch.cat([m[0].weight.t() for m in mods], 0)),      # [sum(cls), dim]: W1_i's columns
                        b1=f(torch.stack([m[0].bias for m in mods])),
                        w2=f(torch.stack([m[2].weight for m in mods])),
                        b2=f(torch.stack([m[2].bias for m in mods])),
                        wf1=f(self.fusion[0].weight), bf1=f(self.fusion[0].bias),
                        wf2=f(self.fusion[2].weight), bf2=f(self.fusion[2].bias))
        return _cached(self, "packed", srcs, build)

    def check_attributes(self, attr):
        """raise ValueError naming the first attribute outside 0..cls_num-1 (F.one_hot rejects those too)"""
        if attr.dim() != 2 or attr.shape[1] != self.attr_num:
            raise ValueError(f"shape attributes must be [B, {self.attr_num}], got {tuple(attr.shape)}")
        if attr.dtype.is_floating_point or attr.dtype == torch.bool:
            raise ValueError(f"shape attributes must be integers, got {attr.dtype}")
        lo, hi = (v.tolist() for v in torch.stack((attr.amin(0), attr.amax(0))).cpu())
        for i, n in enumerate(self.cls_num_list):
            if lo[i] < 0 or hi[i] >= n:
                bad = lo[i] if lo[i] < 0 else hi[i]
                raise ValueError(f"shape attribute {i} has value {bad}, outside its {n} classes 0..{n - 1}")

    @torch.no_grad()
    def forward(self, attr):
        assert not self.training, "inference only"
        self.check_attributes(attr)
        return ops.shape_attr_embed(attr.to(self.fusion[0].weight.device), self._packed())


_DEFAULT_CFGS = dict(conv_cfg=None, norm_cfg=dict(type='BN'), act_cfg=dict(type='ReLU'))


class ShapeUNet(nn.Module):
    """UNet whose every encoder stage also reads the attribute embedding, broadcast over the stage's input
    (unet_arch.py:657-668).  forward(x NCHW, attr_embedding [B, attr_embedding]) -> list of num_stages NCHW maps,
    coarsest first.  Supported: the reference defaults every Text2Human config uses (stride-1 stages, MaxPool2d
    downsampling, dilation 1, InterpConv upsampling, BN + ReLU, no checkpointing / DCN / plugins)."""

    def __init__(self, in_channels=3, base_channels=64, num_stages=5, attr_embedding=128, strides=(1, 1, 1, 1, 1),
                 enc_num_convs=(2, 2, 2, 2, 2), dec_num_convs=(2, 2, 2, 2), downsamples=(True, True, True, True),
                 enc_dilations=(1, 1, 1, 1, 1), dec_dilations=(1, 1, 1, 1), with_cp=False, conv_cfg=None,
                 norm_cfg=dict(type='BN'), act_cfg=dict(type='ReLU'), upsample_cfg=dict(type='InterpConv'),
                 norm_eval=False, dcn=None, plugins=None):
        super().__init__()
        unsupported = (any(s != 1 for s in strides) or not all(downsamples) or any(d != 1 for d in enc_dilations)
                       or any(d != 1 for d in dec_dilations) or with_cp or dcn is not None or plugins is not None
                       or dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg) != _DEFAULT_CFGS
                       or upsample_cfg != dict(type='InterpConv'))
        if unsupported:
            raise NotImplementedError("ShapeUNet: only the reference defaults (stride 1, MaxPool2d, dilation 1, "
                                      "InterpConv, BN + ReLU, no with_cp / dcn / plugins)")
        if len(strides) != num_stages or len(downsamples) != num_stages - 1:
            raise ValueError("strides / downsamples do not match num_stages")
        self.in_channels, self.attr_embedding = in_channels, attr_embedding
        self.norm_eval = norm_eval
        build_unet_stages(self, in_channels, base_channels, num_stages, enc_num_convs, dec_num_convs,
                          extra_in=attr_embedding)

    @torch.no_grad()
    def forward_nhwc(self, x, attr_embedding, nhwc_in=False):
        """x fp32 NCHW (or NHWC with ``nhwc_in``), attr_embedding fp32 [B, attr_embedding] -> list of fp32 NHWC
        maps (dec_outs)"""
        assert not self.training, "inference only: BatchNorm uses its running statistics"
        if not nhwc_in:
            B, C, H, W = x.shape
            # a 1-channel NCHW map (the pose) already is its NHWC layout
            x = x.reshape(B, H, W, 1) if C == 1 else ops.nchw_to_nhwc(x)
        enc = []
        for i, stage in enumerate(self.encoder):
            a = ops.f32_to_planes_bcast(x, attr_embedding, ops.CVT_PLAIN if i == 0 else ops.CVT_MAXPOOL2)
            x = stage[-1].forward_planes(a)
            enc.append(x)
        return unet_decode(self.decoder, enc)

    def forward(self, x, attr_embedding):
        return [ops.nhwc_to_nchw(d) for d in self.forward_nhwc(x, attr_embedding)]


class FCNHead(nn.Module):
    """BaseDecodeHead + FCNHead (fcn_arch.py:7-225) for the configuration the parsing generator uses:
    num_convs=1, concat_input=False, kernel 3 -> a 3x3 ConvModule, Dropout2d (identity in eval), 1x1 conv_seg.
    forward(inputs) -> logits NCHW [B, num_classes, H, W] of inputs[in_index]."""

    def __init__(self, num_convs=2, kernel_size=3, concat_input=True, *, in_channels, channels, num_classes,
                 dropout_ratio=0.1, conv_cfg=None, norm_cfg=dict(type='BN'), act_cfg=dict(type='ReLU'), in_index=-1,
                 input_transform=None, ignore_index=255, align_corners=False):
        super().__init__()
        if (num_convs != 1 or concat_input or kernel_size != 3 or input_transform is not None
                or dict(conv_cfg=conv_cfg, norm_cfg=norm_cfg, act_cfg=act_cfg) != _DEFAULT_CFGS):
            raise NotImplementedError("FCNHead: only num_convs=1, concat_input=False, kernel 3, single input, BN + "
                                      "ReLU (every Text2Human config)")
        self.num_convs, self.kernel_size, self.concat_input = num_convs, kernel_size, concat_input
        self.in_channels, self.channels, self.num_classes = in_channels, channels, num_classes
        self.in_index, self.input_transform = in_index, input_transform
        self.dropout_ratio, self.ignore_index, self.align_corners = dropout_ratio, ignore_index, align_corners
        self.conv_seg = nn.Conv2d(channels, num_classes, kernel_size=1)     # registered first, as in the reference
        self.dropout = nn.Dropout2d(dropout_ratio) if dropout_ratio > 0 else None
        self.convs = nn.Sequential(ConvModule(in_channels, channels, kernel_size, padding=kernel_size // 2))

    def _seg_packed(self):
        t = ops.get_terms()
        return _cached(self, ("seg", t), (self.conv_seg.weight, self.conv_seg.bias),
                       lambda: (ops.pack_conv_weight(self.conv_seg.weight, t), self.conv_seg.bias.detach().float()))

    @torch.no_grad()
    def forward_logits(self, feat_nhwc):
        """fp32 NHWC feature [B,H,W,in_channels] -> fp32 NHWC logits [B,H,W,num_classes]"""
        assert not self.training, "inference only: BatchNorm uses its running statistics"
        y = self.convs[0].forward_planes(ops.f32_to_planes(feat_nhwc), planes_out=True)
        w, b = self._seg_packed()
        return ops.conv3x3(y, w, b, taps=ops._TAPS_1)

    def forward(self, inputs):
        return ops.nhwc_to_nchw(self.forward_logits(ops.nchw_to_nhwc(inputs[self.in_index])))


def parsing_argmax(logits_nhwc):
    """fp32 NHWC logits [B,H,W,n] -> float class-id map [B,1,H,W] (what onehot_to_planes / texture_mask read):
    argmax over the classes, lowest index on ties (torch.argmax)"""
    B, H, W, n = logits_nhwc.shape
    M = B * H * W
    ids = ops.argmax_heads(logits_nhwc.reshape(1, M, n), torch.zeros((M,), dtype=torch.int64,
                                                                       device=logits_nhwc.device))
    return ids.view(B, 1, H, W).float()


@torch.no_grad()
def generate_parsing_map(embedder, unet, head, pose, shape_attr):
    """SampleFromPoseModel.generate_parsing_map (sample_model.py:431-437), batched: pose fp32 [B,1,H,W] and shape
    attributes int [B, n_attr] -> float parsing map [B,1,H,W] of class ids"""
    e = embedder(shape_attr)
    feat = unet.forward_nhwc(pose, e)[head.in_index]
    return parsing_argmax(head.forward_logits(feat))
