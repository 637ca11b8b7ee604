"""H100-native mirror of the index-prediction networks that sit between the sampler and the decoder in
``sample_and_refine``: the UNet guidance encoder (reference models/archs/unet_arch.py:317-481) and the
18-head FCN decoder (models/archs/fcn_arch.py:228-348), inference only (eval-mode BatchNorm).

Same constructor arguments, ``forward`` return structures and ``state_dict`` keys as the reference classes,
so ``index_pred_net.pth`` (``guidance_encoder`` / ``index_decoder``) loads with ``strict=True``.  The reference
builds its layers from ``mmcv.cnn.ConvModule``; the ``ConvModule`` below is a parameter container with the
same attribute names (``conv`` without bias, ``bn``, ``activate``).  Arithmetic runs in libt2h:

* every ConvModule is one wgmma tap-GEMM with the BatchNorm folded into the packed weights / bias and the
  ReLU in the epilogue (3x3 and 1x1 alike);
* ``MaxPool2d(2)`` and the bilinear x2 upsample are modes of the fp32 -> fp16-plane conversion that the next
  conv needs anyway (no extra pass);
* the 18 heads run as ONE 3x3 conv with 18*C output channels followed by ONE batched GEMM (18 groups with
  per-group weights and biases) and a per-position argmax inside the position's own head.
"""
import torch
import torch.nn as nn

from . import ops
from .vqgan_arch import _cached


class ConvModule(nn.Module):
    """conv (no bias) -> BatchNorm2d -> ReLU, as mmcv.cnn.ConvModule builds it for norm_cfg=BN, act_cfg=ReLU"""

    def __init__(self, in_channels, out_channels, kernel_size, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_channels)
        self.activate = nn.ReLU(inplace=True)

    def folded(self):
        """eval-mode BatchNorm folded into the conv: w' = w * g / sqrt(var + eps), b' = beta - mean * g / sqrt(..)"""
        bn = self.bn
        s = bn.weight.detach().float() / torch.sqrt(bn.running_var.float() + bn.eps)
        w = self.conv.weight.detach().float() * s.view(-1, 1, 1, 1)
        b = bn.bias.detach().float() - bn.running_mean.float() * s
        return w, b

    def _packed(self):
        t = ops.get_terms()
        srcs = (self.conv.weight, self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var)

        def build():
            w, b = self.folded()
            return ops.pack_conv_weight(w, t), b.contiguous()
        return _cached(self, ("folded", t), srcs, build)

    def forward_planes(self, a, planes_out):
        """a: planes [T,N,H,W,Cin] -> ReLU(BN(conv(a))) as planes or fp32 NHWC"""
        w, b = self._packed()
        taps = None if self.conv.kernel_size[0] == 3 else ops._TAPS_1
        return ops.conv3x3(a, w, b, planes_out=planes_out, taps=taps, act=ops.ACT_RELU)


class BasicConvBlock(nn.Module):
    """num_convs 3x3 ConvModules (unet_arch.py:113-181; stride 1, dilation 1 on this path)"""

    def __init__(self, in_channels, out_channels, num_convs=2):
        super().__init__()
        self.convs = nn.Sequential(*[ConvModule(in_channels if i == 0 else out_channels, out_channels, 3, padding=1)
                                     for i in range(num_convs)])

    def forward_planes(self, a):
        """planes in -> fp32 NHWC out (the last conv's output feeds a pooling / upsampling conversion)"""
        n = len(self.convs)
        for i, c in enumerate(self.convs):
            a = c.forward_planes(a, planes_out=(i < n - 1))
        return a


class InterpConv(nn.Module):
    """bilinear x2 upsample then a 1x1 ConvModule (unet_arch.py:244-314, conv_first=False)"""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.interp_upsample = nn.Sequential(nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False),
                                             ConvModule(in_channels, out_channels, 1))

    def forward_planes(self, x_nhwc):
        a = ops.f32_to_planes(x_nhwc, ops.CVT_BILINEAR2X)
        return self.interp_upsample[1].forward_planes(a, planes_out=True)


class UpConvBlock(nn.Module):
    """upsample the coarse map, concatenate the skip map, fuse with a conv block (unet_arch.py:12-110)"""

    def __init__(self, in_channels, skip_channels, out_channels, num_convs=2):
        super().__init__()
        self.conv_block = BasicConvBlock(2 * skip_channels, out_channels, num_convs)
        self.upsample = InterpConv(in_channels, skip_channels)

    def forward_planes(self, skip_nhwc, x_nhwc):
        up = self.upsample.forward_planes(x_nhwc)
        skip = ops.f32_to_planes(skip_nhwc)
        return self.conv_block.forward_planes(torch.cat((skip, up), dim=-1))     # torch.cat([skip, x], dim=1) :107


def build_unet_stages(net, in_channels, base_channels, num_stages, enc_num_convs, dec_num_convs, extra_in=0):
    """net.encoder / net.decoder with the reference's stage layout (UNet :420-458, ShapeUNet :619-655): stage i is
    [MaxPool2d(2) for i > 0,] BasicConvBlock(C_in + extra_in -> base * 2**i); ShapeUNet's extra_in is the width of
    the attribute embedding concatenated to every stage's input"""
    assert len(enc_num_convs) == num_stages and len(dec_num_convs) == num_stages - 1
    net.num_stages = num_stages
    net.encoder = nn.ModuleList()
    net.decoder = nn.ModuleList()
    for i in range(num_stages):
        blk = []
        if i != 0:
            blk.append(nn.MaxPool2d(kernel_size=2))
            net.decoder.append(UpConvBlock(base_channels * 2**i, base_channels * 2**(i - 1),
                                           base_channels * 2**(i - 1), dec_num_convs[i - 1]))
        blk.append(BasicConvBlock(in_channels + extra_in, base_channels * 2**i, enc_num_convs[i]))
        net.encoder.append(nn.Sequential(*blk))
        in_channels = base_channels * 2**i


def unet_decode(decoder, enc):
    """the UNet decoder (reference :467-471): fp32 NHWC encoder outputs -> dec_outs, coarsest first"""
    x = enc[-1]
    dec = [x]
    for i in reversed(range(len(decoder))):
        x = decoder[i].forward_planes(enc[i], x)
        dec.append(x)
    return dec


class UNet(nn.Module):
    """UNet backbone with the reference's defaults (stride-1 stages, MaxPool2d(2) between them, InterpConv
    upsampling).  forward(x NCHW) -> list of num_stages NCHW maps, coarsest first (reference :460-471)."""

    def __init__(self, in_channels=3, base_channels=64, num_stages=5, enc_num_convs=(2, 2, 2, 2, 2),
                 dec_num_convs=(2, 2, 2, 2)):
        super().__init__()
        build_unet_stages(self, in_channels, base_channels, num_stages, enc_num_convs, dec_num_convs)

    @torch.no_grad()
    def forward_nhwc(self, x, nhwc_in=False):
        """x fp32 NCHW (or NHWC with ``nhwc_in``) -> list of fp32 NHWC maps (dec_outs)"""
        assert not self.training, "inference only: BatchNorm uses its running statistics"
        a = ops.f32_to_planes(x) if nhwc_in else ops.nchw_to_planes(x)
        enc = []
        x = None
        for i, stage in enumerate(self.encoder):
            if i != 0:
                a = ops.f32_to_planes(x, ops.CVT_MAXPOOL2)
            x = stage[-1].forward_planes(a)
            enc.append(x)
        return unet_decode(self.decoder, enc)

    def forward(self, x):
        return [ops.nhwc_to_nchw(d) for d in self.forward_nhwc(x)]


class MultiHeadFCNHead(nn.Module):
    """num_head independent FCN heads on one feature map (fcn_arch.py:228-348); the configuration the
    reference uses: num_convs=1, concat_input=False, kernel 3, Dropout2d (identity in eval)."""

    def __init__(self, in_channels, channels, *, num_classes, dropout_ratio=0.1, in_index=-1, num_convs=1,
                 kernel_size=3, concat_input=False, num_head=18, align_corners=False, **kwargs):
        super().__init__()
        if num_convs != 1 or concat_input or kernel_size != 3:
            raise NotImplementedError("only num_convs=1, concat_input=False, kernel 3 (every Text2Human config)")
        self.in_channels, self.channels, self.num_classes = in_channels, channels, num_classes
        self.in_index, self.num_head = in_index, num_head
        self.dropout = nn.Dropout2d(dropout_ratio) if dropout_ratio > 0 else None
        self.conv_seg_head_list = nn.ModuleList([nn.Conv2d(channels, num_classes, kernel_size=1)
                                                 for _ in range(num_head)])
        self.convs_list = nn.ModuleList([nn.Sequential(ConvModule(in_channels, channels, 3, padding=1))
                                         for _ in range(num_head)])
        self.conv_cat_list = nn.ModuleList()

    def _packed(self):
        t = ops.get_terms()
        srcs = []
        for seq in self.convs_list:
            cm = seq[0]
            srcs += [cm.conv.weight, cm.bn.weight, cm.bn.bias, cm.bn.running_mean, cm.bn.running_var]
        srcs += [p for c in self.conv_seg_head_list for p in (c.weight, c.bias)]

        def build():
            ws, bs = zip(*[seq[0].folded() for seq in self.convs_list])
            w3 = ops.pack_conv_weight(torch.cat(ws, 0), t)                       # [T,9,num_head*ch,Cin]
            b3 = torch.cat(bs, 0).contiguous()
            w1 = torch.stack([c.weight.detach().float().view(self.num_classes, self.channels)
                              for c in self.conv_seg_head_list])                 # [G,ncls,ch]
            b1 = torch.stack([c.bias.detach().float() for c in self.conv_seg_head_list]).contiguous()
            return w3, b3, ops.split_planes(w1, t), b1
        return _cached(self, ("heads", t), tuple(srcs), build)

    @torch.no_grad()
    def forward_logits(self, feat_nhwc):
        """fp32 NHWC feature [B,H,W,Cin] -> fp32 [num_head, B*H*W, num_classes]"""
        assert not self.training, "inference only: BatchNorm uses its running statistics"
        w3, b3, w1, b1 = self._packed()
        B, H, W, _ = feat_nhwc.shape
        G, ch = self.num_head, self.channels
        y = ops.conv3x3(ops.f32_to_planes(feat_nhwc), w3, b3, planes_out=True, act=ops.ACT_RELU)  # [T,B,H,W,G*ch]
        T = y.shape[0]
        a = y.view(T, B * H * W, G, ch).permute(0, 2, 1, 3)                      # [T,G,M,ch] strided view
        return ops.bmm_nt(a, w1, bias_col=b1)

    def forward(self, inputs):
        x = inputs[self.in_index]
        B, _, H, W = x.shape
        lg = self.forward_logits(ops.nchw_to_nhwc(x))                             # [G, B*H*W, ncls]
        return [lg[k].view(B, H, W, self.num_classes).permute(0, 3, 1, 2) for k in range(self.num_head)]


@torch.no_grad()
def bot_index_prediction(unet, fcn, feature_top, texture_mask, latent_hw=(32, 16), as_list=True, nhwc_in=False):
    """BaseSampleModel.bot_index_prediction (sample_model.py:183-213), batched: per position the argmax of its
    own texture's head.  -> 18 int64 maps [B,h,w] with -1 outside each texture (``as_list``), or the
    (own-codebook index [B,h,w], texture id [B,h,w]) pair the gather kernel consumes."""
    B = feature_top.shape[0]
    h, w = latent_hw
    tex = ops.mask_to_ids(texture_mask, h, w).view(-1).long()
    feat = unet.forward_nhwc(feature_top, nhwc_in)[fcn.in_index]
    own = ops.argmax_heads(fcn.forward_logits(feat), tex)
    if not as_list:
        return own.view(B, h, w), tex.view(B, h, w)
    return [torch.where(tex == k, own, torch.full_like(own, -1)).view(B, h, w) for k in range(fcn.num_head)]
