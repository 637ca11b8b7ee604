"""H100-native mirror of the reference's ``models/archs/vqgan_arch.py``.

Same class names, constructor signatures, ``forward`` signatures and
``state_dict`` keys as the reference (SURVEY.md §8b), so reference checkpoints
load with ``strict=True`` and the reference's model wrappers can construct these
classes unchanged.  torch ``nn.Conv2d`` / ``nn.GroupNorm`` / ``nn.Embedding``
objects are used *only as parameter containers* (same names, shapes and default
initialisation as the reference); their ``forward`` is never called.  All
arithmetic runs in libt2h (``text2human_b200.ops``): wgmma implicit-GEMM convs,
GroupNorm/swish, attention products, softmax and the codebook search.

Every module exposes two entry points:
  * ``forward(x)``       — the reference API: fp32 NCHW in, fp32 NCHW out
  * ``forward_nhwc(x)``  — the fused-pipeline API: fp32 NHWC in/out, no layout
                           round trips between modules (text2human_b200.pipeline)

This round implements the forward (inference) path; kernels run under
``torch.no_grad`` semantics (outputs do not carry autograd history).
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .ops import CVT_PLAIN, CVT_S2D, CVT_UP2X


# ----------------------------------------------------------------------------
# packed-weight cache
# ----------------------------------------------------------------------------
def _cached(owner, key, params, build):
    """Cache a derived (packed fp16-plane) buffer on ``owner``; rebuilt when any
    source parameter was modified in place (``_version``), moved or re-assigned."""
    cache = owner.__dict__.setdefault("_t2h_cache", {})
    sig = tuple((p.data_ptr(), p._version, str(p.device)) for p in params)
    hit = cache.get(key)
    if hit is not None and hit[0] == sig:
        return hit[1]
    with torch.no_grad():
        val = build()
    cache[key] = (sig, val)
    return val


def _conv_w(conv, c_pad=None):
    t = ops.layer_terms(conv)
    return _cached(conv, ("w3", t, c_pad), (conv.weight,),
                   lambda: ops.pack_conv_weight(conv.weight, t, c_pad))


def _lin_w(mod):
    t = ops.get_terms()
    return _cached(mod, ("w1", t), (mod.weight,), lambda: ops.pack_linear_weight(mod.weight, t))


def _f32(p):
    return p.detach()


class _Act:
    """fp32 NHWC activation + (optionally) the GroupNorm(32) statistics of it that the producing
    kernel's epilogue accumulated, so the consumer's GroupNorm skips its statistics pass."""
    __slots__ = ("x", "stats")

    def __init__(self, x, stats=None):
        self.x = x
        self.stats = stats


def conv1x1_nhwc(x, conv, *, residual=None, planes_in=None, want_stats=False):
    """1x1 conv on fp32 NHWC ``x`` (or on planes ``planes_in``) -> fp32 NHWC (and its GN statistics)."""
    if planes_in is None:
        planes_in = ops.f32_to_planes(x, CVT_PLAIN)
    return ops.conv1x1(planes_in, _lin_w(conv), _f32(conv.bias), residual=residual, want_stats=want_stats)


# ----------------------------------------------------------------------------
# building blocks (reference: vqgan_arch.py:510-661)
# ----------------------------------------------------------------------------
def Normalize(in_channels):
    return torch.nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


def _gn_conv3x3(act, norm, conv, *, residual=None, want_stats=False, nchw_out=False):
    """swish(GroupNorm(act)) -> 3x3 conv: the gn_apply pass followed by the conv"""
    a = _gn(act, norm, swish=True, consumer=conv)
    return ops.conv3x3(a, _conv_w(conv), _f32(conv.bias), residual=residual, nchw_out=nchw_out,
                       want_stats=want_stats)


def _gn(act, norm, swish, consumer=None):
    """``consumer``: the conv that reads the planes (decides how many planes are written)"""
    stats = act.stats if norm.num_groups == ops.GN_GROUPS else None
    return ops.group_norm(act.x, _f32(norm.weight), _f32(norm.bias), swish=swish, groups=norm.num_groups,
                          eps=norm.eps, stats=stats,
                          terms=ops.layer_terms(consumer) if consumer is not None else None)


class Upsample(nn.Module):
    """nearest x2 then 3x3 conv (reference :520-534)."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def _fwd(self, act):
        if not self.with_conv:
            raise NotImplementedError("Upsample(with_conv=False) is not on the Text2Human path")
        # nearest x2 + 3x3 conv == four 2x2 convs on the low-resolution input (one per output parity)
        t = ops.get_terms()
        w16 = _cached(self.conv, ("wup", t), (self.conv.weight,),
                      lambda: ops.pack_upsample_conv_weight(self.conv.weight, t))
        a = ops.f32_to_planes(act.x, CVT_PLAIN)
        return _Act(*ops.upsample_conv3x3(a, w16, _f32(self.conv.bias), want_stats=True))

    def forward_nhwc(self, x):
        return self._fwd(_Act(x)).x

    def forward(self, x):
        return ops.nhwc_to_nchw(self.forward_nhwc(ops.nchw_to_nhwc(x)))


class Downsample(nn.Module):
    """pad (0,1,0,1) then 3x3 stride-2 conv (reference :537-554)."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = torch.nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def _fwd(self, act):
        if not self.with_conv:
            raise NotImplementedError("Downsample(with_conv=False) is not on the Text2Human path")
        a = ops.f32_to_planes(act.x, CVT_S2D)
        return _Act(*ops.conv3x3_s2(a, _conv_w(self.conv), _f32(self.conv.bias), want_stats=True))

    def forward_nhwc(self, x):
        return self._fwd(_Act(x)).x

    def forward(self, x):
        return ops.nhwc_to_nchw(self.forward_nhwc(ops.nchw_to_nhwc(x)))


class ResnetBlock(nn.Module):
    """GN-swish-conv3x3-GN-swish-conv3x3 + (1x1) shortcut (reference :557-617)."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout,
                 temb_channels=512):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut

        self.norm1 = Normalize(in_channels)
        self.conv1 = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if temb_channels > 0:
            self.temb_proj = torch.nn.Linear(temb_channels, out_channels)
        self.norm2 = Normalize(out_channels)
        self.dropout = torch.nn.Dropout(dropout)
        self.conv2 = torch.nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                self.conv_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1,
                                                     padding=1)
            else:
                self.nin_shortcut = torch.nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1,
                                                    padding=0)

    def _fwd(self, act):
        assert self.dropout.p == 0.0 or not self.training, "dropout>0 in training is not implemented"
        x = act.x
        # conv1's epilogue accumulates the statistics norm2 needs
        h = _Act(*_gn_conv3x3(act, self.norm1, self.conv1, want_stats=True))
        if self.in_channels != self.out_channels:
            xp = ops.f32_to_planes(x, CVT_PLAIN)
            if self.use_conv_shortcut:
                x = ops.conv3x3(xp, _conv_w(self.conv_shortcut), _f32(self.conv_shortcut.bias))
            else:
                x = conv1x1_nhwc(None, self.nin_shortcut, planes_in=xp)
        # residual add (and the next GroupNorm's statistics) fused into conv2's epilogue
        return _Act(*_gn_conv3x3(h, self.norm2, self.conv2, residual=x, want_stats=True))

    def forward_nhwc(self, x, temb=None):
        assert temb is None, "temb is always None on the Text2Human path (temb_ch=0)"
        return self._fwd(_Act(x)).x

    def forward(self, x, temb=None):
        return ops.nhwc_to_nchw(self.forward_nhwc(ops.nchw_to_nhwc(x), temb))


class AttnBlock(nn.Module):
    """single-head spatial self-attention over h*w tokens (reference :620-661)."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = torch.nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)

    def _qk_packed(self):
        t = ops.get_terms()
        w = _cached(self, ("wqk", t), (self.q.weight, self.k.weight),
                    lambda: ops.pack_linear_weight(torch.cat((self.q.weight, self.k.weight), 0), t))
        b = _cached(self, ("bqk",), (self.q.bias, self.k.bias),
                    lambda: torch.cat((self.q.bias, self.k.bias), 0).float().contiguous())
        return w, b

    def _fwd(self, act):
        x = act.x
        N, H, W, Cc = x.shape
        HW = H * W
        hn = _gn(act, self.norm, swish=False)  # planes [T,N,H,W,C]
        T = hn.shape[0]
        wqk, bqk = self._qk_packed()
        qk = ops.linear(hn.reshape(T, N * HW, Cc), wqk, bqk, planes_out=True).view(T, N, HW, 2 * Cc)
        q, k = qk[..., :Cc], qk[..., Cc:]
        # v^T[b] = Wv @ hn[b]^T  (+ bias per output channel = per row)
        vt = ops.bmm_nt(_lin_w(self.v), hn.view(T, N, HW, Cc), planes_out=True,
                        bias_row=_f32(self.v.bias), a_bcast=True)  # [T,N,C,HW]
        s = ops.bmm_nt(q, k)  # fp32 [N,HW,HW], s[b,i,j] = sum_c q[b,i,c] k[b,j,c]
        p = ops.softmax_rows(s, scale=float(int(Cc) ** (-0.5)))  # planes [T,N,HW,HW]
        o = ops.bmm_nt(p, vt, planes_out=True)  # [T,N,HW,C]
        return _Act(*ops.conv1x1(o.view(T, N, H, W, Cc), _lin_w(self.proj_out), _f32(self.proj_out.bias),
                                 residual=x, want_stats=True))

    def forward_nhwc(self, x):
        return self._fwd(_Act(x)).x

    def forward(self, x):
        return ops.nhwc_to_nchw(self.forward_nhwc(ops.nchw_to_nhwc(x)))


# ----------------------------------------------------------------------------
# Encoder / Decoder / DecoderRes (reference :818-1151)
# ----------------------------------------------------------------------------
def _conv_in_nchw(conv, x):
    """network-entry conv: fp32 NCHW -> (split + NHWC + channel pad) -> 3x3 conv -> fp32 NHWC"""
    a = ops.nchw_to_planes(x)
    return _Act(*ops.conv3x3(a, _conv_w(conv, a.shape[-1]), _f32(conv.bias), want_stats=True))


def _conv_in_nhwc(conv, x):
    a = ops.f32_to_planes(x, CVT_PLAIN)
    return _Act(*ops.conv3x3(a, _conv_w(conv), _f32(conv.bias), want_stats=True))


def _conv_out(norm, conv, act, nchw):
    return _gn_conv3x3(act, norm, conv, nchw_out=nchw)


class Encoder(nn.Module):

    def __init__(self, ch, num_res_blocks, attn_resolutions, in_channels, resolution, z_channels,
                 ch_mult=(1, 2, 4, 8), dropout=0.0, resamp_with_conv=True, double_z=True):
        super().__init__()
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels

        self.conv_in = torch.nn.Conv2d(in_channels, self.ch, kernel_size=3, stride=1, padding=1)

        curr_res = resolution
        in_ch_mult = (1, ) + tuple(ch_mult)
        self.down = nn.ModuleList()
        for i_level in range(self.num_resolutions):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_in = ch * in_ch_mult[i_level]
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out,
                                         temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            down = nn.Module()
            down.block = block
            down.attn = attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
                curr_res = curr_res // 2
            self.down.append(down)

        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)

        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels,
                                        kernel_size=3, stride=1, padding=1)

    def _body(self, h):
        for i_level in range(self.num_resolutions):
            lvl = self.down[i_level]
            for i_block in range(self.num_res_blocks):
                h = lvl.block[i_block]._fwd(h)
                if len(lvl.attn) > 0:
                    h = lvl.attn[i_block]._fwd(h)
            if i_level != self.num_resolutions - 1:
                h = lvl.downsample._fwd(h)
        h = self.mid.block_1._fwd(h)
        h = self.mid.attn_1._fwd(h)
        h = self.mid.block_2._fwd(h)
        return h

    @torch.no_grad()
    def forward_planes(self, a):
        """fp16 planes NHWC [T,N,H,W,c_pad] in (e.g. a one-hot segmentation), fp32 NHWC latent out."""
        h = _Act(*ops.conv3x3(a, _conv_w(self.conv_in, a.shape[-1]), _f32(self.conv_in.bias), want_stats=True))
        return _conv_out(self.norm_out, self.conv_out, self._body(h), nchw=False)

    @torch.no_grad()
    def forward_nhwc(self, x_nchw):
        """fp32 NCHW image in (the network entry is NCHW either way), fp32 NHWC latent out."""
        h = self._body(_conv_in_nchw(self.conv_in, x_nchw))
        return _conv_out(self.norm_out, self.conv_out, h, nchw=False)

    def forward(self, x):
        from . import vqgan_autograd as VA
        if VA.recording(self, x):       # training: one autograd node with the hand-written backward
            return VA.encoder_forward(self, x)
        with torch.no_grad():
            h = self._body(_conv_in_nchw(self.conv_in, x))
            return _conv_out(self.norm_out, self.conv_out, h, nchw=True)


class Decoder(nn.Module):

    def __init__(self, in_channels, resolution, z_channels, ch, out_ch, num_res_blocks, attn_resolutions,
                 ch_mult=(1, 2, 4, 8), dropout=0.0, resamp_with_conv=True, give_pre_end=False):
        super().__init__()
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.give_pre_end = give_pre_end

        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2**(self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res // 2)
        print("Working with z of shape {} = {} dimensions.".format(self.z_shape, np.prod(self.z_shape)))

        self.conv_in = torch.nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)

        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)

        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            attn = nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(self.num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out,
                                         temb_channels=self.temb_ch, dropout=dropout))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block = block
            up.attn = attn
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
                curr_res = curr_res * 2
            self.up.insert(0, up)  # prepend to get consistent order

        self.norm_out = Normalize(block_in)
        self.conv_out = torch.nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)
        # per-layer precision map (ops.set_precision("mixed")): the 3x3 convs of the full-resolution level are the
        # layers whose single-product error is smallest relative to their FLOPs (nearest the output, least amplified)
        for blk in self.up[0].block:
            blk.conv1._t2h_single = blk.conv2._t2h_single = True

    def _trunk(self, h, bot_h=None, stop_after_level=None, mid_h=None):
        h = self.mid.block_1._fwd(h)
        h = self.mid.attn_1._fwd(h)
        h = self.mid.block_2._fwd(h)
        for i_level in reversed(range(self.num_resolutions)):
            lvl = self.up[i_level]
            for i_block in range(self.num_res_blocks + 1):
                h = lvl.block[i_block]._fwd(h)
                if len(lvl.attn) > 0:
                    h = lvl.attn[i_block]._fwd(h)
            if i_level != 0:
                h = lvl.upsample._fwd(h)
            # reference :1023-1024 — the hierarchy residual enters after level 4's upsample
            if i_level == 4 and bot_h is not None:
                h = _Act(ops.add_inplace(h.x, bot_h))  # statistics of the sum are not known
            if i_level == 4 and mid_h is not None:
                h = _Act(ops.add_inplace(h.x, mid_h))
            if stop_after_level is not None and i_level == stop_after_level:
                return h
        return h

    def _finish(self, h, nchw):
        if self.give_pre_end:
            return ops.nhwc_to_nchw(h.x) if nchw else h.x
        return _conv_out(self.norm_out, self.conv_out, h, nchw=nchw)

    @torch.no_grad()
    def forward_nhwc(self, z, bot_h=None, nchw_out=True):
        """z, bot_h: fp32 NHWC.  Output fp32 NCHW image (default) or NHWC."""
        self.last_z_shape = torch.Size((z.shape[0], z.shape[3], z.shape[1], z.shape[2]))
        h = self._trunk(_conv_in_nhwc(self.conv_in, z), bot_h=bot_h)
        return self._finish(h, nchw_out)

    def forward(self, z, bot_h=None):
        self.last_z_shape = z.shape
        from . import vqgan_autograd as VA
        # training: trunk node + (norm_out, conv_out) node.  A bot_h that requires grad takes the nodes in eval mode
        # too: with fix_decoder the reference never calls decoder.train() and back-propagates through the eval-mode
        # decoder into bot_h (no BatchNorm, dropout 0: both modes compute the same)
        if VA.recording(self, z, bot_h) or (bot_h is not None and bot_h.requires_grad and torch.is_grad_enabled()):
            return VA.decoder_forward(self, z, bot_h)
        with torch.no_grad():
            bh = ops.nchw_to_nhwc(bot_h) if bot_h is not None else None
            h = self._trunk(_conv_in_nchw(self.conv_in, z), bot_h=bh)
            return self._finish(h, True)

    @torch.no_grad()
    def get_feature_top(self, z):
        """reference :1035-1059 — activations after level 4's upsample"""
        self.last_z_shape = z.shape
        h = self._trunk(_conv_in_nchw(self.conv_in, z), stop_after_level=4)
        return ops.nhwc_to_nchw(h.x)

    @torch.no_grad()
    def get_feature_middle(self, z, mid_h):
        """reference :1061-1087 — adds mid_h after level 4, returns after level 3"""
        self.last_z_shape = z.shape
        h = self._trunk(_conv_in_nchw(self.conv_in, z), mid_h=ops.nchw_to_nhwc(mid_h), stop_after_level=3)
        return ops.nhwc_to_nchw(h.x)


class DecoderRes(nn.Module):

    def __init__(self, in_channels, resolution, z_channels, ch, num_res_blocks, ch_mult=(1, 2, 4, 8),
                 dropout=0.0, give_pre_end=False):
        super().__init__()
        self.ch = ch
        self.temb_ch = 0
        self.num_resolutions = len(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.resolution = resolution
        self.in_channels = in_channels
        self.give_pre_end = give_pre_end

        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2**(self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res // 2)
        print("Working with z of shape {} = {} dimensions.".format(self.z_shape, np.prod(self.z_shape)))

        self.conv_in = torch.nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in,
                                       temb_channels=self.temb_ch, dropout=dropout)

    def _trunk(self, h):
        h = self.mid.block_1._fwd(h)
        h = self.mid.attn_1._fwd(h)
        return self.mid.block_2._fwd(h).x

    @torch.no_grad()
    def forward_nhwc(self, z):
        self.last_z_shape = torch.Size((z.shape[0], z.shape[3], z.shape[1], z.shape[2]))
        return self._trunk(_conv_in_nhwc(self.conv_in, z))

    def forward(self, z):
        self.last_z_shape = z.shape
        from . import vqgan_autograd as VA
        if VA.recording(self, z):          # training: one autograd node (conv_in + mid) with the hand-written backward
            return VA.decoder_res_forward(self, z)
        with torch.no_grad():
            return ops.nhwc_to_nchw(self._trunk(_conv_in_nchw(self.conv_in, z)))


# ----------------------------------------------------------------------------
# Patch discriminator (reference :1154-1203)
# ----------------------------------------------------------------------------
class Discriminator(nn.Module):
    """conv4x4 s2 + LeakyReLU(0.2) | (n_layers-1) x [conv4x4 s2, BatchNorm, LeakyReLU] | [conv4x4 s1, BatchNorm,
    LeakyReLU] | conv4x4 s1 -> 1 channel.  The nn.Sequential ``main`` only holds the parameters / BatchNorm buffers
    under the reference's state_dict keys; the arithmetic runs in libt2h (``vqgan_train.DiscNet``): 16-tap wgmma
    convs on space-to-depth planes, BatchNorm as one-image GroupNorm(groups=C) kernels with the LeakyReLU fused."""

    def __init__(self, nc, ndf, n_layers=3):
        super().__init__()
        layers = [nn.Conv2d(nc, ndf, kernel_size=4, stride=2, padding=1), nn.LeakyReLU(0.2, True)]
        ndf_mult = 1
        for n in range(1, n_layers):
            ndf_mult_prev, ndf_mult = ndf_mult, min(2**n, 8)
            layers += [nn.Conv2d(ndf * ndf_mult_prev, ndf * ndf_mult, kernel_size=4, stride=2, padding=1, bias=False),
                       nn.BatchNorm2d(ndf * ndf_mult), nn.LeakyReLU(0.2, True)]
        ndf_mult_prev, ndf_mult = ndf_mult, min(2**n_layers, 8)
        layers += [nn.Conv2d(ndf * ndf_mult_prev, ndf * ndf_mult, kernel_size=4, stride=1, padding=1, bias=False),
                   nn.BatchNorm2d(ndf * ndf_mult), nn.LeakyReLU(0.2, True)]
        layers += [nn.Conv2d(ndf * ndf_mult, 1, kernel_size=4, stride=1, padding=1)]
        self.main = nn.Sequential(*layers)

    def forward(self, x):
        """fp32 NCHW [N,3,H,W] -> patch logits fp32 [N,1,h,w].  With autograd enabled the call is recorded as ONE
        autograd node whose backward is the hand-written discriminator backward (``vqgan_autograd``)."""
        from . import vqgan_autograd as VA
        return VA.discriminator_forward(self, x)


# ----------------------------------------------------------------------------
# Quantizers (reference :12-486)
# ----------------------------------------------------------------------------
def _check_gumbel_args(temp, rescale_logits, return_logits):
    assert temp is None or temp == 1.0, "Only for interface compatible with Gumbel"
    assert rescale_logits == False, "Only for interface compatible with Gumbel"  # noqa: E712
    assert return_logits == False, "Only for interface compatible with Gumbel"  # noqa: E712


def _loss_from_sqerr(sqerr, numel, beta):
    # legacy and non-legacy placements of beta have the same forward value:
    # mean((zq.detach()-z)^2) + beta*mean((zq-z.detach())^2) = (1+beta)*mse   (reference :273-278)
    return ((1.0 + beta) * sqerr[0] / numel).to(torch.float32)


class VectorQuantizer(nn.Module):
    """single-codebook L2 nearest neighbour (reference :12-139; segm tokeniser)."""

    def __init__(self, n_e, e_dim, beta, remap=None, unknown_index="random", sane_index_shape=False,
                 legacy=True):
        super().__init__()
        self.n_e = n_e
        self.e_dim = e_dim
        self.beta = beta
        self.legacy = legacy
        self.embedding = nn.Embedding(self.n_e, self.e_dim)
        self.embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)
        if remap is not None:
            raise NotImplementedError("remap is unused on the Text2Human path (remap=None everywhere)")
        self.remap = None
        self.re_embed = n_e
        self.sane_index_shape = sane_index_shape

    def _codebook(self):
        return self.embedding.weight.detach().unsqueeze(0)

    @torch.no_grad()
    def forward_nhwc(self, z):
        """z fp32 NHWC -> dict with zq_nhwc, idx [B,h,w], loss"""
        r = ops.vq_search(z, self._codebook(), None, want_list=False, want_nchw=False)
        r["loss"] = _loss_from_sqerr(r["sqerr"], z.numel(), self.beta)
        return r

    def forward(self, z, temp=None, rescale_logits=False, return_logits=False):
        _check_gumbel_args(temp, rescale_logits, return_logits)
        from . import vqgan_autograd as VA
        if VA.recording(self, z):          # training: straight-through + codebook-loss gradients
            return VA.quantizer_forward(self, z)
        with torch.no_grad():
            zh = ops.nchw_to_nhwc(z)
            r = ops.vq_search(zh, self._codebook(), None, want_list=False, want_nhwc=False)
            loss = _loss_from_sqerr(r["sqerr"], z.numel(), self.beta)
            idx = r["idx"]
            if not self.sane_index_shape:
                idx = idx.reshape(-1)
            return r["zq_nchw"], loss, (None, None, idx)

    @torch.no_grad()
    def get_codebook_entry(self, indices, shape):
        # shape = (batch, height, width, channel)
        if shape is None:
            return self.embedding.weight.detach()[indices]
        B, H, W, Cc = shape
        _, zq = ops.vq_gather(self._codebook(), indices.reshape(-1), None, B=B, Hz=H, Wz=W, Cz=Cc)
        return zq


class _TextureQuantizerBase(nn.Module):
    NUM_BOOKS = 18

    def _codebook(self):
        ws = tuple(e.weight for e in self.embedding_list)
        return _cached(self, ("cb",), ws, lambda: torch.stack([w.detach().float() for w in ws]).contiguous())

    def _resolve_indices(self, indices_list, ids):
        """pick, per position, the entry of the list its texture id selects (reference :297-303); a single
        tensor is taken as the already-resolved own-codebook index map"""
        if torch.is_tensor(indices_list):
            return indices_list.reshape(ids.shape)
        stacked = torch.stack([i.reshape(ids.shape) for i in indices_list])  # [18,B,h,w]
        sel = ids.clamp(0, self.NUM_BOOKS - 1).long().unsqueeze(0)
        return stacked.gather(0, sel).squeeze(0)


class VectorQuantizerTexture(_TextureQuantizerBase):
    """18 texture-selected codebooks (reference :142-309)."""

    def __init__(self, n_e, e_dim, beta, remap=None, unknown_index="random", sane_index_shape=False,
                 legacy=True):
        super().__init__()
        self.n_e = n_e
        self.e_dim = e_dim
        self.beta = beta
        self.legacy = legacy
        self.embedding_list = nn.ModuleList([nn.Embedding(self.n_e, self.e_dim) for _ in range(18)])
        for embedding in self.embedding_list:
            embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)
        if remap is not None:
            raise NotImplementedError("remap is unused on the Text2Human path (remap=None everywhere)")
        self.remap = None
        self.re_embed = n_e
        self.sane_index_shape = sane_index_shape

    @torch.no_grad()
    def forward_nhwc(self, z, segm_map, want_nchw=False):
        B, H, W, _ = z.shape
        ids = ops.mask_to_ids(segm_map, H, W)
        # the reference hard-codes 1024 as the continual-index stride (:262)
        r = ops.vq_search(z, self._codebook(), ids, cont_stride=1024, want_nchw=want_nchw)
        r["loss"] = _loss_from_sqerr(r["sqerr"], z.numel(), self.beta)
        r["ids"] = ids
        return r

    def forward(self, z, segm_map, temp=None, rescale_logits=False, return_logits=False):
        _check_gumbel_args(temp, rescale_logits, return_logits)
        from . import vqgan_autograd as VA
        if VA.recording(self, z):          # training: straight-through + codebook-loss gradients
            return VA.quantizer_texture_forward(self, z, segm_map)
        with torch.no_grad():
            r = self.forward_nhwc(ops.nchw_to_nhwc(z), segm_map, want_nchw=True)
            return r["zq_nchw"], r["loss"], (None, r["idx_cont"], list(r["idx_list"].unbind(0)))

    @torch.no_grad()
    def get_codebook_entry(self, indices_list, segm_map, shape, nhwc=False):
        B, H, W, Cc = shape
        ids = ops.mask_to_ids(segm_map, H, W)
        idx = self._resolve_indices(indices_list, ids)
        zq_nhwc, zq_nchw = ops.vq_gather(self._codebook(), idx, ids, B=B, Hz=H, Wz=W, Cz=self.e_dim,
                                         want_nchw=not nhwc, want_nhwc=nhwc)
        return zq_nhwc if nhwc else zq_nchw


class VectorQuantizerSpatialTextureAware(_TextureQuantizerBase):
    """18 texture-selected codebooks over 2x2 patches (reference :329-486)."""

    def __init__(self, n_e, e_dim, beta, spatial_size, remap=None, unknown_index="random",
                 sane_index_shape=False, legacy=True):
        super().__init__()
        self.n_e = n_e
        self.e_dim = e_dim * spatial_size * spatial_size
        self.beta = beta
        self.legacy = legacy
        self.spatial_size = spatial_size
        self.embedding_list = nn.ModuleList([nn.Embedding(self.n_e, self.e_dim) for _ in range(18)])
        for embedding in self.embedding_list:
            embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)
        if remap is not None:
            raise NotImplementedError("remap is unused on the Text2Human path (remap=None everywhere)")
        self.remap = None
        self.re_embed = n_e
        self.sane_index_shape = sane_index_shape

    @torch.no_grad()
    def forward_nhwc(self, z, segm_map, want_nchw=False):
        B, H, W, _ = z.shape
        ps = self.spatial_size
        ids = ops.mask_to_ids(segm_map, H // ps, W // ps)
        r = ops.vq_search(z, self._codebook(), ids, ps=ps, cont_stride=self.n_e, want_nchw=want_nchw)
        r["loss"] = _loss_from_sqerr(r["sqerr"], z.numel(), self.beta)
        r["ids"] = ids
        return r

    def forward(self, z, segm_map, temp=None, rescale_logits=False, return_logits=False):
        _check_gumbel_args(temp, rescale_logits, return_logits)
        ps = self.spatial_size
        if z.dim() != 4 or z.shape[2] % ps or z.shape[3] % ps:
            raise ValueError(f"latent {tuple(z.shape)}: H and W must be multiples of the patch size {ps}")
        from . import vqgan_autograd as VA
        if VA.recording(self, z):          # training: straight-through + codebook-loss gradients
            return VA.quantizer_spatial_forward(self, z, segm_map)
        with torch.no_grad():
            r = self.forward_nhwc(ops.nchw_to_nhwc(z), segm_map, want_nchw=True)
            # unlike the top quantizer, the reference returns the continual indices flat here (:460)
            return r["zq_nchw"], r["loss"], (None, r["idx_cont"].reshape(-1), list(r["idx_list"].unbind(0)))

    @torch.no_grad()
    def get_codebook_entry(self, indices_list, segm_map, shape, nhwc=False):
        # the reference ignores shape[3] and uses e_dim (:480-481)
        B, Hp, Wp = shape[0], shape[1], shape[2]
        ps = self.spatial_size
        ids = ops.mask_to_ids(segm_map, Hp, Wp)
        idx = self._resolve_indices(indices_list, ids)
        cz = self.e_dim // (ps * ps)
        zq_nhwc, zq_nchw = ops.vq_gather(self._codebook(), idx, ids, B=B, Hz=Hp * ps, Wz=Wp * ps, Cz=cz,
                                         ps=ps, want_nchw=not nhwc, want_nhwc=nhwc)
        return zq_nhwc if nhwc else zq_nchw
