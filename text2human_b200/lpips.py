"""LPIPS perceptual distance (lpips==0.1.4, ``LPIPS(net="vgg", version="0.1")`` in eval mode) on the H100 kernels.

The reference trains both VQGANs with ``p_loss = self.perceptual(x, xrec)`` (models/vqgan_model.py:427,450,
models/hierarchy_vqgan_model.py:90,253).  ``LPIPS`` here is a mirror of that module: the same ``state_dict`` keys
(so a checkpoint taken from a real ``lpips.LPIPS`` instance loads with ``strict=True``), the same forward, and its
weights only from files the caller names.

Network (lpips/pretrained_networks.py ``vgg16``, lpips/lpips.py ``LPIPS.forward``):
  ScalingLayer (x - shift) / scale  ->  VGG16 ``features`` cut after indices 3, 8, 15, 22, 29 (relu1_2 .. relu5_3)
  -> per slice: unit-normalise each pixel's channel vector (eps 1e-10), squared difference, 1x1 ``lin`` conv to one
  channel (no bias; its Dropout is inactive in eval mode), spatial mean; the five means are summed -> [B,1,1,1].

Execution: in0 and in1 run through the trunk as ONE batch of 2B images (each weight tile is read once per call and
the deep slices, which have few pixels, fill more tiles).  The 3x3 convs and their data gradients run on the
tap-GEMM (``conv_grad``) with a ReLU epilogue; the scaling, the five heads and the ReLU backward are csrc/lpips.cu.
Because the loss is a scalar per image and in0 is constant, the gradient with respect to in1 is computed in the same
call as the value ("gradient at forward"): every head folds its own backward and the mask of its slice's last ReLU
into one pass, and the data gradients walk the trunk back to the image.  The autograd node only scales that map by
``grad_output[b]``, so it can run its backward any number of times (``retain_graph``).
"""
import math

import torch
import torch.nn as nn

from . import conv_grad as G
from . import ops
from .ops import ACT_RELU, CVT_MAXPOOL2

# torchvision vgg16 ``features``: 'M' = MaxPool2d(2, 2), int = Conv2d(cin, n, 3, padding=1) + ReLU(inplace=True)
VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M")
SLICE_ENDS = (4, 9, 16, 23, 30)          # lpips vgg16: slice k holds features[SLICE_ENDS[k-1]:SLICE_ENDS[k]]
CHNS = (64, 128, 256, 512, 512)
SHIFT = (-.030, -.088, -.188)            # lpips ScalingLayer
SCALE = (.458, .448, .450)
VGG_FILE = "vgg16-397923af.pth"          # torchvision's ImageNet VGG16 weights (features.N.weight / .bias)
LIN_FILE = "weights/v0.1/vgg.pth"        # lpips' learned heads (lin0..lin4.model.1.weight)


def vgg16_features():
    """the modules of torchvision's ``vgg16().features`` (31 entries), in order"""
    layers, cin = [], 3
    for v in VGG16_CFG:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            cin = v
    return layers


def grad_scale(H, W):
    """power-of-two factor carried by the gradient planes inside the trunk's backward, undone when the gradient is
    added to the image gradient: keeps the head gradients (~ gscale / (h w) per pixel) in fp16's normal range"""
    return 2.0 ** (math.floor(math.log2(H * W)) + 6)


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.tensor(SHIFT)[None, :, None, None])
        self.register_buffer("scale", torch.tensor(SCALE)[None, :, None, None])


class VGG16Slices(nn.Module):
    """lpips.pretrained_networks.vgg16: slice1..slice5 keep torchvision's ``features`` indices as module names"""

    def __init__(self):
        super().__init__()
        feats = vgg16_features()
        start = 0
        for k, end in enumerate(SLICE_ENDS):
            s = nn.Sequential()
            for i in range(start, end):
                s.add_module(str(i), feats[i])
            setattr(self, f"slice{k + 1}", s)
            start = end
        self.N_slices = 5

    def slice_convs(self):
        """[[Conv2d, ...] per slice]"""
        return [[m for m in getattr(self, f"slice{k + 1}") if isinstance(m, nn.Conv2d)] for k in range(5)]


class NetLinLayer(nn.Module):
    """lpips NetLinLayer(chn_in, use_dropout=True): Dropout (inactive in eval mode) + 1x1 conv to one channel"""

    def __init__(self, chn_in):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn_in, 1, 1, stride=1, padding=0, bias=False))


def _map_vgg_features(sd):
    """torchvision ``features.N.*`` keys -> ``net.sliceK.N.*``"""
    out = {}
    for key, v in sd.items():
        if not key.startswith("features."):
            continue
        i = int(key.split(".")[1])
        k = next(j for j, end in enumerate(SLICE_ENDS) if i < end)
        out[f"net.slice{k + 1}." + key[len("features."):]] = v
    return out


class _Fn(torch.autograd.Function):
    """p_loss = LPIPS(in0, in1) with the gradient wrt in1 computed in the forward (see the module docstring)"""

    @staticmethod
    def forward(ctx, in1, in0, mod):
        g = torch.zeros(in1.shape, dtype=torch.float32, device=in1.device)
        val = mod.run(in0, in1, g=g, alpha=1.0)
        ctx.save_for_backward(g)
        return val.float().view(-1, 1, 1, 1).to(in1.dtype)

    @staticmethod
    def backward(ctx, dv):
        (g,) = ctx.saved_tensors
        return (g * dv.reshape(-1, 1, 1, 1).to(g.dtype)).to(dv.dtype), None, None


class LPIPS(nn.Module):
    """Mirror of ``lpips.LPIPS(net="vgg", version="0.1")`` in eval mode, on libt2h.

    ``pretrained=True`` loads ``vgg_path`` (torchvision's ``vgg16-397923af.pth``) into the trunk and ``model_path``
    (lpips' ``weights/v0.1/vgg.pth``) into the heads; nothing is downloaded.  ``pretrained=False`` leaves random
    parameters, for tests and for ``load_state_dict``.  The parameters never require grad: the loss is used frozen.
    Only ``in1`` may require grad (the reconstruction, as the VQGAN trainers call it)."""

    def __init__(self, pretrained=True, net="vgg", version="0.1", lpips=True, spatial=False, model_path=None,
                 vgg_path=None):
        super().__init__()
        if net != "vgg":
            raise NotImplementedError(f"LPIPS net={net!r}: only 'vgg' is implemented")
        if version != "0.1":
            raise NotImplementedError(f"LPIPS version={version!r}: only '0.1' is implemented")
        if not lpips:
            raise NotImplementedError("LPIPS lpips=False (the non-learned variant) is not implemented")
        if spatial:
            raise NotImplementedError("LPIPS spatial=True is not implemented")
        self.scaling_layer = ScalingLayer()
        self.net = VGG16Slices()
        self.L = 5
        for k, c in enumerate(CHNS):
            setattr(self, f"lin{k}", NetLinLayer(c))
        self.lins = nn.ModuleList([getattr(self, f"lin{k}") for k in range(5)])   # lpips registers both names
        if pretrained:
            missing = [f"{what} ({name})" for what, name, p in (("vgg_path", VGG_FILE, vgg_path),
                                                               ("model_path", LIN_FILE, model_path)) if p is None]
            if missing:
                raise FileNotFoundError(
                    f"LPIPS(pretrained=True) loads its weights only from named files: torchvision's {VGG_FILE} "
                    f"(vgg_path=) and lpips' {LIN_FILE} (model_path=); missing: {', '.join(missing)}")
            self.load_pretrained(vgg_path, model_path)
        self.requires_grad_(False)
        self.eval()
        self._packed = None

    def load_pretrained(self, vgg_path, model_path):
        """torchvision's VGG16 state dict into the trunk and lpips' lin weights into the heads (strict)"""
        vgg = torch.load(vgg_path, map_location="cpu")
        lin = torch.load(model_path, map_location="cpu")
        sd = _map_vgg_features(vgg)
        for k in range(5):
            sd[f"lin{k}.model.1.weight"] = lin[f"lin{k}.model.1.weight"]
            sd[f"lins.{k}.model.1.weight"] = lin[f"lin{k}.model.1.weight"]
        sd["scaling_layer.shift"] = self.scaling_layer.shift
        sd["scaling_layer.scale"] = self.scaling_layer.scale
        self.load_state_dict(sd, strict=True)

    # ---- packed weights (frozen; repacked when a parameter changes or the precision mode does)
    def _pack(self):
        params = list(self.parameters()) + list(self.buffers())
        key = (ops.get_terms(), tuple((p.device, p.data_ptr(), p._version) for p in params))
        if self._packed is not None and self._packed[0] == key:
            return self._packed[1]
        ops._need_cuda(*params)
        terms = ops.get_terms()
        slices = []
        for convs in self.net.slice_convs():
            packs = []
            for conv in convs:
                wn, wt = G.weight_planes(G.oihw_to_master(conv.weight.detach()), terms)
                packs.append((wn, wt, conv.bias.detach().float().contiguous()))
            slices.append(packs)
        lins = [getattr(self, f"lin{k}").model[1].weight.detach().float().reshape(-1).contiguous() for k in range(5)]
        shift = self.scaling_layer.shift.detach().float().reshape(3).contiguous()
        scale = self.scaling_layer.scale.detach().float().reshape(3).contiguous()
        packed = dict(slices=slices, lins=lins, shift=shift, scale=scale)
        self._packed = (key, packed)
        return packed

    @staticmethod
    def check_inputs(in0, in1):
        if in0.shape != in1.shape:
            raise ValueError(f"LPIPS: in0 {tuple(in0.shape)} and in1 {tuple(in1.shape)} differ")
        if in1.dim() != 4 or in1.shape[1] != 3:
            raise ValueError(f"LPIPS: inputs must be [B,3,H,W], got {tuple(in1.shape)}")
        if in1.shape[2] % 16 or in1.shape[3] % 16:
            raise ValueError(f"LPIPS: H and W must be multiples of 16 (four 2x2 max-pools), got {tuple(in1.shape)}")

    def run(self, in0, in1, g=None, alpha=1.0):
        """-> p_loss fp64 [B].  With ``g`` (fp32 NCHW like in1): g += alpha * d p_loss[b] / d in1, per image."""
        self.check_inputs(in0, in1)
        ops._need_cuda(in0, in1)
        pk = self._pack()
        B, _, H, W = in1.shape
        n = 2 * B
        want = g is not None
        sigma = grad_scale(H, W)
        h = ops.lpips_scale_fwd(in0, in1, pk["shift"], pk["scale"])
        feats, saved = [], []
        hh, ww = H, W
        for k, packs in enumerate(pk["slices"]):
            if k > 0:
                h = ops.f32_to_planes(feats[-1], CVT_MAXPOOL2)
                hh, ww = hh // 2, ww // 2
            mids = []
            for j, (wn, _, b) in enumerate(packs):
                last = j == len(packs) - 1
                h = G.forward("k3", h, wn, b, n=n, in_hw=(hh, ww), planes_out=not last, act=ACT_RELU)
                if not last and want:
                    mids.append(h[0, B:])           # the in1 half's hi plane: the ReLU mask of the backward
            feats.append(h)
            saved.append(mids)
        acc = torch.zeros(B, dtype=torch.float64, device=in1.device)
        gin = None
        for k in reversed(range(5)):
            f = feats[k]
            planes = ops.lpips_head(f[:B], f[B:], pk["lins"][k], acc, gscale=sigma / (f.shape[1] * f.shape[2]),
                                    gin=gin, want_grad=want)
            if not want:
                continue
            fh, fw = f.shape[1:3]
            packs = pk["slices"][k]
            for j in reversed(range(len(packs))):
                d = G.dgrad("k3", planes, packs[j][1], n=B, in_hw=(fh, fw))
                if j > 0:
                    planes = ops.relu_bwd(saved[k].pop(), d)
            feats[k] = planes = None
            if k > 0:
                prev = feats[k - 1][B:]
                gin = torch.empty_like(prev)
                ops.maxpool2_bcast_bwd(d, prev.shape[-1], 0, x=prev, dx=gin)
            else:
                ops.lpips_scale_bwd(d, pk["scale"], alpha / sigma, g)
        return acc

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        if normalize:
            raise NotImplementedError("LPIPS normalize=True (inputs in [0, 1]) is not implemented: pass [-1, 1]")
        if retPerLayer:
            raise NotImplementedError("LPIPS retPerLayer=True is not implemented")
        if in0.requires_grad and torch.is_grad_enabled():
            raise NotImplementedError("LPIPS: the gradient with respect to in0 is not implemented")
        self.check_inputs(in0, in1)
        ops._need_cuda(in0, in1)
        in0 = in0.detach()
        if torch.is_grad_enabled() and in1.requires_grad:
            return _Fn.apply(in1, in0, self)
        with torch.no_grad():
            return self.run(in0, in1.detach()).float().view(-1, 1, 1, 1).to(in1.dtype)
