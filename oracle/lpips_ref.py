"""Plain-torch restatement of LPIPS (lpips==0.1.4, ``lpips.LPIPS(net="vgg", version="0.1")`` in eval mode), used as
the fp64 CPU oracle of ``text2human_b200.lpips`` and as ``self.perceptual`` of the reference training step in
oracle/make_golden_lpips_train.py.  The lpips package is not installed here, so this restatement is written from
lpips 0.1.4's source and is not itself checked against the package; where each constant comes from:

  * ScalingLayer shift [-.030, -.088, -.188], scale [.458, .448, .450]:   lpips/lpips.py ``ScalingLayer``
  * VGG16 trunk = torchvision ``vgg16().features`` cut into slices [0:4], [4:9], [9:16], [16:23], [23:30]
    (relu1_2, relu2_2, relu3_3, relu4_3, relu5_3):                          lpips/pretrained_networks.py ``vgg16``
  * channels (64, 128, 256, 512, 512):                                     lpips/lpips.py ``LPIPS.__init__`` chns
  * normalize_tensor: x / (sqrt(sum_c x^2) + 1e-10):                       lpips/__init__.py ``normalize_tensor``
  * head: NetLinLayer = Dropout (identity in eval mode) + Conv2d(C, 1, 1, bias=False); spatial_average =
    mean over (H, W) with keepdim; the five averages summed:               lpips/lpips.py ``NetLinLayer``, ``forward``

``sd`` is a state dict with the mirror's (= lpips') keys: scaling_layer.*, net.sliceK.N.{weight,bias},
lin{k}.model.1.weight.
"""
import torch
import torch.nn.functional as F

SLICE_ENDS = (4, 9, 16, 23, 30)
CONV_IDX = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))


def _slice_key(i):
    k = next(j for j, end in enumerate(SLICE_ENDS) if i < end)
    return f"net.slice{k + 1}.{i}"


def slices(sd, x):
    """the five slice outputs of the VGG16 trunk on an (already scaled) input"""
    outs, h = [], x
    for k, idxs in enumerate(CONV_IDX):
        if k > 0:
            h = F.max_pool2d(h, kernel_size=2, stride=2)
        for i in idxs:
            p = _slice_key(i)
            h = F.relu(F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], padding=1))
        outs.append(h)
    return outs


def normalize_tensor(x, eps=1e-10):
    return x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + eps)


def lpips(sd, in0, in1):
    """-> [B,1,1,1], autograd-capable in every argument"""
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    o0 = slices(sd, (in0 - shift) / scale)
    o1 = slices(sd, (in1 - shift) / scale)
    val = 0
    for k in range(5):
        d = (normalize_tensor(o0[k]) - normalize_tensor(o1[k])) ** 2
        val = val + F.conv2d(d, sd[f"lin{k}.model.1.weight"]).mean([2, 3], keepdim=True)
    return val


def pool_windows(x):
    """[N,C,H,W] -> [N,C,H/2,W/2,4]: each 2x2 window of MaxPool2d(2) row-major (torch's order of first maxima)"""
    N, C, H, W = x.shape
    return x.reshape(N, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(N, C, H // 2, W // 2, 4)


def choices(sd, in0, in1):
    """the discrete choices of an fp64 forward of the 2B images (in0's first): (masks, picks) as
    ``lpips_conditioned`` takes them -- pre-activation > 0 per conv, first maximum per max-pool window"""
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    h = torch.cat([(in0 - shift) / scale, (in1 - shift) / scale])
    masks, picks = [], []
    for k, idxs in enumerate(CONV_IDX):
        if k > 0:
            picks.append(pool_windows(h).argmax(-1))
            h = F.max_pool2d(h, kernel_size=2, stride=2)
        for i in idxs:
            p = _slice_key(i)
            u = F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], padding=1)
            masks.append(u > 0)
            h = F.relu(u)
    return masks, picks


def lpips_conditioned(sd, in0, in1, masks, picks, trace=None):
    """``lpips`` with every discrete choice imposed: conv i's ReLU multiplies by ``masks[i]`` (bool [2B,C,h,w], the 13
    convs in CONV_IDX order, in0's images first) and the max-pool before slice k+2 takes the window element at
    ``picks[k]`` (int [2B,C,h/2,w/2] in 0..3, row-major).  Away from every kink and tie, with fp64's own choices
    (``choices``), this is ``lpips``.  -> [B,1,1,1], autograd-capable; ``trace`` (a list) receives, in order, each
    max-pool's input and each conv's (input, pre-activation)."""
    shift, scale = sd["scaling_layer.shift"], sd["scaling_layer.scale"]
    B = in1.shape[0]
    h = torch.cat([(in0 - shift) / scale, (in1 - shift) / scale])
    outs, m = [], iter(masks)
    for k, idxs in enumerate(CONV_IDX):
        if k > 0:
            if trace is not None:
                trace.append(h.detach())
            h = pool_windows(h).gather(-1, picks[k - 1].unsqueeze(-1)).squeeze(-1)
        for i in idxs:
            p = _slice_key(i)
            u = F.conv2d(h, sd[p + ".weight"], sd[p + ".bias"], padding=1)
            if trace is not None:
                trace.append((h.detach(), u.detach()))
            h = u * next(m).to(u.dtype)
        outs.append(h)
    val = 0
    for k in range(5):
        d = (normalize_tensor(outs[k][:B]) - normalize_tensor(outs[k][B:])) ** 2
        val = val + F.conv2d(d, sd[f"lin{k}.model.1.weight"]).mean([2, 3], keepdim=True)
    return val


class LPIPSRef(torch.nn.Module):
    """nn.Module wrapper of ``lpips`` on a fixed state dict (the reference step calls ``self.perceptual(x, xrec)``)"""

    def __init__(self, sd):
        super().__init__()
        self.sd = sd

    def forward(self, in0, in1):
        sd = {k: v.to(device=in1.device, dtype=in1.dtype) for k, v in self.sd.items()}
        return lpips(sd, in0, in1)
