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


class LPIPSRef(torch.nn.Module):
    """nn.Module wrapper of ``lpips`` on a fixed state dict (the reference step calls ``self.perceptual(x, xrec)``)"""

    def __init__(self, sd):
        super().__init__()
        self.sd = sd

    def forward(self, in0, in1):
        sd = {k: v.to(device=in1.device, dtype=in1.dtype) for k, v in self.sd.items()}
        return lpips(sd, in0, in1)
