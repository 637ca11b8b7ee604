"""Plain-PyTorch fp32 restatement of one parsing-generator training step (ParsingGenModel.optimize_parameters,
/root/reference/models/parsing_gen_model.py:80-95), with the Dropout2d draw as an input.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Training-mode counterparts of oracle/parsing_gen_ref.py over reference-keyed state dicts: mmcv's ConvModule with
BatchNorm2d on batch statistics (F.batch_norm(training=True, momentum 0.1, eps 1e-5), which also updates the
running statistics it is given), ShapeUNet (unet_arch.py:657-674), FCNHead (fcn_arch.py:151-156, 218-225; Dropout2d
= input * mask / (1-p) with one mask entry per image and channel), and CrossEntropyLoss
(cross_entropy_loss.py: F.cross_entropy(reduction='none', ignore_index=-100) then .mean()).
"""
import torch
import torch.nn.functional as F

from oracle.indexpred_ref import _n


class Margins:
    """How far one forward pass stays from the points where the backward pass is discontinuous: the smallest |u| of
    a pre-activation in front of a (Leaky)ReLU, and the smallest relative gap between the largest and the second
    largest value of a max-pool window whose maximum is positive.  A value within rounding of such a point is a
    kink / tie that two correct fp32 implementations may resolve differently (routing a pixel's gradient elsewhere,
    or scaling it by 0.01 instead of 1); a fixture whose margins are wide has no such value."""

    def __init__(self):
        self.relu = float("inf")
        self.lrelu = float("inf")
        self.pool = float("inf")

    def pre_act(self, u, leaky=False):
        m = float(u.detach().abs().min())
        if leaky:
            self.lrelu = min(self.lrelu, m)
        else:
            self.relu = min(self.relu, m)

    def max_pool(self, x):
        B, C, H, W = x.shape
        w = x.detach()[:, :, :H // 2 * 2, :W // 2 * 2].reshape(B, C, H // 2, 2, W // 2, 2)
        w = w.permute(0, 1, 2, 4, 3, 5).reshape(-1, 4)
        top = w.topk(2, dim=1).values
        pos = top[:, 0] > 0
        if bool(pos.any()):
            self.pool = min(self.pool, float(((top[pos, 0] - top[pos, 1]) / top[pos, 0]).min()))


def shape_attr_embedding(sd, attr, cls_num_list, probe=None):
    """oracle.parsing_gen_ref.shape_attr_embedding in the state dict's dtype (fp64 checks of the fp32 arithmetic)"""
    hs = []
    for i, n in enumerate(cls_num_list):
        h = F.one_hot(attr[:, i], num_classes=n).to(sd[f"attr_{i}.0.weight"].dtype)
        u = F.linear(h, sd[f"attr_{i}.0.weight"], sd[f"attr_{i}.0.bias"])
        if probe is not None:
            probe.pre_act(u, leaky=True)
        hs.append(F.linear(F.leaky_relu(u, 0.01), sd[f"attr_{i}.2.weight"], sd[f"attr_{i}.2.bias"]))
    u = F.linear(torch.cat(hs, 1), sd["fusion.0.weight"], sd["fusion.0.bias"])
    if probe is not None:
        probe.pre_act(u, leaky=True)
    return F.linear(F.leaky_relu(u, 0.01), sd["fusion.2.weight"], sd["fusion.2.bias"])


def conv_module(sd, p, x, padding, running, probe=None):
    """ConvModule in training mode; running[p + "bn.running_mean" / "bn.running_var"] are updated in place"""
    x = F.conv2d(x, sd[p + "conv.weight"], None, padding=padding)
    x = F.batch_norm(x, running[p + "bn.running_mean"], running[p + "bn.running_var"], sd[p + "bn.weight"],
                     sd[p + "bn.bias"], True, 0.1, 1e-5)
    if probe is not None:
        probe.pre_act(x)
    return F.relu(x)


def running_stats(*sds):
    """fresh copies of the BatchNorm running statistics of state dicts, keyed like them (prefixes kept apart by
    the caller)"""
    return {k: v.detach().clone() for sd in sds for k, v in sd.items() if k.endswith(("running_mean", "running_var"))}


def shape_unet(sd, x, e, running, probe=None):
    n_stage = _n(sd, r"encoder\.(\d+)\.")
    B, Ce = e.shape
    enc_outs = []
    for i in range(n_stage):
        _, _, H, W = x.shape
        if i != 0 and probe is not None:
            probe.max_pool(x)           # the broadcast channels are constant: their windows tie by construction
        x = torch.cat([x, e.view(B, Ce, 1, 1).expand(B, Ce, H, W)], dim=1)
        if i != 0:
            x = F.max_pool2d(x, 2)
        blk = f"encoder.{i}.{0 if i == 0 else 1}.convs."
        for j in range(_n(sd, rf"encoder\.{i}\.\d+\.convs\.(\d+)\.")):
            x = conv_module(sd, f"{blk}{j}.", x, 1, running, probe)
        enc_outs.append(x)
    dec_outs = [x]
    for i in reversed(range(n_stage - 1)):
        p = f"decoder.{i}."
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
        x = conv_module(sd, p + "upsample.interp_upsample.1.", x, 0, running, probe)
        x = torch.cat([enc_outs[i], x], dim=1)
        for j in range(_n(sd, rf"decoder\.{i}\.conv_block\.convs\.(\d+)\.")):
            x = conv_module(sd, f"{p}conv_block.convs.{j}.", x, 1, running, probe)
        dec_outs.append(x)
    return dec_outs


def fcn_head(sd, inputs, mask, running, p_drop=0.1, in_index=4, probe=None):
    y = conv_module(sd, "convs.0.", inputs[in_index], 1, running, probe)
    if mask is not None:
        B, C = mask.shape
        y = y * mask.to(y.dtype).div(1 - p_drop).view(B, C, 1, 1)
    return F.conv2d(y, sd["conv_seg.weight"], sd["conv_seg.bias"])


def train_loss(sd_emb, sd_unet, sd_head, data, mask, cls_num_list, running_unet, running_head, p_drop=0.1,
               in_index=4, probe=None):
    """-> (loss, logits): the forward of optimize_parameters (:85-89) in training mode; the running statistics in
    running_unet / running_head (keyed like sd_unet / sd_head) are updated as the reference's BatchNorm2d does.
    ``probe`` (a Margins) records the distances of the pass from its kinks and ties."""
    e = shape_attr_embedding(sd_emb, data["attr"], cls_num_list, probe)
    logits = fcn_head(sd_head, shape_unet(sd_unet, data["densepose"], e, running_unet, probe), mask, running_head,
                      p_drop, in_index, probe)
    segm = data["segm"]
    if segm.dim() == 4:
        segm = segm.squeeze(1)
    return F.cross_entropy(logits, segm, reduction="none", ignore_index=-100).mean(), logits
