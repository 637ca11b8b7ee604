"""Plain-PyTorch fp32 restatement of one index-prediction training step
(VQGANTextureAwareSpatialHierarchyInferenceModel.optimize_parameters, /root/reference/models/
hierarchy_inference_model.py:227-245), with the 18 Dropout2d draws as an input, and of its validation metric
(``inference``, :247-298).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Training-mode counterparts of oracle/indexpred_ref.py over reference-keyed state dicts: UNet (unet_arch.py:460-471)
and MultiHeadFCNHead (fcn_arch.py:335-348: per head a ConvModule, the shared Dropout2d called once per head, so one
[B, channels] mask per head in head order, then the head's conv_seg), with mmcv's ConvModule on batch statistics
(parsing_gen_train_ref.conv_module), and the loss sum over heads of CrossEntropyLoss(ignore_index=-1)
(cross_entropy_loss.py: F.cross_entropy(reduction='none') then .mean() over all positions).
"""
import torch
import torch.nn.functional as F

from oracle import indexpred_ref
from oracle.indexpred_ref import _n
from oracle.parsing_gen_train_ref import Margins, conv_module, running_stats  # noqa: F401 (re-exported)


def unet(sd, x, running, probe=None):
    """UNet.forward in training mode -> dec_outs (coarsest first)"""
    n_stage = _n(sd, r"encoder\.(\d+)\.")
    enc_outs = []
    for i in range(n_stage):
        if i != 0:
            if probe is not None:
                probe.max_pool(x)
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


def fcn_heads(sd, inputs, masks, running, p_drop=0.1, in_index=4, probe=None):
    """MultiHeadFCNHead.forward in training mode; masks[k] [B, channels] is head k's Dropout2d draw (None: no
    dropout) -> the 18 logit maps"""
    x = inputs[in_index]
    out = []
    for k in range(_n(sd, r"conv_seg_head_list\.(\d+)\.")):
        y = conv_module(sd, f"convs_list.{k}.0.", x, 1, running, probe)
        if masks is not None:
            B, C = masks[k].shape
            y = y * masks[k].to(y.dtype).div(1 - p_drop).view(B, C, 1, 1)
        out.append(F.conv2d(y, sd[f"conv_seg_head_list.{k}.weight"], sd[f"conv_seg_head_list.{k}.bias"]))
    return out


def gt_indices_list(own, tex, n_head=18):
    """the bottom quantizer's per-texture index maps: own index where tex == k, -1 elsewhere"""
    return [torch.where(tex == k, own, torch.full_like(own, -1)) for k in range(n_head)]


def train_loss(sd_unet, sd_fcn, feature_t, gt_list, masks, running_unet, running_fcn, p_drop=0.1, in_index=4,
               probe=None):
    """-> (loss, logits list): the forward of optimize_parameters (:231-239); the running statistics in
    running_unet / running_fcn (keyed like the state dicts) are updated as the reference's BatchNorm2d does"""
    logits = fcn_heads(sd_fcn, unet(sd_unet, feature_t, running_unet, probe), masks, running_fcn, p_drop, in_index,
                       probe)
    loss = 0
    for lg, gt in zip(logits, gt_list):
        loss = loss + F.cross_entropy(lg, gt, reduction="none", ignore_index=-1).mean()
    return loss, logits


def accuracy(sd_unet, sd_fcn, feature_t, own, tex, in_index=4):
    """inference's metric (:247-298) on one batch, eval-mode nets: (correct own-head argmaxes) / (h*w) / B summed
    as the reference does, i.e. the share of all B*h*w positions"""
    with torch.no_grad():
        logits = indexpred_ref.fcn_heads(sd_fcn, indexpred_ref.unet(sd_unet, feature_t), in_index)
    B, h, w = own.shape
    correct = 0
    for k, lg in enumerate(logits):
        roi = tex == k
        correct += int((lg.argmax(1)[roi] == own[roi]).sum())
    return correct / (B * h * w)
