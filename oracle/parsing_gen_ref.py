"""Plain-PyTorch fp32 restatement of the parsing generator of sample_from_pose (pose + shape attributes -> parsing
map), and the loader that makes the reference's own `models.*` package see text2human_b200's parsing-generator
mirrors.

TEST / BASELINE INFRASTRUCTURE ONLY (see oracle/__init__.py).

Restates /root/reference/models/archs/shape_attr_embedding_arch.py (ShapeAttrEmbedding),
/root/reference/models/archs/unet_arch.py (ShapeUNet :503-674; its decoder is UNet's) and
/root/reference/models/archs/fcn_arch.py (FCNHead :159-225) and sample_model.py generate_parsing_map (:431-437),
functionally over reference-keyed state dicts, in eval mode.  mmcv's ConvModule is `indexpred_ref.conv_module`.
"""
import sys
import types

import torch
import torch.nn.functional as F

from oracle import ref_loader as RL
from oracle.indexpred_ref import _n, conv_module


def shape_attr_embedding(sd, attr, cls_num_list):
    """ShapeAttrEmbedding.forward (shape_attr_embedding_arch.py:23-36): per attribute one_hot -> Linear -> LeakyReLU
    -> Linear, concatenated, then Linear -> LeakyReLU -> Linear.  attr int64 [B, n_attr] -> [B, out_dim]"""
    hs = []
    for i, n in enumerate(cls_num_list):
        h = F.one_hot(attr[:, i], num_classes=n).to(torch.float32)
        h = F.leaky_relu(F.linear(h, sd[f"attr_{i}.0.weight"], sd[f"attr_{i}.0.bias"]), 0.01)
        hs.append(F.linear(h, sd[f"attr_{i}.2.weight"], sd[f"attr_{i}.2.bias"]))
    h = F.leaky_relu(F.linear(torch.cat(hs, 1), sd["fusion.0.weight"], sd["fusion.0.bias"]), 0.01)
    return F.linear(h, sd["fusion.2.weight"], sd["fusion.2.bias"])


def shape_unet(sd, x, e):
    """ShapeUNet.forward (unet_arch.py:657-674) with the defaults: every encoder stage reads
    cat([x, e broadcast over H, W]) -- pooled by the stage's MaxPool2d(2) for stages 1..4 -- then the UNet
    decoder (bilinear x2 + 1x1 ConvModule, skip concatenation, two 3x3 ConvModules).  Returns dec_outs, coarsest
    first."""
    n_stage = _n(sd, r"encoder\.(\d+)\.")
    B, Ce = e.shape
    enc_outs = []
    for i in range(n_stage):
        _, _, H, W = x.shape
        x = torch.cat([x, e.view(B, Ce, 1, 1).expand(B, Ce, H, W)], dim=1)   # :661-667
        if i != 0:
            x = F.max_pool2d(x, 2)
        blk = f"encoder.{i}.{0 if i == 0 else 1}.convs."
        for j in range(_n(sd, rf"encoder\.{i}\.\d+\.convs\.(\d+)\.")):
            x = conv_module(sd, f"{blk}{j}.", x, 1)
        enc_outs.append(x)
    dec_outs = [x]
    for i in reversed(range(n_stage - 1)):                                   # :669-672
        p = f"decoder.{i}."
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
        x = conv_module(sd, p + "upsample.interp_upsample.1.", x, 0)
        x = torch.cat([enc_outs[i], x], dim=1)
        for j in range(_n(sd, rf"decoder\.{i}\.conv_block\.convs\.(\d+)\.")):
            x = conv_module(sd, f"{p}conv_block.convs.{j}.", x, 1)
        dec_outs.append(x)
    return dec_outs


def fcn_head(sd, inputs, in_index=4):
    """FCNHead.forward (fcn_arch.py:218-225), num_convs=1, concat_input=False, eval (Dropout2d is identity):
    3x3 ConvModule then the 1x1 conv_seg -> [B, num_classes, H, W]"""
    y = conv_module(sd, "convs.0.", inputs[in_index], 1)
    return F.conv2d(y, sd["conv_seg.weight"], sd["conv_seg.bias"])


def generate_parsing_map(sd_emb, sd_unet, sd_head, pose, shape_attr, cls_num_list, in_index=4):
    """SampleFromPoseModel.generate_parsing_map (sample_model.py:431-437) -> (logits, int64 parsing map [B,1,H,W])"""
    logits = fcn_head(sd_head, shape_unet(sd_unet, pose, shape_attr_embedding(sd_emb, shape_attr, cls_num_list)),
                      in_index)
    return logits, logits.argmax(dim=1, keepdim=True)


def install(archs="reference", wrappers=()):
    """ref_loader.install, plus the parsing generator: with archs="mirror" the mirror ShapeUNet / FCNHead replace the
    placeholders of `models.archs.unet_arch` / `.fcn_arch` and the mirror ShapeAttrEmbedding is installed as
    `models.archs.shape_attr_embedding_arch`, before the (unmodified) wrapper files are loaded, so that e.g.
    `models/sample_model.py`'s SampleFromPoseModel methods run on them.  ns.shape_attr_embedding_arch is set in
    both modes."""
    ns = RL.install(archs, wrappers=())
    if archs == "mirror":
        import text2human_b200.parsing_gen_arch as pg
        ns.unet_arch.ShapeUNet = pg.ShapeUNet
        ns.fcn_arch.FCNHead = pg.FCNHead
        sae = types.ModuleType("models.archs.shape_attr_embedding_arch")
        sae.ShapeAttrEmbedding = pg.ShapeAttrEmbedding
        sys.modules[sae.__name__] = sae
    ns.shape_attr_embedding_arch = sys.modules["models.archs.shape_attr_embedding_arch"]
    for w in wrappers:
        setattr(ns, w, RL._exec(f"models.{w}", f"{ns.root}/models/{w}.py"))
    return ns
