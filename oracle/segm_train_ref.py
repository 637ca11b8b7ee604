"""Plain-PyTorch fp32 restatement of the parsing tokenizer's training step, as a pure function of explicit state dicts.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  The product package never imports this file.

Restates /root/reference/models/vqgan_model.py VQSegmentationModel.training_step (:177-182) with VQModel.feed_data
(:117-124: F.one_hot of the parsing map), encode / decode / forward_step (:97-115), VectorQuantizer.forward
(models/archs/vqgan_arch.py:79-122: nearest code, legacy-beta loss, straight-through) and BCELossWithQuant
(models/losses/segmentation_loss.py:12-25, codebook_weight 1).  Encoder / Decoder are oracle/vqgan_ref's.
Pinned against the real reference by tests/test_segm_train_oracle.py (fixture: oracle/make_golden_segm_train.py).
"""
import torch
import torch.nn.functional as F

from . import vqgan_ref as V


def quantize_train(codebook, z, beta=0.25, legacy=True):
    """VectorQuantizer.forward with its autograd semantics -> (z_q NCHW, loss, idx [b,h,w])"""
    b, c, hh, ww = z.shape
    zp = z.permute(0, 2, 3, 1).contiguous()
    rows = zp.view(-1, c)
    d = torch.sum(rows ** 2, dim=1, keepdim=True) + torch.sum(codebook ** 2, dim=1) - 2 * (rows @ codebook.t())
    idx = torch.argmin(d, dim=1)
    zq = codebook[idx].view(zp.shape)
    if legacy:
        loss = torch.mean((zq.detach() - zp) ** 2) + beta * torch.mean((zq - zp.detach()) ** 2)
    else:
        loss = beta * torch.mean((zq.detach() - zp) ** 2) + torch.mean((zq - zp.detach()) ** 2)
    zq = zp + (zq - zp).detach()
    return zq.permute(0, 3, 1, 2).contiguous(), loss, idx.view(b, hh, ww)


def segm_training_step(sd, codebook, segm, n_classes=24, beta=0.25):
    """sd: encoder.* / decoder.* / quant_conv.* / post_quant_conv.* tensors; codebook [n_e, D]; segm int [B,H,W].
    -> dict(total_loss, bce_loss, quant_loss, xrec, idx); tensors that require grad receive loss.backward()'s
    gradients as the reference's optimiser sees them."""
    x = F.one_hot(segm.long(), num_classes=n_classes).permute(0, 3, 1, 2).contiguous().float()
    h = V.conv(sd, "quant_conv", V.encoder(sd, x, "encoder."), padding=0)
    quant, qloss, idx = quantize_train(codebook, h, beta)
    xrec = V.decoder(sd, V.conv(sd, "post_quant_conv", quant, padding=0), "decoder.")
    bce = F.binary_cross_entropy_with_logits(xrec, x)
    return dict(total_loss=bce + qloss, bce_loss=bce, quant_loss=qloss, xrec=xrec, idx=idx)
