"""Plain-PyTorch restatement of the hierarchical VQGAN's bottom-level training step, as a pure function of explicit
state dicts and the torch RNG (fp32 or fp64: the dtype of the tensors passed in).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Restates models/hierarchy_vqgan_model.py HierarchyVQSpatialTextureAwareModel.training_step (:250-291) with
forward_step (:233-238), top_encode / bot_encode / decode (:211-231), the legacy-beta straight-through loss of
VectorQuantizerSpatialTextureAware.forward (models/archs/vqgan_arch.py:375-461) and the GAN losses of
models/losses/vqgan_loss.py.  LPIPS enters as zero, as in oracle/vqgan_train_ref.py.
"""
import torch
import torch.nn.functional as F

from . import vqgan_ref as V
from . import vqgan_train_ref as TR


def quantize_spatial_train(codebooks, z, segm_map, ps=2, beta=0.25, probe=None):
    """VectorQuantizerSpatialTextureAware.forward with its autograd semantics over F.unfold's ps x ps patches ->
    (straight-through z_q, codebook loss, continual indices [rows] (idx + n_e * book, -1 without a codebook)).
    ``probe`` (list): per selected row, the gap between its second-best and best distance, relative to the best."""
    b, c, hh, ww = z.shape
    hp, wp = hh // ps, ww // ps
    seg = F.interpolate(segm_map, size=(hp, wp), mode="nearest").reshape(-1)
    rows = F.unfold(z, (ps, ps), stride=ps).permute(0, 2, 1).reshape(-1, c * ps * ps)
    zq = torch.zeros_like(rows)
    cont = torch.full((rows.shape[0],), -1, dtype=torch.long, device=z.device)
    for k in range(len(codebooks)):
        sel = seg == k
        if sel.any():
            e = codebooks[k]
            d = torch.sum(rows[sel] ** 2, dim=1, keepdim=True) + torch.sum(e ** 2, dim=1) - 2 * (rows[sel] @ e.t())
            i = torch.argmin(d, dim=1)
            zq = zq.index_put((sel.nonzero(as_tuple=True)[0],), e[i])
            cont[sel] = i + e.shape[0] * k
            if probe is not None:
                two = torch.topk(d.detach(), 2, dim=1, largest=False).values
                probe.append(((two[:, 1] - two[:, 0]) / two[:, 0].abs().clamp_min(1e-12)).min())
    zq = F.fold(zq.view(b, hp * wp, -1).permute(0, 2, 1), (hh, ww), kernel_size=(ps, ps), stride=ps)
    loss = torch.mean((zq.detach() - z) ** 2) + beta * torch.mean((zq - z.detach()) ** 2)
    return z + (zq - z).detach(), loss, cont


def disc_kink_margin(sd, x, n_layers=3):
    """the smallest |pre-activation| of the discriminator's LeakyReLUs on ``x`` and the smallest distance of its
    logits from the hinge kinks at +-1 (TR.discriminator in training mode, restated layer by layer)"""
    p = "main."
    h = F.conv2d(x, sd[p + "0.weight"], sd[p + "0.bias"], stride=2, padding=1)
    m = float(h.abs().min())
    h = F.leaky_relu(h, 0.2)
    i = 2
    for n in range(1, n_layers + 1):
        h = F.conv2d(h, sd[f"{p}{i}.weight"], None, stride=2 if n < n_layers else 1, padding=1)
        bn = f"{p}{i + 1}."
        h = F.batch_norm(h, sd[bn + "running_mean"].clone(), sd[bn + "running_var"].clone(), sd[bn + "weight"],
                         sd[bn + "bias"], True, 0.1, 1e-5)
        m = min(m, float(h.abs().min()))
        h = F.leaky_relu(h, 0.2)
        i += 3
    logits = F.conv2d(h, sd[f"{p}{i}.weight"], sd[f"{p}{i}.bias"], stride=1, padding=1)
    return m, float(torch.minimum((logits - 1).abs(), (logits + 1).abs()).min())


def training_step(sd, top_books, bot_books, sd_disc, x, mask, step, *, disc_start_step=1, disc_weight_max=1.0,
                  diff_aug=True, disc_layers=3, probe=None, disc_masks=None):
    """-> dict(loss, d_loss or None, nll_loss, g_loss, d_weight, codebook_loss, bot_idx, xrec).  sd keys:
    top_encoder.*, top_quant_conv.*, top_post_quant_conv.*, decoder.*, bot_encoder.*, bot_quant_conv.*,
    bot_post_quant_conv.*, bot_decoder_res.*; top_books [18, 1024, D] (frozen), bot_books: 18 [n_e, 4 D] (requires
    grad for the codebook gradient).  ``probe`` (dict): 'argmin' (relative second-best gaps of both quantizers) and
    'kink' (discriminator margins of the three passes) for the fixture's seed scan.  ``disc_masks``: per
    discriminator pass the LeakyReLU masks TR.discriminator imposes (fake image, real image, detached fake image)."""
    masks = list(disc_masks) if disc_masks is not None else [None] * 3
    with torch.no_grad():                                                   # forward_step :236-237
        ht = V.conv(sd, "top_quant_conv", V.encoder(sd, x, "top_encoder."), padding=0)
        quant_top, _, _, _ = V.quantize_texture(top_books, ht, mask)
        quant_top = V.conv(sd, "top_post_quant_conv", quant_top, padding=0)
        if probe is not None:
            tp = []
            quantize_spatial_train(list(top_books), ht, mask, ps=1, probe=tp)
            probe["argmin"] = tp
    hb = V.conv(sd, "bot_quant_conv", V.encoder(sd, x, "bot_encoder."), padding=0)
    qb, codebook_loss, bot_idx = quantize_spatial_train(bot_books, hb, mask,
                                                        probe=probe["argmin"] if probe is not None else None)
    bot_h = V.decoder_res(sd, V.conv(sd, "bot_post_quant_conv", qb, padding=0), "bot_decoder_res.")
    xrec = V.decoder(sd, quant_top, "decoder.", bot_h=bot_h)
    # training_step :253-291, as the top step (oracle/vqgan_train_ref.training_step)
    nll_loss = torch.mean(torch.abs(x - xrec))
    xr = TR.diff_augment(xrec) if diff_aug else xrec
    g_loss = -torch.mean(TR.discriminator(sd_disc, xr, n_layers=disc_layers, masks=masks[0]))
    last = sd["decoder.conv_out.weight"]
    rg = torch.autograd.grad(nll_loss, last, retain_graph=True)[0]
    gg = torch.autograd.grad(g_loss, last, retain_graph=True)[0]
    d_weight = torch.clamp(torch.norm(rg) / (torch.norm(gg) + 1e-4), 0.0, disc_weight_max).detach()
    d_weight = d_weight * (1 if step >= disc_start_step else 0.0)
    loss = nll_loss + d_weight * g_loss + codebook_loss
    d_loss = None
    if step > disc_start_step:
        real_in = TR.diff_augment(x.detach()) if diff_aug else x.detach()
        lr_ = TR.discriminator(sd_disc, real_in, n_layers=disc_layers, masks=masks[1])
        lf_ = TR.discriminator(sd_disc, xr.detach(), n_layers=disc_layers, masks=masks[2])
        d_loss = 0.5 * (torch.mean(F.relu(1.0 - lr_)) + torch.mean(F.relu(1.0 + lf_)))
        if probe is not None:
            probe["kink"] = [disc_kink_margin(sd_disc, t.detach(), disc_layers) for t in (xr, real_in)]
    return dict(loss=loss, d_loss=d_loss, nll_loss=nll_loss, g_loss=g_loss, d_weight=d_weight,
                codebook_loss=codebook_loss, bot_idx=bot_idx, xrec=xrec)
