"""Plain-PyTorch fp32 restatement of the VQGAN training step (SURVEY a18 / BASELINE config 5): generator loss with
the adaptive discriminator weight, hinge discriminator loss, DiffAugment, as a pure function of explicit state
dicts and the torch RNG.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  The CUDA path for this step is NOT built yet (DESIGN §5); this
file and tests/golden/vqgan_train.npz pin what it will have to reproduce.

Restates /root/reference/models/vqgan_model.py VQImageSegmTextureModel.training_step (:438-488, same body as
VQModel.training_step :289-327) with forward_step (:532-551), /root/reference/models/losses/vqgan_loss.py
(calculate_adaptive_weight :5-12, adopt_weight :15-18, hinge_d_loss :21-26, DiffAugment 'color,translation'
:29-80), Discriminator (models/archs/vqgan_arch.py:1155-1203, BatchNorm in training mode) and the straight-through
/ legacy-beta codebook loss of VectorQuantizerTexture.forward (:270-281).

Third-party: `lpips.LPIPS(net="vgg")` (lpips==0.1.4, downloads VGG weights: unavailable offline).  It enters as
``perceptual(x, xrec) -> [B,1,1,1]``; the fixture uses the zero function (perceptual_weight therefore has no effect),
as BASELINE config 5 states ("LPIPS stubbed").
"""
import torch
import torch.nn.functional as F

from . import vqgan_ref as V


def quantize_texture_train(codebooks, z, segm_map, beta=0.25, idx=None, info=None):
    """VectorQuantizerTexture.forward with its autograd semantics: nearest codes per texture, legacy loss
    mean((zq.detach()-z)^2) + beta*mean((zq-z.detach())^2), straight-through z + (zq - z).detach().
    codebooks: list/tensor of 18 [n_e, D] (requires_grad for the codebook gradient).
    ``idx``: per-row code indices (NHWC row order, any shape with B*H*W elements) used instead of the argmin, so that
    an implementation's own picks can be imposed.  ``info`` (dict): receives ``dist`` [rows, n_e], each row's
    distances to the codes of its texture's codebook in z's dtype (inf for rows of no texture), and ``argmin``
    [rows] (-1 for rows of no texture), ``rows`` [rows, D], z's rows themselves, and ``seg`` [rows], each row's
    texture id."""
    b, c, hh, ww = z.shape
    seg = F.interpolate(segm_map, size=(hh, ww), mode="nearest").reshape(-1)
    zp = z.permute(0, 2, 3, 1).contiguous()
    rows = zp.view(-1, c)
    # fp32 codes with autocast's fp16 latent: the quantized rows stay in the wider type
    zq = torch.zeros(rows.shape, dtype=torch.promote_types(rows.dtype, codebooks[0].dtype), device=rows.device)
    if info is not None:
        info["dist"] = torch.full((rows.shape[0], codebooks[0].shape[0]), float("inf"), dtype=rows.dtype,
                                  device=rows.device)
        info["argmin"] = torch.full((rows.shape[0],), -1, dtype=torch.long, device=rows.device)
        info["rows"] = rows.detach()
        info["seg"] = seg
    for k in range(len(codebooks)):
        sel = seg == k
        if sel.any():
            e = codebooks[k]
            d = torch.sum(rows[sel] ** 2, dim=1, keepdim=True) + torch.sum(e ** 2, dim=1) - 2 * (rows[sel] @ e.t())
            pick = torch.argmin(d, dim=1)
            if info is not None:
                info["dist"][sel] = d.detach().to(rows.dtype)
                info["argmin"][sel] = pick
            if idx is not None:
                pick = idx.reshape(-1).to(rows.device)[sel].long()
            zq = zq.index_put((sel.nonzero(as_tuple=True)[0],), e[pick])
    zq = zq.view(zp.shape)
    loss = torch.mean((zq.detach() - zp) ** 2) + beta * torch.mean((zq - zp.detach()) ** 2)
    zq = zp + (zq - zp).detach()
    return zq.permute(0, 3, 1, 2).contiguous(), loss


def _lrelu(h, masks, trace):
    if trace is not None:
        trace.append(h.detach())
    if masks is None:
        return F.leaky_relu(h, 0.2)
    return torch.where(next(masks), h, 0.2 * h)


def discriminator(sd, x, prefix="main.", n_layers=3, train=True, bn_state=None, masks=None, trace=None):
    """Discriminator.forward (:1200-1203): conv4x4 s2 + LeakyReLU, (n_layers-1) x [conv4x4 s2, BN, LeakyReLU],
    [conv4x4 s1, BN, LeakyReLU], conv4x4 s1 -> 1 channel.  BatchNorm uses batch statistics when ``train``;
    running-statistic updates are returned in ``bn_state`` (dict) if given, starting from the statistics already
    there (so consecutive passes chain), else from ``sd``'s.  ``masks``: one bool tensor per LeakyReLU (shaped like
    its input) imposing which elements take slope 1, so that an implementation's own kink decisions can be imposed;
    ``trace`` (list): receives every LeakyReLU's input."""
    masks = iter(masks) if masks is not None else None
    i = 0
    h = _lrelu(F.conv2d(x, sd[f"{prefix}{i}.weight"], sd[f"{prefix}{i}.bias"], stride=2, padding=1), masks, trace)
    i = 2
    for n in range(1, n_layers + 1):
        stride = 2 if n < n_layers else 1
        h = F.conv2d(h, sd[f"{prefix}{i}.weight"], None, stride=stride, padding=1)
        bn = f"{prefix}{i + 1}."
        src = bn_state if bn_state is not None and bn + "running_mean" in bn_state else sd
        rm, rv = src[bn + "running_mean"].clone(), src[bn + "running_var"].clone()
        h = F.batch_norm(h, rm, rv, sd[bn + "weight"], sd[bn + "bias"], train, 0.1, 1e-5)
        if bn_state is not None:
            bn_state[bn + "running_mean"], bn_state[bn + "running_var"] = rm, rv
        h = _lrelu(h, masks, trace)
        i += 3
    return F.conv2d(h, sd[f"{prefix}{i}.weight"], sd[f"{prefix}{i}.bias"], stride=1, padding=1)


def rng_draws(b, h, w, dtype, device):
    """DiffAugment's random draws from the global RNG in the reference's call order: three torch.rand(B,1,1,1)
    (brightness, saturation, contrast) then two torch.randint translations -> (r [B,3], t [B,2] int64), the layout
    of ``VQGANTrainer._aug_draws``"""
    r = [torch.rand(b, 1, 1, 1, dtype=dtype, device=device).view(b, 1) for _ in range(3)]
    sx, sy = int(h * 0.125 + 0.5), int(w * 0.125 + 0.5)
    tx = torch.randint(-sx, sx + 1, size=[b, 1, 1], device=device).view(b, 1)
    ty = torch.randint(-sy, sy + 1, size=[b, 1, 1], device=device).view(b, 1)
    return torch.cat(r, 1), torch.cat([tx, ty], 1)


def diff_augment(x, draws=None):
    """DiffAugment(x, 'color,translation'); ``draws``: (r [B,3], t [B,2] int) as ``rng_draws`` returns them, else
    drawn from the global RNG"""
    b = x.size(0)
    r, t = draws if draws is not None else rng_draws(b, x.size(2), x.size(3), x.dtype, x.device)
    r, t = r.to(x.device, x.dtype), t.to(x.device).long()
    x = x + (r[:, 0].view(b, 1, 1, 1) - 0.5)
    m = x.mean(dim=1, keepdim=True)
    x = (x - m) * (r[:, 1].view(b, 1, 1, 1) * 2) + m
    m = x.mean(dim=[1, 2, 3], keepdim=True)
    x = (x - m) * (r[:, 2].view(b, 1, 1, 1) + 0.5) + m
    tx, ty = t[:, 0].view(b, 1, 1), t[:, 1].view(b, 1, 1)
    gb, gx, gy = torch.meshgrid(torch.arange(b, device=x.device), torch.arange(x.size(2), device=x.device),
                                torch.arange(x.size(3), device=x.device), indexing="ij")
    gx = torch.clamp(gx + tx + 1, 0, x.size(2) + 1)
    gy = torch.clamp(gy + ty + 1, 0, x.size(3) + 1)
    xp = F.pad(x, [1, 1, 1, 1, 0, 0, 0, 0])
    return xp.permute(0, 2, 3, 1).contiguous()[gb, gx, gy].permute(0, 3, 1, 2).contiguous()


def training_step(sd, codebooks, sd_disc, x, mask, step, *, perceptual=None, perceptual_weight=1.0,
                  disc_start_step=0, disc_weight_max=1.0, diff_aug=True, disc_layers=3, draws=None, idx=None,
                  bn_state=None, loss_scale=1.0, d_weight=None, disc_masks=None, disc_trace=None):
    """-> dict(loss, d_loss or None, nll_loss, g_loss, d_weight, codebook_loss, xrec, l1, perceptual, ratio, vq).
    ``sd`` / ``codebooks`` / ``sd_disc`` tensors that require grad receive gradients from loss.backward() /
    d_loss.backward() exactly as the reference's two optimisers see them (the discriminator's parameters also collect
    the generator loss's gradient in the reference, until disc_optimizer.zero_grad() clears it: not restated).

    ``draws``: (fake pass's, real pass's) DiffAugment draws, each (r [B,3], t [B,2]) as ``rng_draws`` returns them,
    instead of the global RNG.  ``idx``: code indices imposed on the quantizer (``quantize_texture_train``); ``vq``
    holds its distances and argmin.  ``bn_state`` (dict): the discriminator's BatchNorm running statistics are carried
    through its passes in the reference's order (fake image for g_loss, real image, detached fake image) and left
    there with ``num_batches_tracked``; ``bn_passes`` counts the passes.  ``loss_scale``: the adaptive weight's two
    gradients are taken of the losses times this static scale and unscaled before their norms (for fp16 autocast;
    ``ratio`` is the adaptive weight before its clamp).  ``d_weight``: a value imposed on the adaptive weight (after
    its clamp and start-step factor), so that an implementation's own weight can be imposed like its codebook picks.
    ``disc_masks``: per discriminator pass (in the order above) the LeakyReLU masks ``discriminator`` imposes;
    ``disc_trace`` (list): receives per pass the list of its LeakyReLU inputs.
    """
    draws = draws or (None, None)
    n_pass = 0

    def disc(inp):
        nonlocal n_pass
        masks = disc_masks[n_pass] if disc_masks is not None else None
        trace = None
        if disc_trace is not None:
            trace = []
            disc_trace.append(trace)
        n_pass += 1
        return discriminator(sd_disc, inp, n_layers=disc_layers, bn_state=bn_state, masks=masks, trace=trace)

    h = V.conv(sd, "quant_conv", V.encoder(sd, x, "encoder."), padding=0)
    vq = {}
    quant, codebook_loss = quantize_texture_train(codebooks, h, mask, idx=idx, info=vq)
    xrec = V.decoder(sd, V.conv(sd, "post_quant_conv", quant, padding=0), "decoder.")
    recon = torch.abs(x - xrec)
    p_loss = perceptual(x, xrec) if perceptual is not None else torch.zeros(x.size(0), 1, 1, 1, dtype=recon.dtype,
                                                                              device=x.device)
    nll_loss = torch.mean(recon + perceptual_weight * p_loss)
    xr = diff_augment(xrec, draws[0]) if diff_aug else xrec
    g_loss = -torch.mean(disc(xr))
    last = sd["decoder.conv_out.weight"]
    if loss_scale != 1.0:
        rg = torch.autograd.grad(nll_loss * loss_scale, last, retain_graph=True)[0] / loss_scale
        gg = torch.autograd.grad(g_loss * loss_scale, last, retain_graph=True)[0] / loss_scale
    else:
        rg = torch.autograd.grad(nll_loss, last, retain_graph=True)[0]
        gg = torch.autograd.grad(g_loss, last, retain_graph=True)[0]
    ratio = (torch.norm(rg) / (torch.norm(gg) + 1e-4)).detach()
    if d_weight is None:
        d_weight = torch.clamp(ratio, 0.0, disc_weight_max)
        d_weight = d_weight * (1 if step >= disc_start_step else 0.0)
    else:
        d_weight = torch.as_tensor(d_weight, dtype=ratio.dtype, device=ratio.device)
    loss = nll_loss + d_weight * g_loss + codebook_loss
    d_loss = None
    if step > disc_start_step:
        real_in = diff_augment(x.detach(), draws[1]) if diff_aug else x.detach()
        lr_ = disc(real_in)
        lf_ = disc(xr.detach())
        d_loss = 0.5 * (torch.mean(F.relu(1.0 - lr_)) + torch.mean(F.relu(1.0 + lf_)))
    if bn_state is not None:
        for k in [k for k in bn_state if k.endswith("running_mean")]:
            nbt = k[:-len("running_mean")] + "num_batches_tracked"
            bn_state[nbt] = sd_disc[nbt] + n_pass
    return dict(loss=loss, d_loss=d_loss, nll_loss=nll_loss, g_loss=g_loss, d_weight=d_weight,
                codebook_loss=codebook_loss, xrec=xrec, l1=torch.mean(recon), perceptual=torch.mean(p_loss),
                ratio=ratio, vq=vq, bn_state=bn_state, bn_passes=n_pass)
