"""Training step of the hierarchical VQGAN's bottom level on the H100 kernels.

Mirrors ``HierarchyVQSpatialTextureAwareModel.optimize_parameters`` / ``training_step`` (models/
hierarchy_vqgan_model.py:196-291) with the optimiser membership of ``configure_optimizers`` (:127-159).  The GAN
micro-step (L1, DiffAugment, discriminator backward into the image, adaptive weight, hinge discriminator update), the
loss scales, ``losses()``, Adam and checkpointing are ``VQGANTrainer``'s; this class replaces the generator:

  frozen top path   top_encoder -> top_quant_conv -> VectorQuantizerTexture -> top_post_quant_conv -> decoder
                    conv_in, mid and level 4 up to its upsample: forward only on the inference path, no saved
                    activations (the reference computes gradients there and never steps them)
  bottom path       bot_encoder -> bot_quant_conv -> VectorQuantizerSpatialTextureAware (2x2 patches) ->
                    bot_post_quant_conv -> DecoderRes = bot_h
  decoder           (top features + bot_h) -> levels 3..0 -> norm_out -> conv_out

Adam steps the bottom nets, the 18 codebooks and the decoder's levels 0..3 (``up.0`` .. ``up.3``, unless
``fix_decoder``).  ``norm_out`` / ``conv_out`` (and with ``fix_decoder`` levels 0..3) live in a second ParamSpace,
``fixed``: their gradients are computed (conv_out's feeds the adaptive weight) but never stepped, all-reduced,
broadcast or saved as optimiser state.  The discriminator is loaded from the top checkpoint and trained as in the
top step.
"""
import torch

from . import ops
from .flat_params import ParamSpace
from .train_layers import Grad
from .vqgan_arch import _conv_in_nhwc
from .vqgan_train import (Act, ConvL, Lin1x1L, NormConvOutL, Seq, VQGANTrainer, decoder_up_layers, decoder_up_order,
                          encoder_layers, encoder_order, mid_layers, mid_order)

NETS = ("bot_encoder", "bot_decoder_res", "decoder", "bot_quantize", "bot_quant_conv", "bot_post_quant_conv")
RES_LEVEL = 4       # the decoder adds bot_h after this level's upsample (vqgan_arch.py:1023)


class HierarchyVQGANTrainer(VQGANTrainer):
    """Owns a ``pipeline.HierarchyVQSpatialTextureAwareModel`` whose top nets are already loaded and a
    ``Discriminator``; ``optimize_parameters(data, step)`` is one reference training step.  Keyword arguments are
    ``VQGANTrainer``'s plus ``fix_decoder`` (configs/vqvae_bottom.yml)."""

    def __init__(self, model, disc, fix_decoder=False, **kw):
        self.fix_decoder = bool(fix_decoder)
        super().__init__(model, disc, **kw)

    def _build(self, model, bucket_bytes):
        dec = model.decoder
        assert dec.num_resolutions == RES_LEVEL + 1, "the bot_h residual needs a decoder of 5 levels"
        top = RES_LEVEL - 1
        self.enc_in, self.enc_body, self.enc_out = encoder_layers(self, model.bot_encoder)
        self.qconv, self.pqconv = Lin1x1L(self, model.bot_quant_conv), Lin1x1L(self, model.bot_post_quant_conv)
        dres = model.bot_decoder_res
        self.dres_in, self.dres_body = ConvL(self, dres.conv_in, "k3"), Seq(mid_layers(self, dres.mid))
        self.dec_body = Seq(decoder_up_layers(self, dec, top))
        self.dec_out = NormConvOutL(self, dec.norm_out, dec.conv_out, nchw=True)
        up = decoder_up_order(dec, top)
        fixed = [dec.conv_out, dec.norm_out] + (up if self.fix_decoder else [])
        self.fixed = ParamSpace(fixed, self.device, bucket_bytes)
        q = model.bot_quantize
        order = ([] if self.fix_decoder else up) + mid_order(dres.mid) + [dres.conv_in]
        order += [model.bot_post_quant_conv] + list(q.embedding_list) + [model.bot_quant_conv]
        return order + encoder_order(model.bot_encoder), q

    def training_step(self, data, step, generator=None):
        x, mask = data['image'], data['texture_mask']
        if x.dim() != 4 or x.shape[2] % 16 or x.shape[3] % 16:
            raise ValueError(f"image {tuple(x.shape)}: H and W must be multiples of 16 (four downsamplings in the top "
                             "encoder, three and a 2x2 patch in the bottom one)")
        if mask.dim() != 4 or mask.shape[0] != x.shape[0] or mask.shape[1] != 1 or mask.shape[2:] != x.shape[2:]:
            raise ValueError(f"texture_mask {tuple(mask.shape)} does not match image {tuple(x.shape)}: "
                             "expected [B,1,H,W]")
        return super().training_step(data, step, generator)

    def gen_forward(self, x, mask):
        m = self.model
        with torch.no_grad():
            quant_top, _ = m.top_encode_nhwc(x, mask)
            h_top = m.decoder._trunk(_conv_in_nhwc(m.decoder.conv_in, quant_top), stop_after_level=RES_LEVEL).x
        h = self.enc_out.fwd(self.enc_body.fwd(self.enc_in.fwd(x)))          # fp32 NHWC latent
        z = self.qconv.fwd(h)
        B, Hz, Wz, D = z.shape
        q = self.quantizer
        ps = q.spatial_size
        ids = ops.mask_to_ids(mask, Hz // ps, Wz // ps)
        r = ops.vq_search(z, self.codebook, ids, ps=ps, cont_stride=q.n_e, want_list=False, want_nchw=False)
        self._vq = (z, r["idx"], ids)
        self.bot_idx = r["idx_cont"]
        bot_h = self.dres_body.fwd(self.dres_in.fwd(Act(self.pqconv.fwd(r["zq_nhwc"])))).x
        xrec = self.dec_out.fwd(self.dec_body.fwd(Act(ops.add_inplace(h_top, bot_h))))
        return xrec, r["sqerr"], z.numel()

    def gen_backward(self, dxrec, cb_scale, conv_out_gw=None):
        # the gradient leaving the decoder's first level-3 block is d bot_h (the top features are constant)
        g = self.dec_body.bwd(self.dec_out.bwd(dxrec, gw_known=conv_out_gw))
        g = self.pqconv.bwd(self.dres_in.bwd(self.dres_body.bwd(g)))
        z, idx, ids = self._vq
        nel = z.numel()
        dz = ops.vq_bwd_patch(z, self.codebook, idx, ids, g.g, self.g_codebook, 2.0 * cb_scale / nel,
                              2.0 * self.beta * cb_scale / nel, ps=self.quantizer.spatial_size)
        for e in self.quantizer.embedding_list:
            self.gen.done(e)
        g = self.qconv.bwd(Grad(dz))
        self.enc_in.bwd(self.enc_body.bwd(self.enc_out.bwd(g.g)))
        self._vq = None

    def _nets(self):
        return dict({k: getattr(self.model, k) for k in NETS}, discriminator=self.disc)
