"""Reduced hierarchical VQGAN + discriminator for the bottom-level training-step fixture
(oracle/make_golden_vqgan_bottom_train.py), and the seeded weights / batch shared by the generating script and the
tests.  Real: configs/vqvae_bottom.yml (top ch 128 x [1,1,2,2,4], bottom ch 128 x [1,1,2,4], embed_dim 256,
bot_n_embed 512, ndf 64).  The decoder keeps its 5 levels because the bot_h residual is added after level 4, and the
widths meet there: top ch 32 x 4 = bottom DecoderRes ch 32 x 4 = 128 channels at 8 x 4.
"""
import contextlib
import io

import torch

import golden_recipes as R

OPT = dict(embed_dim=32, n_embed=1024, codebook_spatial_size=2,
           bot_n_embed=64, bot_double_z=False, bot_z_channels=32, bot_resolution=64, bot_in_channels=3,
           bot_out_ch=3, bot_ch=32, bot_ch_mult=[1, 1, 2, 4], bot_num_res_blocks=1, bot_attn_resolutions=[8],
           bot_dropout=0.0,
           top_double_z=False, top_z_channels=32, top_resolution=64, top_in_channels=3, top_out_ch=3, top_ch=32,
           top_ch_mult=[1, 1, 2, 2, 4], top_num_res_blocks=1, top_attn_resolutions=[4], top_dropout=0.0)
NDF, DISC_LAYERS, DISC_START_STEP, STEP, BATCH, H, W = 16, 3, 1, 5, 2, 64, 32

# Module seeds of the weights (golden_recipes.fill_state_dict) and of the two codebook sets.
SEEDS = dict(top_encoder=201, decoder=202, top_quant_conv=203, top_post_quant_conv=204, bot_encoder=205,
             bot_decoder_res=206, bot_quant_conv=207, bot_post_quant_conv=208, disc=209, top_books=210, bot_books=211)
# Data and DiffAugment seeds, chosen by a scan (data seeds 301..320, then DiffAugment seeds 400..499) with the fp64
# restatement (make_golden_vqgan_bottom_train.py --scan): the step's gradient is discontinuous where a quantizer's
# argmin changes and at the discriminator's LeakyReLU / hinge kinks.  With these seeds every argmin (both quantizers) has its second-best distance at least ARGMIN_MARGIN
# (relative) above the best, and every discriminator pre-activation is at least KINK_MARGIN away from its kink, so an
# fp32-equivalent implementation cannot land on the other side of either.
DATA_SEED = 301
AUG_SEED = 406
ARGMIN_MARGIN = 4e-3
KINK_MARGIN = 7e-5


def batch():
    return dict(image=R.image(DATA_SEED, BATCH, 3, H, W), texture_mask=R.blocky_mask(DATA_SEED + 1, BATCH, H, W, 8))


def modules():
    """the seeded nets of pipeline.HierarchyVQSpatialTextureAwareModel and the Discriminator (CPU, fp32)"""
    from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
    from text2human_b200.vqgan_arch import Discriminator
    with contextlib.redirect_stdout(io.StringIO()):
        m = HierarchyVQSpatialTextureAwareModel(OPT)
    for name in ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv", "bot_encoder", "bot_decoder_res",
                 "bot_quant_conv", "bot_post_quant_conv"):
        mod = getattr(m, name)
        mod.load_state_dict(R.fill_state_dict(R.spec_of(mod), SEEDS[name]), strict=True)
    for q, key, n_e, d in ((m.top_quantize, "top_books", 1024, OPT["embed_dim"]),
                           (m.bot_quantize, "bot_books", OPT["bot_n_embed"], 4 * OPT["embed_dim"])):
        cb = R.codebooks(SEEDS[key], 18, n_e, d, "trained")
        for k, e in enumerate(q.embedding_list):
            e.weight.data.copy_(cb[k])
    disc = Discriminator(3, NDF, n_layers=DISC_LAYERS)
    disc.load_state_dict(R.fill_state_dict(R.spec_of(disc), SEEDS["disc"]), strict=True)
    return m, disc


def stepped(name):
    """is generator tensor ``name`` (``<net>.<key>``) in the reference's Adam (configure_optimizers, :127-159)?"""
    if name.startswith("bot_"):
        return True
    return name.startswith("decoder.") and any(f"up.{i}" in name for i in range(4))


def restatement_state(dtype=torch.float32):
    """-> (sd, top_books, bot_books list, sd_disc) for oracle.vqgan_bottom_train_ref.training_step; tensors of stepped
    generator tensors, the bottom codebooks and the disc's parameters require grad"""
    m, disc = modules()
    sd = {}
    for net in ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv", "bot_encoder", "bot_decoder_res",
                "bot_quant_conv", "bot_post_quant_conv"):
        for k, v in getattr(m, net).state_dict().items():
            sd[f"{net}.{k}"] = v.detach().to(dtype).clone()
    for k in sd:
        if stepped(k) or k == "decoder.conv_out.weight":
            sd[k].requires_grad_(True)
    top = torch.stack([e.weight.detach() for e in m.top_quantize.embedding_list]).to(dtype)
    bot = [e.weight.detach().to(dtype).clone().requires_grad_(True) for e in m.bot_quantize.embedding_list]
    sdd = {}
    for k, v in disc.state_dict().items():
        v = v.detach().clone()
        if v.is_floating_point():
            v = v.to(dtype)
            if "running" not in k:
                v.requires_grad_(True)
        sdd[k] = v
    return sd, top, bot, sdd


def gen_grads(sd, bot):
    """{fixture name: gradient} of every stepped generator tensor after loss.backward() (zeros for a codebook no
    position selects)"""
    out = {k: sd[k].grad for k in sd if stepped(k)}
    for k, e in enumerate(bot):
        out[f"bot_quantize.embedding_list.{k}.weight"] = e.grad if e.grad is not None else torch.zeros_like(e)
    return out
