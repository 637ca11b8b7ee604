"""Deterministic recipes for the parsing-tokenizer training-step fixture, shared by
oracle/make_golden_segm_train.py (which runs the real reference on them) and the tests (which re-create the same
tensors without the reference).  Built on golden_recipes' seeded generators."""
import golden_recipes as R

# reduced parsing tokenizer (real: configs/parsing_token.yml, 512 x 256).  ch 64 keeps two channels per GroupNorm
# group and the real level widths; 24 one-hot input / logit channels; the real 1024 x 32 codebook (rows ~ N(0,1), so
# that no code distances are near ties)
TINY_SEGM_TRAIN = dict(ch=64, num_res_blocks=1, attn_resolutions=[16], ch_mult=[1, 1, 2, 2, 4], in_channels=24,
                       out_ch=24, resolution=64, z_channels=32, double_z=False, dropout=0.0, n_embed=1024,
                       embed_dim=32, num_segm_classes=24, lr=4.5e-05, batch=2)
SEGM_TRAIN_SEEDS = dict(encoder=201, decoder=202, quant_conv=203, post_quant_conv=204, codebook=205, labels=206)


def segm_labels(seed, b, h, w, tile=4, n_ids=24):
    """integer parsing map [b,h,w] (MaskDataset's 'segm'), constant on tile x tile blocks"""
    return R.blocky_mask(seed, b, h, w, tile, n_ids=n_ids).squeeze(1).long()
