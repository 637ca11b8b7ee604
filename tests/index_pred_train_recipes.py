"""Deterministic recipes for the index-prediction training fixture, shared by oracle/make_golden_index_pred_train.py
(which runs the real reference training step on them) and the tests (which re-create the same tensors without the
reference).  The nets are golden_recipes.TINY_UNET / TINY_FCN (base 8, 18 heads of 16 classes)."""
import torch

import golden_recipes as R

N_HEAD = R.TINY_FCN["num_head"]
N_CLASSES = R.TINY_FCN["num_classes"]
TRAIN_SHAPE = (2, 32, 16)          # B, h, w: the latent grid of a 512x256 image
# The feature seed is chosen so that the step's gradient is continuous at rounding level: fp64 gradients of weights
# perturbed by 3e-7 relative noise move by at most 4e-5 per tensor (tests/test_index_pred_train_oracle.py holds the
# fixture to 1e-4 there).  At B = 2 the UNet's bottleneck BatchNorms normalise 4 values per channel and each head's
# gradient lives on its own texture's ~50 positions, so a ReLU kink within amplified rounding would move a gradient by
# percents; at 1e-6 relative noise every seed tried (B = 2, 4 and 8) shows such a jump in some draw.
SEEDS = dict(unet=411, fcn=412, feature=627, tex=414, own=415)
ABSENT_HEAD = 7                    # no position of the fixture has this texture: its head gets zero gradient
OUT_OF_RANGE = (18, 21)            # texture ids that select no head (ignored in every head)
LR = 1e-4                          # configs/index_pred_net.yml


def state_dicts(unet, fcn, seeds=SEEDS):
    return R.fill_state_dict(R.spec_of(unet), seeds["unet"]), R.fill_state_dict(R.spec_of(fcn), seeds["fcn"])


def feature_t(seed=SEEDS["feature"], shape=TRAIN_SHAPE, channels=R.TINY_UNET["in_channels"]):
    b, h, w = shape
    return R.latent(seed, (b, channels, h, w), 1.0, "feature_t")


def texture_ids(seed=SEEDS["tex"], shape=TRAIN_SHAPE, absent=(ABSENT_HEAD,), extra=OUT_OF_RANGE, n_head=N_HEAD,
                tile=2):
    """int64 [B,h,w] texture ids constant on tile x tile blocks, uniform over the heads not in ``absent`` and the
    out-of-range ids ``extra``"""
    b, h, w = shape
    pool = [k for k in range(n_head) if k not in absent] + list(extra)
    pick = R.blocky_mask(seed, b, h, w, tile, n_ids=len(pool))[:, 0].long()
    return torch.tensor(pool, dtype=torch.int64)[pick]


def own_indices(seed=SEEDS["own"], shape=TRAIN_SHAPE, n_classes=N_CLASSES):
    """int64 [B,h,w] own-codebook indices, uniform"""
    return torch.randint(0, n_classes, shape, generator=R._gen(seed, "own"))


def batch(seeds=SEEDS, shape=TRAIN_SHAPE, absent=(ABSENT_HEAD,)):
    """(feature_t [B,C,h,w], own [B,h,w], tex [B,h,w])"""
    return feature_t(seeds["feature"], shape), own_indices(seeds["own"], shape), \
        texture_ids(seeds["tex"], shape, absent)
