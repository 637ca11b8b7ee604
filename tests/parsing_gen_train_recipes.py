"""Deterministic recipes for the parsing-generator training fixture, shared by
oracle/make_golden_parsing_gen_train.py (which runs the real reference training step on them) and the tests (which
re-create the same tensors without the reference).  The nets are the reduced ones of parsing_gen_recipes."""
import torch

import golden_recipes as R
import parsing_gen_recipes as P

N_CLASSES = P.TINY_FCN_HEAD["num_classes"]
# The fixture's shape and pose seed are chosen so that the reference's forward pass stays clear of every kink and
# tie (oracle/parsing_gen_train_ref.Margins: no BatchNorm output within 9e-5 of its ReLU's kink, no pooled window's
# two largest values within 1.6e-4 of each other), where two correct fp32 implementations could route a gradient
# differently; tests/test_parsing_gen_train_oracle.py holds the fixture to that.
TRAIN_SHAPE = (2, 32, 16)          # B, H, W
TRAIN_SEEDS = dict(P.SEEDS, pose=1350, attr=312, labels=313)
LR = 1e-4                          # configs/parsing_gen.yml


def segm_labels(seed, b, h, w, n_cls=N_CLASSES, tile=2, n_ignored=23, absent=()):
    """int64 parsing labels [b,h,w]: class ids constant on tile x tile blocks, uniform over the classes not in
    ``absent``, plus ``n_ignored`` pixels (per batch) set to ignore_index -100"""
    pool = [c for c in range(n_cls) if c not in absent]
    ids = R.blocky_mask(seed, b, h, w, tile, n_ids=len(pool))[:, 0].long()
    lab = torch.tensor(pool, dtype=torch.int64)[ids]
    g = R._gen(seed, "ignored")
    flat = lab.view(-1)
    flat[torch.randperm(flat.numel(), generator=g)[:n_ignored]] = -100
    return lab


def pose(seed, b, h, w):
    """the densepose input of parsing_gen_recipes plus N(0, 0.05^2) noise: a piecewise-constant pose makes whole
    regions of equal activations, whose max-pool windows are ties that the two implementations break on rounding
    noise (routing the gradient to different pixels); with the noise no window is tied"""
    return P.pose(seed, b, h, w) + 0.05 * torch.randn((b, 1, h, w), generator=R._gen(seed, "pose_noise"))


def batch(seeds=TRAIN_SEEDS, shape=TRAIN_SHAPE, absent=()):
    """the reference's batch dict (densepose [B,1,H,W], attr [B,15], segm [B,H,W])"""
    b, h, w = shape
    return dict(densepose=pose(seeds["pose"], b, h, w), attr=P.shape_attrs(seeds["attr"], b),
                segm=segm_labels(seeds["labels"], b, h, w, absent=absent))
