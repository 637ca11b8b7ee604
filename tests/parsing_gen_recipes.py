"""Deterministic recipes for the parsing-generator fixture (pose + shape attributes -> parsing map), shared by
oracle/make_golden_parsing_gen.py (which runs the real reference classes on them) and the tests (which re-create
the same tensors without the reference).  Built on golden_recipes' seeded generators."""
import torch

import golden_recipes as R

# configs/sample_from_pose.yml:112-126
CLS_NUM = [2, 4, 6, 5, 4, 3, 5, 5, 3, 2, 2, 2, 2, 2, 2]
REAL_EMBEDDER = dict(dim=8, out_dim=128, cls_num_list=CLS_NUM)
REAL_SHAPE_UNET = dict(in_channels=1)                     # base 64, 5 stages, attr_embedding 128
REAL_FCN_HEAD = dict(in_channels=64, in_index=4, channels=64, num_convs=1, concat_input=False, dropout_ratio=0.1,
                     num_classes=24, align_corners=False)
# reduced nets for the fixture: the real attribute lists, widths cut by 8
TINY_EMBEDDER = dict(dim=4, out_dim=16, cls_num_list=CLS_NUM)
TINY_SHAPE_UNET = dict(in_channels=1, base_channels=8, attr_embedding=16)
TINY_FCN_HEAD = dict(REAL_FCN_HEAD, in_channels=8, channels=8)
TINY_POSE = (2, 64, 32)          # B, H, W of the 1-channel pose
SEEDS = dict(embedder=301, encoder=302, decoder=303, pose=304, attr=305)


def pose(seed, b, h, w, tile=8):
    """densepose input as DeepFashionAttrPoseDataset yields it: part index 0..24 (constant on tile x tile blocks)
    / 12 - 1, [b,1,h,w] fp32"""
    return R.blocky_mask(seed, b, h, w, tile, n_ids=25) / 12.0 - 1.0


def shape_attrs(seed, b, cls_num=CLS_NUM):
    """int64 [b, 15], attribute i uniform in 0..cls_num[i]-1"""
    g = R._gen(seed, "shape_attr")
    return torch.stack([torch.randint(0, n, (b,), generator=g) for n in cls_num], 1)


def every_class_attrs(cls_num=CLS_NUM):
    """int64 [max(cls_num), 15]: row r sets attribute i to r mod cls_num[i], so every class of every attribute
    appears"""
    rows = max(cls_num)
    return torch.tensor([[r % n for n in cls_num] for r in range(rows)], dtype=torch.int64)


def state_dicts(emb, unet, head, seeds=SEEDS):
    return (R.fill_state_dict(R.spec_of(emb), seeds["embedder"]), R.fill_state_dict(R.spec_of(unet), seeds["encoder"]),
            R.fill_state_dict(R.spec_of(head), seeds["decoder"]))
