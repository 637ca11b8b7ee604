"""Seeded LPIPS weights shared by oracle/make_golden_lpips_train.py and the tests: VGG16 weights N(0, 1/fan_in) and
biases 0.1 N(0, 1) (``golden_recipes.fill_state_dict``), lin weights |N(0, 1)| / C (lpips' learned heads are
non-negative)."""
import torch

import golden_recipes as R

SEED = 401
CHNS = (64, 128, 256, 512, 512)
# (conv index in torchvision's vgg16 features, cin, cout), per slice
CONVS = (((0, 3, 64), (2, 64, 64)), ((5, 64, 128), (7, 128, 128)),
         ((10, 128, 256), (12, 256, 256), (14, 256, 256)), ((17, 256, 512), (19, 512, 512), (21, 512, 512)),
         ((24, 512, 512), (26, 512, 512), (28, 512, 512)))


def spec():
    """(key, shape) of every tensor of the lpips state dict, lin weights under their lin{k} names only"""
    out = [("scaling_layer.shift", (1, 3, 1, 1)), ("scaling_layer.scale", (1, 3, 1, 1))]
    for k, convs in enumerate(CONVS):
        for i, cin, cout in convs:
            out += [(f"net.slice{k + 1}.{i}.weight", (cout, cin, 3, 3)), (f"net.slice{k + 1}.{i}.bias", (cout,))]
    out += [(f"lin{k}.model.1.weight", (1, c, 1, 1)) for k, c in enumerate(CHNS)]
    return out


def state_dict(seed=SEED, dead_slice5=False):
    """the oracle's state dict (lin{k} keys); ``dead_slice5``: conv5_3's biases so negative that relu5_3 is zero at
    every pixel"""
    sd = R.fill_state_dict([s for s in spec() if not s[0].startswith("scaling_layer")], seed)
    sd["scaling_layer.shift"] = torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1)
    sd["scaling_layer.scale"] = torch.tensor([.458, .448, .450]).view(1, 3, 1, 1)
    for k, c in enumerate(CHNS):
        g = R._gen(seed, f"lin{k}")
        sd[f"lin{k}.model.1.weight"] = torch.randn((1, c, 1, 1), generator=g).abs() / c
    if dead_slice5:
        sd["net.slice5.28.bias"] = torch.full((512,), -1e4)
    return sd


def mirror_state_dict(sd):
    """the oracle's state dict plus the ``lins.{k}`` aliases lpips.LPIPS also registers"""
    out = dict(sd)
    for k in range(5):
        out[f"lins.{k}.model.1.weight"] = sd[f"lin{k}.model.1.weight"]
    return out


def mirror(device, seed=SEED, dead_slice5=False):
    from text2human_b200.lpips import LPIPS
    m = LPIPS(pretrained=False)
    m.load_state_dict(mirror_state_dict(state_dict(seed, dead_slice5)), strict=True)
    return m.to(device)
