"""Generate tests/golden/parsing_gen.npz by running the REAL reference ShapeAttrEmbedding, ShapeUNet and FCNHead
(/root/reference/models/archs/shape_attr_embedding_arch.py, unet_arch.py, fcn_arch.py) on the deterministic
recipes of tests/parsing_gen_recipes.py.

unet_arch.py / fcn_arch.py import mmcv / mmseg (absent here); the stand-ins of oracle/make_golden_indexpred.py are
registered before the files are loaded by path.  Everything structural (attribute embedding, broadcast concatenation,
pooling, upsampling, skips, head) is the reference's code.

Run in the build container only:  python oracle/make_golden_parsing_gen.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parsing_gen_recipes as P  # noqa: E402
from oracle.make_golden_indexpred import OUT, _load, _stub_modules  # noqa: E402


def build(emb_cfg, unet_cfg, head_cfg, load=True):
    _stub_modules()
    sa, un, fc = _load("shape_attr_embedding_arch"), _load("unet_arch"), _load("fcn_arch")
    emb, unet, head = sa.ShapeAttrEmbedding(**emb_cfg), un.ShapeUNet(**unet_cfg), fc.FCNHead(**head_cfg)
    if load:
        for m, sd in zip((emb, unet, head), P.state_dicts(emb, unet, head)):
            m.load_state_dict(sd, strict=True)
    return emb.eval(), unet.eval(), head.eval()


def _listing(m):
    return np.array([f"{k}:{tuple(v.shape)}" for k, v in m.state_dict().items()])


def main():
    torch.set_num_threads(8)
    emb, unet, head = build(P.TINY_EMBEDDER, P.TINY_SHAPE_UNET, P.TINY_FCN_HEAD)
    B = P.TINY_POSE[0]
    pose = P.pose(P.SEEDS["pose"], *P.TINY_POSE)
    attr = P.shape_attrs(P.SEEDS["attr"], B)
    with torch.no_grad():
        e = emb(attr)
        dec = unet(pose, e)
        logits = head(dec)
    out = {"attr": attr.numpy(), "pose": pose.numpy(), "embedding": e.numpy(), "logits": logits.numpy(),
           "argmax": logits.argmax(dim=1).unsqueeze(1).numpy()}
    for i, d in enumerate(dec):
        out[f"dec{i}"] = d.numpy()
    # key/shape listings of the real-size nets (the parsing_gen.pth layout the mirrors must keep)
    emb_r, unet_r, head_r = build(P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD, load=False)
    out["embedder_keys"], out["encoder_keys"], out["decoder_keys"] = map(_listing, (emb_r, unet_r, head_r))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "parsing_gen.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), [tuple(d.shape) for d in dec], tuple(logits.shape),
          [len(out[k]) for k in ("embedder_keys", "encoder_keys", "decoder_keys")])


if __name__ == "__main__":
    main()
