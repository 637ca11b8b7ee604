"""Generate tests/golden/index_pred_train.npz by running the REAL reference index-prediction training step
(/root/reference/models/hierarchy_inference_model.py VQGANTextureAwareSpatialHierarchyInferenceModel.
init_training_settings / optimize_parameters, unbound, on a stand-in ``self`` carrying the attributes they read,
device CPU) around the REAL UNet / MultiHeadFCNHead (loaded by path with the mmcv stand-ins of
oracle/make_golden_indexpred.py) and the REAL CrossEntropyLoss, on the reduced nets and the ground truth of
tests/index_pred_train_recipes.py (feature_t, and gt_indices_list built from own indices and texture ids as the
bottom quantizer returns them: the own index where the texture is k, -1 elsewhere).

The fixture stores the loss, the 18 Dropout2d masks the reference drew (a forward hook fires once per head), per
parameter tensor the gradient's norm, its first 8 entries and its first 8 entries after the Adam step, and every
BatchNorm's running statistics after the step.
Run in the build container only:  python oracle/make_golden_index_pred_train.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import index_pred_train_recipes as IT  # noqa: E402
from oracle.index_pred_train_ref import gt_indices_list  # noqa: E402
from oracle.make_golden_indexpred import OUT, _stub_modules  # noqa: E402
from oracle.make_golden_vqgan_train import REF, _load  # noqa: E402

NETS = dict(guidance_encoder="guidance_encoder", index_decoder="index_decoder")


def load_reference():
    _stub_modules()
    for name in ("models", "models.archs", "models.losses"):
        sys.modules.setdefault(name, types.ModuleType(name))
    # the model file imports the VQGAN classes and torchvision's save_image for paths this step never runs
    vq = types.ModuleType("models.archs.vqgan_arch")
    vq.Decoder = vq.DecoderRes = vq.Encoder = None
    vq.VectorQuantizerSpatialTextureAware = vq.VectorQuantizerTexture = None
    sys.modules["models.archs.vqgan_arch"] = vq
    if "torchvision" not in sys.modules:
        tv, tvu = types.ModuleType("torchvision"), types.ModuleType("torchvision.utils")
        tvu.save_image = lambda *a, **k: None
        tv.utils = tvu
        sys.modules.setdefault("torchvision", tv)
        sys.modules.setdefault("torchvision.utils", tvu)
    mods = {}
    for sub in ("archs.unet_arch", "archs.fcn_arch", "losses.accuracy", "losses.cross_entropy_loss"):
        mods[sub] = _load("models." + sub, os.path.join(REF, *sub.split(".")) + ".py")
    mods["model"] = _load("models.hierarchy_inference_model", os.path.join(REF, "hierarchy_inference_model.py"))
    return mods


def make_fake(mods, seeds=IT.SEEDS):
    unet = mods["archs.unet_arch"].UNet(**R.TINY_UNET)
    fcn = mods["archs.fcn_arch"].MultiHeadFCNHead(**R.TINY_FCN)
    for m, sd in zip((unet, fcn), IT.state_dicts(unet, fcn, seeds)):
        m.load_state_dict(sd, strict=True)
    fake = types.SimpleNamespace(opt=dict(optimizer="Adam", lr=IT.LR, weight_decay=0, loss_function="cross_entropy"),
                                 device=torch.device("cpu"), guidance_encoder=unet, index_decoder=fcn)
    Model = mods["model"].VQGANTextureAwareSpatialHierarchyInferenceModel
    for name in ("init_training_settings", "optimize_parameters"):
        setattr(fake, name, types.MethodType(getattr(Model, name), fake))
    return fake


def main():
    torch.set_num_threads(8)
    mods = load_reference()
    fake = make_fake(mods)
    feature, own, tex = IT.batch()
    masks = []

    def hook(mod, inp, out):
        x, y = inp[0].detach(), out.detach()
        kept = (y != 0).flatten(2).any(2)
        # a channel whose input is all zero keeps no trace of its draw; it has no effect either way: call it kept
        masks.append((kept | ~(x != 0).flatten(2).any(2)).float())
    fake.index_decoder.dropout.register_forward_hook(hook)
    torch.manual_seed(2021)                     # configs/index_pred_net.yml manual_seed
    fake.init_training_settings()
    fake.feature_t = feature                    # feed_data's outputs (:178-197)
    fake.gt_indices_list = gt_indices_list(own, tex, IT.N_HEAD)
    params = {f"{k}.{n}": p for k, attr in NETS.items() for n, p in getattr(fake, attr).named_parameters()}
    fake.optimize_parameters()
    assert len(masks) == IT.N_HEAD
    out = {"loss_total": np.float64(float(fake.log_dict["loss_total"].detach())),
           "dropout_mask": torch.stack(masks).numpy()}
    for k, p in params.items():
        out["gnorm/" + k] = p.grad.norm().numpy()
        out["ghead/" + k] = p.grad.reshape(-1)[:8].numpy().copy()
        out["phead/" + k] = p.detach().reshape(-1)[:8].numpy().copy()
    for k, attr in NETS.items():
        for n, b in getattr(fake, attr).named_buffers():
            if n.endswith(("running_mean", "running_var")):
                out[f"buf/{k}.{n}"] = b.numpy().copy()
    path = os.path.join(OUT, "index_pred_train.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), float(out["loss_total"]), len(params), "parameter tensors",
          int(out["dropout_mask"].sum()), "of", out["dropout_mask"].size, "channels kept")


if __name__ == "__main__":
    main()
