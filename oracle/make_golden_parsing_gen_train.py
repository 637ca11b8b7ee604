"""Generate tests/golden/parsing_gen_train.npz by running the REAL reference parsing-generator training step
(/root/reference/models/parsing_gen_model.py ParsingGenModel.init_training_settings / feed_data /
optimize_parameters, unbound, on a stand-in ``self`` carrying the attributes they read, device CPU) around the REAL
ShapeAttrEmbedding / ShapeUNet / FCNHead (loaded by path with the mmcv stand-ins of oracle/make_golden_indexpred.py)
and the REAL CrossEntropyLoss, on the reduced nets of tests/parsing_gen_recipes.py and the labels of
tests/parsing_gen_train_recipes.py.

The fixture stores the loss, the Dropout2d mask the reference drew (captured with a forward hook), per parameter
tensor the gradient's norm, its first 8 entries and its first 8 entries after the Adam step, and every BatchNorm's
running statistics after the step.
Run in the build container only:  python oracle/make_golden_parsing_gen_train.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parsing_gen_recipes as P  # noqa: E402
import parsing_gen_train_recipes as PT  # noqa: E402
from oracle.make_golden_indexpred import OUT, _stub_modules  # noqa: E402
from oracle.make_golden_vqgan_train import REF, _load  # noqa: E402

NETS = dict(embedder="attr_embedder", encoder="parsing_encoder", decoder="parsing_decoder")


def load_reference():
    _stub_modules()
    for name in ("models", "models.archs", "models.losses"):
        sys.modules.setdefault(name, types.ModuleType(name))
    mods = {}
    for sub in ("archs.shape_attr_embedding_arch", "archs.unet_arch", "archs.fcn_arch", "losses.accuracy",
                "losses.cross_entropy_loss"):
        mods[sub] = _load("models." + sub, os.path.join(REF, *sub.split(".")) + ".py")
    sys.modules["mmcv"].imwrite = lambda *a, **k: None
    mods["model"] = _load("models.parsing_gen_model", os.path.join(REF, "parsing_gen_model.py"))
    return mods


def make_fake(mods, seeds=PT.TRAIN_SEEDS):
    emb = mods["archs.shape_attr_embedding_arch"].ShapeAttrEmbedding(**P.TINY_EMBEDDER)
    unet = mods["archs.unet_arch"].ShapeUNet(**P.TINY_SHAPE_UNET)
    head = mods["archs.fcn_arch"].FCNHead(**P.TINY_FCN_HEAD)
    for m, sd in zip((emb, unet, head), P.state_dicts(emb, unet, head, seeds)):
        m.load_state_dict(sd, strict=True)
    fake = types.SimpleNamespace(opt=dict(lr=PT.LR, weight_decay=0), device=torch.device("cpu"), attr_embedder=emb,
                                 parsing_encoder=unet, parsing_decoder=head)
    Model = mods["model"].ParsingGenModel
    for name in ("init_training_settings", "feed_data", "optimize_parameters"):
        setattr(fake, name, types.MethodType(getattr(Model, name), fake))
    return fake


def main():
    torch.set_num_threads(8)
    mods = load_reference()
    fake = make_fake(mods)
    data = PT.batch()
    masks = []

    def hook(mod, inp, out):
        x, y = inp[0].detach(), out.detach()
        kept = (y != 0).flatten(2).any(2)
        # a channel whose input is all zero keeps no trace of its draw; it has no effect either way: call it kept
        masks.append((kept | ~(x != 0).flatten(2).any(2)).float())
    fake.parsing_decoder.dropout.register_forward_hook(hook)
    torch.manual_seed(2021)                     # configs/parsing_gen.yml manual_seed
    fake.init_training_settings()
    fake.feed_data(data)
    params = {f"{k}.{n}": p for k, attr in NETS.items() for n, p in getattr(fake, attr).named_parameters()}
    fake.optimize_parameters()
    out = {"loss_total": np.float64(float(fake.log_dict["loss_total"].detach())), "dropout_mask": masks[0].numpy()}
    for k, p in params.items():
        out["gnorm/" + k] = p.grad.norm().numpy()
        out["ghead/" + k] = p.grad.reshape(-1)[:8].numpy().copy()
        out["phead/" + k] = p.detach().reshape(-1)[:8].numpy().copy()
    for k, attr in NETS.items():
        for n, b in getattr(fake, attr).named_buffers():
            if n.endswith(("running_mean", "running_var")):
                out[f"buf/{k}.{n}"] = b.numpy().copy()
    path = os.path.join(OUT, "parsing_gen_train.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), float(out["loss_total"]), len(params), "parameter tensors",
          int(masks[0].sum()), "of", masks[0].numel(), "channels kept")


if __name__ == "__main__":
    main()
