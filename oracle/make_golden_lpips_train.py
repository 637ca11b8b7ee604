"""Generate tests/golden/vqgan_lpips_train.npz: the REAL reference GAN training steps with the perceptual loss on.

Both recipes of the existing GAN-step fixtures are rerun unchanged, except that ``self.perceptual`` is the LPIPS
restatement (oracle/lpips_ref.py) carrying the seeded weights of tests/lpips_recipes.py instead of a zero stub:
  * top:    VQImageSegmTextureModel.training_step on TINY_VQGAN_TRAIN (the loader of make_golden_vqgan_train.py),
  * bottom: HierarchyVQSpatialTextureAwareModel.training_step on the vqgan_bottom_train recipe (the loader of
            make_golden_vqgan_bottom_train.py),
each followed by ``loss.backward()`` and ``d_loss.backward()``.  Keys are those of the existing fixtures behind a
"top_" / "bot_" prefix (losses, d_weight, per parameter tensor the gradient's norm and first 8 entries), plus the
reference's logged "l1" and "perceptual".
Run in the build container only:  python oracle/make_golden_lpips_train.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import lpips_recipes as LR  # noqa: E402
import vqgan_bottom_train_recipes as BR  # noqa: E402
from oracle import lpips_ref  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _record(out, prefix, f, loss, d_loss, gen_params):
    loss.backward()
    out[prefix + "loss"] = loss.detach().numpy()
    out[prefix + "d_loss"] = d_loss.detach().numpy()
    for k in ("nll_loss", "g_loss", "codebook_loss", "l1", "perceptual"):
        out[prefix + k] = np.float32(f.log_dict[k])
    out[prefix + "d_weight"] = np.asarray(f.log_dict["d_weight"].detach().numpy())
    for k, p in gen_params.items():
        g = p.grad if p.grad is not None else torch.zeros_like(p)
        out[prefix + "gnorm/" + k] = g.norm().numpy()
        out[prefix + "ghead/" + k] = g.reshape(-1)[:8].numpy().copy()
    f.disc.zero_grad()          # disc_optimizer.zero_grad() before d_loss.backward()
    d_loss.backward()
    for k, p in f.disc.named_parameters():
        out[prefix + "dnorm/" + k] = p.grad.norm().numpy()
        out[prefix + "dhead/" + k] = p.grad.reshape(-1)[:8].numpy().copy()


def top(out):
    from oracle import make_golden_vqgan_train as T
    vq, vm = T.build()
    cfg = R.TINY_VQGAN_TRAIN
    f = T.make_fake(vq, vm, cfg)
    f.perceptual = lpips_ref.LPIPSRef(LR.state_dict())
    for name, seed in (("encoder", 101), ("decoder", 102), ("quant_conv", 103), ("post_quant_conv", 104), ("disc", 105)):
        mod = getattr(f, name)
        mod.load_state_dict(R.fill_state_dict(R.spec_of(mod), seed), strict=True)
    cb = R.codebooks(106, 18, cfg["n_embed"], cfg["embed_dim"], "trained")
    for k, e in enumerate(f.quantize.embedding_list):
        e.weight.data.copy_(cb[k])
    for m in (f.encoder, f.decoder, f.quantize, f.quant_conv, f.post_quant_conv, f.disc):
        m.train()
    B, H, W = cfg["batch"], cfg["enc"]["resolution"], cfg["enc"]["resolution"] // 2
    data = dict(image=R.image(107, B, 3, H, W), texture_mask=R.blocky_mask(108, B, H, W, 8))
    torch.manual_seed(R.VQGAN_TRAIN_AUG_SEED)
    loss, d_loss = f.training_step(data, cfg["step"])
    params = {}
    for name in ("encoder", "decoder", "quant_conv", "post_quant_conv"):
        for k, p in getattr(f, name).named_parameters():
            params[f"{name}.{k}"] = p
    for k, e in enumerate(f.quantize.embedding_list):
        params[f"quantize.embedding_list.{k}.weight"] = e.weight
    _record(out, "top_", f, loss, d_loss, params)


def bottom(out):
    from oracle import make_golden_vqgan_bottom_train as BT
    from oracle import ref_loader
    ns = ref_loader.install(archs="reference", wrappers=("hierarchy_vqgan_model",))
    f = BT.stand_in(ns)
    f.perceptual = lpips_ref.LPIPSRef(LR.state_dict())
    data = BR.batch()
    params = BT.stepped_params(f)
    torch.manual_seed(BR.AUG_SEED)
    loss, d_loss = f.training_step(data, BR.STEP)
    _record(out, "bot_", f, loss, d_loss, params)


def main():
    torch.set_num_threads(8)
    out = {}
    top(out)
    bottom(out)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "vqgan_lpips_train.npz")
    np.savez_compressed(path, **out)
    for p in ("top_", "bot_"):
        print(p, {k: float(out[p + k]) for k in ("loss", "d_loss", "nll_loss", "l1", "perceptual", "d_weight")})
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
