"""Generate tests/golden/segm_train.npz by running the REAL reference parsing-tokenizer training step
(/root/reference/models/vqgan_model.py VQSegmentationModel.feed_data / encode / decode / forward_step /
training_step / configure_optimizers, unbound, on a stand-in ``self`` carrying the attributes they read) around the
REAL reference Encoder / Decoder / VectorQuantizer and BCELossWithQuant, followed by ``loss.backward()`` and one
``torch.optim.Adam(lr=4.5e-5, betas=(0.5, 0.9))`` step.  (VQSegmentationModel.__init__ hard-codes the CUDA device.)

The fixture stores the three logged losses and, per parameter tensor, the gradient's norm, its first 8 entries and
the first 8 entries of the parameter after the Adam step.
Run in the build container only:  python oracle/make_golden_segm_train.py
"""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import segm_recipes as SG  # noqa: E402
from oracle.make_golden_vqgan_train import OUT, build  # noqa: E402

NETS = ("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv")


def make_fake(vq, vm, cfg):
    import models.losses.segmentation_loss as SL
    Model = vm.VQSegmentationModel
    fake = types.SimpleNamespace(opt=dict(cfg), device="cpu", log_dict={}, loss=SL.BCELossWithQuant())
    with contextlib.redirect_stdout(io.StringIO()):
        fake.encoder = vq.Encoder(ch=cfg['ch'], num_res_blocks=cfg['num_res_blocks'],
                                  attn_resolutions=cfg['attn_resolutions'], ch_mult=cfg['ch_mult'],
                                  in_channels=cfg['in_channels'], resolution=cfg['resolution'],
                                  z_channels=cfg['z_channels'], double_z=cfg['double_z'], dropout=cfg['dropout'])
        fake.decoder = vq.Decoder(in_channels=cfg['in_channels'], resolution=cfg['resolution'],
                                  z_channels=cfg['z_channels'], ch=cfg['ch'], out_ch=cfg['out_ch'],
                                  num_res_blocks=cfg['num_res_blocks'], attn_resolutions=cfg['attn_resolutions'],
                                  ch_mult=cfg['ch_mult'], dropout=cfg['dropout'], resamp_with_conv=True,
                                  give_pre_end=False)
    fake.quantize = vq.VectorQuantizer(cfg['n_embed'], cfg['embed_dim'], beta=0.25)
    fake.quant_conv = torch.nn.Conv2d(cfg["z_channels"], cfg['embed_dim'], 1)
    fake.post_quant_conv = torch.nn.Conv2d(cfg['embed_dim'], cfg["z_channels"], 1)
    for name in ("feed_data", "encode", "decode", "forward_step", "training_step", "configure_optimizers"):
        setattr(fake, name, types.MethodType(getattr(Model, name), fake))
    return fake


def load_weights(fake, cfg):
    S = SG.SEGM_TRAIN_SEEDS
    for name in ("encoder", "decoder", "quant_conv", "post_quant_conv"):
        mod = getattr(fake, name)
        mod.load_state_dict(R.fill_state_dict(R.spec_of(mod), S[name]), strict=True)
    cb = R.codebooks(S["codebook"], 1, cfg["n_embed"], cfg["embed_dim"], "trained")[0]
    fake.quantize.embedding.weight.data.copy_(cb)


def main():
    torch.set_num_threads(8)
    vq, vm = build()
    cfg = SG.TINY_SEGM_TRAIN
    fake = make_fake(vq, vm, cfg)
    load_weights(fake, cfg)
    B, H, W = cfg["batch"], cfg["resolution"], cfg["resolution"] // 2
    segm = SG.segm_labels(SG.SEGM_TRAIN_SEEDS["labels"], B, H, W)
    assert segm.unique().numel() == cfg["num_segm_classes"], "every class id should occur in the fixture's labels"
    params = {f"{n}.{k}": p for n in NETS for k, p in getattr(fake, n).named_parameters()}
    # optimize_parameters (vqgan_model.py:86-96): train mode, training_step, zero_grad, backward, Adam step
    for n in NETS:
        getattr(fake, n).train()
    fake.configure_optimizers()
    loss = fake.training_step(dict(segm=segm))
    fake.optimizer.zero_grad()
    loss.backward()
    out = {k.split("/")[1]: np.float64(float(v)) for k, v in fake.log_dict.items()}
    for k, p in params.items():
        out["gnorm/" + k] = p.grad.norm().numpy()
        out["ghead/" + k] = p.grad.reshape(-1)[:8].numpy().copy()
    fake.optimizer.step()
    for k, p in params.items():
        out["phead/" + k] = p.detach().reshape(-1)[:8].numpy().copy()
    path = os.path.join(OUT, "segm_train.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), {k: float(out[k]) for k in ("total_loss", "bce_loss", "quant_loss")},
          len(params), "parameter tensors")


if __name__ == "__main__":
    main()
