"""CPU: the parsing-tokenizer training-step restatement (oracle/segm_train_ref.segm_training_step) against the fixture
made from the real reference `VQSegmentationModel.training_step` + `loss.backward()` + Adam step
(oracle/make_golden_segm_train.py): losses, every parameter gradient and the parameters after one Adam step."""
import contextlib
import io
import os

import numpy as np
import torch

import golden_recipes as R
import segm_recipes as SG
from oracle import segm_train_ref as SR

GOLD = os.path.join(os.path.dirname(__file__), "golden", "segm_train.npz")


def segm_state(cfg=None):
    """the fixture's seeded weights keyed as the reference checkpoint ('encoder.*', ..., codebook [n_e, D])"""
    from text2human_b200.segm_train import SegmTokenizerModel
    cfg = cfg or SG.TINY_SEGM_TRAIN
    with contextlib.redirect_stdout(io.StringIO()):
        m = SegmTokenizerModel(cfg)
    sd = {}
    for name in ("encoder", "decoder", "quant_conv", "post_quant_conv"):
        for k, v in R.fill_state_dict(R.spec_of(getattr(m, name)), SG.SEGM_TRAIN_SEEDS[name]).items():
            sd[f"{name}.{k}"] = v
    cb = R.codebooks(SG.SEGM_TRAIN_SEEDS["codebook"], 1, cfg["n_embed"], cfg["embed_dim"], "trained")[0]
    return sd, cb


def test_segm_training_step_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    cfg = SG.TINY_SEGM_TRAIN
    sd, cb = segm_state()
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    cb = cb.clone().requires_grad_(True)
    B, H, W = cfg["batch"], cfg["resolution"], cfg["resolution"] // 2
    r = SR.segm_training_step(sd, cb, SG.segm_labels(SG.SEGM_TRAIN_SEEDS["labels"], B, H, W))
    for k in ("total_loss", "bce_loss", "quant_loss"):
        got = float(r[k].detach())
        assert abs(got - float(gold[k])) <= 1e-5 * abs(float(gold[k])), (k, got, float(gold[k]))
    r["total_loss"].backward()
    named = dict(sd)
    named["quantize.embedding.weight"] = cb
    gmax = max(float(gold[k]) for k in gold.files if k.startswith("gnorm/"))
    params = [(k, named[k]) for k in named]
    opt = torch.optim.Adam([p for _, p in params], lr=cfg["lr"], betas=(0.5, 0.9))
    n = 0
    for name, p in params:
        want = float(gold["gnorm/" + name])
        err = max(abs(float(p.grad.norm()) - want),
                  float((p.grad.reshape(-1)[:8] - torch.from_numpy(gold["ghead/" + name])).abs().max()))
        # gradients that vanish in exact arithmetic (a conv bias in front of a GroupNorm) are rounding noise in
        # the reference as well: absolute floor
        assert err <= 1e-5 * want or err <= 1e-9 * gmax, (name, err, want)
        n += 1
    assert n == len([k for k in gold.files if k.startswith("gnorm/")]) == 243
    opt.step()
    for name, p in params:
        got = p.detach().reshape(-1)[:8]
        want = torch.from_numpy(gold["phead/" + name])
        g = torch.from_numpy(gold["ghead/" + name]).abs()
        # one Adam step moves a parameter by ~lr * sign(g): where g is rounding noise its sign is arbitrary
        tol = torch.where(g > 1e-9 * gmax, torch.full_like(g, 1e-3 * cfg["lr"]), torch.full_like(g, 2.5 * cfg["lr"]))
        assert bool(((got - want).abs() <= tol + 1e-7 * want.abs()).all()), name
