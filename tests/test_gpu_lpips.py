"""GPU checks of the native LPIPS (text2human_b200/lpips.py, csrc/lpips.cu) against the fp64 restatement
(oracle/lpips_ref.py), and of both VQGAN trainers with ``perceptual=`` against the fixture recorded from the REAL
reference training steps with the restatement as ``self.perceptual`` (oracle/make_golden_lpips_train.py)."""
import os
import sys

import numpy as np
import pytest
import torch

import golden_recipes as R
import lpips_recipes as LR
import vqgan_bottom_train_recipes as BR
from oracle import lpips_ref

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "vqgan_lpips_train.npz")


def _oracle(in0, in1, dead=False):
    sd = {k: v.double() for k, v in LR.state_dict(dead_slice5=dead).items()}
    x1 = in1.detach().cpu().double().requires_grad_(True)
    v = lpips_ref.lpips(sd, in0.detach().cpu().double(), x1)
    v.sum().backward()
    return v.detach(), x1.grad


def _native(m, in0, in1):
    x1 = in1.clone().requires_grad_(True)
    v = m(in0, x1)
    v.sum().backward()
    torch.cuda.synchronize()
    return v.detach().double().cpu(), x1.grad.double().cpu()


def _inputs(cuda, B, H, W, seed):
    return R.image(seed, B, 3, H, W).to(cuda), R.image(seed + 1, B, 3, H, W).to(cuda)


# The gradient is discontinuous at every ReLU kink and max-pool tie of the trunk: an element whose pre-activation (or
# window runner-up) lies within rounding of the kink lands on either side in any fp32 computation, and moves a whole
# gradient element.  That is the whole gap measured here on an H100 80GB HBM3 (700 W): 3.1e-4 (norm) / 1.3e-3 (worst
# element) at 2 x 64 x 32 and 1.2e-3 / 3.4e-2 at 3 x 256 x 128.  test_gpu_lpips_kernels.py::
# test_lpips_stages_and_conditioned runs the same inputs against the fp64 restatement conditioned on the native ReLU
# masks and max-pool picks: the gradient then agrees to 5e-6, and the elements whose mask differs from fp64's sign
# (5 at 2 x 64 x 32, within 1.4 fp32 rounding units of their kink; 74 masks and 16 picks at 3 x 256 x 128, within 30)
# are rounding-level kink flips.  The value is a fixed-order fp64 sum of fp32 per-pixel terms: within 3.1e-7.
@pytest.mark.parametrize("B,H,W,gtol,wtol", [(2, 64, 32, 1e-3, 3e-3), (3, 256, 128, 3e-3, 6e-2)])
def test_value_and_gradient_match_fp64(cuda, B, H, W, gtol, wtol):
    from text2human_b200 import ops
    ops.set_precision("fp32")
    m = LR.mirror(cuda)
    in0, in1 = _inputs(cuda, B, H, W, 500 + H)
    v, g = _native(m, in0, in1)
    wv, wg = _oracle(in0, in1)
    assert v.shape == (B, 1, 1, 1)
    verr = float(((v - wv).abs() / wv.abs()).max())
    gnorm = float((g - wg).norm() / wg.norm())
    gmax = float((g - wg).abs().max() / wg.abs().max())
    print(f"[lpips {B}x{H}x{W}] value rel {verr:.2e}, grad norm rel {gnorm:.2e}, worst element / largest {gmax:.2e}")
    assert verr <= 1e-6 and gnorm <= gtol and gmax <= wtol, (verr, gnorm, gmax)
    # the no_grad path (forward only) gives the same values
    with torch.no_grad():
        v2 = m(in0, in1).double().cpu()
    assert torch.equal(v2, v)


def test_dead_slice5_pixels(cuda):
    """relu5_3 zero at every pixel: the value equals the oracle's, the gradient is finite and equals the oracle's"""
    from text2human_b200 import ops
    ops.set_precision("fp32")
    m = LR.mirror(cuda, dead_slice5=True)
    in0, in1 = _inputs(cuda, 2, 64, 32, 610)
    v, g = _native(m, in0, in1)
    wv, wg = _oracle(in0, in1, dead=True)
    assert torch.isfinite(g).all()
    assert float(((v - wv).abs() / wv.abs()).max()) <= 1e-4
    # (bounds: see test_value_and_gradient_match_fp64; measured 5.5e-4 / 1.9e-3)
    assert float((g - wg).norm() / wg.norm()) <= 1e-3 and float((g - wg).abs().max() / wg.abs().max()) <= 3e-3


def test_fp16_mode_tracks_fp32(cuda):
    from text2human_b200 import ops
    in0, in1 = _inputs(cuda, 2, 128, 64, 620)
    res = {}
    try:
        for mode in ("fp32", "fp16"):
            ops.set_precision(mode)
            res[mode] = _native(LR.mirror(cuda), in0, in1)
    finally:
        ops.set_precision("fp32")
    (v32, g32), (v16, g16) = res["fp32"], res["fp16"]
    cos = float((g32 * g16).sum() / (g32.norm() * g16.norm()))
    verr = float(((v16 - v32).abs() / v32.abs()).max())
    print(f"[lpips fp16] value rel {verr:.2e}, gradient cosine {cos:.5f}")
    assert verr <= 2e-2 and cos >= 0.98


def test_backward_runs_twice_and_repacks_after_load(cuda):
    """retain_graph: the node's backward can run twice; load_state_dict changes the packed weights"""
    from text2human_b200 import ops
    ops.set_precision("fp32")
    m = LR.mirror(cuda)
    in0, in1 = _inputs(cuda, 2, 64, 32, 630)
    x1 = in1.clone().requires_grad_(True)
    v = m(in0, x1)
    (g1,) = torch.autograd.grad(v.sum(), x1, retain_graph=True)
    (3.0 * v).sum().backward()
    assert torch.allclose(x1.grad, 3.0 * g1, rtol=1e-6, atol=0)
    with torch.no_grad():
        before = m(in0, in1)
        m.load_state_dict(LR.mirror_state_dict(LR.state_dict(seed=LR.SEED + 1)), strict=True)
        after = m(in0, in1)
    sd = {k: v_.double() for k, v_ in LR.state_dict(seed=LR.SEED + 1).items()}
    want = lpips_ref.lpips(sd, in0.cpu().double(), in1.cpu().double())
    assert not torch.equal(before, after)
    assert float(((after.double().cpu() - want).abs() / want.abs()).max()) <= 1e-4


# ----------------------------------------------------------------------------
# the trainers with perceptual=
# ----------------------------------------------------------------------------
def _check(gold, prefix, named, scale, tol):
    from test_gpu_vqgan_train import _check_grads
    return _check_grads(gold, prefix, named, scale, tol)


def _top(cuda, **kw):
    from test_gpu_vqgan_train import build, recorded_draws
    from text2human_b200.vqgan_train import VQGANTrainer
    m, disc, cfg = build(cuda)
    tr = VQGANTrainer(m, disc, disc_start_step=cfg["disc_start_step"], **kw)
    tr.aug_draw_fn = recorded_draws(R.VQGAN_TRAIN_AUG_SEED)
    B, H, W = cfg["batch"], cfg["enc"]["resolution"], cfg["enc"]["resolution"] // 2
    data = dict(image=R.image(107, B, 3, H, W), texture_mask=R.blocky_mask(108, B, H, W, 8))
    named = {f"{n}.{k}": p for n in ("encoder", "decoder", "quant_conv", "post_quant_conv")
             for k, p in getattr(m, n).named_parameters()}
    for k, e in enumerate(m.quantize.embedding_list):
        named[f"quantize.embedding_list.{k}.weight"] = e.weight
    return tr, data, cfg["step"], named, disc


def _bottom(cuda, **kw):
    from test_gpu_vqgan_bottom_train import build, named_gen
    from test_gpu_vqgan_train import recorded_draws
    m, disc, tr = build(cuda, **kw)
    tr.aug_draw_fn = recorded_draws(BR.AUG_SEED)
    return tr, BR.batch(), BR.STEP, named_gen(m), disc


@pytest.mark.parametrize("which", ["top", "bot"])
def test_trainer_with_perceptual_matches_reference_fixture(cuda, which):
    from text2human_b200 import ops
    ops.set_precision("fp32")
    gold = np.load(GOLD)
    p = which + "_"
    tr, data, step, named, disc = (_top if which == "top" else _bottom)(cuda, perceptual=LR.mirror(cuda))
    tr.training_step(data, step)
    torch.cuda.synchronize()
    got = tr.losses()
    for k in ("nll_loss", "g_loss", "codebook_loss", "d_weight", "loss", "d_loss", "l1", "perceptual"):
        want = float(gold[p + k])
        assert abs(got[k] - want) <= 2e-4 * max(1.0, abs(want)), (k, got[k], want)
    worst_g, n_g = _check(gold, p + "g", named, tr.loss_scale, 1e-3)
    worst_d, n_d = _check(gold, p + "d", dict(disc.named_parameters()), tr.disc_scale, 1e-3)
    print(f"[{which} step + LPIPS] worst gradient rel err {worst_g:.2e} ({n_g}) / {worst_d:.2e} ({n_d}); {got}")
    assert n_g > 50 and n_d >= 10


@pytest.mark.parametrize("which", ["top", "bot"])
def test_trainer_without_perceptual_is_unchanged(cuda, which):
    """perceptual=None is the step without the perceptual term: the same gradients as a step whose LPIPS runs with
    perceptual_weight 0 (it then adds exact zeros) up to the run-to-run summation order of the split weight-gradient
    reductions, and nll_loss is the L1 term alone"""
    from text2human_b200 import ops
    ops.set_precision("fp32")
    build = _top if which == "top" else _bottom
    res = []
    for kw in (dict(perceptual=None), dict(perceptual=LR.mirror(cuda), perceptual_weight=0.0)):
        tr, data, step, _, _ = build(cuda, **kw)
        tr.training_step(data, step)
        torch.cuda.synchronize()
        res.append((tr.gen.flat_g.clone(), tr.dsc.flat_g.clone(), tr.losses()))
    for a, b in ((res[0][0], res[1][0]), (res[0][1], res[1][1])):
        assert float((a - b).norm() / b.norm()) <= 1e-5          # measured 2.0e-6 run to run
    assert res[0][2]["perceptual"] == 0.0 and res[0][2]["nll_loss"] == res[0][2]["l1"]
    assert res[1][2]["perceptual"] > 0.0
    for k in ("nll_loss", "g_loss", "codebook_loss", "d_weight", "loss", "d_loss"):
        assert abs(res[0][2][k] - res[1][2][k]) <= 1e-6 * max(1.0, abs(res[1][2][k])), k


def test_micro_batches_sum_single_image_steps(cuda):
    """two micro-batches of 1 == the sum of the two single-image steps (each micro-batch its own adaptive weight)"""
    from text2human_b200 import ops
    ops.set_precision("fp32")
    lp = LR.mirror(cuda)
    tr, data, step, _, _ = _top(cuda, perceptual=lp, micro_batch=1, diff_aug=False)
    tr.force_no_reduce = True
    tr.training_step(data, step)
    torch.cuda.synchronize()
    both = tr.gen.flat_g.clone()
    single = torch.zeros_like(both)
    ps = []
    for i in range(2):
        tr1, _, _, _, _ = _top(cuda, perceptual=lp, diff_aug=False)
        tr1.force_no_reduce = True
        tr1.training_step({k: v[i:i + 1] for k, v in data.items()}, step)
        torch.cuda.synchronize()
        single += tr1.gen.flat_g
        ps.append(tr1.losses()["perceptual"])
    err = float((both - single).norm() / single.norm())
    assert err <= 1e-5, err
    assert abs(tr.losses()["perceptual"] - sum(ps) / 2) <= 1e-6 * abs(sum(ps))


def test_unmodified_reference_wrapper_with_mirror_installed_as_lpips(cuda, monkeypatch):
    """The reference's own VQImageSegmTextureModel (its __init__ calls ``lpips.LPIPS(net="vgg")``, its
    training_step the perceptual loss) on the mirrors, with the LPIPS mirror installed as ``lpips.LPIPS`` inside
    this test only, against the same wrapper on the reference arch classes with the oracle LPIPS."""
    import contextlib
    import io
    from test_gpu_boundary import _fill, _loader, _rel, _tiny_opt
    from text2human_b200 import ops
    ops.set_precision("fp32")
    RL = _loader()
    opt = _tiny_opt()
    B, H, W = 2, 64, 32
    data = dict(image=R.image(107, B, 3, H, W), texture_mask=R.blocky_mask(108, B, H, W, 8))
    sd = LR.state_dict()
    wrappers = []
    for archs, factory in (("mirror", lambda net="vgg": LR.mirror(cuda)),
                           ("reference", lambda net="vgg": lpips_ref.LPIPSRef(sd))):
        ns = RL.install(archs, wrappers=("vqgan_model",))
        monkeypatch.setattr(sys.modules["lpips"], "LPIPS", factory)
        with contextlib.redirect_stdout(io.StringIO()):
            w = ns.vqgan_model.VQImageSegmTextureModel(opt)
        _fill(w)
        for n in ("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv", "disc"):
            getattr(w, n).train()
        wrappers.append(w)
    wm, wr = wrappers
    assert type(wm.perceptual).__module__ == "text2human_b200.lpips"
    # a DiffAugment seed under which no discriminator pre-activation of the reference run is within 1e-4 of a kink
    margins = []
    hooks = [mod.register_forward_pre_hook(lambda m_, inp: margins.append(float(inp[0].detach().abs().min())))
             for mod in wr.disc.main if isinstance(mod, torch.nn.LeakyReLU)]
    best = (0.0, None)
    for cand in range(31, 51):
        margins.clear()
        torch.manual_seed(cand)
        wr.training_step(data, opt["disc_start_step"] + 5)
        best = max(best, (min(margins), cand))
    for h_ in hooks:
        h_.remove()
    assert best[0] > 3e-5
    res = []
    for w in (wm, wr):
        torch.manual_seed(best[1])
        loss, d_loss = w.training_step(data, opt["disc_start_step"] + 5)
        loss.backward()
        res.append({k: p.grad.detach().clone() for k, p in w.decoder.named_parameters() if p.grad is not None})
    for k in ("nll_loss", "g_loss", "codebook_loss", "l1", "perceptual"):
        assert abs(wm.log_dict[k] - wr.log_dict[k]) <= 2e-4 * max(1.0, abs(wr.log_dict[k])), k
    assert wm.log_dict["perceptual"] > 0
    assert abs(float(wm.log_dict["d_weight"]) - float(wr.log_dict["d_weight"])) <= 2e-3 * float(wr.log_dict["d_weight"])
    gmax = max(float(g.abs().max()) for g in res[1].values())
    worst = 0.0
    for k, gr in res[1].items():
        if float(gr.abs().max()) < 1e-6 * gmax:
            continue
        worst = max(worst, _rel(res[0][k], gr))
    print(f"[lpips boundary] reference training_step with the LPIPS mirror: worst decoder gradient rel err {worst:.2e}")
    assert worst < 1e-3
