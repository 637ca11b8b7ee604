"""CPU: the fp32 restatement of the index-prediction training step (oracle/index_pred_train_ref.py) reproduces the
fixture recorded from the REAL reference optimize_parameters (oracle/make_golden_index_pred_train.py): loss, every
gradient (norm and first entries), the parameters after Adam and the BatchNorm running statistics."""
import os

import numpy as np
import torch

import golden_recipes as R
import index_pred_train_recipes as IT
from oracle import index_pred_train_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden", "index_pred_train.npz")
NETS = ("guidance_encoder", "index_decoder")


def reference_state(seeds=IT.SEEDS, cfgs=(R.TINY_UNET, R.TINY_FCN)):
    """the fixture's initial state dicts (guidance_encoder, index_decoder), from the mirrors' key layout"""
    from text2human_b200.index_pred_arch import MultiHeadFCNHead, UNet
    return IT.state_dicts(UNet(**cfgs[0]), MultiHeadFCNHead(**cfgs[1]), seeds)


def restated_step(sds, batch, masks, lr=IT.LR):
    """-> (loss, {name: grad}, {name: param after Adam}, {name: running stat}) with names '<net>.<key>'"""
    feature, own, tex = batch
    params = {f"{net}.{k}": v.clone().float().requires_grad_(True) for net, sd in zip(NETS, sds)
              for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    view = lambda net: {k[len(net) + 1:]: v for k, v in params.items() if k.startswith(net + ".")}  # noqa: E731
    ru, rf = TR.running_stats(sds[0]), TR.running_stats(sds[1])
    loss, _ = TR.train_loss(dict(view(NETS[0]), **ru), dict(view(NETS[1]), **rf), feature,
                            TR.gt_indices_list(own, tex), masks, ru, rf)
    opt = torch.optim.Adam(list(params.values()), lr, weight_decay=0)
    opt.zero_grad()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in params.items()}
    opt.step()
    running = {f"{NETS[0]}.{k}": v for k, v in ru.items()}
    running.update({f"{NETS[1]}.{k}": v for k, v in rf.items()})
    return float(loss.detach()), grads, {k: p.detach() for k, p in params.items()}, running


def test_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    torch.set_num_threads(4)
    loss, grads, after, running = restated_step(reference_state(), IT.batch(),
                                                torch.from_numpy(gold["dropout_mask"]))
    assert abs(loss - float(gold["loss_total"])) <= 1e-5 * abs(float(gold["loss_total"]))
    names = [k[len("gnorm/"):] for k in gold.files if k.startswith("gnorm/")]
    assert sorted(names) == sorted(grads) and len(names) == 156
    for k in names:
        g, want = grads[k], float(gold["gnorm/" + k])
        assert abs(float(g.norm()) - want) <= 1e-5 * want + 1e-12, k
        assert np.allclose(g.reshape(-1)[:8].numpy(), gold["ghead/" + k], rtol=1e-5, atol=1e-5 * want + 1e-12), k
        assert np.allclose(after[k].reshape(-1)[:8].numpy(), gold["phead/" + k], rtol=0, atol=1e-6), k
    bufs = [k[len("buf/"):] for k in gold.files if k.startswith("buf/")]
    assert sorted(bufs) == sorted(running)
    for k in bufs:
        assert np.allclose(running[k].numpy(), gold["buf/" + k], rtol=1e-5, atol=1e-6), k


def test_fixture_has_an_absent_head_and_ignored_positions():
    """one texture has no position (its head's gradient is exactly zero), some ids select no head, every other head
    has positions, and the 18 Dropout2d draws differ"""
    gold = np.load(GOLD)
    _, own, tex = IT.batch()
    present = set(tex.unique().tolist())
    assert IT.ABSENT_HEAD not in present
    assert set(range(IT.N_HEAD)) - present == {IT.ABSENT_HEAD}
    assert int((tex >= IT.N_HEAD).sum()) > 0
    k = IT.ABSENT_HEAD
    for p in (f"index_decoder.conv_seg_head_list.{k}.weight", f"index_decoder.conv_seg_head_list.{k}.bias",
              f"index_decoder.convs_list.{k}.0.conv.weight", f"index_decoder.convs_list.{k}.0.bn.weight"):
        assert float(gold["gnorm/" + p]) == 0.0, p
    masks = gold["dropout_mask"]
    assert masks.shape == (IT.N_HEAD, 2, R.TINY_FCN["channels"]) and len({m.tobytes() for m in masks}) > 1


def _gradients(sds, batch, masks):
    """fp64 gradients of the restated step (names '<net>.<key>')"""
    feature, own, tex = batch
    params = {f"{net}.{k}": v.double().requires_grad_(True) for net, sd in zip(NETS, sds) for k, v in sd.items()
              if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    view = lambda net: {k[len(net) + 1:]: v for k, v in params.items() if k.startswith(net + ".")}  # noqa: E731
    run = [{k: v.double() for k, v in TR.running_stats(sd).items()} for sd in sds]
    loss, _ = TR.train_loss(dict(view(NETS[0]), **run[0]), dict(view(NETS[1]), **run[1]), feature.double(),
                            TR.gt_indices_list(own, tex), masks.double(), run[0], run[1])
    return dict(zip(params, torch.autograd.grad(loss, list(params.values()))))


def test_fixture_gradient_is_stable_under_rounding_level_noise():
    """A BatchNorm output within rounding of its ReLU kink (amplified by 1/sigma where a BatchNorm sees few values)
    would let two correct fp32 implementations route a gradient differently.  The direct test: fp64 gradients of the
    fixture's weights perturbed by 3e-7 relative noise (several times fp32 rounding) move by at most 1e-4 per tensor,
    a tenth of the native step's bar, in every one of 8 draws."""
    torch.set_num_threads(4)
    sds = reference_state()
    batch = IT.batch()
    masks = torch.from_numpy(np.load(GOLD)["dropout_mask"])
    g0 = _gradients(sds, batch, masks)
    worst = 0.0
    for s in range(8):
        gen = torch.Generator().manual_seed(100 + s)
        sdp = [{k: v.double() * (1 + 3e-7 * torch.randn(v.shape, generator=gen, dtype=torch.float64))
                if v.is_floating_point() else v for k, v in sd.items()} for sd in sds]
        gp = _gradients(sdp, batch, masks)
        for k, g in g0.items():
            if float(g.norm()) > 0:
                worst = max(worst, float((gp[k] - g).norm() / g.norm()))
    assert worst <= 1e-4, worst


def test_fixture_stays_clear_of_kinks_and_ties():
    """no max-pool window's two largest values are within rounding of each other (the backward routes to the first
    maximum, so a tie could be broken differently); ReLU kinks, whose distance in BatchNorm-output units says little
    where a BatchNorm sees few values, are covered by the noise test above"""
    sds = reference_state()
    feature, own, tex = IT.batch()
    probe = TR.Margins()
    with torch.no_grad():
        TR.train_loss(dict(sds[0]), dict(sds[1]), feature, TR.gt_indices_list(own, tex), None,
                      TR.running_stats(sds[0]), TR.running_stats(sds[1]), probe=probe)
    assert probe.pool >= 2e-4, probe.pool
