"""CPU: the fp32 restatement of the parsing-generator training step (oracle/parsing_gen_train_ref.py) reproduces the
fixture recorded from the REAL reference ParsingGenModel.optimize_parameters (oracle/make_golden_parsing_gen_train.py):
loss, every gradient (norm and first entries), the parameters after Adam and the BatchNorm running statistics."""
import os

import numpy as np
import torch

import parsing_gen_recipes as P
import parsing_gen_train_recipes as PT
from oracle import parsing_gen_train_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden", "parsing_gen_train.npz")


def reference_state(seeds=PT.TRAIN_SEEDS, cfgs=(P.TINY_EMBEDDER, P.TINY_SHAPE_UNET, P.TINY_FCN_HEAD)):
    """the fixture's initial state dicts (embedder, encoder, decoder), from the mirrors' key layout"""
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    nets = ShapeAttrEmbedding(**cfgs[0]), ShapeUNet(**cfgs[1]), FCNHead(**cfgs[2])
    return P.state_dicts(*nets, seeds)


def restated_step(sds, data, mask, lr=PT.LR, cls_num=P.CLS_NUM):
    """-> (loss, {name: grad}, {name: param after Adam}, {name: running stat}) with names '<net>.<key>'"""
    params = {f"{net}.{k}": v.clone().float().requires_grad_(True) for net, sd in zip(("embedder", "encoder", "decoder"), sds)
              for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    view = lambda net: {k[len(net) + 1:]: v for k, v in params.items() if k.startswith(net + ".")}  # noqa: E731
    ru, rh = TR.running_stats(sds[1]), TR.running_stats(sds[2])
    sd_u, sd_h = dict(view("encoder"), **ru), dict(view("decoder"), **rh)
    loss, _ = TR.train_loss(view("embedder"), sd_u, sd_h, data, mask, cls_num, ru, rh)
    opt = torch.optim.Adam(list(params.values()), lr, weight_decay=0)
    opt.zero_grad()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in params.items()}
    opt.step()
    running = {f"encoder.{k}": v for k, v in ru.items()}
    running.update({f"decoder.{k}": v for k, v in rh.items()})
    return float(loss.detach()), grads, {k: p.detach() for k, p in params.items()}, running


def test_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    torch.set_num_threads(4)
    loss, grads, after, running = restated_step(reference_state(), PT.batch(), torch.from_numpy(gold["dropout_mask"]))
    assert abs(loss - float(gold["loss_total"])) <= 1e-5 * abs(float(gold["loss_total"]))
    names = [k[len("gnorm/"):] for k in gold.files if k.startswith("gnorm/")]
    assert sorted(names) == sorted(grads) and len(names) == 135
    for k in names:
        g, want = grads[k], float(gold["gnorm/" + k])
        assert abs(float(g.norm()) - want) <= 1e-5 * want + 1e-12, k
        assert np.allclose(g.reshape(-1)[:8].numpy(), gold["ghead/" + k], rtol=1e-5, atol=1e-5 * want + 1e-12), k
        assert np.allclose(after[k].reshape(-1)[:8].numpy(), gold["phead/" + k], rtol=0, atol=1e-6), k
    bufs = [k[len("buf/"):] for k in gold.files if k.startswith("buf/")]
    assert sorted(bufs) == sorted(running)
    for k in bufs:
        assert np.allclose(running[k].numpy(), gold["buf/" + k], rtol=1e-5, atol=1e-6), k


def test_fixture_labels_hold_ignored_pixels_and_every_class():
    segm = PT.batch()["segm"]
    assert int((segm == -100).sum()) == 23
    assert set(segm.unique().tolist()) - {-100} == set(range(PT.N_CLASSES))


def test_fixture_stays_clear_of_kinks_and_ties():
    """the fixture's forward pass (the reference's arithmetic, fp32) has no pre-activation within rounding of a
    (Leaky)ReLU kink and no max-pool window within rounding of a tie, so the native step must route every gradient
    as the reference did"""
    sds = reference_state()
    probe = TR.Margins()
    with torch.no_grad():
        TR.train_loss(sds[0], dict(sds[1]), dict(sds[2]), PT.batch(), None, P.CLS_NUM, TR.running_stats(sds[1]),
                      TR.running_stats(sds[2]), probe=probe)
    assert min(probe.relu, probe.lrelu, probe.pool) >= 5e-5, (probe.relu, probe.lrelu, probe.pool)
