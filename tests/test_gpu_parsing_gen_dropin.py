"""The parsing generator through the reference's own ``ParsingGenModel`` (models/parsing_gen_model.py, unmodified, built
by its own ``__init__``) on the mirrors: ShapeAttrEmbedding, ShapeUNet and FCNHead as autograd nodes
(parsing_gen_autograd), against the same wrapper on the reference's arch classes (stock PyTorch) on the same GPU, the
native ``ParsingGenTrainer`` and the fixture recorded from the real reference step.

The wrapper's ``__init__`` builds ShapeUNet at its default widths; for the reduced nets of parsing_gen_recipes the
classes it finds are wrapped with the reduced widths (``functools.partial``), in both arms alike.  The reduced batch
and seeds are those of parsing_gen_train_recipes, whose forward pass stays clear of every ReLU kink and max-pool tie
(oracle/parsing_gen_train_ref.Margins).
"""
import contextlib
import copy
import functools
import io
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import parsing_gen_recipes as P
import parsing_gen_train_recipes as PT

pytestmark = pytest.mark.gpu
NETS = dict(embedder="attr_embedder", encoder="parsing_encoder", decoder="parsing_decoder")
GOLD = os.path.join(os.path.dirname(__file__), "golden", "parsing_gen_train.npz")
TINY = (P.TINY_EMBEDDER, P.TINY_SHAPE_UNET, P.TINY_FCN_HEAD)
REAL = (P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD)


@pytest.fixture(autouse=True)
def _fp32():
    from text2human_b200 import ops
    ops.set_precision("fp32")
    yield
    ops.set_precision("fp32")


def _loader():
    from oracle import ref_loader as RL
    if not RL.available():
        pytest.skip("reference sources not staged (run oracle/make_ref.py in the build container)")
    return RL


def _rel(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def arch_classes(archs):
    """(ShapeAttrEmbedding, ShapeUNet, FCNHead) of ``archs``: the mirrors, or the reference's classes on the mmcv
    stand-ins"""
    if archs == "mirror":
        from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
        return ShapeAttrEmbedding, ShapeUNet, FCNHead
    ns = _loader().install("reference", wrappers=())
    return (sys.modules["models.archs.shape_attr_embedding_arch"].ShapeAttrEmbedding, ns.unet_arch.ShapeUNet,
            ns.fcn_arch.FCNHead)


def opt_for(cfgs=TINY, **kw):
    e, u, h = cfgs
    o = dict(is_train=True, embedder_dim=e["dim"], embedder_out_dim=e["out_dim"], attr_class_num=e["cls_num_list"],
             encoder_in_channels=u["in_channels"], fc_in_channels=h["in_channels"], fc_in_index=h["in_index"],
             fc_channels=h["channels"], fc_num_convs=h["num_convs"], fc_concat_input=h["concat_input"],
             fc_dropout_ratio=h["dropout_ratio"], fc_num_classes=h["num_classes"],
             fc_align_corners=h["align_corners"], lr=PT.LR, weight_decay=0, lr_decay="step", gamma=0.5, step=1)
    o.update(kw)
    return o


def wrapper(archs, opt, cfgs=TINY, seeds=PT.TRAIN_SEEDS, images=None):
    """the reference's ParsingGenModel built by its own __init__ on ``archs`` ("mirror" / "reference"), with the nets
    of parsing_gen_recipes; ``images`` collects what ``inference`` writes through mmcv.imwrite"""
    RL = _loader()
    emb_cls, unet_cls, head_cls = arch_classes(archs)
    if archs == "mirror":
        RL.install("mirror", wrappers=())
        sys.modules["models.archs.unet_arch"].ShapeUNet = unet_cls
        sys.modules["models.archs.fcn_arch"].FCNHead = head_cls
        sae = types.ModuleType("models.archs.shape_attr_embedding_arch")
        sae.ShapeAttrEmbedding = emb_cls
        sys.modules[sae.__name__] = sae
    store = {} if images is None else images
    sys.modules["mmcv"].imwrite = lambda img, path: store.__setitem__(os.path.basename(path), np.array(img))
    pg = RL._exec("models.parsing_gen_model", os.path.join(RL.ref_root(), "models", "parsing_gen_model.py"))
    if cfgs is TINY:
        u = {k: v for k, v in cfgs[1].items() if k != "in_channels"}
        pg.ShapeUNet = functools.partial(unet_cls, **u)
    w = pg.ParsingGenModel(opt)
    for m, sd in zip((w.attr_embedder, w.parsing_encoder, w.parsing_decoder),
                     P.state_dicts(w.attr_embedder, w.parsing_encoder, w.parsing_decoder, seeds)):
        m.load_state_dict(sd, strict=True)
    return w


def pair(cfgs=TINY, **kw):
    opt = opt_for(cfgs, **kw)
    wm, wr = wrapper("mirror", opt, cfgs), wrapper("reference", opt, cfgs)
    from text2human_b200 import parsing_gen_arch as A
    assert isinstance(wm.parsing_encoder, A.ShapeUNet) and not isinstance(wr.parsing_encoder, A.ShapeUNet)
    assert isinstance(wm.attr_embedder, A.ShapeAttrEmbedding) and isinstance(wm.parsing_decoder, A.FCNHead)
    return wm, wr


BROADCAST_SUMS = ("embedder.", "encoder.encoder.0.0.convs.0.conv.weight")


def grad_tol(k, later=False):
    """the gradient bound of tensor ``k`` (of its own max; of the embedder's largest gradient for an embedder tensor,
    see check_grads): 1e-3; 3e-3 for the embedder.  The embedder's gradients and the embedding columns of the first
    conv's weight gradient are per-image sums over H x W of broadcast-channel gradients that largely cancel
    (test_gpu_parsing_gen_train), which amplifies rounding, the more so once Adam has moved the weights off the
    recipe's: from the second step on (``later``) the embedder's tensors and the first conv's whole weight gradient are
    held to 1e-2 (measured on an H100 80GB HBM3 from kink-free batches: up to 1.5e-3 at the first step; 3.2e-3 for the
    embedder and 2.2e-3 for the first conv at the second, every other tensor within 7e-4)"""
    if later and k.startswith(BROADCAST_SUMS):
        return 1e-2
    return 3e-3 if k.startswith("embedder.") else 1e-3


def check_grads(gm, gr, later=False):
    """every gradient within grad_tol of its tensor's max; the same tensors are None in both.  A gradient below 1e-6 of
    the largest (one that vanishes in exact arithmetic is rounding noise in the reference too) is held to 1e-5 of the
    largest, absolutely -- the conditioning of test_gpu_vqgan_bottom_dropin.check_grads.  The embedder's gradients all
    come from the embedding's, a per-image sum over H x W of broadcast-channel gradients that largely cancel
    (test_gpu_parsing_gen_train): its rounding error reaches every embedder tensor alike, so they are held to 3e-3 of
    the largest embedder gradient (measured on an H100 80GB HBM3: up to 1.5e-3 of a tensor's own max)"""
    assert gm.keys() == gr.keys()
    for k in gr:
        assert (gm[k] is None) == (gr[k] is None), k
    keys = [k for k in gr if gr[k] is not None]
    gmax = max(float(gr[k].abs().max()) for k in keys)
    emax = max(float(gr[k].abs().max()) for k in keys if k.startswith("embedder."))
    worst = (0.0, None)
    for k in keys:
        if float(gr[k].abs().max()) < 1e-6 * gmax:
            assert float((gm[k] - gr[k]).abs().max()) < 1e-5 * gmax, k
            continue
        e = _rel(gm[k], gr[k]) if not k.startswith("embedder.") else \
            float((gm[k] - gr[k]).abs().max()) / emax
        assert e < grad_tol(k, later), (k, e)
        worst = max(worst, (e, k))
    return worst


def grads(w):
    return {f"{k}.{n}": p.grad for k, a in NETS.items() for n, p in getattr(w, a).named_parameters()}


def params(w):
    return {f"{k}.{n}": p.detach().clone() for k, a in NETS.items() for n, p in getattr(w, a).named_parameters()}


def bn_buffers(w):
    return {f"{k}.{n}": b for k, a in NETS.items() for n, b in getattr(w, a).named_buffers()}


def check_buffers(wm, wr, tol=1e-4):
    """running statistics to ``tol`` of each tensor's max (measured on an H100 80GB HBM3: 3.2e-5 for the BatchNorm of the
    coarsest decoder block's upsample, whose input comes out of a BatchNorm over 4 values per channel at this size;
    every other tensor within 1e-5); step counters equal"""
    bm, br = bn_buffers(wm), bn_buffers(wr)
    assert bm.keys() == br.keys()
    for k in br:
        if k.endswith("num_batches_tracked"):
            assert int(bm[k]) == int(br[k]), k
        else:
            assert _rel(bm[k], br[k]) <= tol, k


def sync(wm, wr):
    """give the mirror arm the reference arm's parameters, running statistics and Adam state.  Adam's first steps move
    a parameter by about lr * sign(g), so entries whose gradient is within rounding of zero move either way, and two
    correct fp32 runs drift apart step by step; each step is compared from the same state instead."""
    for a in NETS.values():
        getattr(wm, a).load_state_dict(getattr(wr, a).state_dict(), strict=True)
    # (a copy: load_state_dict keeps the very moment tensors it is given, which the other arm's steps update)
    wm.optimizer.load_state_dict(copy.deepcopy(wr.optimizer.state_dict()))


def check_adam_moves(pm, pr, p0, g, lr, later=False):
    """parameters after an Adam step.  Adam moves an entry by at most about lr, by lr * sign(g) at the first step; at
    later steps the move changes by about lr * dg / |g| for a gradient error dg, so an entry whose gradient is small
    beside its tensor's max (where grad_tol bounds dg) may move differently: each entry is held to
    min(2.5 lr, 10 lr grad_tol max|g| / |g|), and to 1e-3 lr at least"""
    for k in pr:
        ga = g[k].abs()
        scale = max(float(g[j].abs().max()) for j in g if j.startswith("embedder.")) if k.startswith("embedder.") \
            else float(ga.max())
        tol = torch.clamp(10 * lr * grad_tol(k, later) * scale / ga.clamp_min(1e-30), max=2.5 * lr)
        err = (pm[k] - pr[k]).abs()
        assert bool((err <= tol + 1e-3 * lr + 1e-6 * p0[k].abs()).all()), (k, float(err.max()))


# the smallest |pre-activation| and relative max-pool gap a batch may have.  At these sizes the deepest ShapeUNet stage
# normalises over 4 values per channel, which amplifies rounding: with margins of 1e-5 .. 4e-5, one step in three
# differed from the reference by 1.5e-3 .. 6e-3 in some gradient (measured on an H100 80GB HBM3), and at the
# fixture's own margins (7.5e-5 and 1.7e-4 on the reference's GPU forward) or above 6e-5 and 1e-4 no step did.  So few
# batches are that clear (the fixture's seed was found by such a scan) that thousands of seeds may be needed.
RELU_MARGIN, POOL_MARGIN = 5e-5, 1e-4


def margins(w, data):
    """oracle.parsing_gen_train_ref.Margins of the reference arm's forward pass on ``data`` in training mode, taken with
    hooks in front of every (Leaky)ReLU and MaxPool2d; the running statistics the pass moves are restored.  A ShapeUNet
    stage pools cat([x, embedding broadcast over H, W]): the broadcast channels tie in every window, and whichever
    position takes their gradient, the embedding's gradient is the same sum, so only x's channels are probed."""
    from oracle import parsing_gen_train_ref as TR
    probe = TR.Margins()
    nets = [getattr(w, a) for a in NETS.values()]
    bufs = [b for m in nets for b in m.buffers()]
    keep = [b.clone() for b in bufs]
    ce = w.attr_embedder.fusion[2].out_features
    hooks = []
    for m in nets:
        for mod in m.modules():
            if isinstance(mod, torch.nn.LeakyReLU):
                hooks.append(mod.register_forward_pre_hook(lambda m_, inp: probe.pre_act(inp[0], leaky=True)))
            elif isinstance(mod, torch.nn.ReLU):
                hooks.append(mod.register_forward_pre_hook(lambda m_, inp: probe.pre_act(inp[0])))
            elif isinstance(mod, torch.nn.MaxPool2d):
                hooks.append(mod.register_forward_pre_hook(
                    lambda m_, inp: probe.max_pool(inp[0][:, :inp[0].shape[1] - ce])))
    try:
        emb, unet, head = nets
        dev = next(emb.parameters()).device
        for m in nets:
            m.train()
        with torch.no_grad():
            head(unet(data["densepose"].to(dev), emb(data["attr"].to(dev))))
    finally:
        for h in hooks:
            h.remove()
        with torch.no_grad():
            for b, k in zip(bufs, keep):
                b.copy_(k)
    return probe


def kink_free_batch(wr, seeds=(PT.TRAIN_SEEDS["pose"],) + tuple(range(2000, 6000))):
    """The step's gradient is discontinuous at ReLU / LeakyReLU kinks and max-pool ties: an element within rounding of
    one may fall on different sides in two correct fp32 implementations and route its gradient differently.  The
    fixture's batch is clear of them at the recipe's weights only; after Adam steps (every weight moved by about lr)
    the batch is chosen again, scanning the pose-noise seed until the reference arm's forward at its current weights
    keeps every pre-activation and every max-pool gap at least RELU_MARGIN / POOL_MARGIN from its kink"""
    best = (0.0, None)
    for seed in seeds:
        data = PT.batch(dict(PT.TRAIN_SEEDS, pose=seed))
        pr = margins(wr, data)
        best = max(best, (min(pr.relu / RELU_MARGIN, pr.lrelu / RELU_MARGIN, pr.pool / POOL_MARGIN), seed))
        if min(pr.relu, pr.lrelu) >= RELU_MARGIN and pr.pool >= POOL_MARGIN:
            print(f"[parsing gen drop-in] pose seed {seed}: margins relu {pr.relu:.1e} leaky relu {pr.lrelu:.1e} "
                  f"max-pool {pr.pool:.1e}")
            return data
    raise AssertionError(f"no kink-free batch among the candidate seeds; best {best}")


def step(w, data, seed):
    w.feed_data(data)
    torch.cuda.manual_seed(seed)
    w.optimize_parameters()
    return float(w.log_dict["loss_total"].detach())


# ----------------------------------------------------------------------------- 1. three steps against the reference
def test_three_steps_match_reference_wrapper(cuda):
    wm, wr = pair()
    for s in range(3):
        data = kink_free_batch(wr)
        p0 = params(wr)
        lm, lr_ = step(wm, data, 100 + s), step(wr, data, 100 + s)
        assert abs(lm - lr_) <= 2e-4 * abs(lr_), (s, lm, lr_)
        gm, gr = grads(wm), grads(wr)
        worst = check_grads(gm, gr, later=s > 0)
        check_buffers(wm, wr)
        check_adam_moves(params(wm), params(wr), p0, gr, wm.optimizer.param_groups[0]["lr"], later=s > 0)
        print(f"[parsing gen drop-in] step {s + 1}: loss {lm:.6f} (ref {lr_:.6f}), worst gradient rel err "
              f"{worst[0]:.2e} ({worst[1]})")
        assert wm.update_learning_rate(s + 1) == wr.update_learning_rate(s + 1)
        sync(wm, wr)


# ----------------------------------------------------------------------------- 2. the nodes against the native step
def _nets(cuda, cfgs=TINY, seeds=PT.TRAIN_SEEDS):
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    nets = [ShapeAttrEmbedding(**cfgs[0]), ShapeUNet(**cfgs[1]), FCNHead(**cfgs[2])]
    for m, sd in zip(nets, P.state_dicts(*nets, seeds)):
        m.load_state_dict(sd, strict=True)
    return [m.to(cuda) for m in nets]


def _node_loss(emb, unet, head, data, cuda):
    logits = head(unet(data["densepose"].to(cuda), emb(data["attr"].to(cuda))))
    # CrossEntropyLoss of the reference: per-pixel cross-entropy, mean over every pixel (ignored ones included)
    return F.cross_entropy(logits, data["segm"].to(cuda), reduction="none", ignore_index=-100).mean()


def test_nodes_match_native_step_and_run_its_kernels(cuda):
    from text2human_b200 import _lib
    from text2human_b200.parsing_gen_train import ParsingGenTrainer
    calls, real_load = [], _lib.load

    class Rec:
        def __init__(self, lib):
            self.lib = lib

        def __getattr__(self, name):
            calls.append(name)
            return getattr(self.lib, name)

    data = PT.batch()
    tr = ParsingGenTrainer(*[m.eval() for m in _nets(cuda)])
    nets = [m.train() for m in _nets(cuda)]
    _lib.load = lambda: Rec(real_load())
    try:
        torch.cuda.manual_seed(7)
        tr.training_step(data)
        native = list(calls)
        torch.cuda.manual_seed(7)
        loss = _node_loss(*nets, data, cuda)
        calls.clear()
        loss.backward()
        node = list(calls)
    finally:
        _lib.load = real_load
    torch.cuda.synchronize()
    ln = tr.losses()["loss_total"]
    assert abs(float(loss.detach()) - ln) <= 1e-5 * ln, (float(loss.detach()), ln)
    gn = {f"{k}.{n}": p.grad / tr.loss_scale for k, m in zip(NETS, (tr.embedder, tr.unet, tr.head))
          for n, p in m.named_parameters()}
    gd = {f"{k}.{n}": p.grad for k, m in zip(NETS, nets) for n, p in m.named_parameters()}
    top = max(float(g.abs().max()) for g in gn.values())
    worst = max((float((gd[k] - gn[k]).abs().max()) / top, k) for k in gn)
    print(f"[parsing gen drop-in vs native] loss {float(loss.detach()):.7f} vs {ln:.7f}; worst gradient err {worst[0]:.1e} "
          f"of the largest gradient ({worst[1]})")
    # the nodes' logit gradient is torch's log-softmax backward, the native one ce_logits' fused softmax: they differ by
    # rounding (~1e-7 of each entry), carried through ~25 BatchNorm'd layers (measured on an H100 80GB HBM3: 2.1e-5 of
    # the largest gradient, at the first conv, whose weight gradient sums the embedding's broadcast channels)
    assert worst[0] <= 5e-5, worst
    # below the loss: the native backward's launches, plus the conversions at the node boundaries
    boundary = {"t2h_nchw_grad_to_planes", "t2h_nchw_to_nhwc", "t2h_nhwc_to_nchw"}
    tail = native[native.index("t2h_ce_logits") + 2:]      # after the loss kernel and the bias-gradient add
    assert node[0] == "t2h_nchw_grad_to_planes"
    assert [c for c in node if c not in boundary] == tail


# ----------------------------------------------------------------------------- 3. the fixture of the real reference
def test_step_matches_reference_fixture(cuda, monkeypatch):
    """the wrapper's step on the mirrors with the fixture's Dropout2d draw, held to what test_gpu_parsing_gen_train
    holds the native step to"""
    from text2human_b200 import parsing_gen_autograd as PA
    gold = np.load(GOLD)
    mask = torch.from_numpy(gold["dropout_mask"])
    monkeypatch.setattr(PA, "dropout2d_mask", lambda B, C, p, device, generator=None: mask.to(device).clone())
    w = wrapper("mirror", opt_for())
    loss = step(w, PT.batch(), 0)
    assert abs(loss - float(gold["loss_total"])) <= 1e-3 * float(gold["loss_total"]), loss
    g = grads(w)
    assert len(g) == 135
    errs = {}
    for k, gk in g.items():
        want, head = float(gold["gnorm/" + k]), torch.from_numpy(gold["ghead/" + k])
        gk = gk.detach().cpu()
        errs[k] = max(abs(float(gk.norm()) - want), float((gk.reshape(-1)[:8] - head).abs().max())) / want
    bad = {k: v for k, v in errs.items() if v > 1e-3}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])
    gmax = max(float(gold[k]) for k in gold.files if k.startswith("gnorm/"))
    for k, p in params(w).items():
        want = torch.from_numpy(gold["phead/" + k])
        gh = torch.from_numpy(gold["ghead/" + k]).abs()
        small = gh <= 1e-3 * max(float(gold["gnorm/" + k]), 1e-6 * gmax)
        tol = torch.where(small, torch.full_like(gh, 2.5 * PT.LR), torch.full_like(gh, 1e-3 * PT.LR))
        err = (p.cpu().reshape(-1)[:8] - want).abs()
        assert bool((err <= tol + 1e-6 * want.abs()).all()), (k, err)
    bufs = {k: b for k, b in bn_buffers(w).items() if k.endswith(("running_mean", "running_var"))}
    bworst = max(_rel(b.cpu(), torch.from_numpy(gold["buf/" + k])) for k, b in bufs.items())
    assert bworst <= 1e-3, bworst
    print(f"[parsing gen drop-in vs fixture] loss {loss:.6f}; worst gradient rel err {max(errs.values()):.2e}; "
          f"running stats {bworst:.2e}")


# ----------------------------------------------------------------------------- 4. real widths
def _glob(a, b, keys=None):
    keys = list(b) if keys is None else keys
    return float(torch.stack([(a[k].double() - b[k].double()).norm() for k in keys]).norm() /
                 torch.stack([b[k].double().norm() for k in keys]).norm())


def test_real_widths_step_against_reference_and_fp16(cuda):
    """configs/parsing_gen.yml's widths, B 8, 256 x 128 (Dropout2d off, so that every arm, fp64 included, runs the same
    function): one step of the wrapper on the mirrors in fp32 mode against the same wrapper on the reference's classes
    in fp64, held to the reference's own fp32 error as test_gpu_parsing_gen_train holds the native step (ReLU kinks and
    max-pool ties that flip at fp32 rounding, and the embedding's gradient, a per-image sum of broadcast-channel
    gradients that largely cancel, make any two fp32 implementations differ); fp16 mode against fp32 mode within the
    native trainer's fp16 bounds"""
    from text2human_b200 import ops
    data = PT.batch(PT.TRAIN_SEEDS, (8, 256, 128))
    opt = opt_for(REAL, fc_dropout_ratio=0.0)
    res = {}
    for arm in ("fp64", "reference", "fp32", "fp16"):
        ops.set_precision("fp16" if arm == "fp16" else "fp32")
        w = wrapper("mirror" if arm in ("fp32", "fp16") else "reference", opt, REAL)
        d = data
        if arm == "fp64":
            for a in NETS.values():
                getattr(w, a).double()
            for i in range(w.attr_embedder.attr_num):       # the one-hot codes are made in fp32 (.to(torch.float32))
                getattr(w.attr_embedder, f"attr_{i}").register_forward_pre_hook(lambda m_, inp: (inp[0].double(),))
            d = dict(data, densepose=data["densepose"].double())
        loss = step(w, d, 5)
        res[arm] = (loss, {k: g.detach().clone() for k, g in grads(w).items()})
        del w
    ops.set_precision("fp32")
    (l64, g64), (lr_, gr), (l32, g32), (l16, g16) = res["fp64"], res["reference"], res["fp32"], res["fp16"]
    net = [k for k in g64 if not k.startswith("embedder.")]
    ours, ref, e16 = _glob(g32, g64), _glob(gr, g64), _glob(g16, g32)
    ours_n, ref_n = _glob(g32, g64, net), _glob(gr, g64, net)
    print(f"[parsing gen drop-in real widths B=8 256x128] loss mirror {l32:.7f} ref fp32 {lr_:.7f} fp64 {l64:.7f} "
          f"fp16 {l16:.6f}; gradient rel err vs fp64 (global norm): mirror {ours:.2e}, reference fp32 {ref:.2e}; "
          f"without the embedder: mirror {ours_n:.2e}, reference fp32 {ref_n:.2e}; fp16 vs fp32 {e16:.2e}")
    assert abs(l32 - l64) <= 1e-4 * l64 and abs(lr_ - l64) <= 1e-4 * l64
    assert ours <= max(1e-3, 5 * ref), (ours, ref)
    assert ours_n <= max(1e-3, 5 * ref_n), (ours_n, ref_n)
    assert abs(l16 - l32) <= 5e-3 * l32 and e16 <= 0.35, (l16, l32, e16)


# ----------------------------------------------------------------------------- 5. validation and checkpoints
def test_inference_after_training_matches_reference(cuda):
    """one training step, then the wrapper's own validation loop: the eval-mode caches see the trained weights and
    the updated running statistics"""
    data = PT.batch()
    loader = [dict(densepose=data["densepose"][i:i + 1], attr=data["attr"][i:i + 1], segm=data["segm"][i:i + 1],
                   img_name=[f"img{i}.png"]) for i in range(2)]
    out = []
    opt = opt_for()
    for archs in ("mirror", "reference"):
        images = {}
        w = wrapper(archs, opt, images=images)
        acc0 = w.inference(loader, "val")
        step(w, data, 11)
        acc = w.inference(loader, "val")
        assert w.parsing_encoder.training and w.parsing_decoder.training
        w.attr_embedder.eval(), w.parsing_encoder.eval(), w.parsing_decoder.eval()
        with torch.no_grad():
            logits = w.parsing_decoder(w.parsing_encoder(data["densepose"].to(cuda),
                                                         w.attr_embedder(data["attr"].to(cuda))))
        out.append((acc0, acc, images, logits))
    (a0m, am, im, lm), (a0r, ar, ir, lr_) = out
    top2 = lr_.topk(2, dim=1).values
    clear = top2[:, 0] - top2[:, 1] > 1e-3                      # [B, H, W]
    n_unclear = int((~clear).sum())
    print(f"[parsing gen drop-in inference] accuracy before {a0m:.4f} / {a0r:.4f}, after one step {am:.4f} / "
          f"{ar:.4f}; {n_unclear} pixels within 1e-3 of a tie")
    tol = 100.0 * n_unclear / clear.numel() + 1e-4
    assert abs(a0m - a0r) <= tol and abs(am - ar) <= tol
    assert _rel(lm, lr_) <= 1e-4
    assert sorted(im) == sorted(ir) == ["img0.png", "img1.png"]
    W = data["densepose"].shape[3]
    for i in range(2):
        a, b = im[f"img{i}.png"], ir[f"img{i}.png"]
        assert a.shape == b.shape
        pred = slice(W, 2 * W)                                    # concat(pose, prediction, label) along W
        c = clear[i].cpu().numpy()
        assert np.array_equal(a[:, pred][c], b[:, pred][c]), i
        assert np.array_equal(np.delete(a, np.s_[W:2 * W], 1), np.delete(b, np.s_[W:2 * W], 1))


def test_save_load_network_and_sample_from_pose(cuda, tmp_path):
    from test_gpu_parsing_gen import _pose_opt
    from text2human_b200.pipeline import SampleFromPoseModel
    path = str(tmp_path / "parsing_gen.pth")
    data = PT.batch(PT.TRAIN_SEEDS, (2, 128, 64))
    w = wrapper("mirror", opt_for(REAL, pretrained_parsing_gen=path), REAL)
    step(w, data, 12)
    w.save_network(path)
    assert set(torch.load(path)) == {"embedder", "encoder", "decoder"}
    w2 = wrapper("mirror", opt_for(REAL, pretrained_parsing_gen=path), REAL,
                 seeds=dict(PT.TRAIN_SEEDS, embedder=1, encoder=2, decoder=3))
    w2.load_network()                                            # strict=True
    for a in NETS.values():
        s1, s2 = getattr(w, a).state_dict(), getattr(w2, a).state_dict()
        assert all(torch.equal(s1[k], s2[k]) for k in s1), a
    with contextlib.redirect_stdout(io.StringIO()):
        m = SampleFromPoseModel(_pose_opt())
    m.load_shape_generation_models(path)
    m = m.to(cuda)
    got = m.generate_parsing_map(data["densepose"].to(cuda), data["attr"].to(cuda))
    w.attr_embedder.eval(), w.parsing_encoder.eval(), w.parsing_decoder.eval()
    with torch.no_grad():
        logits = w.parsing_decoder(w.parsing_encoder(data["densepose"].to(cuda),
                                                     w.attr_embedder(data["attr"].to(cuda))))
    top2 = logits.topk(2, dim=1).values
    clear = top2[:, 0] - top2[:, 1] > 1e-3
    assert bool((got.long()[:, 0] == logits.argmax(1))[clear].all()) and float(clear.float().mean()) > 0.99


# ----------------------------------------------------------------------------- 6. extra capabilities
def test_weight_decay_matches_reference(cuda):
    wm, wr = pair(weight_decay=1e-4)
    for s in range(2):
        data = kink_free_batch(wr)
        p0 = params(wr)
        lm, lr_ = step(wm, data, 20 + s), step(wr, data, 20 + s)
        assert abs(lm - lr_) <= 2e-4 * abs(lr_)
        check_grads(grads(wm), grads(wr), later=s > 0)
        check_adam_moves(params(wm), params(wr), p0, grads(wr), PT.LR, later=s > 0)
        sync(wm, wr)


def _module_pair(cuda):
    out = []
    for archs in ("mirror", "reference"):
        emb_cls, unet_cls, head_cls = arch_classes(archs)
        nets = [emb_cls(**TINY[0]), unet_cls(**TINY[1]), head_cls(**TINY[2])]
        for m, sd in zip(nets, P.state_dicts(*nets, PT.TRAIN_SEEDS)):
            m.load_state_dict(sd, strict=True)
        out.append([m.to(cuda).train() for m in nets])
    return out


def _module_grads(nets):
    return {f"{k}.{n}": p.grad for k, m in zip(NETS, nets) for n, p in m.named_parameters()}


def test_loss_over_every_unet_output_matches(cuda):
    """a loss on all five ShapeUNet outputs (and the head's logits): the coarser outputs' gradients enter the UNet's
    backward where the reference's do"""
    data = PT.batch()
    res = []
    for nets in _module_pair(cuda):
        emb, unet, head = nets
        torch.cuda.manual_seed(31)
        outs = unet(data["densepose"].to(cuda), emb(data["attr"].to(cuda)))
        assert len(outs) == 5
        wts = [torch.randn(o.shape, generator=torch.Generator().manual_seed(40 + i)).to(cuda) * 1e-3
               for i, o in enumerate(outs)]
        loss = F.cross_entropy(head(outs), data["segm"].to(cuda), reduction="none", ignore_index=-100).mean()
        loss = loss + sum((o * w).sum() for o, w in zip(outs, wts))
        loss.backward()
        res.append((float(loss), _module_grads(nets), [b.clone() for n, b in unet.named_buffers()]))
    (lm, gm, bm), (lr_, gr, br) = res
    assert abs(lm - lr_) <= 2e-4 * abs(lr_)
    worst = check_grads(gm, gr)
    print(f"[parsing gen drop-in all five outputs] worst gradient rel err {worst[0]:.2e} ({worst[1]})")
    for a, b in zip(bm, br):
        assert _rel(a, b) <= 1e-5


def test_retain_graph_replay_reproduces_gradients(cuda):
    nets = _module_pair(cuda)[0]
    data = PT.batch()
    torch.cuda.manual_seed(32)
    loss = _node_loss(*nets, data, cuda)
    ps = [p for m in nets for p in m.parameters()]
    g1 = torch.autograd.grad(loss, ps, retain_graph=True)
    g2 = torch.autograd.grad(loss, ps)
    top = max(float(b.abs().max()) for b in g2)
    # the weight gradients sum with fp32 atomics: a replay agrees to their arrival order
    for a, b in zip(g1, g2):
        assert float((a - b).abs().max()) <= 1e-5 * top


def test_train_mode_under_no_grad_updates_running_stats(cuda):
    data = PT.batch()
    res = []
    for nets in _module_pair(cuda):
        emb, unet, head = nets
        torch.cuda.manual_seed(33)
        with torch.no_grad():
            logits = head(unet(data["densepose"].to(cuda), emb(data["attr"].to(cuda))))
        assert not logits.requires_grad
        res.append((logits, {f"{k}.{n}": b.clone() for k, m in zip(NETS, nets) for n, b in m.named_buffers()}))
    (lm, bm), (lr_, br) = res
    assert _rel(lm, lr_) <= 1e-4                                # the same channels dropped
    for k in br:
        if k.endswith("num_batches_tracked"):
            assert int(bm[k]) == int(br[k]) == 1, k
        else:
            assert _rel(bm[k], br[k]) <= 1e-5, k


# ----------------------------------------------------------------------------- 7. validation before any launch
def test_invalid_inputs_raise_before_any_launch(cuda):
    from text2human_b200 import ops
    emb, unet, head = _module_pair(cuda)[0]
    data = PT.batch()
    bad = data["attr"].clone()
    bad[0, 2] = 6
    for attr in (bad, data["attr"].float(), data["attr"][:, :14]):
        n0 = ops.COUNTERS["launches"]
        with pytest.raises(ValueError):
            emb(attr.to(cuda))
        assert ops.COUNTERS["launches"] == n0
    e = torch.zeros((2, TINY[0]["out_dim"]), device=cuda, requires_grad=True)
    pose = data["densepose"].to(cuda).requires_grad_(True)
    n0 = ops.COUNTERS["launches"]
    with pytest.raises(NotImplementedError):
        unet(pose, e)
    assert ops.COUNTERS["launches"] == n0


# ----------------------------------------------------------------------------- 8. the boundary kernel
@pytest.mark.parametrize("N,C,H,W", [(2, 5, 7, 9), (3, 24, 13, 11), (1, 130, 5, 7)])
@pytest.mark.parametrize("mode", ["fp32", "fp16"])
def test_nchw_grad_to_planes_kernel(cuda, N, C, H, W, mode):
    from text2human_b200 import ops
    ops.set_precision(mode)
    g = torch.Generator().manual_seed(N * 1000 + C * 10 + H)
    x = torch.randn((N, C, H, W), generator=g) * 1e-3
    x.view(-1)[::17] *= 1e3                                      # a spread of magnitudes
    c_pad = (C + 7) // 8 * 8
    s = 2.0 ** 9
    planes, sums = ops.nchw_grad_to_planes(x.to(cuda), c_pad, s)
    planes2, sums2 = ops.nchw_grad_to_planes(x.to(cuda), c_pad, s)
    torch.cuda.synchronize()
    T = 2 if mode == "fp32" else 1
    assert planes.shape == (T, N, H, W, c_pad) and sums.shape == (c_pad,)
    want = s * x.double().permute(0, 2, 3, 1)
    got = planes.double().sum(0).cpu()
    if c_pad > C:
        assert float(got[..., C:].abs().max()) == 0.0 and float(sums[C:].abs().max()) == 0.0
    # hi + lo: fp16 split resolution (2^-22 of each value, 2^-24 absolute near fp16's subnormals); hi alone: 2^-11
    rel = 2.0 ** -21 if T == 2 else 2.0 ** -10
    assert bool(((got[..., :C] - want).abs() <= rel * want.abs() + 2.0 ** -24).all())
    ws = want.sum((0, 1, 2))
    assert float(((sums[:C].cpu().double() - ws).abs() / ws.abs().clamp_min(1e-30)).max()) <= 1e-6
    assert torch.equal(sums, sums2) and torch.equal(planes, planes2)
