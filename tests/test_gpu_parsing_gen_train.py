"""GPU: training the parsing generator (ShapeAttrEmbedding + ShapeUNet + FCNHead, configs/parsing_gen.yml) on libt2h.

  * every new kernel against fp64 torch: BatchNorm apply / backward with ReLU (and the Dropout2d factor), max-pool +
    broadcast-concat backward, bilinear x2 backward, pixel cross-entropy, the embedding backward;
  * the native ParsingGenTrainer against the fixture recorded from the REAL reference optimize_parameters
    (oracle/make_golden_parsing_gen_train.py), against autograd of the restatement (oracle/parsing_gen_train_ref.py)
    at other shapes and at the real widths, fp16 against fp32 mode, five steps against restatement + torch Adam;
  * save -> load -> resume, and the checkpoint in SampleFromPoseModel; invalid inputs."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import parsing_gen_recipes as P
import parsing_gen_train_recipes as PT
from oracle import parsing_gen_ref as PR
from oracle import parsing_gen_train_ref as TR
from test_parsing_gen_train_oracle import GOLD

pytestmark = pytest.mark.gpu
NETS = ("embedder", "encoder", "decoder")
REAL = (P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD)
TINY = (P.TINY_EMBEDDER, P.TINY_SHAPE_UNET, P.TINY_FCN_HEAD)


def _ops():
    from text2human_b200 import ops
    ops.set_precision("fp32")
    return ops


def build(cuda, cfgs=TINY, seeds=PT.TRAIN_SEEDS, lr=PT.LR):
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    from text2human_b200.parsing_gen_train import ParsingGenTrainer
    nets = [ShapeAttrEmbedding(**cfgs[0]), ShapeUNet(**cfgs[1]), FCNHead(**cfgs[2])]
    sds = P.state_dicts(*nets, seeds)
    for m, sd in zip(nets, sds):
        m.load_state_dict(sd, strict=True)
    nets = [m.to(cuda).eval() for m in nets]
    return ParsingGenTrainer(*nets, lr=lr), sds


def named(tr):
    return {f"{k}.{n}": p for k, m in zip(NETS, (tr.embedder, tr.unet, tr.head)) for n, p in m.named_parameters()}


def multi_step_batch():
    """the batch of the tests that follow the step beyond one exact comparison (fp16 mode, several Adam steps): 4x the
    fixture's pixels, so that the few activations that flip across a ReLU kink or max-pool tie -- at fp16 precision,
    or once Adam has moved the weights off the fixture's margins -- weigh on the gradient as they do in training,
    not as a large share of a 1024-pixel batch"""
    return PT.batch(dict(PT.TRAIN_SEEDS, pose=311), P.TINY_POSE)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


# ---------------------------------------------------------------------------- 1. kernels
@pytest.mark.parametrize("N,H,W,C", [(3, 13, 7, 16), (2, 32, 16, 64)])
def test_bn_relu_apply_and_backward_with_dropout(cuda, N, H, W, C):
    ops = _ops()
    g = torch.Generator().manual_seed(N * 100 + C)
    x = torch.randn((N, H, W, C), generator=g) * 2 + 0.3
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=g), 0.3 * torch.randn(C, generator=g)
    dy = torch.randn((N, H, W, C), generator=g)
    mask = (torch.rand((N, C), generator=g) > 0.2).float()
    drop = mask / 0.9
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    for dr in (None, drop):
        y = F.relu(F.batch_norm(xd, None, None, gd, bd, True, 0.1, 1e-5))
        if dr is not None:
            y = y * dr.double().view(N, C, 1, 1)
        gx, gg, gb = torch.autograd.grad(y, (xd, gd, bd), dy.double().permute(0, 3, 1, 2))
        xc = x.to(cuda)
        st = ops.norm_stats(xc, C, n=1)
        f, p = ops.norm_apply_ex(xc, st, gamma.to(cuda), beta.to(cuda), act="relu", groups=C, eps=1e-5, n=1,
                                 drop=None if dr is None else dr.to(cuda), want_planes=True)
        want_y = y.detach().permute(0, 2, 3, 1)
        assert _rel(f.cpu(), want_y) <= 1e-5
        assert _rel(p.double().sum(0).cpu(), want_y) <= 1e-5
        if dr is None:
            p2 = ops.norm_apply(xc, st, gamma.to(cuda), beta.to(cuda), act="relu", groups=C, eps=1e-5, n=1)
            assert torch.equal(p2, p)
        dg, db = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
        dx, dxp = ops.norm_bwd(xc, st, gamma.to(cuda), beta.to(cuda), dy.to(cuda), act="relu", groups=C, eps=1e-5,
                               dgamma=dg, dbeta=db, want_planes=True, n=1,
                               dy_scale=None if dr is None else dr.to(cuda))
        torch.cuda.synchronize()
        ex, eg, eb = _rel(dx.cpu(), gx.permute(0, 2, 3, 1)), _rel(dg.cpu(), gg), _rel(db.cpu(), gb)
        assert max(ex, eg, eb) <= 1e-4, (ex, eg, eb)
        print(f"[bn relu {N}x{H}x{W}x{C} drop={dr is not None}] dx {ex:.1e} dgamma {eg:.1e} dbeta {eb:.1e}")


@pytest.mark.parametrize("N,H,W,C,Ce,pool", [(2, 8, 6, 5, 3, True), (3, 9, 7, 8, 16, True), (2, 6, 4, 1, 16, False),
                                             (1, 16, 8, 24, 128, True)])
def test_maxpool_bcast_backward(cuda, N, H, W, C, Ce, pool):
    ops = _ops()
    g = torch.Generator().manual_seed(H * 10 + C)
    x = torch.randn((N, C, H, W), generator=g)
    x[:, :, :4, :4] = 0.5                                    # tied windows: constant ...
    x[0, :, 4:6, :4] = 0.0                                   # ... and all zero
    e = torch.randn((N, Ce), generator=g)
    xd, ed = x.double().requires_grad_(True), e.double().requires_grad_(True)
    cat = torch.cat([xd, ed.view(N, Ce, 1, 1).expand(N, Ce, H, W)], 1)
    out = F.max_pool2d(cat, 2) if pool else cat
    ld = (C + Ce + 7) // 8 * 8
    da = torch.zeros(out.shape[0], out.shape[2], out.shape[3], ld)
    da[..., :C + Ce] = torch.randn(out.permute(0, 2, 3, 1).shape, generator=g)
    gx, ge = torch.autograd.grad(out, (xd, ed), da[..., :C + Ce].double().permute(0, 3, 1, 2))
    base = torch.randn((N, H, W, C), generator=g)
    dx = base.clone().to(cuda)
    de = torch.ones((N, Ce), device=cuda)
    ops.maxpool2_bcast_bwd(da.to(cuda), C, Ce, x=x.permute(0, 2, 3, 1).contiguous().to(cuda), dx=dx, de=de,
                           pool=pool, in_hw=(H, W), accumulate=True)
    torch.cuda.synchronize()
    assert _rel(dx.cpu() - base, gx.permute(0, 2, 3, 1)) <= 1e-6
    assert _rel(de.cpu() - 1, ge) <= 1e-5
    de2 = torch.empty((N, Ce), device=cuda)
    ops.maxpool2_bcast_bwd(da.to(cuda), C, Ce, de=de2, pool=pool, in_hw=(H, W))
    de3 = torch.empty((N, Ce), device=cuda)
    ops.maxpool2_bcast_bwd(da.to(cuda), C, Ce, de=de3, pool=pool, in_hw=(H, W))
    assert torch.equal(de2, de3)                            # fixed-order sums: bitwise reproducible


@pytest.mark.parametrize("N,H,W,C", [(2, 5, 3, 8), (1, 16, 8, 64), (3, 1, 2, 4)])
def test_bilinear_backward_is_the_adjoint(cuda, N, H, W, C):
    ops = _ops()
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn((N, C, H, W), dtype=torch.float64, requires_grad=True)
    dy = torch.randn((N, 2 * H, 2 * W, C), generator=g)
    y = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    (gx,) = torch.autograd.grad(y, x, dy.double().permute(0, 3, 1, 2))
    got = ops.bilinear2x_bwd(dy.to(cuda))
    assert _rel(got.cpu(), gx.permute(0, 2, 3, 1)) <= 1e-6


@pytest.mark.parametrize("N,H,W,C", [(2, 13, 7, 24), (1, 9, 5, 5), (2, 4, 4, 130)])
def test_ce_logits_kernel(cuda, N, H, W, C):
    ops = _ops()
    g = torch.Generator().manual_seed(N * H + C)
    x = torch.randn((N, H, W, C), generator=g) * 3
    flat = x.view(-1)
    flat[:C], flat[C:2 * C] = 30.0, -30.0
    lab = torch.randint(0, C, (N, H, W), generator=g)
    lab.view(-1)[::11] = -100
    npix = N * H * W
    gscale = 2.0 ** int(np.floor(np.log2(npix))) / npix
    xd = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    loss = F.cross_entropy(xd, lab, reduction="none", ignore_index=-100).sum()
    (gx,) = torch.autograd.grad(loss, xd)
    want_g = gscale * gx.permute(0, 2, 3, 1)
    for terms in (2, 1):
        acc = torch.zeros(1, dtype=torch.float64, device=cuda)
        cs = torch.zeros(C, device=cuda)
        p = ops.ce_logits(x.to(cuda), lab.to(cuda), acc, gscale=gscale, colsum_out=cs, terms=terms)
        torch.cuda.synchronize()
        cp = (C + 7) // 8 * 8
        assert p.shape == (terms, N, H, W, cp) and (cp == C or float(p[..., C:].abs().max()) == 0.0)
        assert float(p.sum(0)[(lab == -100).to(cuda)].abs().max()) == 0.0
        assert abs(float(acc[0]) - float(loss.detach())) <= 1e-6 * float(loss.detach())
        assert _rel(p.double().sum(0)[..., :C].cpu(), want_g) <= (1e-6 if terms == 2 else 1e-3)
        assert _rel(cs.cpu(), want_g.sum((0, 1, 2))) <= 1e-5
    bad = lab.clone()
    bad[0, 0, 0] = C
    with pytest.raises(ValueError):
        ops.ce_logits(x.to(cuda), bad.to(cuda), torch.zeros(1, dtype=torch.float64, device=cuda))


def test_embedding_backward_matches_autograd(cuda):
    ops = _ops()
    from text2human_b200.flat_params import ParamSpace
    from text2human_b200.parsing_gen_arch import ShapeAttrEmbedding
    from text2human_b200.parsing_gen_train import embedder_linears
    for cfg in (P.TINY_EMBEDDER, P.REAL_EMBEDDER):
        emb = ShapeAttrEmbedding(**cfg)
        sd = R.fill_state_dict(R.spec_of(emb), 77)
        emb.load_state_dict(sd, strict=True)
        emb = emb.to(cuda).eval()
        attr = torch.cat([P.every_class_attrs(), P.shape_attrs(78, 5)])
        B = attr.shape[0]
        d = torch.randn((B, cfg["out_dim"]), generator=torch.Generator().manual_seed(79))
        sdr = {k: v.float().requires_grad_(True) for k, v in sd.items()}
        out = PR.shape_attr_embedding(sdr, attr, cfg["cls_num_list"])
        grads = torch.autograd.grad(out, list(sdr.values()), d.double())
        sp = ParamSpace(embedder_linears(emb), cuda)
        goff = torch.tensor([sp.g(p).storage_offset() for m in embedder_linears(emb) for p in (m.weight, m.bias)],
                            dtype=torch.int64, device=cuda)
        ops.shape_attr_embed_bwd(attr.to(cuda), emb._packed(), d.to(cuda), sp.flat_g, goff)
        torch.cuda.synchronize()
        got = dict(emb.named_parameters())
        worst = max(_rel(got[k].grad.cpu(), g) for k, g in zip(sdr, grads))
        assert worst <= 2e-5, worst
        print(f"[embedding bwd out_dim={cfg['out_dim']}] worst rel err {worst:.1e}")


# ---------------------------------------------------------------------------- 2. the step against the fixture
def test_native_step_matches_reference_fixture(cuda):
    _ops()
    gold = np.load(GOLD)
    tr, _ = build(cuda)
    tr.training_step(PT.batch(), dropout_mask=torch.from_numpy(gold["dropout_mask"]))
    torch.cuda.synchronize()
    loss = tr.losses()["loss_total"]
    assert abs(loss - float(gold["loss_total"])) <= 1e-3 * float(gold["loss_total"]), loss
    params = named(tr)
    assert len(params) == 135
    errs = {}
    for k, p in params.items():
        g, want = p.grad.detach().cpu() / tr.loss_scale, float(gold["gnorm/" + k])
        head = torch.from_numpy(gold["ghead/" + k])
        errs[k] = max(abs(float(g.norm()) - want), float((g.reshape(-1)[:8] - head).abs().max())) / want
    bad = {k: v for k, v in errs.items() if v > 1e-3}
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])
    worst = max(errs.values())
    tr.adam_step()
    torch.cuda.synchronize()
    gmax = max(float(gold[k]) for k in gold.files if k.startswith("gnorm/"))
    for k, p in params.items():
        want = torch.from_numpy(gold["phead/" + k])
        gh = torch.from_numpy(gold["ghead/" + k]).abs()
        # Adam's first step is ~lr * sign(g): an entry whose gradient is within rounding of zero may move either way
        small = gh <= 1e-3 * max(float(gold["gnorm/" + k]), 1e-6 * gmax)
        tol = torch.where(small, torch.full_like(gh, 2.5 * PT.LR), torch.full_like(gh, 1e-3 * PT.LR))
        err = (p.detach().cpu().reshape(-1)[:8] - want).abs()
        assert bool((err <= tol + 1e-6 * want.abs()).all()), (k, err)
    bufs = {f"{k}.{n}": b for k, m in zip(NETS, (tr.embedder, tr.unet, tr.head)) for n, b in m.named_buffers()
            if n.endswith(("running_mean", "running_var"))}
    bworst = max(_rel(b.cpu(), torch.from_numpy(gold["buf/" + k])) for k, b in bufs.items())
    assert bworst <= 1e-3, bworst
    print(f"[parsing gen train fp32] loss {loss:.6f} (ref {float(gold['loss_total']):.6f}); worst gradient rel err "
          f"{worst:.2e}; running stats {bworst:.2e}")


# ---------------------------------------------------------------------------- 3. against autograd of the restatement
def _restated(sds, data, mask, dtype=torch.float32):
    """restatement forward + backward on the same initial state -> (loss, {name: grad}, params)"""
    params = {f"{n}.{k}": v.clone().to(dtype).requires_grad_(True) for n, sd in zip(NETS, sds) for k, v in sd.items()
              if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    view = lambda n: {k[len(n) + 1:]: v for k, v in params.items() if k.startswith(n + ".")}  # noqa: E731
    ru = {k: v.to(dtype) for k, v in TR.running_stats(sds[1]).items()}
    rh = {k: v.to(dtype) for k, v in TR.running_stats(sds[2]).items()}
    d = dict(data, densepose=data["densepose"].to(dtype))
    m = None if mask is None else mask.to(dtype)
    loss, _ = TR.train_loss(view("embedder"), dict(view("encoder"), **ru), dict(view("decoder"), **rh), d, m,
                            P.CLS_NUM, ru, rh)
    grads = dict(zip(params, torch.autograd.grad(loss, list(params.values()))))
    return float(loss.detach()), grads, params


def _errors(got, want):
    """Frobenius-norm relative errors of a gradient set: (over all tensors, {tensor: error})"""
    num = sum(float((got[k].double() - want[k]).norm()) ** 2 for k in want) ** 0.5
    glob = num / sum(float(g.norm()) ** 2 for g in want.values()) ** 0.5
    return glob, {k: float((got[k].double() - want[k]).norm() / max(float(want[k].norm()), 1e-30)) for k in want}


def _compare_full(tr, sds, data, mask, tag):
    """The native step's full gradients against fp64 autograd of the restatement, measured against the spread of the
    restatement's own fp32 gradients (CPU) around the same fp64 values.  A few BatchNorm outputs within rounding of a
    ReLU kink and max-pool windows within rounding of a tie make any two fp32 implementations differ at those pixels,
    and the embedding's gradient (a per-image sum of broadcast-channel gradients that largely cancel) amplifies
    rounding: the yardstick is what fp32 itself achieves, not a fixed number."""
    loss64, g64, _ = _restated(sds, data, mask, torch.float64)
    _, g32, _ = _restated(sds, data, mask)
    tr.training_step(data, dropout_mask=mask)
    torch.cuda.synchronize()
    loss = tr.losses()["loss_total"]
    assert abs(loss - loss64) <= 1e-4 * loss64, (loss, loss64)
    got = {k: p.grad.detach().cpu() / tr.loss_scale for k, p in named(tr).items()}
    ours, ours_per = _errors(got, g64)
    ref, ref_per = _errors(g32, g64)
    worst = sorted(ours_per.items(), key=lambda kv: -kv[1])[:3]
    print(f"[{tag}] loss {loss:.6f}; gradient rel err vs fp64: native {ours:.2e}, fp32 restatement {ref:.2e}; "
          f"worst native tensors {[(k, f'{v:.1e}') for k, v in worst]}")
    assert ours <= max(1e-3, 5 * ref), (ours, ref)
    net = [k for k in g64 if not k.startswith("embedder.")]
    assert max(ours_per[k] for k in net) <= max(1e-2, 5 * max(ref_per[k] for k in net))


def test_native_step_full_gradients_second_shape(cuda):
    _ops()
    seeds = dict(PT.TRAIN_SEEDS, pose=321, attr=322, labels=323)
    tr, sds = build(cuda, seeds=seeds)
    data = PT.batch(seeds, (3, 96, 48), absent=(5,))
    mask = tr.draw_dropout_mask(3, torch.Generator(device=cuda).manual_seed(3)).cpu()
    _compare_full(tr, sds, data, mask, "parsing gen train B=3 96x48")


def test_native_step_real_widths(cuda):
    _ops()
    tr, sds = build(cuda, cfgs=REAL)
    data = PT.batch(PT.TRAIN_SEEDS, (2, 128, 64))
    mask = tr.draw_dropout_mask(2, torch.Generator(device=cuda).manual_seed(4)).cpu()
    _compare_full(tr, sds, data, mask, "parsing gen train real widths B=2 128x64")


def test_fp16_mode_tracks_fp32_mode(cuda):
    ops = _ops()
    gold = np.load(GOLD)
    mask = torch.from_numpy(gold["dropout_mask"])
    out = {}
    try:
        for mode in ("fp32", "fp16"):
            ops.set_precision(mode)
            tr, _ = build(cuda)
            tr.training_step(multi_step_batch(), dropout_mask=mask)
            torch.cuda.synchronize()
            out[mode] = (tr.losses()["loss_total"], {k: p.grad.detach().clone() / tr.loss_scale
                                                     for k, p in named(tr).items()})
    finally:
        ops.set_precision("fp32")
    (l32, g32), (l16, g16) = out["fp32"], out["fp16"]
    # single-product fp16 operands (10-bit mantissa, like TF32) through ~25 layers of a tiny net, whose many near-kink
    # / near-tie pixels flip at that precision: a loose bound on the loss, a looser one on the gradient as a whole
    assert abs(l16 - l32) <= 5e-3 * l32
    rel = float(torch.stack([(g16[k] - g32[k]).norm() for k in g32]).norm() /
                torch.stack([g.norm() for g in g32.values()]).norm())
    assert rel <= 0.35, rel
    print(f"[parsing gen train fp16 vs fp32] loss {l16:.6f} vs {l32:.6f}, gradient rel err (global norm) {rel:.2e}")


def _restated_losses(sds, data, masks, dtype):
    """the loss of each of len(masks) consecutive steps of the restatement + torch.optim.Adam in ``dtype``"""
    _, _, params = _restated(sds, data, None, dtype)
    opt = torch.optim.Adam(list(params.values()), PT.LR)
    ru = {k: v.to(dtype) for k, v in TR.running_stats(sds[1]).items()}
    rh = {k: v.to(dtype) for k, v in TR.running_stats(sds[2]).items()}
    view = lambda n: {k[len(n) + 1:]: v for k, v in params.items() if k.startswith(n + ".")}  # noqa: E731
    d = dict(data, densepose=data["densepose"].to(dtype))
    out = []
    for m in masks:
        loss, _ = TR.train_loss(view("embedder"), dict(view("encoder"), **ru), dict(view("decoder"), **rh), d,
                                m.to(dtype), P.CLS_NUM, ru, rh)
        opt.zero_grad()
        loss.backward()
        opt.step()
        out.append(float(loss.detach()))
    return out


def test_five_steps_track_restatement_with_torch_adam(cuda):
    """Five steps (masks replayed) against the restatement + torch Adam in fp64.  Adam's first steps move every
    parameter by about lr * sign(gradient), so gradients within rounding of zero move their parameters either way and
    any two fp32 runs drift apart step by step: the restatement's own fp32 trajectory is the yardstick (on this
    batch it is ~1.2e-3 off fp64 at step 5).  The first loss precedes any update and is held tightly."""
    _ops()
    tr, sds = build(cuda)
    data = multi_step_batch()
    masks = [tr.draw_dropout_mask(2, torch.Generator(device=cuda).manual_seed(10 + s)).cpu() for s in range(5)]
    got = []
    for m in masks:
        tr.optimize_parameters(data, dropout_mask=m)
        got.append(tr.losses()["loss_total"])
    want = _restated_losses(sds, data, masks, torch.float64)
    fp32 = _restated_losses(sds, data, masks, torch.float32)
    err = [abs(a - b) / b for a, b in zip(got, want)]
    ref = [abs(a - b) / b for a, b in zip(fp32, want)]
    print(f"[parsing gen train 5 steps] native {[f'{v:.5f}' for v in got]} fp64 {[f'{v:.5f}' for v in want]}; "
          f"rel err native {[f'{v:.1e}' for v in err]}, fp32 restatement {[f'{v:.1e}' for v in ref]}")
    assert err[0] <= 1e-5, err
    assert max(err) <= max(1e-3, 3 * max(ref)), (err, ref)
    assert want[-1] < want[0]


# ---------------------------------------------------------------------------- 4. checkpoints, inputs
def test_save_load_resume_and_sample_from_pose(cuda, tmp_path):
    _ops()
    from test_gpu_parsing_gen import _pose_opt
    from text2human_b200.pipeline import SampleFromPoseModel
    tr, _ = build(cuda, cfgs=REAL)
    data = PT.batch(PT.TRAIN_SEEDS, (2, 128, 64))
    mask = torch.ones((2, 64))
    tr.optimize_parameters(data, dropout_mask=mask)
    path = str(tmp_path / "parsing_gen.pth")
    tr.save(path)
    tr.optimize_parameters(data, dropout_mask=mask)
    tr.losses()
    after_a = {k: p.detach().clone() for k, p in named(tr).items()}
    tr2, _ = build(cuda, cfgs=REAL, seeds=dict(PT.TRAIN_SEEDS, embedder=1, encoder=2, decoder=3))
    tr2.load(path)
    tr2.optimize_parameters(data, dropout_mask=mask)
    # the same step from the checkpoint: equal up to Adam's sign-like second step on gradients within rounding of 0
    worst = max(float((p.detach() - after_a[k]).abs().max()) for k, p in named(tr2).items())
    assert worst <= 2.5 * PT.LR, worst
    ck = torch.load(path, map_location="cpu")
    assert set(ck) == {"embedder", "encoder", "decoder", "optimizer"}
    with contextlib.redirect_stdout(io.StringIO()):
        m = SampleFromPoseModel(_pose_opt())
    m.load_shape_generation_models(path)
    m = m.to(cuda)
    pose, attr = data["densepose"], data["attr"]
    got = m.generate_parsing_map(pose.to(cuda), attr.to(cuda)).cpu()
    logits, want = PR.generate_parsing_map({k: v.float() for k, v in ck["embedder"].items()}, ck["encoder"],
                                           ck["decoder"], pose, attr, P.CLS_NUM)
    top2 = logits.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1] > 1e-3).unsqueeze(1)
    assert bool((got.long() == want)[clear].all()) and float(clear.float().mean()) > 0.99


def test_invalid_inputs_raise_before_any_launch(cuda):
    ops = _ops()
    tr, _ = build(cuda)
    data = PT.batch()
    for key, bad in (("segm", lambda s: s.index_put_((torch.tensor([0]), torch.tensor([0]), torch.tensor([0])),
                                                    torch.tensor(PT.N_CLASSES))),
                     ("segm", lambda s: s.index_put_((torch.tensor([1]), torch.tensor([2]), torch.tensor([3])),
                                                    torch.tensor(-1))),
                     ("attr", lambda a: a.index_put_((torch.tensor([0]), torch.tensor([2])), torch.tensor(6)))):
        d = dict(data)
        d[key] = bad(d[key].clone())
        n0 = ops.COUNTERS["launches"]
        with pytest.raises(ValueError):
            tr.training_step(d)
        assert ops.COUNTERS["launches"] == n0
    with pytest.raises(NotImplementedError):
        from text2human_b200.parsing_gen_train import ParsingGenTrainer
        ParsingGenTrainer(tr.embedder, tr.unet, tr.head, weight_decay=1e-4)
