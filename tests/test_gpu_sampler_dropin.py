"""The sampler's drop-in training path: ``TransformerMultiHead.forward`` as one autograd node (transformer_train
``_SamplerNode``) under the reference's own ``TransformerTextureAwareModel.optimize_parameters``.

  A  t2h_head_grads_to_planes / t2h_head_grads_absmax element by element against f32_to_planes_rows of the
     concatenated gradients, on the strides torch's loss really produces, contiguous, mixed and null heads
  B  the node under the reference's loss arithmetic against the native SamplerTrainer at the real widths
  C  the reference wrapper, unmodified, on the mirrors against the same wrapper on the reference's arch classes
  D  replay under retain_graph, memory release, weight caches after torch.optim.Adam
  E  the dropout guard
"""
import contextlib
import io
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
REAL = dict(codebook_size=18 * 1024, segm_codebook_size=1024, texture_codebook_size=18, bert_n_emb=512,
            bert_n_layers=2, bert_n_head=8, block_size=512, latent_shape=[32, 16], embd_pdrop=0.0, resid_pdrop=0.0,
            attn_pdrop=0.0, num_head=18)
MID = dict(R.TINY_TRANSFORMER, codebook_size=18 * 64, bert_n_emb=128, bert_n_layers=3, bert_n_head=8, block_size=160,
           latent_shape=[16, 10])


@pytest.fixture(autouse=True)
def _fp32():
    from text2human_b200 import ops
    ops.set_precision("fp32")
    yield
    ops.set_precision("fp32")


def _make(cfg, seed):
    from text2human_b200.transformer_arch import TransformerMultiHead
    net = TransformerMultiHead(**cfg)
    sd = R.fill_state_dict(R.spec_of(net), seed)
    net.load_state_dict(sd, strict=True)
    return net.to(DEV), sd


def _batch(cfg, seed, B):
    x_0, gt_list, segm, tex = R.sampler_train_batch(seed, B=B, cfg=cfg)
    g = R._gen(seed + 1, "t")
    t = torch.randint(1, 1001, (B,), generator=g)
    mask = torch.rand(x_0.shape, generator=g) < (t.float().unsqueeze(-1) / 1000)
    return [v.to(DEV) for v in (x_0, segm, tex, t, mask)] + [[v.to(DEV) for v in gt_list]]


def _ref_loss(outs, gt_list, mask, t, loss_type="reweighted_elbo"):
    """the arithmetic of the reference's _train_loss (models/transformer_model.py:232-270) on the 18 logit tensors"""
    ce = 0
    for lg, gt in zip(outs, gt_list):
        ce = ce + F.cross_entropy(lg.permute(0, 2, 1), torch.where(mask, gt, torch.full_like(gt, -1)),
                                  ignore_index=-1, reduction="none").sum(1)
    T = mask.shape[1]
    vb = ce / t / (1.0 / 1000) / (math.log(2) * T)
    if loss_type == "elbo":
        loss = vb
    elif loss_type == "mlm":
        denom = mask.float().sum(1)
        denom[denom == 0] = 1
        loss = ce / denom
    else:
        loss = (1 - t / 1000) * ce / (math.log(2) * T)
    return loss.mean(), vb.mean()


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _grad_errors(named_got, named_want):
    """test_gpu_train._grad_report's rule: error relative to the tensor's max; gradients that vanish in exact
    arithmetic (key.bias) are held to 5 % of the median tensor's scale instead"""
    typical = float(np.median([float(w.abs().max()) for w in named_want.values()]))
    out = {}
    for k, want in named_want.items():
        got = named_got[k]
        assert got is not None, k
        out[k] = float((got.double() - want.double()).abs().max()) / max(float(want.abs().max()), 0.05 * typical)
    return out


# ----------------------------------------------------------------------------- A. the conversion kernels
def _loss_layout_grads(B, T, ncls, nh, seed):
    """the 18 logit gradients as the reference's F.cross_entropy(logits.permute(0, 2, 1), ...) hands them over"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    heads = [(3 * torch.randn(B, T, ncls, device=DEV, generator=g)).requires_grad_(True) for _ in range(nh)]
    tgt = torch.randint(-1, ncls, (nh, B, T), device=DEV, generator=g)
    loss = sum(F.cross_entropy(h.permute(0, 2, 1), tgt[k], ignore_index=-1, reduction="none").sum(1).mean()
               for k, h in enumerate(heads))
    return list(torch.autograd.grad(loss, heads))


@pytest.mark.parametrize("terms", [2, 1])
@pytest.mark.parametrize("B,T,ncls", [(2, 512, 1024), (3, 100, 70), (1, 33, 129), (2, 64, 64)])
def test_head_grads_to_planes_matches_plane_split_of_the_concatenation(B, T, ncls, terms):
    from text2human_b200 import ops
    from text2human_b200.transformer_train import head_grad_scale
    nh = 18
    grads = _loss_layout_grads(B, T, ncls, nh, seed=B * T + ncls)
    if T > 1 and ncls > 1:
        assert all(g.stride() == (T * ncls, 1, T) for g in grads), grads[0].stride()   # class-major, as measured
    wide = torch.randn(B, T, 2 * ncls, device=DEV)
    layouts = {
        "loss": grads,
        "contiguous": [g.contiguous() for g in grads],
        "mixed": [g if k % 3 == 0 else g.contiguous() if k % 3 == 1 else None for k, g in enumerate(grads)],
        "strided": [(wide * (k + 1))[:, :, :ncls] if k % 2 else g for k, g in enumerate(grads)],
        "null": [None] * (nh - 1) + [grads[-1]],
    }
    for name, heads in layouts.items():
        table, shape = ops.head_grads_table(heads)
        assert shape == (B, T, ncls)
        dense = torch.cat([h if h is not None else torch.zeros(B, T, ncls, device=DEV) for h in heads], -1)
        amax = float(ops.head_grads_absmax(table, shape)[0])
        assert amax == float(dense.abs().max()), name
        for s in (head_grad_scale(amax), 1.0, 2.0 ** -20):
            got = ops.head_grads_to_planes(table, shape, s, terms=terms)
            want = ops.f32_to_planes_rows((s * dense).reshape(B * T, nh * ncls).contiguous(), terms=terms)
            assert got.shape == want.shape and torch.equal(got, want), (name, s)
        assert head_grad_scale(amax) * amax <= 256.0 < 2 * head_grad_scale(amax) * amax


# ----------------------------------------------------------------------------- B. node against the native trainer
def _node_and_native(cfg, B, seed, loss_type="reweighted_elbo"):
    from text2human_b200.transformer_train import SamplerTrainer, targets_from_gt_list
    net_n, _ = _make(cfg, seed)
    net_d, _ = _make(cfg, seed)
    x_0, segm, tex, t, mask, gt_list = _batch(cfg, seed + 1, B)
    tr = SamplerTrainer(net_n, loss_type=loss_type)
    loss_n, vb_n = tr.loss_and_grads(x_0, targets_from_gt_list(gt_list), segm, tex, t, mask=mask)
    want = {k: p.grad / tr.loss_scale for k, p in net_n.named_parameters()}
    x_t = torch.where(mask, torch.full_like(x_0, cfg["codebook_size"]), x_0)
    net_d.train()
    outs = net_d(x_t, segm, tex, t=t)
    assert len(outs) == cfg["num_head"] and outs[0].shape == (B, cfg["block_size"], cfg["codebook_size"] // 18)
    with torch.no_grad():
        ref = net_d.forward_logits(x_t, segm, tex)
    out_err = _rel(torch.stack(outs, 2).detach(), ref)
    loss, vb = _ref_loss(outs, gt_list, mask, t, loss_type)
    loss.backward()
    assert net_d.start_tok.grad is None
    got = {k: p.grad for k, p in net_d.named_parameters() if k != "start_tok"}
    want.pop("start_tok")
    return dict(loss=(float(loss), float(loss_n)), vb=(float(vb), float(vb_n)), out_err=out_err,
                errs=_grad_errors(got, want))


# fp16 mode (one fp16 plane per operand): the node and the native trainer apply different power-of-two loss scales,
# so the fp16 roundings of every gradient operand differ.  Measured on an H100 80 GB: worst per-tensor gradient
# error 4.0e-4 (blocks.0.mlp.0.weight); the node's logits against forward_logits (fused attention, split-K
# projections: other rounding points) 3.2e-4.  Bounds at about 2.5x.
FP16_BOUND = 1e-3
FP16_OUT_BOUND = 1e-3


@pytest.mark.parametrize("mode", ["fp32", "fp16"])
def test_node_matches_native_trainer_at_real_widths(mode):
    from text2human_b200 import ops
    ops.set_precision(mode)
    r = _node_and_native(REAL, B=2, seed=301)
    worst = max(r["errs"].values())
    print(f"[dropin] {mode}: node vs native worst gradient rel err {worst:.2e} "
          f"({max(r['errs'], key=r['errs'].get)}), outputs vs forward_logits {r['out_err']:.1e}")
    assert r["out_err"] <= (1e-5 if mode == "fp32" else FP16_OUT_BOUND)
    for a, b in (r["loss"], r["vb"]):
        assert abs(a - b) <= (1e-4 if mode == "fp32" else 2e-3) * abs(b)
    assert worst <= (1e-4 if mode == "fp32" else FP16_BOUND), r["errs"]


def test_node_and_native_run_the_same_backward_launches():
    """below the logits, the node and the native trainer issue the same library calls in the same order"""
    from text2human_b200 import _lib
    from text2human_b200.transformer_train import SamplerTrainer, targets_from_gt_list
    calls, real_load = [], _lib.load

    class Rec:
        def __init__(self, lib):
            self.lib = lib

        def __getattr__(self, name):
            calls.append(name)
            return getattr(self.lib, name)

    cfg = MID
    x_0, segm, tex, t, mask, gt_list = _batch(cfg, 7, 2)
    net_n, _ = _make(cfg, 5)
    tr = SamplerTrainer(net_n)
    net_d, _ = _make(cfg, 5)
    x_t = torch.where(mask, torch.full_like(x_0, cfg["codebook_size"]), x_0)
    _lib.load = lambda: Rec(real_load())
    try:
        tr.loss_and_grads(x_0, targets_from_gt_list(gt_list), segm, tex, t, mask=mask)
        native = list(calls)
        calls.clear()
        outs = net_d(x_t, segm, tex)
        loss, _ = _ref_loss(outs, gt_list, mask, t)
        calls.clear()
        loss.backward()
        node = list(calls)
    finally:
        _lib.load = real_load
    tail = native[native.index("t2h_ce_heads") + 2:]          # after the loss kernel and the dlogits conversion
    assert node[:2] == ["t2h_head_grads_absmax", "t2h_head_grads_to_planes"]
    assert node[2:] == tail


BEFORE = os.path.join(os.path.dirname(__file__), "golden", "sampler_native_before_shared_backward.npz")


def test_native_step_unchanged_by_the_shared_backward():
    """SamplerTrainer.loss_and_grads against its own output recorded (on an H100) before its backward became
    transformer_train.backward_from_planes, on test_gpu_train's reference-fixture inputs: loss and vb_loss bit for
    bit, every gradient within 1e-6 of its tensor's max.  The gradients cannot be held bit for bit: the backward sums
    with fp32 atomics (split-K weight gradients, column, LayerNorm-parameter and embedding sums), and two runs of the
    same code differ by up to 1.5e-7 there.  A gradient landing in another parameter's slot would be off by O(1)."""
    from text2human_b200.transformer_train import SamplerTrainer, targets_from_gt_list
    gold, before = np.load(os.path.join(os.path.dirname(__file__), "golden", "sampler_train.npz")), np.load(BEFORE)
    net, _ = _make(R.TINY_TRANSFORMER, 71)
    x_0, gt_list, segm, tex = [t.to(DEV) if torch.is_tensor(t) else [g.to(DEV) for g in t]
                               for t in R.sampler_train_batch(72)]
    tr = SamplerTrainer(net)
    loss, vb = tr.loss_and_grads(x_0, targets_from_gt_list(gt_list), segm, tex, torch.from_numpy(gold["t"]).to(DEV),
                                 mask=torch.from_numpy(gold["mask"]).to(DEV))
    assert tr.loss_scale == float(before["loss_scale"])
    assert np.float32(float(loss)) == before["loss"] and np.float32(float(vb)) == before["vb_loss"]
    errs = _grad_errors({k: p.grad for k, p in net.named_parameters()},
                        {k: torch.from_numpy(before["grad/" + k]).to(DEV) for k, _ in net.named_parameters()})
    assert max(errs.values()) <= 1e-6, errs


# ----------------------------------------------------------------------------- D. replay, lifetime, weight caches
def test_replay_release_and_weight_caches_after_torch_adam():
    cfg = MID
    net, _ = _make(cfg, 11)
    x_0, segm, tex, t, mask, gt_list = _batch(cfg, 12, 2)
    x_t = torch.where(mask, torch.full_like(x_0, cfg["codebook_size"]), x_0)
    params = [p for n, p in net.named_parameters() if n != "start_tok"]
    # one step first, so that the baseline is taken in steady state
    _ref_loss(net(x_t, segm, tex), gt_list, mask, t)[0].backward()
    for p in params:
        p.grad = None
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    outs = net(x_t, segm, tex)
    loss = _ref_loss(outs, gt_list, mask, t)[0]
    g1 = torch.autograd.grad(loss, params, retain_graph=True)
    g2 = torch.autograd.grad(loss, params, retain_graph=True)
    loss.backward()
    # the backward reduces with fp32 atomics (split-K weight gradients, column and LayerNorm parameter sums), so two
    # passes agree to the arrival order of those sums: rounding level
    names = [n for n, _ in net.named_parameters() if n != "start_tok"]
    first = dict(zip(names, g1))
    for again in (dict(zip(names, g2)), {n: p.grad for n, p in zip(names, params)}):
        errs = _grad_errors(again, first)
        assert max(errs.values()) <= 1e-6, errs
    assert net.start_tok.grad is None
    # a .grad a caller still holds is not written by the next backward
    held = [p.grad for p in params]
    snap = [h.clone() for h in held]
    for p in params:
        p.grad = None
    outs2 = net(x_t, segm, tex)
    _ref_loss(outs2, gt_list, mask, t)[0].backward()
    assert all(torch.equal(h, s) for h, s in zip(held, snap))
    del outs, outs2, loss, g1, g2, first, again, errs, held, snap
    for p in params:
        p.grad = None
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == mem0
    # torch.optim.Adam steps the parameters in place: the eval path must see the new weights with no extra call
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    net.eval()
    with torch.no_grad():
        before = torch.stack(net(x_t, segm, tex))
    net.train()
    _ref_loss(net(x_t, segm, tex), gt_list, mask, t)[0].backward()
    opt.step()
    net.eval()
    with torch.no_grad():
        after = torch.stack(net(x_t, segm, tex))
    from oracle import transformer_ref as TR
    sd1 = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    want = torch.stack(TR.transformer_logits(sd1, x_t.cpu(), segm.cpu(), tex.cpu(), cfg["bert_n_head"]))
    assert not torch.equal(before, after)
    assert _rel(after.cpu(), want) < 1e-4


# ----------------------------------------------------------------------------- E. dropout guard
@pytest.mark.parametrize("which", ["embd_pdrop", "resid_pdrop", "attn_pdrop"])
def test_dropout_guard_raises_before_any_launch(which):
    from text2human_b200 import ops
    cfg = dict(MID, **{which: 0.1})
    net, _ = _make(cfg, 21)
    x_0, segm, tex, t, mask, gt_list = _batch(cfg, 22, 2)
    n0 = ops.COUNTERS["launches"]
    with pytest.raises(NotImplementedError):
        net(x_0, segm, tex)
    assert ops.COUNTERS["launches"] == n0
    with torch.no_grad():
        a = torch.stack(net(x_0, segm, tex))
    net.eval()
    b = torch.stack(net(x_0, segm, tex))
    assert torch.equal(a, b) and not b.requires_grad


# ----------------------------------------------------------------------------- C. the reference wrapper, unmodified
def _loader():
    from oracle import ref_loader as RL
    if not RL.available():
        pytest.skip("reference sources not staged (run oracle/make_ref.py in the build container)")
    return RL


def _vae_checkpoints(tmp_path):
    """tiny image / segm VAE checkpoints whose 64x32 inputs give the transformer's 8x4 latent; 1024 entries per
    texture codebook, so that every index the sampler draws decodes"""
    from text2human_b200 import vqgan_arch as va
    e = R.TINY_VQGAN_TRAIN["enc"]
    img = dict(encoder=va.Encoder(**e), decoder=va.Decoder(**R.TINY_VQGAN_TRAIN["dec"]),
               quantize=va.VectorQuantizerTexture(1024, 32, beta=0.25), quant_conv=torch.nn.Conv2d(32, 32, 1),
               post_quant_conv=torch.nn.Conv2d(32, 32, 1))
    ck = {}
    for i, (k, mod) in enumerate(img.items()):
        ck[k] = R.fill_state_dict(R.spec_of(mod), 401 + i)
    cb = R.codebooks(406, 18, 1024, 32, "trained")
    ck["quantize"] = {f"embedding_list.{k}.weight": cb[k] for k in range(18)}
    torch.save(ck, tmp_path / "img.pth")
    se = dict(e, in_channels=24, z_channels=16)
    seg = dict(encoder=va.Encoder(**se), quantize=va.VectorQuantizer(32, 16, beta=0.25, sane_index_shape=True),
               quant_conv=torch.nn.Conv2d(16, 16, 1))
    sck = {k: R.fill_state_dict(R.spec_of(mod), 411 + i) for i, (k, mod) in enumerate(seg.items())}
    sck["quantize"] = {"embedding.weight": R.codebooks(414, 1, 32, 16, "trained")[0]}
    torch.save(sck, tmp_path / "segm.pth")
    e = R.TINY_VQGAN_TRAIN["enc"]
    return dict(img_ch=e["ch"], img_num_res_blocks=e["num_res_blocks"], img_attn_resolutions=e["attn_resolutions"],
                img_ch_mult=e["ch_mult"], img_in_channels=3, img_resolution=e["resolution"], img_z_channels=32,
                img_double_z=False, img_dropout=0.0, img_n_embed=1024, img_embed_dim=32, img_out_ch=3,
                img_ae_path=str(tmp_path / "img.pth"),
                segm_ch=e["ch"], segm_num_res_blocks=e["num_res_blocks"], segm_attn_resolutions=e["attn_resolutions"],
                segm_ch_mult=e["ch_mult"], segm_in_channels=24, segm_resolution=e["resolution"], segm_z_channels=16,
                segm_double_z=False, segm_dropout=0.0, segm_n_embed=32, segm_embed_dim=16,
                segm_num_segm_classes=24, segm_ae_path=str(tmp_path / "segm.pth"))


def _wrapper(ns, opt, sd):
    with contextlib.redirect_stdout(io.StringIO()):
        w = ns.transformer_model.TransformerTextureAwareModel(opt)
    w._denoise_fn.load_state_dict({k: v.to(DEV) for k, v in sd.items()}, strict=True)
    return w


@pytest.mark.parametrize("loss_type", ["reweighted_elbo", "elbo", "mlm"])
@pytest.mark.parametrize("shape", ["tiny", "mid"])
def test_reference_sampler_wrapper_runs_unmodified_on_the_mirrors(cuda, tmp_path, loss_type, shape):
    RL = _loader()
    tcfg = dict(R.TINY_TRANSFORMER, codebook_size=18 * 1024)
    if shape == "mid":
        tcfg.update(bert_n_emb=256, bert_n_layers=4, bert_n_head=8)
    opt = dict(_vae_checkpoints(tmp_path), **{k: v for k, v in tcfg.items()}, loss_type=loss_type,
               mask_schedule="random", sample_steps=4, is_train=True, lr=1e-3, weight_decay=0)
    from text2human_b200.transformer_arch import TransformerMultiHead
    sd = R.fill_state_dict(R.spec_of(TransformerMultiHead(**tcfg)), 421)
    ns_m = RL.install("mirror", wrappers=("transformer_model",))
    wm = _wrapper(ns_m, opt, sd)
    assert isinstance(wm._denoise_fn, TransformerMultiHead)
    ns_r = RL.install("reference", wrappers=("transformer_model",))
    wr = _wrapper(ns_r, opt, sd)
    B = 2
    data = dict(image=R.image(422, B, 3, 64, 32), segm=R.blocky_mask(423, B, 64, 32, 8, n_ids=24),
                texture_mask=R.blocky_mask(424, B, 64, 32, 8), img_name=["a.png", "b.png"])
    wm.feed_data(data)
    wr.feed_data(data)
    agree = float((wm.input_indices == wr.input_indices).float().mean())
    print(f"[dropin] tokenizers on the mirrors vs the reference: {100 * agree:.2f} % of image tokens identical")
    # the transformer comparison starts from the same tokens
    wr.input_indices, wr.gt_indices_list = wm.input_indices.clone(), [g.clone() for g in wm.gt_indices_list]
    wr.segm_tokens, wr.texture_tokens = wm.segm_tokens.clone(), wm.texture_tokens.clone()
    prev_grads = None
    for step in range(2):
        snap = [{k: p.detach().clone() for k, p in w._denoise_fn.named_parameters()} for w in (wm, wr)]
        for w in (wm, wr):
            torch.manual_seed(431 + step)
            w.optimize_parameters()
        for k in ("loss", "vb_loss"):
            a, b = float(wm.log_dict[k]), float(wr.log_dict[k])
            assert abs(a - b) <= 1e-4 * abs(b), (step, k, a, b)
        pm, pr = dict(wm._denoise_fn.named_parameters()), dict(wr._denoise_fn.named_parameters())
        assert pm["start_tok"].grad is None and pr["start_tok"].grad is None
        want = {k: p.grad.clone() for k, p in pr.items() if p.grad is not None}
        errs = _grad_errors({k: pm[k].grad for k in want}, want)
        assert max(errs.values()) <= 1e-3, (step, errs)
        # each Adam step's parameter moves agree where a gradient exists.  The first step uses test_gpu_train's rule.
        # From the second step on Adam divides by the gradient's history, so an element whose gradient is small
        # against its tensor's max in either step moves by up to ~lr on a gradient difference inside the 1e-3
        # tolerance: there the elements compared are those at >= 10 % of their tensor's max in both steps, in
        # tensors whose gradient does not vanish in exact arithmetic (key.bias: rounding noise in both builds).
        typical = float(np.median([float(g.abs().max()) for g in want.values()]))
        for k, g in want.items():
            g = g.abs()
            if step == 0:
                sel = (g > 1e-3 * g.max()) & (g > 1e-4 * typical)
            else:
                gp = prev_grads[k].abs()
                sel = (g > 0.1 * g.max()) & (gp > 0.1 * gp.max()) & (g.max() >= 0.05 * typical)
            if sel.any():
                d = (pm[k].detach() - snap[0][k]) - (pr[k].detach() - snap[1][k])
                assert float(d[sel].abs().max()) <= 0.02 * opt["lr"], (step, k, float(d[sel].abs().max()))
        prev_grads = want
    assert not wm._denoise_fn.training
    with torch.no_grad():
        lm = torch.stack(wm._denoise_fn(wm.input_indices, wm.segm_tokens, wm.texture_tokens))
        lr = torch.stack(wr._denoise_fn(wm.input_indices, wm.segm_tokens, wm.texture_tokens))
    assert _rel(lm, lr) <= 1e-3
    # the validation loop of train_sampler.py: sample_fn + decode_image_indices + get_vis, one file per sample
    out = tmp_path / "val"
    out.mkdir()
    wm.inference([data], str(out))
    assert sorted(p.name for p in out.iterdir()) == ["a.png", "b.png"]
