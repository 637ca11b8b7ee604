"""GPU checks of the hierarchical VQGAN's bottom-level training step (HierarchyVQGANTrainer): the patch quantizer
backward against fp64, AttnL at 2048 tokens against fp64 autograd, the whole step against the fixture recorded from
the REAL reference `training_step` + `loss.backward()` + `d_loss.backward()` (oracle/make_golden_vqgan_bottom_train.py)
and, at real widths, against the fp64 restatement; the fp16 mode, frozen tensors and fix_decoder, Adam,
micro-batches, resume, the checkpoint layout, input validation and two NCCL ranks."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import vqgan_bottom_train_recipes as BR
from test_gpu_vqgan_train import _check_grads, recorded_draws

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "vqgan_bottom_train.npz")


# ---------------------------------------------------------------- the patch quantizer backward
def _vq_bwd_fp64(z, cb, idx, book, dzq, coef_z, coef_e, ps):
    B, Hz, Wz, Cz = z.shape
    nb, ne, D = cb.shape
    rows = F.unfold(z.double().permute(0, 3, 1, 2), (ps, ps), stride=ps).permute(0, 2, 1).reshape(-1, D)
    b, i = book.reshape(-1).long(), idx.reshape(-1)
    ok = (b >= 0) & (b < nb) & (i >= 0) & (i < ne)
    e = torch.zeros_like(rows)
    e[ok] = cb.double()[b[ok], i[ok]]
    drow = coef_z * (rows - e)
    dz = F.fold(drow.view(B, -1, D).permute(0, 2, 1), (Hz, Wz), kernel_size=(ps, ps), stride=ps)
    dz = dz.permute(0, 2, 3, 1) + dzq.double()
    terms = coef_e * (e - rows)
    dcb = torch.zeros((nb, ne, D), dtype=torch.float64, device=z.device)
    mag = torch.zeros_like(dcb)
    cnt = torch.zeros((nb, ne, 1), dtype=torch.float64, device=z.device)
    dcb.index_put_((b[ok], i[ok]), terms[ok], accumulate=True)
    mag.index_put_((b[ok], i[ok]), terms[ok].abs(), accumulate=True)
    cnt.index_put_((b[ok], i[ok]), torch.ones_like(terms[ok][:, :1]), accumulate=True)
    dz_mag = dzq.double().abs() + coef_z * F.fold((rows.abs() + e.abs()).view(B, -1, D).permute(0, 2, 1), (Hz, Wz),
                                                  kernel_size=(ps, ps), stride=ps).permute(0, 2, 3, 1)
    return dz, dcb, dz_mag, mag, cnt


# (B, Hz, Wz, Cz, ps, n_e, case): the real bottom quantizer is [B*512 rows, 1024] x 18 x 512
VQ_CASES = [(4, 64, 32, 256, 2, 512, "real"), (2, 8, 4, 32, 2, 64, "tiny"), (3, 16, 12, 16, 2, 40, "outside_ids"),
            (2, 32, 16, 64, 2, 128, "repeated_codes"), (2, 8, 8, 64, 1, 96, "ps1")]


@pytest.mark.parametrize("case", VQ_CASES, ids=[c[-1] for c in VQ_CASES])
def test_vq_bwd_patch_matches_fp64(cuda, case):
    from text2human_b200 import ops
    B, Hz, Wz, Cz, ps, ne, kind = case
    g = torch.Generator().manual_seed(sum(map(ord, kind)))
    Hp, Wp = Hz // ps, Wz // ps
    z = torch.randn(B, Hz, Wz, Cz, generator=g)
    dzq = torch.randn(B, Hz, Wz, Cz, generator=g) * 1e-3
    cb = torch.randn(18, ne, Cz * ps * ps, generator=g)
    book = torch.randint(0, 18, (B, Hp, Wp), generator=g, dtype=torch.int32)
    idx = torch.randint(0, ne, (B, Hp, Wp), generator=g)
    if kind == "outside_ids":
        book[:, ::3] = torch.tensor([-1, 18, 25], dtype=torch.int32)[torch.randint(0, 3, book[:, ::3].shape, generator=g)]
    if kind == "repeated_codes":
        book[:] = 2
        idx = torch.randint(0, 3, (B, Hp, Wp), generator=g)
    coef_z, coef_e = 2.0 / z.numel() * 4096, 0.5 / z.numel() * 4096
    dcb0 = torch.randn(cb.shape, generator=g) * 1e-3                 # gradients accumulate into the buffer
    zc, cbc, ic, bc, dqc = (t.to(cuda) for t in (z, cb, idx, book, dzq))
    outs = []
    for _ in range(2):
        dcb = dcb0.to(cuda)
        dz = ops.vq_bwd_patch(zc, cbc, ic, bc, dqc, dcb, coef_z, coef_e, ps=ps)
        outs.append((dz, dcb))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "reruns differ"
    dz, dcb = outs[0]
    wdz, wdcb, dz_mag, mag, cnt = _vq_bwd_fp64(zc, cbc, ic, bc, dqc, coef_z, coef_e, ps)
    wdcb = wdcb + dcb0.to(cuda).double()
    assert float(((dz.double() - wdz).abs() - 4e-7 * dz_mag).max()) <= 1e-30
    bound = 1.2e-7 * (cnt + 2) * (mag + dcb0.to(cuda).double().abs()) + 1e-30
    assert bool(((dcb.double() - wdcb).abs() <= bound).all()), float(((dcb.double() - wdcb).abs() / bound).max())
    untouched = (cnt == 0).expand_as(dcb)
    assert torch.equal(dcb[untouched], dcb0.to(cuda)[untouched])     # codes no row chose are left bit for bit


# ---------------------------------------------------------------- AttnL at 2048 tokens
def test_attn_layer_at_2048_tokens_matches_fp64(cuda):
    """the bottom encoder's and DecoderRes's AttnBlock at 64 x 32 tokens, 512 channels: output, input gradient and
    every parameter gradient against fp64 autograd of oracle.vqgan_ref.attn_block"""
    from oracle import vqgan_ref
    from text2human_b200 import ops
    from text2human_b200.flat_params import ParamSpace
    from text2human_b200.train_layers import Grad
    from text2human_b200.vqgan_arch import AttnBlock
    from text2human_b200.vqgan_train import Act, AttnL
    ops.set_precision("fp32")
    C, H, W, N = 512, 64, 32, 2
    blk = AttnBlock(C)
    blk.load_state_dict(R.fill_state_dict(R.spec_of(blk), 41), strict=True)
    sd = {k: v.double().to(cuda).requires_grad_(True) for k, v in blk.state_dict().items()}
    blk = blk.to(cuda)

    class Host:
        def space_of(self, m):
            return sp

        def space_of_param(self, p):
            return sp
    sp = ParamSpace([blk.proj_out, (blk.q, blk.k, blk.v), blk.norm], cuda)
    layer = AttnL(Host(), blk)
    x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(3)).to(cuda)
    dy = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(4)).to(cuda)
    sp.prepare(ops.get_terms())
    y = layer.fwd(Act(x.permute(0, 2, 3, 1).contiguous()))
    dx = layer.bwd(Grad(dy.permute(0, 2, 3, 1).contiguous())).g
    xd = x.double().requires_grad_(True)
    yd = vqgan_ref.attn_block(sd, "", xd)
    yd.backward(dy.double())
    errs = {"y": float((y.x.permute(0, 3, 1, 2) - yd).abs().max() / yd.abs().max()),
            "dx": float((dx.permute(0, 3, 1, 2) - xd.grad).abs().max() / xd.grad.abs().max())}
    top = max(float(sd[k].grad.abs().max()) for k, _ in blk.named_parameters())
    for k, p in blk.named_parameters():
        want = sd[k].grad
        err = float((sp.g(p).reshape(want.shape) - want).abs().max())
        # the key bias's gradient is zero in exact arithmetic (softmax is invariant to it): what is left is the
        # cancellation residue of a sum over 2048 tokens, held to 1e-6 of the largest parameter gradient
        errs[k] = err / top * 1e3 if k == "k.bias" else err / float(want.abs().max())
    print(f"[AttnL 2048 tokens x 512] {errs}")
    assert max(errs.values()) < 1e-3, errs


# ---------------------------------------------------------------- the whole step
def build(cuda, **kw):
    from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer
    m, disc = BR.modules()
    m, disc = m.to(cuda), disc.to(cuda)
    kw.setdefault("disc_start_step", BR.DISC_START_STEP)
    return m, disc, HierarchyVQGANTrainer(m, disc, **kw)


def named_gen(m):
    out = {}
    for net in ("bot_encoder", "bot_decoder_res", "bot_quant_conv", "bot_post_quant_conv", "bot_quantize", "decoder"):
        for k, p in getattr(m, net).named_parameters():
            out[f"{net}.{k}"] = p
    return out


def test_step_matches_reference_fixture(cuda):
    from text2human_b200 import ops
    gold = np.load(GOLD)
    ops.set_precision("fp32")
    m, disc, tr = build(cuda)
    tr.aug_draw_fn = recorded_draws(BR.AUG_SEED)
    tr.training_step(BR.batch(), BR.STEP)
    torch.cuda.synchronize()
    got = tr.losses()
    for k in ("nll_loss", "g_loss", "codebook_loss", "d_weight", "loss", "d_loss"):
        assert abs(got[k] - float(gold[k])) <= 2e-4 * max(1.0, abs(float(gold[k]))), (k, got[k], float(gold[k]))
    assert np.array_equal(tr.bot_idx.reshape(-1).cpu().numpy(), gold["bot_idx"])
    worst_g, n_g = _check_grads(gold, "g", named_gen(m), tr.loss_scale, 1e-3)
    worst_d, n_d = _check_grads(gold, "d", dict(disc.named_parameters()), tr.disc_scale, 1e-3)
    print(f"[vqgan bottom train fp32] {n_g} generator / {n_d} discriminator gradient tensors, worst rel err "
          f"{worst_g:.2e} / {worst_d:.2e}; losses {got}")
    assert n_g > 150 and n_d >= 10


def test_fp16_mode_tracks_fp32(cuda):
    from text2human_b200 import ops
    res = {}
    try:
        for mode in ("fp32", "fp16"):
            ops.set_precision(mode)
            m, disc, tr = build(cuda)
            tr.aug_draw_fn = recorded_draws(BR.AUG_SEED)
            tr.training_step(BR.batch(), BR.STEP)
            res[mode] = (tr.losses(), tr.gen.flat_g.clone() / tr.loss_scale, tr.dsc.flat_g.clone() / tr.disc_scale)
    finally:
        ops.set_precision("fp32")
    (l32, g32, d32), (l16, g16, d16) = res["fp32"], res["fp16"]
    for k in ("nll_loss", "g_loss", "codebook_loss", "loss", "d_loss"):
        assert abs(l16[k] - l32[k]) <= 2e-2 * max(1.0, abs(l32[k])), (k, l16[k], l32[k])
    cg = float(F.cosine_similarity(g16.double(), g32.double(), dim=0))
    cd = float(F.cosine_similarity(d16.double(), d32.double(), dim=0))
    print(f"[vqgan bottom train fp16 vs fp32] gradient cosine generator {cg:.5f} discriminator {cd:.5f}")
    assert cg > 0.98 and cd > 0.98


def test_frozen_tensors_fix_decoder_and_adam(cuda):
    """three Adam steps leave the top nets, the never-stepped decoder tensors and (fix_decoder) the whole decoder
    bitwise unchanged; the bottom gradients do not depend on fix_decoder; one step equals torch.optim.Adam"""
    from text2human_b200 import ops
    ops.set_precision("fp32")
    bot_g = {}
    for run, fix in enumerate((False, True, False)):
        m, disc, tr = build(cuda, fix_decoder=fix)
        before = {n: p.detach().clone() for n, p in m.named_parameters()}
        for s in range(3):
            tr.aug_draw_fn = recorded_draws(BR.AUG_SEED + s)
            tr.training_step(BR.batch(), BR.STEP)
            if s == 0:
                bot_g[run] = {n: p.grad.detach().clone() / tr.loss_scale for n, p in named_gen(m).items()
                              if n.startswith("bot_")}
                p0 = tr.gen.flat_p.clone()
                ref_p = p0.clone().requires_grad_(True)
                opt = torch.optim.Adam([ref_p], lr=tr.lr)
                ref_p.grad = tr.gen.flat_g.clone() / (tr.n_micro * tr.loss_scale)
                opt.step()
                tr.adam_step()
                assert float((tr.gen.flat_p - ref_p.detach()).abs().max()) < 2e-7
            else:
                tr.adam_step()
        torch.cuda.synchronize()
        n_moved = 0
        for n, p in m.named_parameters():
            frozen = not BR.stepped(n) or (fix and n.startswith("decoder."))
            same = torch.equal(p.detach(), before[n])
            assert same or not frozen, (fix, n)     # (a stepped codebook no position selects stays put too)
            n_moved += not same
        assert n_moved > 100
    # the whole bottom gradient, relative in norm; the split weight-gradient reductions add in a run-dependent order,
    # so two runs of the same step (0 and 2) set the noise level the fix_decoder run (1) is held to
    def rel(i, j):
        a = torch.cat([g.reshape(-1) for g in bot_g[i].values()]).double()
        b = torch.cat([bot_g[j][n].reshape(-1) for n in bot_g[i]]).double()
        return float((b - a).norm() / a.norm())
    worst, noise = rel(0, 1), rel(0, 2)
    print(f"[fix_decoder] bottom gradient difference {worst:.2e}, run-to-run {noise:.2e}")
    assert worst <= max(1e-6, 4 * noise) and worst < 1e-5, (worst, noise)


def test_micro_batches_resume_and_checkpoint(cuda, tmp_path):
    from oracle import vqgan_ref
    from text2human_b200 import ops
    from text2human_b200.vqgan_arch import Discriminator
    ops.set_precision("fp32")
    data = BR.batch()
    x, mask = data["image"].to(cuda), data["texture_mask"].to(cuda)
    m, disc, tr = build(cuda, micro_batch=1, lr=1e-3)
    dec0, _ = m.forward_step(x, mask)
    tr.aug_draw_fn = recorded_draws(5)
    tr.training_step(data, 3)
    g_both = tr.gen.flat_g.clone()
    tr.micro_batch = None
    tr.aug_draw_fn = recorded_draws(5)
    gsum = torch.zeros_like(g_both)
    for i in range(2):
        tr.training_step({k: v[i:i + 1] for k, v in data.items()}, 3)
        gsum += tr.gen.flat_g
    assert float((g_both - gsum).abs().max() / gsum.abs().max()) < 1e-4
    # save -> load -> identical optimiser state and next step
    tr.micro_batch = 1
    tr.aug_draw_fn = recorded_draws(6)
    tr.optimize_parameters(data, 3)
    path = os.path.join(tmp_path, "bot.pth")
    tr.save(path)
    ck = torch.load(path, map_location=cuda)
    assert set(ck) == {"bot_encoder", "bot_decoder_res", "decoder", "bot_quantize", "bot_quant_conv",
                       "bot_post_quant_conv", "discriminator", "optimizer"}
    tr.aug_draw_fn = recorded_draws(7)
    tr.optimize_parameters(data, 4)
    want = tr.gen.flat_p.clone()
    m2, disc2, tr2 = build(cuda, micro_batch=1, lr=1e-3)
    tr2.load(path)
    for sp2, key in ((tr2.gen, "gen"), (tr2.dsc, "disc")):
        assert torch.equal(sp2.flat_m, ck["optimizer"][key]["flat_m"]) and sp2.step_count == 1
    tr2.aug_draw_fn = recorded_draws(7)
    tr2.optimize_parameters(data, 4)
    dev_ = (tr2.gen.flat_p - want).abs()
    assert float(dev_.max()) <= 2.5 * tr.lr and float((dev_ > 1e-6).float().mean()) < 0.01
    # the checkpoint loads strict=True into fresh mirrors, and the inference path sees the stepped weights
    fresh, _ = BR.modules()
    for k in ("bot_encoder", "bot_decoder_res", "decoder", "bot_quantize", "bot_quant_conv", "bot_post_quant_conv"):
        getattr(fresh, k).load_state_dict(ck[k], strict=True)
    with contextlib.redirect_stdout(io.StringIO()):
        Discriminator(3, BR.NDF, n_layers=BR.DISC_LAYERS).load_state_dict(ck["discriminator"], strict=True)
    dec, _ = m.forward_step(x, mask)
    sd = {f"{n}.{k}": v.detach() for n in ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv",
                                           "bot_encoder", "bot_decoder_res", "bot_quant_conv", "bot_post_quant_conv")
          for k, v in getattr(m, n).state_dict().items()}
    top = torch.stack([e.weight.detach() for e in m.top_quantize.embedding_list])
    bot = torch.stack([e.weight.detach() for e in m.bot_quantize.embedding_list])
    with torch.no_grad():
        want_dec = vqgan_ref.hierarchy_forward_step(sd, top, bot, x, mask)["dec"]
    err = float((dec - want_dec).abs().max() / want_dec.abs().max())
    moved = float((dec - dec0).abs().max() / want_dec.abs().max())
    assert err < 1e-3 and moved > 10 * err, (err, moved)       # forward_step sees the stepped weights


def test_invalid_inputs_raise_before_any_launch(cuda):
    from text2human_b200 import ops
    m, disc, tr = build(cuda)
    x = torch.zeros(1, 3, 64, 32)
    for data in (dict(image=torch.zeros(1, 3, 56, 32), texture_mask=torch.zeros(1, 1, 56, 32)),
                 dict(image=torch.zeros(1, 3, 64, 40), texture_mask=torch.zeros(1, 1, 64, 40)),
                 dict(image=x, texture_mask=torch.zeros(1, 1, 32, 16)),
                 dict(image=x, texture_mask=torch.zeros(2, 1, 64, 32))):
        n0 = ops.COUNTERS["launches"]
        with pytest.raises(ValueError):
            tr.training_step(data, 2)
        assert ops.COUNTERS["launches"] == n0


# ---------------------------------------------------------------- real widths
def test_real_width_step_against_fp64_restatement(cuda, monkeypatch):
    """configs/vqvae_bottom.yml widths, B = 1, 512 x 256: the native fp32 step and the fp32 restatement, each against
    the fp64 restatement on the GPU.  The generator's gradient through the discriminator is discontinuous at its
    LeakyReLU kinks, some of which lie within rounding of a pre-activation at this size: both restatements take the
    native step's own masks (recorded first), as test_gpu_vqgan_train_widths does."""
    from test_gpu_vqgan_train_widths import disc_masks, record_disc_passes
    from oracle import vqgan_bottom_train_ref as BT
    from text2human_b200 import ops
    from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
    from text2human_b200.vqgan_arch import Discriminator
    from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    ops.set_precision("fp32")
    opt = dict(BR.OPT, embed_dim=256, bot_n_embed=512, bot_z_channels=256, bot_resolution=512, bot_ch=128,
               bot_num_res_blocks=2, bot_attn_resolutions=[64], top_z_channels=256, top_resolution=512, top_ch=128,
               top_num_res_blocks=2, top_attn_resolutions=[32])
    with contextlib.redirect_stdout(io.StringIO()):
        m = HierarchyVQSpatialTextureAwareModel(opt)
    seeds = dict(BR.SEEDS)
    for name in ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv", "bot_encoder", "bot_decoder_res",
                 "bot_quant_conv", "bot_post_quant_conv"):
        getattr(m, name).load_state_dict(R.fill_state_dict(R.spec_of(getattr(m, name)), seeds[name]), strict=True)
    for q, key, ne, d in ((m.top_quantize, "top_books", 1024, 256), (m.bot_quantize, "bot_books", 512, 1024)):
        cb = R.codebooks(seeds[key], 18, ne, d, "trained")
        for k, e in enumerate(q.embedding_list):
            e.weight.data.copy_(cb[k])
    disc = Discriminator(3, 64, n_layers=3)
    disc.load_state_dict(R.fill_state_dict(R.spec_of(disc), seeds["disc"]), strict=True)
    x, mask = R.image(11, 1, 3, 512, 256), R.blocky_mask(12, 1, 512, 256, 32)
    passes = record_disc_passes(monkeypatch)
    tr = HierarchyVQGANTrainer(m.to(cuda), disc.to(cuda), disc_start_step=1, diff_aug=False)
    tr.training_step(dict(image=x, texture_mask=mask), BR.STEP)
    torch.cuda.synchronize()
    got = tr.losses()
    masks = disc_masks(passes)
    del passes
    ref = {}
    for dt in (torch.float64, torch.float32):
        sd = {f"{n}.{k}": v.detach().to(cuda, dt).clone() for n in
              ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv", "bot_encoder", "bot_decoder_res",
               "bot_quant_conv", "bot_post_quant_conv") for k, v in getattr(m, n).state_dict().items()}
        for k in sd:
            if BR.stepped(k) or k == "decoder.conv_out.weight":
                sd[k].requires_grad_(True)
        top = torch.stack([e.weight.detach() for e in m.top_quantize.embedding_list]).to(cuda, dt)
        bot = [e.weight.detach().to(cuda, dt).clone().requires_grad_(True) for e in m.bot_quantize.embedding_list]
        sdd = {k: (v.detach().to(cuda, dt).clone().requires_grad_("running" not in k) if v.is_floating_point()
                   else v.detach().to(cuda).clone()) for k, v in disc.state_dict().items()}
        r_ = BT.training_step(sd, top, bot, sdd, x.to(cuda, dt), mask.to(cuda), BR.STEP, disc_start_step=1,
                              diff_aug=False, disc_masks=masks)
        r_["loss"].backward()
        ref[dt] = ({k: float(r_[k]) for k in ("nll_loss", "g_loss", "codebook_loss", "d_weight")},
                   {k: g.detach().double() for k, g in BR.gen_grads(sd, bot).items()}, r_["bot_idx"])
        del sd, sdd, bot, r_
    named = named_gen(m)
    l64, g64, i64 = ref[torch.float64]

    def worst(grads):
        floor = 1e-6 * max(float(g.norm()) for g in g64.values())
        w = (0.0, None)
        for k, g in g64.items():
            if float(g.norm()) > floor:
                e = float((grads[k] - g).norm() / g.norm())
                w = max(w, (e, k))
        return w
    nat = worst({k: named[k].grad.double() / tr.loss_scale for k in g64})
    r32 = worst(ref[torch.float32][1])
    n_idx = int((tr.bot_idx.reshape(-1) != i64).sum())
    print(f"[real widths B=1 512x256] native fp32 worst gradient {nat[0]:.2e} ({nat[1]}); fp32 restatement "
          f"{r32[0]:.2e} ({r32[1]}); bottom indices differing {n_idx}; losses {got} vs fp64 {l64}")
    assert n_idx == 0
    for k in l64:
        assert abs(got[k] - l64[k]) <= 1e-3 * max(1.0, abs(l64[k])), k
    assert nat[0] < 1e-2


# ---------------------------------------------------------------- two ranks
def _nccl_worker(rank, world, port, q):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import vqgan_bottom_train_recipes as BR
    from test_gpu_vqgan_train import recorded_draws
    from text2human_b200 import dist as D
    from text2human_b200 import ops
    from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    D.init("nccl")
    ops.set_precision("fp32")
    m, disc = BR.modules()
    dev = torch.device("cuda", rank)
    tr = HierarchyVQGANTrainer(m.to(dev), disc.to(dev), disc_start_step=BR.DISC_START_STEP)
    tr.aug_draw_fn = recorded_draws(BR.AUG_SEED + rank)
    data = {k: v[rank:rank + 1] for k, v in BR.batch().items()}
    tr.optimize_parameters(data, BR.STEP)
    torch.cuda.synchronize()
    q.put((rank, float(tr.gen.flat_p.double().sum()), float(tr.dsc.flat_p.double().sum())))
    torch.distributed.destroy_process_group()


def test_two_rank_nccl_step():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket

    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert res[0][1:] == res[1][1:]          # the replicas stepped with the same all-reduced gradients
