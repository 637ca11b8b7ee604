"""The hierarchy's bottom level through the reference's own ``HierarchyVQSpatialTextureAwareModel`` (models/
hierarchy_vqgan_model.py, unmodified, built by its own ``__init__``) on the mirrors: ``VectorQuantizerSpatialTextureAware``,
``DecoderRes`` and ``Decoder(z, bot_h)`` as autograd nodes (vqgan_autograd), against the same wrapper on the
reference's arch classes (stock PyTorch) on the same GPU.

The constructor reads ``top_vae_path`` twice (top nets, discriminator): each test writes that checkpoint from
vqgan_bottom_train_recipes.modules() to its tmp_path and loads the bottom nets and codebooks into both wrappers from
the same recipe.
"""
import contextlib
import io
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import vqgan_bottom_train_recipes as BR

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "vqgan_bottom_train.npz")
BOT = ("bot_encoder", "bot_decoder_res", "bot_quantize", "bot_quant_conv", "bot_post_quant_conv")
GEN = BOT + ("decoder",)


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


def opt_for(tmp_path, base=None, **kw):
    o = dict(base or BR.OPT, n_channels=3, ndf=BR.NDF, disc_layers=BR.DISC_LAYERS, perceptual_weight=1.0,
             disc_start_step=BR.DISC_START_STEP, disc_weight_max=1.0, diff_aug=True, fix_decoder=False, lr=1e-4,
             top_vae_path=str(tmp_path / "vqvae_top.pth"))
    o.update(kw)
    return o


def write_top(path, m, disc):
    """the top checkpoint the wrapper's constructor reads: the top nets and the discriminator"""
    torch.save(dict(encoder=m.top_encoder.state_dict(), decoder=m.decoder.state_dict(),
                    quantize=m.top_quantize.state_dict(), quant_conv=m.top_quant_conv.state_dict(),
                    post_quant_conv=m.top_post_quant_conv.state_dict(), discriminator=disc.state_dict()), path)


def wrapper(archs, opt, m):
    """the reference's HierarchyVQSpatialTextureAwareModel built by its own __init__ on ``archs`` ("mirror" /
    "reference"), with the bottom nets and codebooks of ``m``"""
    ns = _loader().install(archs, wrappers=("hierarchy_vqgan_model",))
    with contextlib.redirect_stdout(io.StringIO()):
        w = ns.hierarchy_vqgan_model.HierarchyVQSpatialTextureAwareModel(opt)
    for n in BOT:
        getattr(w, n).load_state_dict(getattr(m, n).state_dict(), strict=True)
    return w


def pair(tmp_path, **kw):
    m, disc = BR.modules()
    opt = opt_for(tmp_path, **kw)
    write_top(opt["top_vae_path"], m, disc)
    wm = wrapper("mirror", opt, m)
    wr = wrapper("reference", opt, m)
    from text2human_b200 import vqgan_arch
    assert isinstance(wm.bot_decoder_res, vqgan_arch.DecoderRes) and not isinstance(wr.decoder, vqgan_arch.Decoder)
    return wm, wr, opt


def kink_free_seed(wr, data, step, seeds=range(31, 71)):
    """DiffAugment draws from the CUDA RNG: scan seeds until the reference run has no discriminator pre-activation
    within 3e-5 of its LeakyReLU kink (the step's gradient is discontinuous there).  The discriminator's BatchNorm
    running statistics the scan moves are restored."""
    keep = {k: v.clone() for k, v in wr.disc.state_dict().items()}
    margins = []
    hooks = [mod.register_forward_pre_hook(lambda m_, inp: margins.append(float(inp[0].detach().abs().min())))
             for mod in wr.disc.main if isinstance(mod, torch.nn.LeakyReLU)]
    best = (0.0, None)
    try:
        for cand in seeds:
            margins.clear()
            torch.manual_seed(cand)
            wr.training_step(data, step)
            best = max(best, (min(margins), cand))
            if best[0] > 1e-4:
                break
    finally:
        for h_ in hooks:
            h_.remove()
        wr.disc.load_state_dict(keep)
    print(f"[bottom drop-in] DiffAugment seed {best[1]}: discriminator pre-activation margin {best[0]:.2e}")
    assert best[0] > 3e-5
    return best[1]


def capture_bot_idx(w):
    """the bottom continual indices of every bot_quantize call (the wrapper itself discards them)"""
    got = []
    h = w.bot_quantize.register_forward_hook(lambda m_, i_, o: got.append(o[2][1].detach().clone()))
    return got, h


def grads(w, nets=GEN + ("disc",)):
    return {f"{n}.{k}": p.grad for n in nets for k, p in getattr(w, n).named_parameters()}


def check_grads(gm, gr, tol=1e-3):
    """every gradient within ``tol`` of its tensor's max; the same tensors are None in both.  Gradients that vanish in
    exact arithmetic (a conv bias in front of a one-channel-per-group GroupNorm) are rounding noise in the reference
    as well: below 1e-6 of the largest gradient of their net group they are held to 1e-5 of it, absolutely."""
    assert gm.keys() == gr.keys()
    for k in gr:
        assert (gm[k] is None) == (gr[k] is None), k
    worst = (0.0, None)
    for grp in ("gen", "disc"):
        keys = [k for k in gr if gr[k] is not None and k.startswith("disc.") == (grp == "disc")]
        gmax = max(float(gr[k].abs().max()) for k in keys)
        for k in keys:
            if float(gr[k].abs().max()) < 1e-6 * gmax:
                assert float((gm[k] - gr[k]).abs().max()) < 1e-5 * gmax, k
                continue
            worst = max(worst, (_rel(gm[k], gr[k]), k))
    assert worst[0] < tol, worst
    return worst


def check_losses(wm, wr, keys=("nll_loss", "g_loss", "codebook_loss"), tol=2e-4):
    for k in keys:
        a, b = float(wm.log_dict[k]), float(wr.log_dict[k])
        assert abs(a - b) <= tol * max(1.0, abs(b)), (k, a, b)
    a, b = float(wm.log_dict["d_weight"]), float(wr.log_dict["d_weight"])
    assert abs(a - b) <= 10 * tol * abs(b), ("d_weight", a, b)
    assert abs(float(wm.log_dict["d_loss"]) - float(wr.log_dict["d_loss"])) <= tol


# ----------------------------------------------------------------------------- 1. one step against the reference
def test_step_matches_reference_wrapper_and_fixture(cuda, tmp_path):
    wm, wr, _ = pair(tmp_path)
    data = BR.batch()
    seed = kink_free_seed(wr, data, BR.STEP)
    idx = []
    for w in (wm, wr):
        got, h = capture_bot_idx(w)
        torch.manual_seed(seed)
        w.optimize_parameters(data, BR.STEP)
        h.remove()
        idx.append(got[-1])
    check_losses(wm, wr)
    assert torch.equal(idx[0], idx[1])
    gm, gr = grads(wm), grads(wr)
    # the unstepped decoder tensors get gradients too (the reference's loss.backward() fills them)
    for k in ("decoder.conv_in.weight", "decoder.mid.attn_1.q.weight", "decoder.up.4.block.0.conv1.weight",
              "decoder.norm_out.weight", "decoder.conv_out.weight", "decoder.up.0.block.0.conv2.weight"):
        assert gm[k] is not None and gr[k] is not None, k
    worst = check_grads(gm, gr)
    print(f"[bottom drop-in] reduced shape fp32: worst gradient rel err {worst[0]:.2e} ({worst[1]})")
    # what does not depend on DiffAugment equals the fixture recorded from the real reference
    gold = np.load(GOLD)
    assert np.array_equal(idx[0].cpu().numpy(), gold["bot_idx"])
    for k in ("nll_loss", "codebook_loss"):
        assert abs(float(wm.log_dict[k]) - float(gold[k])) <= 2e-4 * max(1.0, abs(float(gold[k]))), k


# ----------------------------------------------------------------------------- 2. codebooks no patch selects
def _books_used(mask, hz, wz):
    """the books the reference's quantizer looks up: F.interpolate(mask, latent / 2, nearest) == k (:385-416)"""
    ids = F.interpolate(mask, size=(hz // 2, wz // 2), mode="nearest").reshape(-1)
    return {int(k) for k in ids.unique() if 0 <= int(k) < 18}


def argmin_margin(q, z, segm):
    """the smallest relative gap between a patch's nearest and second-nearest code of its book (fp64, the
    reference's patch layout): an fp32-equivalent search cannot pick the other code when this is well above rounding"""
    ps = q.spatial_size
    ids = F.interpolate(segm, size=(z.shape[2] // ps, z.shape[3] // ps), mode="nearest").reshape(-1).long()
    rows = F.unfold(z.detach().double(), (ps, ps), stride=ps).permute(0, 2, 1).reshape(-1, q.e_dim)
    best = float("inf")
    for k in ids.unique().tolist():
        if 0 <= k < 18:
            d = torch.cdist(rows[ids == k], q.embedding_list[k].weight.detach().double()) ** 2
            top2 = d.topk(2, largest=False).values
            best = min(best, float(((top2[:, 1] - top2[:, 0]) / top2[:, 1].clamp_min(1e-30)).min()))
    return best


def test_three_steps_with_changing_textures(cuda, tmp_path):
    """three optimize_parameters calls whose masks change which textures appear: every step's gradients against the
    reference wrapper's (check_grads), a codebook no patch selects has .grad None in both, and one that step 1
    selects and step 2 does not is left bitwise alone by step 2's Adam (a zero gradient would move it by its first
    moment)"""
    wm, wr, _ = pair(tmp_path)
    x = BR.batch()["image"]
    hz, wz = BR.H // 8, BR.W // 8
    masks = [BR.batch()["texture_mask"]]
    masks.append(torch.where(masks[0] < 9, masks[0] + 9, masks[0] - 9))      # swaps the two halves of the ids
    masks.append(R.blocky_mask(BR.DATA_SEED + 7, BR.BATCH, BR.H, BR.W, 8))
    used = [_books_used(mk, hz, wz) for mk in masks]
    gone = sorted(used[0] - used[1])
    assert gone and all(len(u) < 18 for u in used), used
    init = [e.weight.detach().to(cuda) for e in BR.modules()[0].bot_quantize.embedding_list]
    snaps = []
    for step, mk in enumerate(masks):
        data = dict(image=x, texture_mask=mk)
        seed = kink_free_seed(wr, data, BR.STEP)
        zin = []
        hq = wr.bot_quantize.register_forward_pre_hook(lambda m_, inp: zin.append((inp[0].detach(), inp[1])))
        idx = []
        for w in (wm, wr):
            got, h = capture_bot_idx(w)
            torch.manual_seed(seed)
            w.optimize_parameters(data, BR.STEP)
            h.remove()
            idx.append(got[-1])
            for k, e in enumerate(w.bot_quantize.embedding_list):
                assert (e.weight.grad is None) == (k not in used[step]), (step, k)
        hq.remove()
        margin = argmin_margin(wr.bot_quantize, *zin[-1])
        check_losses(wm, wr)
        assert torch.equal(idx[0], idx[1]), (step, margin)
        worst = check_grads(grads(wm), grads(wr))
        print(f"[bottom drop-in] step {step + 1}: books {sorted(used[step])}, argmin margin {margin:.1e}, worst "
              f"gradient rel err {worst[0]:.2e} ({worst[1]})")
        snaps.append([{k: e.weight.detach().clone() for k, e in enumerate(w.bot_quantize.embedding_list)}
                      for w in (wm, wr)])
    for i in range(2):
        for k in gone:
            # selected in step 1, not in step 2: step 2 leaves it bitwise alone
            assert torch.equal(snaps[1][i][k], snaps[0][i][k]), (i, k)
        for k in sorted(used[0]):
            assert not torch.equal(snaps[0][i][k], init[k])


# ----------------------------------------------------------------------------- 3. fix_decoder after inference()
def test_fix_decoder_after_inference(cuda, tmp_path):
    wm, wr, _ = pair(tmp_path, fix_decoder=True)
    data = BR.batch()
    loader = [dict(image=data["image"][i:i + 1], texture_mask=data["texture_mask"][i:i + 1], img_name=[f"img{i}"])
              for i in range(2)]
    seed = kink_free_seed(wr, data, BR.STEP)
    for i, w in enumerate((wm, wr)):
        out = tmp_path / f"val{i}"
        out.mkdir()
        w.inference(loader, str(out))
        assert sorted(p.name for p in out.iterdir()) == ["img0.png", "img1.png"]
        assert not w.decoder.training
        before = {k: v.clone() for k, v in w.decoder.state_dict().items()}
        torch.manual_seed(seed)
        w.optimize_parameters(data, BR.STEP)
        assert not w.decoder.training
        assert all(torch.equal(before[k], v) for k, v in w.decoder.state_dict().items())
    check_losses(wm, wr)
    worst = check_grads(grads(wm), grads(wr))
    print(f"[bottom drop-in] fix_decoder, eval-mode decoder: worst gradient rel err {worst[0]:.2e} ({worst[1]})")


# ----------------------------------------------------------------------------- 4. fp16 mode
def test_fp16_mode_tracks_fp32(cuda, tmp_path):
    from text2human_b200 import ops
    m, disc = BR.modules()
    opt = opt_for(tmp_path)
    write_top(opt["top_vae_path"], m, disc)
    res = {}
    for mode in ("fp32", "fp16"):
        ops.set_precision(mode)
        w = wrapper("mirror", opt, m)
        torch.manual_seed(43)
        w.optimize_parameters(BR.batch(), BR.STEP)
        g = grads(w)
        flat = [torch.cat([g[k].reshape(-1) for k in sorted(g) if g[k] is not None and k.startswith("disc.") == d])
                for d in (False, True)]
        res[mode] = ({k: float(w.log_dict[k]) for k in ("nll_loss", "g_loss", "codebook_loss", "loss", "d_loss")},
                     flat)
        del w
    (l32, (g32, d32)), (l16, (g16, d16)) = res["fp32"], res["fp16"]
    for k in l32:
        assert abs(l16[k] - l32[k]) <= 2e-2 * max(1.0, abs(l32[k])), (k, l16[k], l32[k])
    cg = float(F.cosine_similarity(g16.double(), g32.double(), dim=0))
    cd = float(F.cosine_similarity(d16.double(), d32.double(), dim=0))
    print(f"[bottom drop-in fp16 vs fp32] gradient cosine generator {cg:.5f} discriminator {cd:.5f}")
    assert cg > 0.98 and cd > 0.98


# ----------------------------------------------------------------------------- 5. the real LPIPS path
def test_with_lpips_mirror_installed_as_lpips(cuda, tmp_path, monkeypatch):
    import lpips_recipes as LR
    from oracle import lpips_ref
    _loader()
    sd = LR.state_dict()
    m, disc = BR.modules()
    opt = opt_for(tmp_path)
    write_top(opt["top_vae_path"], m, disc)
    ws = []
    for archs, factory in (("mirror", lambda net="vgg": LR.mirror(cuda)),
                           ("reference", lambda net="vgg": lpips_ref.LPIPSRef(sd))):
        _loader().install(archs, wrappers=())
        monkeypatch.setattr(sys.modules["lpips"], "LPIPS", factory)
        ws.append(wrapper(archs, opt, m))
    wm, wr = ws
    assert type(wm.perceptual).__module__ == "text2human_b200.lpips"
    data = BR.batch()
    seed = kink_free_seed(wr, data, BR.STEP)
    for w in (wm, wr):
        torch.manual_seed(seed)
        w.optimize_parameters(data, BR.STEP)
    check_losses(wm, wr, keys=("nll_loss", "g_loss", "codebook_loss", "l1", "perceptual"))
    assert wm.log_dict["perceptual"] > 0
    worst = check_grads(grads(wm), grads(wr))
    print(f"[bottom drop-in] with LPIPS: worst gradient rel err {worst[0]:.2e} ({worst[1]})")


# ----------------------------------------------------------------------------- 6. checkpoints
def test_save_and_load_network_round_trip(cuda, tmp_path):
    m, disc = BR.modules()
    path = str(tmp_path / "bottom.pth")
    opt = opt_for(tmp_path, pretrained_models=path)
    write_top(opt["top_vae_path"], m, disc)
    w = wrapper("mirror", opt, m)
    torch.manual_seed(44)
    w.optimize_parameters(BR.batch(), BR.STEP)
    w.save_network(path)
    assert set(torch.load(path)) == {"bot_encoder", "bot_decoder_res", "decoder", "bot_quantize", "bot_quant_conv",
                                     "bot_post_quant_conv", "discriminator"}
    w2 = wrapper("mirror", opt, BR.modules()[0])
    w2.load_network()
    x, mask = w.feed_data(BR.batch())
    outs = []
    for v in (w, w2):
        for n in GEN:
            getattr(v, n).eval()
        with torch.no_grad():
            outs.append(v.forward_step(x, mask))
    for n in GEN:
        s1, s2 = getattr(w, n).state_dict(), getattr(w2, n).state_dict()
        assert all(torch.equal(s1[k], s2[k]) for k in s1), n
    # the GroupNorm statistics ride in the conv epilogues as fp32 atomics: two forward passes of the same weights
    # agree to the arrival order of those sums (measured on an H100 80GB HBM3: 1.5e-6 of the image's max)
    (d1, c1), (d2, c2) = outs
    assert _rel(d2, d1) <= 1e-5 and abs(float(c2) - float(c1)) <= 1e-5 * abs(float(c1))


# ----------------------------------------------------------------------------- 7. real widths
REAL = dict(BR.OPT, embed_dim=256, bot_n_embed=512, bot_z_channels=256, bot_resolution=512, bot_ch=128,
            bot_num_res_blocks=2, bot_attn_resolutions=[64], top_z_channels=256, top_resolution=512, top_ch=128,
            top_num_res_blocks=2, top_attn_resolutions=[32])


def test_real_width_step_against_reference_wrapper(cuda, tmp_path):
    """configs/vqvae_bottom.yml's widths, B = 2, 512 x 256, seeded weights.  The step's gradient is discontinuous
    wherever a value sits on a kink: the bottom quantizer's argmin (a flipped index changes the patch's z_q by a whole
    code difference), the L1 term's sign(xrec - x) and the discriminator's LeakyReLUs (a flipped element moves a whole
    element of the image gradient).  The bound on indices allows one flip in 1024 patches.  On an H100 80GB HBM3 no
    index flipped, but 5 of the 786 432 L1 signs did and 209 of the reference discriminator's pre-activations lie
    within 1e-6 (relative) of the kink; each net's gradient then differs by 1.3e-3 .. 4.3e-3 in relative norm, and
    bot_post_quant_conv's by 1.1e-2 (bot_quantize's, mostly the continuous codebook-loss term, by 7.6e-6).  The
    gradient bound is 3e-2, that measurement with a margin of about 2.5."""
    from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
    from text2human_b200.vqgan_arch import Discriminator
    with contextlib.redirect_stdout(io.StringIO()):
        m = HierarchyVQSpatialTextureAwareModel(REAL)
    for name in ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv") + BOT[:2] + BOT[3:]:
        getattr(m, name).load_state_dict(R.fill_state_dict(R.spec_of(getattr(m, name)), BR.SEEDS[name]), strict=True)
    for q, key, ne, d in ((m.top_quantize, "top_books", 1024, 256), (m.bot_quantize, "bot_books", 512, 1024)):
        cb = R.codebooks(BR.SEEDS[key], 18, ne, d, "trained")
        for k, e in enumerate(q.embedding_list):
            e.weight.data.copy_(cb[k])
    disc = Discriminator(3, 64, n_layers=3)
    disc.load_state_dict(R.fill_state_dict(R.spec_of(disc), BR.SEEDS["disc"]), strict=True)
    opt = opt_for(tmp_path, base=REAL, ndf=64)
    write_top(opt["top_vae_path"], m, disc)
    wm = wrapper("mirror", opt, m)
    wr = wrapper("reference", opt, m)
    del m, disc
    data = dict(image=R.image(11, 2, 3, 512, 256), texture_mask=R.blocky_mask(12, 2, 512, 256, 32))
    idx, xrec = [], []
    pre = []
    kinks = [mod.register_forward_pre_hook(lambda m_, inp: pre.append(inp[0].detach().abs().flatten()))
             for mod in wr.disc.main if isinstance(mod, torch.nn.LeakyReLU)]
    for w in (wm, wr):
        got, h = capture_bot_idx(w)
        hx = w.decoder.register_forward_hook(lambda m_, i_, o: xrec.append(o.detach().clone()))
        torch.manual_seed(45)
        w.optimize_parameters(data, BR.STEP)
        h.remove()
        hx.remove()
        idx.append(got[-1])
    for h_ in kinks:
        h_.remove()
    agree = float((idx[0] == idx[1]).double().mean())
    # the elements on the other side of a kink: the L1 term's sign(xrec - x), and the reference discriminator's
    # pre-activations within 1e-6 (relative) of the LeakyReLU kink
    x = data["image"].to(cuda)
    l1_flips = int(((xrec[0] - x).sign() != (xrec[1] - x).sign()).sum())
    near_kink = sum(int((p < 1e-6 * p.max()).sum()) for p in pre)
    del pre
    losses = {k: (float(wm.log_dict[k]), float(wr.log_dict[k])) for k in ("nll_loss", "g_loss", "codebook_loss")}
    errs = {}
    for n in GEN + ("disc",):
        gm, gr = grads(wm, (n,)), grads(wr, (n,))
        keys = [k for k in gr if gr[k] is not None]
        assert all(gm[k] is not None for k in keys) and all(gm[k] is None for k in gr if gr[k] is None), n
        a = torch.cat([gm[k].reshape(-1) for k in keys]).double()
        b = torch.cat([gr[k].reshape(-1) for k in keys]).double()
        errs[n] = float((a - b).norm() / b.norm())
    print(f"[bottom drop-in real widths B=2] {100 * agree:.2f} % of bottom indices agree; L1 signs flipped "
          f"{l1_flips}; reference discriminator pre-activations near a kink {near_kink}; losses {losses}; "
          f"gradient rel norm err {errs}")
    assert agree >= 0.999
    for k, (a, b) in losses.items():
        assert abs(a - b) <= 1e-3 * max(1.0, abs(b)), k
    assert max(errs.values()) < 3e-2, errs


# ----------------------------------------------------------------------------- 8. replay and bad input
def test_nodes_replay_under_retain_graph(cuda):
    """DecoderRes and the trunk with the residual keep the snapshot discipline: a second backward of the same graph
    gives the same gradients, to the arrival order of the fp32 atomics in the split weight gradients (measured on an
    H100 80GB HBM3: up to 1.1e-6 of a tensor's max)"""
    m, _ = BR.modules()
    m = m.to(cuda).train()
    q = R.latent(46, (2, BR.OPT["bot_z_channels"], BR.H // 8, BR.W // 8)).to(cuda).requires_grad_(True)
    zt = R.latent(47, (2, BR.OPT["top_z_channels"], BR.H // 16, BR.W // 16)).to(cuda)
    xrec = m.decoder(zt, bot_h=m.bot_decoder_res(q))
    loss = (xrec * R.image(48, 2, 3, BR.H, BR.W).to(cuda)).sum()
    params = [q] + list(m.bot_decoder_res.parameters()) + list(m.decoder.parameters())
    g1 = torch.autograd.grad(loss, params, retain_graph=True)
    g2 = torch.autograd.grad(loss, params)
    top = max(float(b.abs().max()) for b in g2)
    for a, b in zip(g1, g2):
        # a gradient below 1e-3 of the largest (among them those that vanish in exact arithmetic and are rounding
        # noise, whose replay differs by as much as their size) is held to 1e-5 of the largest, absolutely
        bm = float(b.abs().max())
        assert float((a - b).abs().max()) <= 1e-5 * (bm if bm >= 1e-3 * top else top)


@pytest.mark.parametrize("legacy", [True, False])
def test_quantizer_node_matches_reference_quantizer(cuda, legacy):
    """the patch quantizer node alone against the reference's VectorQuantizerSpatialTextureAware (stock PyTorch) on the
    same codebooks, for both placements of beta: z_q, loss, indices, dz and every codebook gradient (None for a book
    no patch selects)"""
    from text2human_b200.vqgan_arch import VectorQuantizerSpatialTextureAware
    ref_cls = _loader().install("reference", wrappers=()).vqgan_arch.VectorQuantizerSpatialTextureAware
    cb = R.codebooks(51, 18, 64, 128, "trained")
    z0 = R.latent(52, (2, 32, 16, 8))
    mask = R.blocky_mask(53, 2, 128, 64, 16).to(cuda)
    g = R.latent(54, (2, 32, 16, 8), name="dzq").to(cuda)
    out = []
    for cls in (VectorQuantizerSpatialTextureAware, ref_cls):
        q = cls(64, 32, beta=0.25, spatial_size=2, legacy=legacy)
        for k, e in enumerate(q.embedding_list):
            e.weight.data.copy_(cb[k])
        q = q.to(cuda).train()
        z = z0.to(cuda).requires_grad_(True)
        zq, loss, (_, cont, lst) = q(z, mask)
        (3.0 * loss + (zq * g).sum()).backward()
        out.append((zq.detach(), float(loss), cont, z.grad, [e.weight.grad for e in q.embedding_list]))
    (zq_m, l_m, c_m, dz_m, gb_m), (zq_r, l_r, c_r, dz_r, gb_r) = out
    assert torch.equal(c_m, c_r) and c_m.dim() == 1
    assert _rel(zq_m, zq_r) <= 1e-6 and abs(l_m - l_r) <= 1e-5 * abs(l_r)
    assert _rel(dz_m, dz_r) <= 1e-5
    for k, (a, b) in enumerate(zip(gb_m, gb_r)):
        assert (a is None) == (b is None), k
        if b is not None:
            assert _rel(a, b) <= 1e-5, k


def test_latent_not_a_multiple_of_the_patch_raises_before_any_launch(cuda):
    from text2human_b200 import ops
    from text2human_b200.vqgan_arch import VectorQuantizerSpatialTextureAware
    q = VectorQuantizerSpatialTextureAware(64, 32, beta=0.25, spatial_size=2).to(cuda).train()
    for shape in ((2, 32, 7, 4), (2, 32, 8, 5)):
        z = torch.randn(shape, device=cuda, requires_grad=True)
        mask = torch.zeros(2, 1, 8 * shape[2], 8 * shape[3], device=cuda)
        n0 = ops.COUNTERS["launches"]
        with pytest.raises(ValueError):
            q(z, mask)
        assert ops.COUNTERS["launches"] == n0
