"""GPU: the VQGAN GAN training step (VQGANTrainer) at configs/vqvae_top.yml's real widths -- ch 128, ch_mult
[1,1,2,2,4], attention at 32, 18 codebooks of 1024 x 256, Discriminator(3, 64, 3), 512 x 256 images, the step that
bench.py's config-5 workload times -- against the fp64 restatement (oracle/vqgan_train_ref.training_step) run on the
GPU.  B = 2 in one micro-batch, so BatchNorm's batch statistics span two images and each image has its own
DiffAugment draws.

The native step's codebook picks, DiffAugment draws (the benchmark's law: ``default_aug_draws`` on a seeded device
generator), adaptive weight and the discriminator's LeakyReLU masks (test_gpu_train_layers.native_masks: the sign each
kernel used) are recorded and imposed on the restatement, so that the comparison is between smooth functions; every
pick that differs from fp64's argmin must be a near-tie the latent's error explains, and the adaptive weight is
checked against fp64's own.  Checked: all losses and the adaptive weight, every generator and discriminator gradient
tensor and the whole flat gradient, which codebook rows receive a gradient, and the discriminator's BatchNorm running
statistics after the step.

  A  the real config's first 30k steps (discriminator off): fp32 mode, LPIPS on both sides
  B  generator + discriminator, the adaptive weight inside its clamp: fp32 mode
  C  as B in the benchmark's fp16 mode, bounded against PyTorch's fp16 autocast of the same restatement
"""
import contextlib
import io
import math

import pytest
import torch

import golden_recipes as R
import lpips_recipes as LR
from test_gpu_train_layers import native_masks

pytestmark = pytest.mark.gpu

VQVAE_TOP = dict(embed_dim=256, n_embed=1024, double_z=False, z_channels=256, resolution=512, in_channels=3,
                 out_ch=3, ch=128, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2, attn_resolutions=[32], dropout=0.0)
B, H, W = 2, 512, 256
NDF, DISC_LAYERS = 64, 3
NETS = ("encoder", "decoder", "quant_conv", "post_quant_conv")
SEEDS = dict(encoder=501, decoder=502, quant_conv=503, post_quant_conv=504, disc=505, books=506, image=507, mask=508,
             aug=509)
LOSSES = ("loss", "nll_loss", "g_loss", "codebook_loss", "d_weight", "l1", "perceptual", "d_loss")


@pytest.fixture(scope="module", autouse=True)
def restore_precision():
    """the restatements run with TF32 off; the trainer's precision mode changes per case"""
    from text2human_b200 import ops
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, dict(ops._PRECISION))
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved[:2]
    ops._PRECISION.update(saved[2])


@pytest.fixture(scope="module")
def state():
    """seeded weights (golden_recipes.fill_state_dict: activations keep unit scale through the real depth, and the
    BatchNorm running statistics start away from 0 / 1), codebooks, images and texture mask, on the CPU"""
    from text2human_b200.pipeline import VQImageSegmTextureModel
    from text2human_b200.vqgan_arch import Discriminator
    with contextlib.redirect_stdout(io.StringIO()):
        m = VQImageSegmTextureModel(VQVAE_TOP)
    sd = {n: R.fill_state_dict(R.spec_of(getattr(m, n)), SEEDS[n]) for n in NETS}
    sdd = R.fill_state_dict(R.spec_of(Discriminator(3, NDF, n_layers=DISC_LAYERS)), SEEDS["disc"])
    return dict(sd=sd, sdd=sdd, books=R.codebooks(SEEDS["books"], 18, 1024, 256, "trained"),
                x=R.image(SEEDS["image"], B, 3, H, W), mask=R.blocky_mask(SEEDS["mask"], B, H, W, 32))


def record_disc_passes(monkeypatch):
    """-> a list that receives, per DiscNet forward of the trainer, its first layer's output planes and the
    (layer, pre-activation, statistics, output) of its three ConvModuleL layers; the library is unchanged"""
    from text2human_b200.train_layers import ConvModuleL
    from text2human_b200.vqgan_train import DiscNet
    passes = []
    disc_fwd, cm_fwd = DiscNet.fwd, ConvModuleL.fwd

    def recording_disc_fwd(self, x):                    # the first layer's output planes carry its mask
        passes.append(dict(mid=[]))
        out = disc_fwd(self, x)
        passes[-1]["y0"] = self.saved[-1][1].clone()
        return out

    def recording_cm_fwd(self, a, out="planes", drop=None):
        y = cm_fwd(self, a, out=out, drop=drop)
        _, pre, st_, _, _, _ = self.saved[-1]
        passes[-1]["mid"].append(dict(layer=self, pre=pre.clone(), st=st_.clone(), y=y, drop=drop))
        return y
    monkeypatch.setattr(DiscNet, "fwd", recording_disc_fwd)
    monkeypatch.setattr(ConvModuleL, "fwd", recording_cm_fwd)
    return passes


def disc_masks(passes):
    """recorded passes -> per pass the masks of its four LeakyReLUs (bool NCHW, True: slope 1), as the kernels used
    them: the sign of the first layer's stored output, and test_gpu_train_layers.native_masks for the others"""
    return [[(p["y0"].float().sum(0) > 0).permute(0, 3, 1, 2)] + native_masks(p["mid"]) for p in passes]


def run_native(st, dev, monkeypatch, mode, step, disc_start_step, disc_weight_max, perceptual):
    """one VQGANTrainer.training_step; -> its losses, gradients (unscaled), BatchNorm buffers, codebook picks,
    DiffAugment draws and per discriminator pass the masks of its four LeakyReLUs (bool NCHW)"""
    from text2human_b200 import ops
    from text2human_b200.pipeline import VQImageSegmTextureModel
    from text2human_b200.vqgan_arch import Discriminator
    from text2human_b200.vqgan_train import VQGANTrainer
    ops.set_precision(mode)
    with contextlib.redirect_stdout(io.StringIO()):
        m = VQImageSegmTextureModel(VQVAE_TOP)
    for n in NETS:
        getattr(m, n).load_state_dict(st["sd"][n], strict=True)
    for k, e in enumerate(m.quantize.embedding_list):
        e.weight.data.copy_(st["books"][k])
    disc = Discriminator(3, NDF, n_layers=DISC_LAYERS)
    disc.load_state_dict(st["sdd"], strict=True)
    m, disc = m.to(dev), disc.to(dev)
    lp = LR.mirror(dev) if perceptual else None
    tr = VQGANTrainer(m, disc, disc_start_step=disc_start_step, disc_weight_max=disc_weight_max, perceptual=lp)
    rec, draws = {}, []
    search = ops.vq_search

    def recording_search(z, codebook, ids, **kw):      # tr._vq is cleared by the end of the step
        r = search(z, codebook, ids, **kw)
        rec.update(z=z.clone(), idx=r["idx"].clone(), ids=ids.clone())
        return r
    monkeypatch.setattr(ops, "vq_search", recording_search)
    passes = record_disc_passes(monkeypatch)
    gen = torch.Generator(device=dev).manual_seed(SEEDS["aug"])

    def draw(b, h, w, device):                           # bench.py's draw law, recorded
        r, t = VQGANTrainer.default_aug_draws(b, h, w, device, gen)
        draws.append((r.clone(), t.clone()))
        return r, t
    tr.aug_draw_fn = draw
    tr.training_step(dict(image=st["x"], texture_mask=st["mask"]), step)
    torch.cuda.synchronize()
    monkeypatch.setattr(ops, "vq_search", search)
    masks = disc_masks(passes)
    del passes
    g = {f"{n}.{k}": p.grad.detach().double() / tr.loss_scale for n in NETS
         for k, p in getattr(m, n).named_parameters()}
    for k, e in enumerate(m.quantize.embedding_list):
        g[f"quantize.embedding_list.{k}.weight"] = e.weight.grad.detach().double() / tr.loss_scale
    d = {k: p.grad.detach().double() / tr.disc_scale for k, p in disc.named_parameters()}
    bn = {k: v.detach().clone() for k, v in disc.state_dict().items() if "running" in k or "num_batches" in k}
    out = dict(losses=tr.losses(), g=g, d=d, bn=bn, rec=rec, draws=draws, masks=masks, loss_scale=tr.loss_scale,
               disc_scale=tr.disc_scale, d_flat_zero=bool((tr.dsc.flat_g == 0).all()))
    del tr, m, disc, lp
    torch.cuda.empty_cache()
    return out


def run_ref(st, dev, dtype, nat, step, disc_start_step, disc_weight_max, perceptual, autocast_scale=None):
    """the restatement in ``dtype`` (with ``autocast_scale``: fp32 under fp16 autocast, the generator's loss scaled by
    it and the discriminator's by the trainer's disc_scale, unscaled after), fed the native picks, draws, adaptive
    weight and LeakyReLU masks.  fp64 also reports its own LeakyReLU inputs (to count the native masks that differ
    from fp64's sign) and its own adaptive weight (``ratio``, before the clamp)."""
    from oracle import lpips_ref
    from oracle import vqgan_train_ref as TR
    sd = {f"{n}.{k}": v.to(dev, dtype).requires_grad_(True) for n in NETS for k, v in st["sd"][n].items()}
    books = [st["books"][k].to(dev, dtype).requires_grad_(True) for k in range(18)]
    sdd = {k: (v.to(dev, dtype).requires_grad_("running" not in k) if v.is_floating_point() else v.to(dev))
           for k, v in st["sdd"].items()}
    plp = None
    if perceptual:
        lsd = {k: v.to(dev, dtype) for k, v in LR.state_dict().items()}

        def plp(a, b):
            return lpips_ref.lpips(lsd, a, b)
    s, sdisc = (autocast_scale, nat["disc_scale"]) if autocast_scale else (1.0, 1.0)
    draws = [tuple(t.to(dev) for t in dr) for dr in nat["draws"]] + [None]
    bn, trace = {}, ([] if dtype == torch.float64 else None)
    with torch.autocast("cuda", torch.float16) if autocast_scale else contextlib.nullcontext():
        r = TR.training_step(sd, books, sdd, st["x"].to(dev, dtype), st["mask"].to(dev), step, perceptual=plp,
                             disc_start_step=disc_start_step, disc_weight_max=disc_weight_max, disc_layers=DISC_LAYERS,
                             draws=(draws[0], draws[1]), idx=nat["rec"]["idx"], bn_state=bn, loss_scale=s,
                             d_weight=nat["losses"]["d_weight"], disc_masks=nat["masks"], disc_trace=trace)
    gen = list(sd) + [f"quantize.embedding_list.{k}.weight" for k in range(18)]
    leaves = list(sd.values()) + books
    gs = torch.autograd.grad(r["loss"] * s, leaves, retain_graph=r["d_loss"] is not None, allow_unused=True)
    g = {k: (v.double() / s if v is not None else torch.zeros_like(p, dtype=torch.float64))
         for k, v, p in zip(gen, gs, leaves)}
    dk = [k for k, v in sdd.items() if v.requires_grad]
    if r["d_loss"] is not None:
        ds = torch.autograd.grad(r["d_loss"] * sdisc, [sdd[k] for k in dk], allow_unused=True)
    else:
        ds = [None] * len(dk)
    d = {k: (v.double() / sdisc if v is not None else torch.zeros_like(sdd[k], dtype=torch.float64))
         for k, v in zip(dk, ds)}
    losses = {k: float(r[k].detach()) for k in LOSSES if r[k] is not None}
    flips = None
    if trace is not None and nat["masks"] is not None:
        flips = sum(int(((u > 0) != mk).sum()) for tp, mp in zip(trace, nat["masks"]) for u, mk in zip(tp, mp))
    out = dict(losses=losses, g=g, d=d, bn=bn, passes=r["bn_passes"], ratio=float(r["ratio"]), flips=flips,
               vq={k: v.detach() for k, v in r["vq"].items()}, sdd_nbt={k: v for k, v in sdd.items() if "num_b" in k})
    del r, sd, sdd, books, gs, ds, leaves, trace
    torch.cuda.empty_cache()
    return out


def grad_errors(got, want):
    """-> (per-tensor list of (relative norm error, norm error, name, norm), floor, flat relative error).  A tensor
    passes at ``tol`` if its relative error is within tol or its error within the floor, 1e-6 of the largest norm
    (gradients that are zero in exact arithmetic, such as a key bias in front of softmax, are rounding residue on
    both sides), as test_gpu_vqgan_train._check_grads"""
    norms = {k: float(w.norm()) for k, w in want.items()}
    floor = 1e-6 * max(norms.values())
    per = []
    for k, w in want.items():
        err = float((got[k] - w).norm())
        per.append((err / max(norms[k], 1e-300), err, k, norms[k]))
    flat_w = torch.cat([w.reshape(-1) for w in want.values()])
    flat_g = torch.cat([got[k].reshape(-1) for k in want])
    return per, floor, float((flat_g - flat_w).norm() / flat_w.norm())


def worst(per, floor, tol=1e-3, only=None):
    """the largest relative error among tensors well above the floor (reporting; ``only``: a name filter)"""
    return max(((rel, k) for rel, _, k, n in per if n > floor / tol and (only is None or only in k)),
               default=(0.0, None))


def failing(per, floor, tol, only=None):
    return [(k, rel, err) for rel, err, k, _ in per if rel > tol and err > floor and (only is None or only in k)]


def check_picks(tag, nat, r64, books):
    """every row whose native pick a differs from fp64's argmin b must be a near-tie the latent's error explains:
    d64(a) - d64(b) <= 2 |z_nat - z64| |e_a - e_b| + 1e-5 (|z|^2 + |e|^2), the last term for the fp32 rounding of
    the distance itself; -> (rows differing, largest margin, largest margin / bound)"""
    rows64 = r64["vq"]["rows"]
    D = rows64.shape[1]
    a = nat["rec"]["idx"].reshape(-1)
    b = r64["vq"]["argmin"]
    ids = nat["rec"]["ids"].reshape(-1).long()
    # the kernel's texture ids (ops.mask_to_ids) and the restatement's nearest-interpolated mask, row for row
    assert torch.equal(ids, r64["vq"]["seg"].long()), int((ids != r64["vq"]["seg"].long()).sum())
    assert bool((b >= 0).all()) and bool(((ids >= 0) & (ids < 18)).all())
    diff = (a != b).nonzero().flatten()
    if diff.numel() == 0:
        return 0, 0.0, 0.0
    cb = books.to(rows64.device, torch.float64)
    z_nat = nat["rec"]["z"].reshape(-1, D).double()[diff]
    z64 = rows64[diff]
    ea, eb = cb[ids[diff], a[diff]], cb[ids[diff], b[diff]]
    dist = r64["vq"]["dist"]
    margin = dist[diff, a[diff]] - dist[diff, b[diff]]
    bound = (2 * (z_nat - z64).norm(dim=1) * (ea - eb).norm(dim=1)
             + 1e-5 * ((z64 ** 2).sum(1) + torch.maximum((ea ** 2).sum(1), (eb ** 2).sum(1))))
    assert bool((margin >= 0).all())
    bad = margin > bound
    assert not bool(bad.any()), (tag, int(bad.sum()), margin[bad][:4].tolist(), bound[bad][:4].tolist())
    return diff.numel(), float(margin.max()), float((margin / bound).max())


def check_codebook_rows(nat):
    """codebook rows with a nonzero gradient are exactly the picked codes"""
    got = torch.stack([nat["g"][f"quantize.embedding_list.{k}.weight"] for k in range(18)])
    picked = torch.zeros(got.shape[:2], dtype=torch.bool, device=got.device)
    picked[nat["rec"]["ids"].reshape(-1).long(), nat["rec"]["idx"].reshape(-1)] = True
    assert torch.equal((got != 0).any(-1), picked), int(((got != 0).any(-1) != picked).sum())
    return int(picked.sum())


def loss_errors(got, want):
    return {k: abs(got[k] - want[k]) / max(abs(want[k]), 1e-30) for k in want if k in got and k != "d_weight"}


def check_draws(draws, n):
    """the native draws fall in the reference's ranges: r in [0, 1), |tx| <= 64 and |ty| <= 32 at 512 x 256"""
    assert len(draws) == n
    for r, t in draws:
        assert r.shape == (B, 3) and t.shape == (B, 2) and t.dtype == torch.int32
        assert bool(((r >= 0) & (r < 1)).all())
        assert int(t[:, 0].abs().max()) <= 64 and int(t[:, 1].abs().max()) <= 32


def bn_errors(got, r64, n_pass):
    """the discriminator's running statistics after the step against fp64's chained passes: num_batches_tracked
    exactly, -> {buffer: norm error relative to the running variance, or for the mean to the running standard
    deviation (the means of bias-free convs are small against the spread they normalise)}"""
    assert r64["passes"] == n_pass
    errs = {}
    for k, w in r64["bn"].items():
        if "num_batches" in k:
            assert int(got[k]) == int(r64["sdd_nbt"][k]) + n_pass == int(w), k
        else:
            var = r64["bn"][k.replace("running_mean", "running_var")]
            errs[k] = float((got[k].double() - w).norm() / (var.sqrt() if "mean" in k else var).norm())
    assert len(errs) == 2 * DISC_LAYERS
    return errs


def run_other(state, cuda, nat, mode, step, disc_start_step, disc_weight_max, perceptual):
    """the yardstick of the same precision: the fp32 restatement (TF32 off), or in fp16 mode the restatement under fp16
    autocast at the trainer's generator loss scale, or the largest smaller power-of-two scale (steps of 2^3) whose
    gradient stays finite (fp16 overflows at 2^19 here)"""
    if mode != "fp16":
        return run_ref(state, cuda, torch.float32, nat, step, disc_start_step, disc_weight_max, perceptual)
    scale = nat["loss_scale"]
    while True:
        other = run_ref(state, cuda, torch.float32, nat, step, disc_start_step, disc_weight_max, perceptual,
                        autocast_scale=scale)
        if all(bool(torch.isfinite(v).all()) for v in list(other["g"].values()) + list(other["d"].values())):
            other["scale"] = scale
            return other
        assert scale > 2.0 ** 4, "fp16 autocast gradients are not finite at any loss scale"
        scale /= 8.0


def run_case(tag, cuda, monkeypatch, state, mode, step, disc_start_step, disc_weight_max, perceptual):
    torch.cuda.reset_peak_memory_stats()
    nat = run_native(state, cuda, monkeypatch, mode, step, disc_start_step, disc_weight_max, perceptual)
    trains_disc = step > disc_start_step
    check_draws(nat["draws"], 2 if trains_disc else 1)
    assert len(nat["masks"]) == (3 if trains_disc else 1)
    r64 = run_ref(state, cuda, torch.float64, nat, step, disc_start_step, disc_weight_max, perceptual)
    other = run_other(state, cuda, nat, mode, step, disc_start_step, disc_weight_max, perceptual)
    n_flip, margin, ratio = check_picks(tag, nat, r64, state["books"])
    n_codes = check_codebook_rows(nat)
    res = dict(nat=nat, r64=r64, other=other)
    want_dw = min(r64["ratio"], disc_weight_max) if step >= disc_start_step else 0.0
    errs = {"d_weight": abs(nat["losses"]["d_weight"] - want_dw) / max(want_dw, 1e-30)}
    for who in ("nat", "other"):
        e = {"losses": loss_errors(res[who]["losses"], r64["losses"]),
             "bn": bn_errors(res[who]["bn"], r64, 3 if trains_disc else 1)}
        for net in ("g", "d") if trains_disc else ("g",):
            e[net] = grad_errors(res[who][net], r64[net])
        errs[who] = e
    what = "fp16 autocast" if mode == "fp16" else "fp32 restatement"
    if mode == "fp16":
        what += f" (loss scale 2^{int(math.log2(other['scale']))})"
    for net in ("g", "d") if trains_disc else ("g",):
        for who, name in (("nat", "native"), ("other", what)):
            per, floor, flat = errs[who][net]
            top = sorted(((rel, k) for rel, _, k, n in per if n > floor / 1e-3), reverse=True)[:3]
            books = worst(per, floor, only="embedding_list")
            print(f"[{tag}] {name} {'generator' if net == 'g' else 'discriminator'}: flat {flat:.2e}, worst "
                  + ", ".join(f"{k} {rel:.2e}" for rel, k in top)
                  + (f"; codebooks {books[0]:.2e}" if net == "g" else "") + f" ({len(per)} tensors)")
    for who, name in (("nat", "native"), ("other", what)):
        print(f"[{tag}] {name} loss errors " + ", ".join(f"{k} {v:.1e}" for k, v in errs[who]["losses"].items()))
        print(f"[{tag}] {name} running statistics " + ", ".join(f"{k} {v:.1e}" for k, v in errs[who]["bn"].items()))
    print(f"[{tag}] losses fp64 {r64['losses']}; adaptive weight before clamp fp64 {r64['ratio']:.6g}, "
          f"native d_weight {nat['losses']['d_weight']:.6g} (error {errs['d_weight']:.1e}); "
          f"{r64['flips']} native LeakyReLU masks differ from fp64's sign")
    print(f"[{tag}] {n_flip} codebook rows differ from fp64's argmin, largest margin {margin:.2e} "
          f"({ratio:.2f} of its bound); {n_codes} codes picked; "
          f"peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    return nat, r64, errs


# Per-tensor bound 1e-3 throughout.  Flat bounds, measured on an H100 80GB HBM3 (700 W), with every discrete choice
# imposed (without the LeakyReLU masks case B's generator was at 8.5e-3 and its discriminator at 3.9e-4, the fp32
# restatement at 2.5e-3 / 9.4e-5: 472 masks differ from fp64's sign there):
# - A: the fp32 mode's hi/lo fp16 planes carry 22 significant bits per operand (11 + 11, the lo x lo product dropped),
#   four times fp32's rounding unit, and the native error is four times the fp32 restatement's: flat 1.06e-4 against
#   2.6e-5, worst tensor 5.1e-4 against 1.3e-4 (encoder.conv_in.weight, the end of the backward pass; the same with
#   LPIPS off).  Bound 2e-4, and at most 6 times the fp32 restatement's.
# - B, generator: flat 3.0e-4 (fp32 restatement 1.75e-5), worst tensors the decoder's norms at 3.7e-4.  The added
#   error is the adaptive-weighted g_loss path: the discriminator's data gradient at the image is within 1.8e-5 of
#   fp64 and DiffAugment's adjoint within 6e-8, and the decoder's backward amplifies the former.  Bound 5e-4.
# - B, discriminator: flat 6.0e-6 (fp32 restatement 1.75e-6).  Bound 1e-4.
FLAT_BOUND = {"A": {"g": 2e-4}, "B": {"g": 5e-4, "d": 1e-4}}
FLAT_RATIO_A = 6.0


def assert_fp32_bounds(case, errs):
    for net, flat_tol in FLAT_BOUND[case].items():
        per, floor, flat = errs["nat"][net]
        bad = failing(per, floor, 1e-3)
        assert not bad, (net, bad[:6], floor)
        assert flat <= flat_tol, (net, flat)
    if case == "A":
        assert errs["nat"]["g"][2] <= FLAT_RATIO_A * errs["other"]["g"][2], (errs["nat"]["g"][2], errs["other"]["g"][2])
    bad = {k: v for k, v in errs["nat"]["losses"].items() if v > 1e-4}
    assert not bad, bad
    assert max(errs["nat"]["bn"].values()) <= 1e-5, errs["nat"]["bn"]
    assert errs["d_weight"] <= 1e-4, errs["d_weight"]


def test_case_a_first_steps_generator_only_with_lpips(cuda, monkeypatch, state):
    """configs/vqvae_top.yml's disc_start_step 30001 at step 1: the adaptive weight is 0, the discriminator runs once
    (g_loss) without a parameter gradient, LPIPS adds to nll_loss on both sides"""
    nat, r64, errs = run_case("A fp32", cuda, monkeypatch, state, "fp32", 1, 30001, 1.0, True)
    assert nat["losses"]["d_weight"] == 0.0 and r64["losses"]["d_weight"] == 0.0
    assert nat["d_flat_zero"] and all(float(v.abs().max()) == 0.0 for v in nat["d"].values())
    assert "d_loss" not in nat["losses"] and "d_loss" not in r64["losses"]
    assert r64["losses"]["perceptual"] > 0
    assert_fp32_bounds("A", errs)


WMAX = 1e6      # far above the adaptive weight's ratio here: the clamp does not bind


def test_case_b_generator_and_discriminator(cuda, monkeypatch, state):
    nat, r64, errs = run_case("B fp32", cuda, monkeypatch, state, "fp32", 2, 0, WMAX, False)
    assert 0 < r64["ratio"] < WMAX
    assert_fp32_bounds("B", errs)


def test_case_c_fp16_mode_against_fp16_autocast(cuda, monkeypatch, state):
    """the benchmark's single-product fp16 mode: no fixed bound exists at these widths, so the native error against
    fp64 is held to twice that of PyTorch's fp16 autocast of the same restatement (same picks, draws, adaptive weight,
    LeakyReLU masks): worst tensor and flat gradient of generator and discriminator, losses, running statistics,
    the adaptive weight, and the codebooks (or 1e-3, whichever is larger)"""
    nat, r64, errs = run_case("C fp16", cuda, monkeypatch, state, "fp16", 2, 0, WMAX, False)
    assert 0 < r64["ratio"] < WMAX
    fails, ratios = [], {}
    for net in ("g", "d"):
        (pn, fl, fn), (pa, fla, fa) = errs["nat"][net], errs["other"][net]
        wn, wa = worst(pn, fl), worst(pa, fla)
        ratios[net] = (wn[0] / wa[0], fn / fa)
        if wn[0] > 2 * wa[0]:
            fails.append((net, "worst tensor", wn, wa))
        if fn > 2 * fa:
            fails.append((net, "flat", fn, fa))
    (pn, fl, _), (pa, fla, _) = errs["nat"]["g"], errs["other"]["g"]
    tol = max(1e-3, 2 * worst(pa, fla, only="embedding_list")[0])
    fails += [("codebook", f) for f in failing(pn, fl, tol, only="embedding_list")]
    ln, la = errs["nat"]["losses"], errs["other"]["losses"]
    fails += [(k, ln[k], la[k]) for k in ln if ln[k] > max(2 * la[k], 1e-3)]
    if errs["d_weight"] > 1e-3:
        fails.append(("d_weight", errs["d_weight"]))
    if max(errs["nat"]["bn"].values()) > 2 * max(errs["other"]["bn"].values()):
        fails.append(("running statistics", errs["nat"]["bn"], errs["other"]["bn"]))
    print("[C fp16] native / autocast (worst tensor, flat): " + ", ".join(
        f"{'generator' if n == 'g' else 'discriminator'} {a:.2f} / {b:.2f}" for n, (a, b) in ratios.items()))
    assert not fails, fails
