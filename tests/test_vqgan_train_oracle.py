"""CPU: the GAN-training-step restatement (oracle/vqgan_train_ref.training_step) against the fixture made from the
real reference `VQImageSegmTextureModel.training_step` + `loss.backward()` + `d_loss.backward()`
(oracle/make_golden_vqgan_train.py).  The CUDA path for this step (SURVEY a18 / config 5) is not built yet; this
pins the oracle it will be measured against."""
import contextlib
import io
import os

import numpy as np
import torch

import golden_recipes as R
from oracle import vqgan_train_ref as TR

GOLD = os.path.join(os.path.dirname(__file__), "golden", "vqgan_train.npz")


def _state():
    """the same seeded weights the generator script loaded into the reference modules, keyed as in state_dict()"""
    from text2human_b200.vqgan_arch import Decoder, Encoder
    cfg = R.TINY_VQGAN_TRAIN
    with contextlib.redirect_stdout(io.StringIO()):
        enc, dec = Encoder(**cfg["enc"]), Decoder(**cfg["dec"])
    sd = {}
    for prefix, mod, seed in (("encoder.", enc, 101), ("decoder.", dec, 102)):
        for k, v in R.fill_state_dict(R.spec_of(mod), seed).items():
            sd[prefix + k] = v
    qc = torch.nn.Conv2d(cfg["enc"]["z_channels"], cfg["embed_dim"], 1)
    pq = torch.nn.Conv2d(cfg["embed_dim"], cfg["enc"]["z_channels"], 1)
    for prefix, mod, seed in (("quant_conv.", qc, 103), ("post_quant_conv.", pq, 104)):
        for k, v in R.fill_state_dict(R.spec_of(mod), seed).items():
            sd[prefix + k] = v
    # the discriminator's keys (nn.Sequential 'main.N'), built from its published layer list
    ndf, spec = cfg["ndf"], []
    spec += [("main.0.weight", (ndf, 3, 4, 4)), ("main.0.bias", (ndf,))]
    i, prev = 2, 1
    for n in range(1, cfg["disc_layers"] + 1):
        mult = min(2 ** n, 8)
        spec += [(f"main.{i}.weight", (ndf * mult, ndf * prev, 4, 4)), (f"main.{i + 1}.weight", (ndf * mult,)),
                 (f"main.{i + 1}.bias", (ndf * mult,)), (f"main.{i + 1}.running_mean", (ndf * mult,)),
                 (f"main.{i + 1}.running_var", (ndf * mult,)), (f"main.{i + 1}.num_batches_tracked", ())]
        prev, i = mult, i + 3
    spec += [(f"main.{i}.weight", (1, ndf * prev, 4, 4)), (f"main.{i}.bias", (1,))]
    sdd = R.fill_state_dict(spec, 105)
    cb = R.codebooks(106, 18, cfg["n_embed"], cfg["embed_dim"], "trained")
    return cfg, sd, sdd, cb


def test_gan_training_step_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    cfg, sd, sdd, cb = _state()
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    sdd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone())
           for k, v in sdd.items()}
    books = [cb[k].clone().requires_grad_(True) for k in range(18)]
    B, H, W = cfg["batch"], cfg["enc"]["resolution"], cfg["enc"]["resolution"] // 2
    x, mask = R.image(107, B, 3, H, W), R.blocky_mask(108, B, H, W, 8)
    torch.manual_seed(R.VQGAN_TRAIN_AUG_SEED)          # the reference's DiffAugment draws, replayed in the same order
    r = TR.training_step(sd, books, sdd, x, mask, cfg["step"], disc_start_step=cfg["disc_start_step"],
                         disc_layers=cfg["disc_layers"])
    for k in ("loss", "d_loss", "nll_loss", "g_loss", "d_weight", "codebook_loss"):
        assert abs(float(r[k]) - float(gold[k])) <= 2e-5 * max(1.0, abs(float(gold[k]))), k
    r["loss"].backward(retain_graph=True)
    n_checked = 0
    for key in gold.files:
        if not key.startswith("gnorm/"):
            continue
        name = key[len("gnorm/"):]
        if name.startswith("quantize.embedding_list."):
            g = books[int(name.split(".")[2])].grad
        else:
            g = sd[name].grad
        g = g if g is not None else torch.zeros(1)
        want = float(gold[key])
        assert abs(float(g.norm()) - want) <= 2e-4 * max(want, 1e-6) + 1e-7, name
        head = torch.from_numpy(gold["ghead/" + name])
        assert (g.reshape(-1)[:8] - head).abs().max() <= 2e-4 * max(want, 1e-6) + 1e-7, name
        n_checked += 1
    assert n_checked > 200
    for p in sdd.values():
        if p.requires_grad:
            p.grad = None                     # disc_optimizer.zero_grad() before d_loss.backward()
    r["d_loss"].backward()
    for key in gold.files:
        if key.startswith("dnorm/"):
            name = key[len("dnorm/"):]
            g, want = sdd[name].grad, float(gold[key])
            assert abs(float(g.norm()) - want) <= 2e-4 * max(want, 1e-6) + 1e-7, name
            assert (g.reshape(-1)[:8] - torch.from_numpy(gold["dhead/" + name])).abs().max() <= 2e-4 * want + 1e-7


def _reference_draws(B, H, W):
    """DiffAugment's draws in the reference's global-RNG call order, drawn here rather than by the restatement"""
    r = torch.cat([torch.rand(B, 1, 1, 1).view(B, 1) for _ in range(3)], 1)
    sx, sy = int(H * 0.125 + 0.5), int(W * 0.125 + 0.5)
    tx = torch.randint(-sx, sx + 1, size=[B, 1, 1]).view(B, 1)
    ty = torch.randint(-sy, sy + 1, size=[B, 1, 1]).view(B, 1)
    return r, torch.cat([tx, ty], 1).int()


def _run(cfg, sd, sdd, cb, x, mask, **kw):
    """one restated step on fresh leaves -> (result, generator gradients, discriminator gradients)"""
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    sdd = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "running" not in k else v.clone())
           for k, v in sdd.items()}
    books = [cb[k].clone().requires_grad_(True) for k in range(18)]
    r = TR.training_step(sd, books, sdd, x, mask, cfg["step"], disc_start_step=cfg["disc_start_step"],
                         disc_layers=cfg["disc_layers"], **kw)
    gen = list(sd.values()) + books
    g = torch.autograd.grad(r["loss"], gen, retain_graph=True, allow_unused=True)
    dl = [v for v in sdd.values() if v.requires_grad]
    d = torch.autograd.grad(r["d_loss"], dl, allow_unused=True)
    return r, g, d


def _same(a, b):
    return (a is None and b is None) or (a is not None and b is not None and torch.equal(a, b))


def test_imposed_picks_and_draws_reproduce_the_default_path_bit_for_bit():
    cfg, sd, sdd, cb = _state()
    B, H, W = cfg["batch"], cfg["enc"]["resolution"], cfg["enc"]["resolution"] // 2
    x, mask = R.image(107, B, 3, H, W), R.blocky_mask(108, B, H, W, 8)
    torch.manual_seed(R.VQGAN_TRAIN_AUG_SEED)
    r0, g0, d0 = _run(cfg, sd, sdd, cb, x, mask)
    torch.manual_seed(R.VQGAN_TRAIN_AUG_SEED)
    draws = (_reference_draws(B, H, W), _reference_draws(B, H, W))
    idx = r0["vq"]["argmin"]
    assert bool((idx >= 0).all()) and torch.equal(idx, r0["vq"]["dist"].argmin(1))
    torch.manual_seed(12345)                          # the imposed path must not read the global RNG
    r1, g1, d1 = _run(cfg, sd, sdd, cb, x, mask, draws=draws, idx=idx.clone())
    for k in ("loss", "d_loss", "nll_loss", "g_loss", "d_weight", "codebook_loss", "xrec"):
        assert torch.equal(r0[k], r1[k]), k
    assert torch.equal(r0["vq"]["dist"], r1["vq"]["dist"])
    assert all(_same(a, b) for a, b in zip(g0, g1)) and all(_same(a, b) for a, b in zip(d0, d1))
    # and the options are not ignored: another code for one row, or another translation, changes the step
    other = idx.clone()
    other[0] = (other[0] + 1) % cfg["n_embed"]
    r2, _, _ = _run(cfg, sd, sdd, cb, x, mask, draws=draws, idx=other)
    assert not torch.equal(r2["codebook_loss"], r0["codebook_loss"])
    (rf, tf), real = draws
    r3, _, _ = _run(cfg, sd, sdd, cb, x, mask, draws=((rf, tf.flip(0)), real), idx=idx)
    assert not torch.equal(r3["g_loss"], r0["g_loss"]) and torch.equal(r3["nll_loss"], r0["nll_loss"])


def _torch_discriminator(cfg, sdd):
    """the Discriminator's layer list from plain torch modules (nn.BatchNorm2d updates its own buffers)"""
    ndf, n_layers = cfg["ndf"], cfg["disc_layers"]
    layers, prev = [torch.nn.Conv2d(3, ndf, 4, 2, 1), torch.nn.LeakyReLU(0.2)], 1
    for n in range(1, n_layers + 1):
        mult = min(2 ** n, 8)
        layers += [torch.nn.Conv2d(ndf * prev, ndf * mult, 4, 2 if n < n_layers else 1, 1, bias=False),
                   torch.nn.BatchNorm2d(ndf * mult), torch.nn.LeakyReLU(0.2)]
        prev = mult
    layers.append(torch.nn.Conv2d(ndf * prev, 1, 4, 1, 1))
    main = torch.nn.Sequential(*layers)
    main.load_state_dict({k[len("main."):]: v.clone() for k, v in sdd.items()}, strict=True)
    return main.train()


def test_chained_running_statistics_equal_sequential_batch_norm_updates():
    """fake image (g_loss), real image, detached fake image: the restatement's chained BatchNorm statistics against
    nn.BatchNorm2d updating its buffers over the same three inputs; one pass when the discriminator does not train"""
    cfg, sd, sdd, cb = _state()
    B, H, W = cfg["batch"], cfg["enc"]["resolution"], cfg["enc"]["resolution"] // 2
    x, mask = R.image(107, B, 3, H, W), R.blocky_mask(108, B, H, W, 8)
    torch.manual_seed(R.VQGAN_TRAIN_AUG_SEED)
    fake, real = _reference_draws(B, H, W), _reference_draws(B, H, W)
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}       # the adaptive weight's autograd.grad
    for step, n_pass in ((cfg["step"], 3), (cfg["disc_start_step"], 1)):
        st = {}
        r = TR.training_step(sd, [cb[k] for k in range(18)], sdd, x, mask, step,
                             disc_start_step=cfg["disc_start_step"], disc_layers=cfg["disc_layers"],
                             draws=(fake, real), bn_state=st)
        assert r["bn_passes"] == n_pass and (r["d_loss"] is None) == (n_pass == 1)
        main = _torch_discriminator(cfg, sdd)
        xr = TR.diff_augment(r["xrec"].detach(), fake)
        with torch.no_grad():
            for inp in (xr, TR.diff_augment(x, real), xr)[:n_pass]:
                main(inp)
        n_bn = 0
        for k, v in main.state_dict().items():
            if "running" in k or "num_batches" in k:
                assert torch.equal(st["main." + k], v), (step, k, float((st["main." + k] - v).abs().max()))
                assert not torch.equal(v, sdd["main." + k]), k
                n_bn += 1
        assert n_bn == 3 * cfg["disc_layers"] and int(st["main.3.num_batches_tracked"]) == n_pass
