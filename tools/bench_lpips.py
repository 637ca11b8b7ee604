"""LPIPS (VGG16, lpips 0.1.4) forward + backward and the VQGAN training steps with and without the perceptual loss,
timed with CUDA events after a warm-up:

  * LPIPS value and d/d in1 at B = 16, 512 x 256: native (text2human_b200.lpips, fp32 3-product and fp16 1-product
    modes) against the eager torch restatement (oracle/lpips_ref.py: F.conv2d on cuDNN) in fp32 with TF32 off and
    with cuDNN TF32;
  * VQGANTrainer.optimize_parameters at config 5's shapes (configs/vqvae_top.yml, 512 x 256, one micro-batch of 8,
    fp16 operands) and HierarchyVQGANTrainer.optimize_parameters (configs/vqvae_bottom.yml, B = 4), each with
    ``perceptual=None`` and with an LPIPS module (seeded weights, tests/lpips_recipes.py);
  * the algorithmic GFLOP of one LPIPS forward + backward (torch FlopCounterMode over the restatement on meta tensors:
    the trunk on in0 and in1, the data gradient for in1).

Prints one JSON line, with the GPU's name, power limit and max SM clock read in the same run.
usage: python tools/bench_lpips.py [--batch 16] [--steps 5] [--warmup 2]"""
import argparse
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import golden_recipes as R  # noqa: E402
import lpips_recipes as LR  # noqa: E402
from bench_vqgan_bottom_train import batch as bot_batch, build_modules as bot_modules, gpu_info, timed  # noqa: E402
from oracle import lpips_ref  # noqa: E402
from text2human_b200 import ops  # noqa: E402

H, W = 512, 256


def lpips_gflop(B):
    from torch.utils.flop_counter import FlopCounterMode
    sd = {k: torch.empty(v.shape, device="meta") for k, v in LR.state_dict().items()}
    x0 = torch.empty((B, 3, H, W), device="meta")
    x1 = torch.empty((B, 3, H, W), device="meta", requires_grad=True)
    with FlopCounterMode(display=False) as fc:
        torch.autograd.grad(lpips_ref.lpips(sd, x0, x1).sum(), x1)
    return fc.get_total_flops() / 1e9


def lpips_arms(B, dev, steps, warmup):
    in0, in1 = R.image(51, B, 3, H, W).to(dev), R.image(52, B, 3, H, W).to(dev)
    out = {}
    for prec in ("fp32", "fp16"):
        ops.set_precision(prec)
        m = LR.mirror(dev)
        g = torch.zeros_like(in1)
        torch.cuda.reset_peak_memory_stats()
        ms = timed(lambda i: m.run(in0, in1, g=g), steps, warmup)
        out[f"native_{prec}"] = dict(ms=ms, img_s=B * 1000.0 / ms, peak_gib=torch.cuda.max_memory_allocated() / 2**30)
        del m
    ops.set_precision("fp32")
    sd = {k: v.to(dev) for k, v in LR.state_dict().items()}

    def eager(_):
        x1 = in1.clone().requires_grad_(True)
        torch.autograd.grad(lpips_ref.lpips(sd, in0, x1).sum(), x1)
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, tf32 in (("eager_fp32", False), ("eager_tf32", True)):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.cuda.reset_peak_memory_stats()
        ms = timed(eager, steps, warmup)
        out[name] = dict(ms=ms, img_s=B * 1000.0 / ms, peak_gib=torch.cuda.max_memory_allocated() / 2**30)
    torch.backends.cudnn.allow_tf32 = False
    return out


def top_step(dev, perceptual, steps, warmup, B=8):
    from bench import VQVAE_TOP
    from text2human_b200.pipeline import VQImageSegmTextureModel
    from text2human_b200.vqgan_arch import Discriminator
    from text2human_b200.vqgan_train import VQGANTrainer
    torch.manual_seed(5)
    with contextlib.redirect_stdout(sys.stderr):
        model = VQImageSegmTextureModel(VQVAE_TOP).to(dev)
    disc = Discriminator(3, 64, n_layers=3).to(dev)
    cb = R.codebooks(7, 18, 1024, 256, "trained")
    with torch.no_grad():
        for k, e in enumerate(model.quantize.embedding_list):
            e.weight.copy_(cb[k])
    tr = VQGANTrainer(model, disc, lr=1e-4, disc_start_step=0, micro_batch=B, perceptual=perceptual)
    data = dict(image=R.image(300, B, 3, H, W).to(dev), texture_mask=R.blocky_mask(300, B, H, W, 32).to(dev))
    gen = torch.Generator(device=dev).manual_seed(17)
    torch.cuda.reset_peak_memory_stats()
    ms = timed(lambda i: tr.optimize_parameters(data, 2 + i, gen), steps, warmup)
    return dict(ms=ms, img_s=B * 1000.0 / ms, peak_gib=torch.cuda.max_memory_allocated() / 2**30,
                perceptual=tr.losses()["perceptual"])


def bottom_step(dev, perceptual, steps, warmup, B=4):
    from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer
    m, disc = bot_modules()
    tr = HierarchyVQGANTrainer(m.to(dev), disc.to(dev), disc_start_step=1, micro_batch=B, perceptual=perceptual)
    data = bot_batch(B, dev)
    torch.cuda.reset_peak_memory_stats()
    ms = timed(lambda i: tr.optimize_parameters(data, 2 + i), steps, warmup)
    return dict(ms=ms, img_s=B * 1000.0 / ms, peak_gib=torch.cuda.max_memory_allocated() / 2**30,
                perceptual=tr.losses()["perceptual"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_lpips.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    res = dict(gpu_info(), batch=a.batch, H=H, W=W, lpips_gflop_per_image=lpips_gflop(1))
    res["lpips_fwd_bwd"] = lpips_arms(a.batch, dev, a.steps, a.warmup)
    res["top_step_fp16_b8"], res["bottom_step_fp16_b4"] = {}, {}
    ops.set_precision("fp16")
    for label, lp in (("no_lpips", None), ("lpips", LR.mirror(dev))):
        res["top_step_fp16_b8"][label] = top_step(dev, lp, a.steps, a.warmup)
        torch.cuda.empty_cache()
        res["bottom_step_fp16_b4"][label] = bottom_step(dev, lp, a.steps, a.warmup)
        torch.cuda.empty_cache()
    ops.set_precision("fp32")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
