"""Hierarchical VQGAN bottom-level training step (configs/vqvae_bottom.yml: top ch 128 x [1,1,2,2,4], bottom ch 128 x
[1,1,2,4], embed_dim 256, 18 x 512 codes of 2x2 x 256, ndf 64, 512 x 256 images) timed with CUDA events after a
warm-up:

  * native: HierarchyVQGANTrainer.optimize_parameters in the fp32 (3-product) and fp16 (1-product) modes, B = 16 in
    micro-batches of 4 (the config's batch);
  * reference: the reference's own HierarchyVQSpatialTextureAwareModel (constructor, configure_optimizers,
    optimize_parameters, LPIPS stubbed to zero) in stock PyTorch eager, fp32 (TF32 off) and with cuDNN convolutions in
    TF32, when oracle/_ref is staged.  Its top checkpoint is written to a temporary directory.

Prints one JSON line: per batch size and arm ms/step, img/s, launches/step (native), peak memory, and the algorithmic
GFLOP of one step (convolution and attention FLOPs counted by torch's FlopCounterMode over the restatement on meta
tensors: the frozen top path forward; the bottom encoder, DecoderRes and decoder levels 3..0 forward and backward;
three discriminator passes and their backward); plus the GPU's name, power limit and max SM clock read in the same run.
usage: python tools/bench_vqgan_bottom_train.py [--batches 4 16] [--steps 5] [--warmup 2] [--no-reference]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel  # noqa: E402
from text2human_b200.vqgan_arch import Discriminator  # noqa: E402
from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer  # noqa: E402

OPT = dict(embed_dim=256, n_embed=1024, codebook_spatial_size=2,
           bot_n_embed=512, bot_double_z=False, bot_z_channels=256, bot_resolution=512, bot_in_channels=3,
           bot_out_ch=3, bot_ch=128, bot_ch_mult=[1, 1, 2, 4], bot_num_res_blocks=2, bot_attn_resolutions=[64],
           bot_dropout=0.0,
           top_double_z=False, top_z_channels=256, top_resolution=512, top_in_channels=3, top_out_ch=3, top_ch=128,
           top_ch_mult=[1, 1, 2, 2, 4], top_num_res_blocks=2, top_attn_resolutions=[32], top_dropout=0.0,
           fix_decoder=False, disc_layers=3, disc_weight_max=1, disc_start_step=1, n_channels=3, ndf=64,
           perceptual_weight=1.0, diff_aug=True, lr=1e-4)
NETS = ("top_encoder", "decoder", "top_quant_conv", "top_post_quant_conv", "bot_encoder", "bot_decoder_res",
        "bot_quant_conv", "bot_post_quant_conv")
H, W, MICRO = 512, 256, 4


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=plim, sm_clock_max=clk)


def algorithmic_flops(B):
    from torch.utils.flop_counter import FlopCounterMode
    from oracle import vqgan_ref as V
    from oracle import vqgan_train_ref as TR
    m, disc = build_modules()

    def meta(mod, prefix, grad):
        return {prefix + k: torch.empty(v.shape, device="meta",
                                        requires_grad=grad and v.is_floating_point() and "running" not in k)
                for k, v in mod.state_dict().items()}
    sd = {}
    for n in NETS:
        sd.update(meta(getattr(m, n), n + ".", n.startswith("bot_") or n == "decoder"))
    sdd = meta(disc, "", True)
    x = torch.empty((B, 3, H, W), device="meta")
    with FlopCounterMode(display=False) as fc:
        with torch.no_grad():
            ht = V.conv(sd, "top_quant_conv", V.encoder(sd, x, "top_encoder."), padding=0)
            h4 = V.decoder(sd, V.conv(sd, "top_post_quant_conv", ht, padding=0), "decoder.", stop_after_level=4)
        hb = V.conv(sd, "bot_quant_conv", V.encoder(sd, x, "bot_encoder."), padding=0)   # the quantizer: no FLOPs
        bot_h = V.decoder_res(sd, V.conv(sd, "bot_post_quant_conv", hb, padding=0), "bot_decoder_res.")
        h = h4.detach() + bot_h
        for lv in reversed(range(4)):
            lp = f"decoder.up.{lv}."
            for bk in range(3):
                h = V.resnet_block(sd, f"{lp}block.{bk}.", h)
            if lv:
                h = V.conv(sd, lp + "upsample.conv", torch.nn.functional.interpolate(h, scale_factor=2.0))
        xrec = V.conv(sd, "decoder.conv_out", V.swish(V.norm(sd, "decoder.norm_out", h)))
        g = TR.discriminator(sdd, xrec, prefix="main.").sum()
        torch.autograd.grad(g + xrec.sum(), [v for v in list(sd.values()) + list(sdd.values()) if v.requires_grad],
                            allow_unused=True)
        for _ in range(2):
            TR.discriminator(sdd, xrec.detach(), prefix="main.").sum().backward()
    return fc.get_total_flops()


def build_modules():
    with contextlib.redirect_stdout(io.StringIO()):
        m = HierarchyVQSpatialTextureAwareModel(OPT)
    for i, n in enumerate(NETS):
        getattr(m, n).load_state_dict(R.fill_state_dict(R.spec_of(getattr(m, n)), 31 + i), strict=True)
    for q, ne, d, s in ((m.top_quantize, 1024, 256, 41), (m.bot_quantize, 512, 1024, 42)):
        cb = R.codebooks(s, 18, ne, d, "trained")
        for k, e in enumerate(q.embedding_list):
            e.weight.data.copy_(cb[k])
    disc = Discriminator(3, OPT["ndf"], n_layers=3)
    disc.load_state_dict(R.fill_state_dict(R.spec_of(disc), 43), strict=True)
    return m, disc


def batch(B, dev):
    return dict(image=R.image(44, B, 3, H, W).to(dev), texture_mask=R.blocky_mask(45, B, H, W, 32).to(dev))


def timed(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(warmup + i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def native(B, prec, dev, steps, warmup):
    ops.set_precision(prec)
    m, disc = build_modules()
    tr = HierarchyVQGANTrainer(m.to(dev), disc.to(dev), disc_start_step=1, micro_batch=min(B, MICRO))
    data = batch(B, dev)
    torch.cuda.reset_peak_memory_stats()
    l0 = ops.COUNTERS["launches"]
    ms = timed(lambda i: tr.optimize_parameters(data, 2 + i), steps, warmup)
    launches = (ops.COUNTERS["launches"] - l0) // (steps + warmup)
    out = dict(ms=ms, launches=launches, losses=tr.losses(), peak_gib=torch.cuda.max_memory_allocated() / 2**30)
    del tr, m, disc
    torch.cuda.empty_cache()
    return out


def reference(B, tf32, dev, steps, warmup):
    from oracle import ref_loader as RL
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ns = RL.install("reference", wrappers=("hierarchy_vqgan_model",))
        m, disc = build_modules()
        with tempfile.TemporaryDirectory() as td:
            top = os.path.join(td, "vqvae_top.pth")
            torch.save(dict(encoder=m.top_encoder.state_dict(), decoder=m.decoder.state_dict(),
                            quantize=m.top_quantize.state_dict(), quant_conv=m.top_quant_conv.state_dict(),
                            post_quant_conv=m.top_post_quant_conv.state_dict(), discriminator=disc.state_dict()), top)
            with contextlib.redirect_stdout(io.StringIO()):
                w = ns.hierarchy_vqgan_model.HierarchyVQSpatialTextureAwareModel(dict(OPT, top_vae_path=top))
        for n in ("bot_encoder", "bot_decoder_res", "bot_quantize", "bot_quant_conv", "bot_post_quant_conv"):
            getattr(w, n).load_state_dict(getattr(m, n).state_dict(), strict=True)
        data = batch(B, dev)
        torch.cuda.reset_peak_memory_stats()
        try:
            ms = timed(lambda i: w.optimize_parameters(data, 2 + i), steps, warmup)
        except torch.cuda.OutOfMemoryError:
            return dict(ms=None, oom=True)
        out = dict(ms=ms, peak_gib=torch.cuda.max_memory_allocated() / 2**30)
        del w
        torch.cuda.empty_cache()
        return out
    finally:
        torch.backends.cudnn.allow_tf32 = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    from oracle import ref_loader as RL
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = dict(gpu_info(), workload=f"vqvae_bottom training step, 512x256, micro-batches of {MICRO}", batches={})
    for B in a.batches:
        flops = algorithmic_flops(B)
        res = {"algorithmic_gflop_per_step": round(flops / 1e9, 1)}
        arms = [("native_fp32", lambda: native(B, "fp32", dev, a.steps, a.warmup)),
                ("native_fp16", lambda: native(B, "fp16", dev, a.steps, a.warmup))]
        if RL.available() and not a.no_reference:
            arms += [("eager_fp32", lambda: reference(B, False, dev, a.steps, a.warmup)),
                     ("eager_tf32", lambda: reference(B, True, dev, a.steps, a.warmup))]
        for name, fn in arms:
            r = fn()
            if r["ms"] is not None:
                r.update(img_per_s=round(B / r["ms"] * 1e3, 2), tflops=round(flops / r["ms"] / 1e9, 2),
                         ms=round(r["ms"], 2))
            res[name] = r
        ops.set_precision("fp32")
        out["batches"][B] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
