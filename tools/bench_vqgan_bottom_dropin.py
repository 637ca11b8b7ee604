"""One training step of the reference's HierarchyVQSpatialTextureAwareModel.optimize_parameters (unmodified, staged
under oracle/_ref/) at configs/vqvae_bottom.yml's shape (B 4, 512 x 256, the real widths, seeded weights, LPIPS
stubbed to zero), four ways:

  mirror      the wrapper's code on the text2human_b200 mirrors (Encoder, the 2x2-patch quantizer, DecoderRes, the
              decoder trunk with the bot_h residual and the Discriminator as autograd nodes)
  reference   the same code on the reference's own arch classes, stock PyTorch eager, fp32 and cuDNN/cuBLAS TF32
  native      text2human_b200.vqgan_bottom_train.HierarchyVQGANTrainer.optimize_parameters

Each way runs in its own process: warm-up steps, then CUDA-event timing over `--steps` synchronised steps, and the
peak allocated memory over the timed steps; the ways alternate `--repeats` times and each reports the median time,
the range and the peak.  The card name, power limit and maximum SM clock are read in the same run and printed with
the numbers (one JSON line).  `--profile` instead prints a torch.profiler table of one mirror step (to stderr).
usage: python tools/bench_vqgan_bottom_dropin.py [--steps 10] [--warmup 3] [--repeats 3] [--precision fp32|fp16]"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_sampler_dropin import gpu_context, timed  # noqa: E402
from bench_vqgan_bottom_train import OPT, batch, build_modules  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer  # noqa: E402

B, STEP = 4, 2
ARMS = ("mirror", "reference_fp32", "reference_tf32", "native")
BOT = ("bot_encoder", "bot_decoder_res", "bot_quantize", "bot_quant_conv", "bot_post_quant_conv")


def wrapper(archs, m, disc, td):
    """the reference wrapper built by its own __init__ (which reads the top checkpoint twice) on ``archs``"""
    ns = RL.install(archs, wrappers=("hierarchy_vqgan_model",))
    top = os.path.join(td, "vqvae_top.pth")
    torch.save(dict(encoder=m.top_encoder.state_dict(), decoder=m.decoder.state_dict(),
                    quantize=m.top_quantize.state_dict(), quant_conv=m.top_quant_conv.state_dict(),
                    post_quant_conv=m.top_post_quant_conv.state_dict(), discriminator=disc.state_dict()), top)
    with contextlib.redirect_stdout(io.StringIO()):
        w = ns.hierarchy_vqgan_model.HierarchyVQSpatialTextureAwareModel(dict(OPT, top_vae_path=top))
    for n in BOT:
        getattr(w, n).load_state_dict(getattr(m, n).state_dict(), strict=True)
    return w


def run_arm(arm, a):
    """one way, in a process of its own: the peak then holds only this arm's model, gradients, optimiser state and
    step temporaries (plus the batch)"""
    dev = torch.device("cuda:0")
    ops.set_precision(a.precision)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = arm == "reference_tf32"
    m, disc = build_modules()
    data = batch(B, dev)
    torch.manual_seed(1)
    if arm == "native":
        tr = HierarchyVQGANTrainer(m.to(dev), disc.to(dev), disc_start_step=OPT["disc_start_step"])
        return timed(lambda: tr.optimize_parameters(data, STEP), a.steps, a.warmup)
    with tempfile.TemporaryDirectory() as td:
        w = wrapper("mirror" if arm == "mirror" else "reference", m, disc, td)
    del m, disc
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for _ in range(a.warmup):
            w.optimize_parameters(data, STEP)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            w.optimize_parameters(data, STEP)
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cpu_time_total", row_limit=40), file=sys.stderr)
        return {}
    return timed(lambda: w.optimize_parameters(data, STEP), a.steps, a.warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--arm", choices=ARMS, help="run one way only (the script runs each in its own process)")
    ap.add_argument("--profile", action="store_true", help="print a torch.profiler table of one mirror step")
    a = ap.parse_args()
    assert torch.cuda.is_available()
    if a.profile:
        a.arm = a.arm or "mirror"
    if a.arm:
        print(json.dumps(run_arm(a.arm, a)))
        return
    res = dict(gpu_context(), shape=dict(B=B, H=512, W=256, config="vqvae_bottom.yml widths"),
               precision=a.precision, steps=a.steps, warmup=a.warmup)
    if not RL.available():
        res["error"] = "reference sources not staged (oracle/make_ref.py)"
        print(json.dumps(res))
        return
    runs = {arm: [] for arm in ARMS}
    for _ in range(a.repeats):            # the ways alternate, so that a slow spell of a shared host hits them all
        for arm in ARMS:
            out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps",
                                           str(a.steps), "--warmup", str(a.warmup), "--precision", a.precision],
                                          text=True)
            runs[arm].append(json.loads(out.strip().splitlines()[-1]))
    for arm, rs in runs.items():
        ms = sorted(r["ms_per_step"] for r in rs)
        res[arm] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_range=[ms[0], ms[-1]],
                        peak_mib=max(r["peak_mib"] for r in rs))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
