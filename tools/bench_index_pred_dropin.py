"""One iteration of train_index_prediction.py -- the reference's VQGANTextureAwareSpatialHierarchyInferenceModel
``feed_data`` + ``optimize_parameters`` (unmodified, staged under oracle/_ref/, built by its own __init__) -- at
configs/index_pred_net.yml's widths (vqvae_top / vqvae_bottom hierarchy, UNet 256 -> base 64, 18 heads of 64 channels
-> 512 classes) with random VQGAN checkpoints written to a temporary directory, four ways:

  mirror           the wrapper's code on the text2human_b200 mirrors (the frozen hierarchy's eval paths; UNet and
                   MultiHeadFCNHead as autograd nodes, NCHW tensors between them)
  reference_fp32   the same code on the reference's own arch classes, stock PyTorch eager
  reference_tf32   the same with cuDNN / cuBLAS TF32
  native           text2human_b200.index_pred_train.IndexPredTrainer: feed_data + optimize_parameters

at each ``--batches`` entry (default 4, the config's, and 16) with 512 x 256 images.  Each way runs in its own
process: warm-up iterations, then CUDA-event timing over ``--steps`` synchronised iterations and the peak allocated
memory; the ways alternate ``--repeats`` times and each reports the median, the range and the peak.  The card name,
power limit and maximum SM clock are read in the same run and printed with the numbers (one JSON line).
usage: python tools/bench_index_pred_dropin.py [--steps 10] [--warmup 3] [--repeats 3] [--precision fp32|fp16]
                                               [--batches 4 16]"""
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
from oracle import ref_loader as RL  # noqa: E402
from test_gpu_modules import HIER_OPT  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from tools.bench_sampler_dropin import gpu_context, timed  # noqa: E402

OPT = dict(HIER_OPT, is_train=True, encoder_in_channels=256, fc_in_channels=64, fc_in_index=4, fc_channels=64,
           fc_num_convs=1, fc_concat_input=False, fc_dropout_ratio=0.1, fc_num_classes=512, fc_align_corners=False,
           optimizer="Adam", lr=1e-4, weight_decay=0, loss_function="cross_entropy")
ARMS = ("mirror", "reference_fp32", "reference_tf32", "native")


def write_checkpoints(d):
    """random vqvae_top / vqvae_bottom checkpoints (codebooks spread like encoder outputs) -> their paths"""
    from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
    torch.manual_seed(7)
    with contextlib.redirect_stdout(io.StringIO()):
        h = HierarchyVQSpatialTextureAwareModel(HIER_OPT)
    cbt = R.codebooks(8, 18, 1024, 256, "trained")
    cbb = R.codebooks(9, 18, 512, 1024, "trained")
    for k in range(18):
        h.top_quantize.embedding_list[k].weight.data.copy_(cbt[k])
        h.bot_quantize.embedding_list[k].weight.data.copy_(cbb[k])
    top, bot = os.path.join(d, "vqvae_top.pth"), os.path.join(d, "vqvae_bottom.pth")
    torch.save(dict(encoder=h.top_encoder.state_dict(), decoder=h.decoder.state_dict(),
                    quantize=h.top_quantize.state_dict(), quant_conv=h.top_quant_conv.state_dict(),
                    post_quant_conv=h.top_post_quant_conv.state_dict()), top)
    torch.save(dict(bot_encoder=h.bot_encoder.state_dict(), bot_decoder_res=h.bot_decoder_res.state_dict(),
                    decoder=h.decoder.state_dict(), bot_quantize=h.bot_quantize.state_dict(),
                    bot_quant_conv=h.bot_quant_conv.state_dict(),
                    bot_post_quant_conv=h.bot_post_quant_conv.state_dict()), bot)
    return top, bot


def build_wrapper(archs, opt):
    ns = RL.install(archs, wrappers=())
    for sub in ("losses.accuracy", "losses.cross_entropy_loss"):
        if "models." + sub not in sys.modules:
            RL._exec("models." + sub, os.path.join(ns.root, "models", *sub.split(".")) + ".py")
    him = RL._exec("models.hierarchy_inference_model", os.path.join(ns.root, "models", "hierarchy_inference_model.py"))
    with contextlib.redirect_stdout(io.StringIO()):
        w = him.VQGANTextureAwareSpatialHierarchyInferenceModel(opt)
    for m, seed in ((w.guidance_encoder, 31), (w.index_decoder, 32)):
        m.load_state_dict(R.fill_state_dict(R.spec_of(m), seed), strict=True)
    return w


def run_arm(arm, B, a):
    ops.set_precision(a.precision)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = arm == "reference_tf32"
    data = dict(image=R.image(41, B, 3, 512, 256), texture_mask=R.blocky_mask(42, B, 512, 256, 16))
    with tempfile.TemporaryDirectory() as d:
        top, bot = write_checkpoints(d)
        w = build_wrapper("reference" if arm.startswith("reference") else "mirror",
                          dict(OPT, top_vae_path=top, bot_vae_path=bot))
    torch.manual_seed(1)
    if arm == "native":
        from text2human_b200.index_pred_train import IndexPredTrainer
        from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
        with contextlib.redirect_stdout(io.StringIO()):
            h = HierarchyVQSpatialTextureAwareModel(HIER_OPT)
        for n in ("top_encoder", "top_quant_conv", "top_quantize", "top_post_quant_conv", "bot_encoder",
                  "bot_quant_conv", "bot_quantize", "decoder", "bot_decoder_res", "bot_post_quant_conv"):
            getattr(h, n).load_state_dict(getattr(w, n).state_dict(), strict=True)
        tr = IndexPredTrainer(w.guidance_encoder.eval(), w.index_decoder.eval(), hierarchy=h.cuda().eval(),
                              lr=OPT["lr"])
        del w
        dev = {k: v.cuda() for k, v in data.items()}
        return timed(lambda: tr.optimize_parameters(dev), a.steps, a.warmup)

    def iteration():
        w.feed_data(data)
        w.optimize_parameters()
    return timed(iteration, a.steps, a.warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", nargs="+", type=int, default=[4, 16])
    ap.add_argument("--arm", choices=ARMS, help="run one way only (the script runs each in its own process)")
    a = ap.parse_args()
    assert torch.cuda.is_available()
    if a.arm:
        print(json.dumps(run_arm(a.arm, a.batches[0], a)))
        return
    res = dict(gpu_context(), precision=a.precision, steps=a.steps, warmup=a.warmup, repeats=a.repeats,
               workload="feed_data + optimize_parameters, index_pred_net.yml, 512x256 images")
    if not RL.available():
        res["error"] = "reference sources not staged (oracle/make_ref.py)"
        print(json.dumps(res))
        return
    for B in a.batches:
        runs = {arm: [] for arm in ARMS}
        for _ in range(a.repeats):            # the ways alternate, so that a slow spell of a shared host hits them all
            for arm in ARMS:
                out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps",
                                               str(a.steps), "--warmup", str(a.warmup), "--precision", a.precision,
                                               "--batches", str(B)], text=True)
                runs[arm].append(json.loads(out.strip().splitlines()[-1]))
                print(f"B {B} {arm}: {runs[arm][-1]}", file=sys.stderr, flush=True)
        key = f"B{B}_512x256"
        res[key] = {}
        for arm, rs in runs.items():
            ms = sorted(r["ms_per_step"] for r in rs)
            res[key][arm] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_range=[ms[0], ms[-1]],
                                 peak_mib=max(r["peak_mib"] for r in rs))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
