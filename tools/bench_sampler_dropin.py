"""One training step of the reference's TransformerTextureAwareModel.optimize_parameters (unmodified, staged under
oracle/_ref/) at configs/sampler.yml's shape (B 4, 512 tokens, 24 layers, 512 wide, 8 heads, 18 x 1024 classes),
three ways:

  mirror      the wrapper's code on the text2human_b200 mirrors (TransformerMultiHead as one autograd node)
  reference   the same code on the reference's own arch classes, stock PyTorch eager, fp32 and cuDNN/cuBLAS TF32
  native      text2human_b200.transformer_train.SamplerTrainer.optimize_parameters

Each way runs in its own process: warm-up steps, then CUDA-event timing over `--steps` synchronised steps, and the
peak allocated memory over the timed steps (model, gradients, optimiser state, batch and step temporaries); the
ways alternate `--repeats` times and each reports the median time, the range and the peak.  The
card name, power limit and maximum SM clock are read in the same run and printed with the numbers (one JSON line).
usage: python tools/bench_sampler_dropin.py [--steps 10] [--warmup 3] [--repeats 3] [--precision fp32|fp16]"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.transformer_train import SamplerTrainer, targets_from_gt_list  # noqa: E402

CFG = dict(codebook_size=18432, segm_codebook_size=1024, texture_codebook_size=18, bert_n_emb=512,
           bert_n_layers=24, bert_n_head=8, block_size=512, latent_shape=[32, 16], embd_pdrop=0.0,
           resid_pdrop=0.0, attn_pdrop=0.0, num_head=18)
B = 4


def gpu_context():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True)
        name, power, clock = [s.strip() for s in out.splitlines()[0].split(",")]
    except (OSError, subprocess.CalledProcessError, ValueError):
        name, power, clock = torch.cuda.get_device_name(), "unknown", "unknown"
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return dict(ms_per_step=round(e0.elapsed_time(e1) / steps, 3),
                peak_mib=round(torch.cuda.max_memory_allocated() / 2 ** 20, 1))


def wrapper(ns, net, batch):
    """a stand-in `self` with exactly the attributes optimize_parameters / _train_loss read (its __init__ would also
    load two VAE checkpoints, which the step does not use); the methods are the reference's own"""
    x_0, gt_list, segm, tex = batch
    w = types.SimpleNamespace(_denoise_fn=net, input_indices=x_0, gt_indices_list=gt_list, segm_tokens=segm,
                              texture_tokens=tex, num_timesteps=1000, mask_id=CFG["codebook_size"],
                              loss_type="reweighted_elbo", mask_schedule="random", log_dict={},
                              optimizer=torch.optim.Adam([p for p in net.parameters() if p.requires_grad], 1e-4,
                                                         weight_decay=0))
    return RL.bind(ns.transformer_model.TransformerTextureAwareModel, w,
                   ["optimize_parameters", "_train_loss", "sample_time", "q_sample"])


ARMS = ("mirror", "reference_fp32", "reference_tf32", "native")


def run_arm(arm, a):
    """one way, in a process of its own: the peak then holds only this arm's model, gradients, optimiser state and
    step temporaries (plus the batch)"""
    dev = torch.device("cuda:0")
    ops.set_precision(a.precision)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = arm == "reference_tf32"
    x_0, gt_list, segm, tex = R.sampler_train_batch(6, B=B, cfg=CFG)
    batch = (x_0.to(dev), [g.to(dev) for g in gt_list], segm.to(dev), tex.to(dev))
    ns = RL.install("mirror" if arm in ("mirror", "native") else "reference", wrappers=("transformer_model",))
    net = ns.transformer_arch.TransformerMultiHead(**CFG)
    net.load_state_dict(R.fill_state_dict(R.spec_of(net), 5), strict=True)
    net.to(dev)
    torch.manual_seed(1)
    if arm == "native":
        tr = SamplerTrainer(net)
        own = targets_from_gt_list(batch[1])
        return timed(lambda: tr.optimize_parameters(batch[0], own, batch[2], batch[3]), a.steps, a.warmup)
    return timed(wrapper(ns, net, batch).optimize_parameters, a.steps, a.warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--arm", choices=ARMS, help="run one way only (the script runs each in its own process)")
    a = ap.parse_args()
    assert torch.cuda.is_available()
    if a.arm:
        print(json.dumps(run_arm(a.arm, a)))
        return
    res = dict(gpu_context(), shape=dict(B=B, T=512, layers=24, width=512, heads=8, classes="18x1024"),
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
