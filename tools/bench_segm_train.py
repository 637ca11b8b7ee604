"""Parsing-tokenizer training step (configs/parsing_token.yml: ch 64, ch_mult [1,1,2,2,4], one res block, 24 classes,
1024 x 32 codebook, 512 x 256 parsing maps) timed with CUDA events after a warm-up:

  * native: SegmTokenizerTrainer.optimize_parameters in the fp32 (3-product) and fp16 (1-product) modes;
  * reference: the reference's own VQSegmentationModel.optimize_parameters in stock PyTorch eager, fp32 (TF32 off)
    and with PyTorch's default TF32 settings (cuDNN convolutions in TF32), when oracle/_ref is staged.

Prints one JSON line: per batch size and arm ms/step, img/s, launches/step (native), algorithmic TFLOP/s (conv and
attention FLOPs of forward + backward, counted by torch's FlopCounterMode over the restatement on meta tensors), and
for the native arms the per-launch tap-GEMM time split (ops.profile_tapgemm, one extra step); plus the GPU's name
and power limit read in the same run.
usage: python tools/bench_segm_train.py [--batches 4 16] [--steps 10] [--warmup 3] [--no-reference]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import segm_recipes as SG  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.segm_train import NETS, SegmTokenizerModel, SegmTokenizerTrainer  # noqa: E402

CFG = dict(ch=64, num_res_blocks=1, attn_resolutions=[16], ch_mult=[1, 1, 2, 2, 4], in_channels=24, out_ch=24,
           resolution=512, z_channels=32, double_z=False, dropout=0.0, n_embed=1024, embed_dim=32,
           num_segm_classes=24, lr=4.5e-05)
H, W = 512, 256


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk = (s.strip() for s in out[0].split(","))
    return dict(gpu=name, power_limit=plim, sm_clock_max=clk)


def algorithmic_flops(B):
    """conv + attention FLOPs of one forward + backward at batch B (the input gets no gradient)"""
    from torch.utils.flop_counter import FlopCounterMode
    from oracle import vqgan_ref as V
    with contextlib.redirect_stdout(io.StringIO()):
        m = SegmTokenizerModel(CFG)
    sd = {f"{n}.{k}": torch.empty(v.shape, device="meta", requires_grad=True)
          for n in ("encoder", "decoder", "quant_conv", "post_quant_conv") for k, v in getattr(m, n).state_dict().items()}
    x = torch.empty((B, 24, H, W), device="meta")
    with FlopCounterMode(display=False) as fc:
        z = V.conv(sd, "quant_conv", V.encoder(sd, x, "encoder."), padding=0)
        y = V.decoder(sd, V.conv(sd, "post_quant_conv", z, padding=0), "decoder.")   # the quantizer: no FLOPs
        y.sum().backward()
    return fc.get_total_flops()


def make_weights(B):
    with contextlib.redirect_stdout(io.StringIO()):
        m = SegmTokenizerModel(CFG)
    sd = {n: R.fill_state_dict(R.spec_of(getattr(m, n)), s) for n, s in
          (("encoder", 11), ("decoder", 12), ("quant_conv", 13), ("post_quant_conv", 14))}
    cb = R.codebooks(15, 1, CFG["n_embed"], CFG["embed_dim"], "trained")[0]
    return sd, cb, SG.segm_labels(16, B, H, W, tile=16)


def load(obj, sd, cb, dev):
    for n, d in sd.items():
        getattr(obj, n).load_state_dict({k: v.to(dev) for k, v in d.items()}, strict=True)
    with torch.no_grad():
        obj.quantize.embedding.weight.copy_(cb)


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def native(B, prec, sd, cb, segm, dev, steps, warmup):
    ops.set_precision(prec)
    m = SegmTokenizerModel(CFG).to(dev)
    load(m, sd, cb, dev)
    tr = SegmTokenizerTrainer(m, lr=CFG["lr"])
    data = dict(segm=segm.to(dev))
    tr.optimize_parameters(data)
    torch.cuda.synchronize()
    l0 = ops.COUNTERS["launches"]
    ms = timed(lambda: tr.optimize_parameters(data), steps, warmup)
    launches = (ops.COUNTERS["launches"] - l0) // (steps + warmup)
    losses = tr.losses()
    # per-launch split of the tap-GEMM / weight-gradient time, one profiled step
    ops.profile_tapgemm(True)
    tr.optimize_parameters(data)
    torch.cuda.synchronize()
    recs = ops.profile_records()
    ops.profile_tapgemm(False)
    by_shape = defaultdict(lambda: [0, 0.0, 0.0])
    for algo, _, s0, s1, shape in recs:
        t = s0.elapsed_time(s1)
        e = by_shape[str(shape)]
        e[0] += 1
        e[1] += t
        e[2] += algo
    top = sorted(by_shape.items(), key=lambda kv: -kv[1][1])[:8]
    gemm_ms = sum(v[1] for v in by_shape.values())
    del tr, m
    torch.cuda.empty_cache()
    return dict(ms=ms, launches=launches, losses=losses, gemm_ms_profiled=gemm_ms, gemm_launches=len(recs),
                top_gemm=[dict(shape=k, n=v[0], ms=round(v[1], 3), tflops=round(v[2] / v[1] / 1e9, 1))
                          for k, v in top])


def reference(B, tf32, sd, cb, segm, dev, steps, warmup):
    from oracle import ref_loader as RL
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False      # PyTorch's default either way
    try:
        ns = RL.install("reference", wrappers=("vqgan_model",))
        with contextlib.redirect_stdout(io.StringIO()):
            w = ns.vqgan_model.VQSegmentationModel(CFG)
        load(w, sd, cb, dev)
        data = dict(segm=segm.to(dev))
        ms = timed(lambda: w.optimize_parameters(data, 0), steps, warmup)
        losses = {k.split("/")[1]: float(v) for k, v in w.log_dict.items()}
        del w
        torch.cuda.empty_cache()
        return dict(ms=ms, losses=losses)
    finally:
        torch.backends.cudnn.allow_tf32 = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    from oracle import ref_loader as RL
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = dict(gpu_info(), workload="parsing tokenizer training step, 512x256, ch 64", batches={})
    for B in a.batches:
        sd, cb, segm = make_weights(B)
        flops = algorithmic_flops(B)
        res = {"algorithmic_gflop_per_step": round(flops / 1e9, 1)}
        arms = [("native_fp32", lambda: native(B, "fp32", sd, cb, segm, dev, a.steps, a.warmup)),
                ("native_fp16", lambda: native(B, "fp16", sd, cb, segm, dev, a.steps, a.warmup))]
        if RL.available() and not a.no_reference:
            arms += [("eager_fp32", lambda: reference(B, False, sd, cb, segm, dev, a.steps, a.warmup)),
                     ("eager_tf32", lambda: reference(B, True, sd, cb, segm, dev, a.steps, a.warmup))]
        for name, fn in arms:
            r = fn()
            r.update(img_per_s=round(B / r["ms"] * 1e3, 2), tflops=round(flops / r["ms"] / 1e9, 2),
                     ms=round(r["ms"], 3))
            res[name] = r
        ops.set_precision("fp32")
        out["batches"][B] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
