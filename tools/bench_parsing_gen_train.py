"""Parsing-generator training step (configs/parsing_gen.yml: ShapeAttrEmbedding dim 8 -> 128, ShapeUNet base 64 with
5 stages, FCNHead 64 channels -> 24 classes) timed with CUDA events after a warm-up, at the reference's training
shape (batch 8, 256 x 128: 512 x 256 parsing maps with downsample_factor 2) and at batch 16, 512 x 256:

  * native: ParsingGenTrainer.optimize_parameters in the fp32 (3-product) and fp16 (1-product) modes;
  * reference: the reference's own ParsingGenModel.optimize_parameters in stock PyTorch eager, fp32 (TF32 off) and
    with cuDNN convolutions in TF32, when oracle/_ref is staged.

Prints one JSON line: per shape and arm ms/step, img/s, launches/step (native), algorithmic TFLOP/s (conv FLOPs of
forward + backward, counted by torch's FlopCounterMode over the restatement on meta tensors), for the native arms the
per-launch tap-GEMM time split of one profiled step; plus the GPU's name, power limit and maximum SM clock read in the
same run.
usage: python tools/bench_parsing_gen_train.py [--shapes 8x256x128 16x512x256] [--steps 10] [--warmup 3]"""
import argparse
import contextlib
import io
import json
import os
import sys
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import parsing_gen_recipes as P  # noqa: E402
import parsing_gen_train_recipes as PT  # noqa: E402
from bench_segm_train import gpu_info, timed  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.parsing_gen_train import ParsingGenNets, ParsingGenTrainer  # noqa: E402

OPT = dict(embedder_dim=8, embedder_out_dim=128, attr_class_num=P.CLS_NUM, encoder_in_channels=1, fc_in_channels=64,
           fc_in_index=4, fc_channels=64, fc_num_convs=1, fc_concat_input=False, fc_dropout_ratio=0.1,
           fc_num_classes=24, fc_align_corners=False, lr=1e-4, weight_decay=0, is_train=True)
PARTS = ("attr_embedder", "parsing_encoder", "parsing_decoder")


def algorithmic_flops(B, H, W):
    from torch.utils.flop_counter import FlopCounterMode
    from oracle import parsing_gen_train_ref as TR
    nets = ParsingGenNets(OPT)
    sds = [{k: torch.empty(v.shape, device="meta", requires_grad=not k.endswith(("running_mean", "running_var",
                                                                                "num_batches_tracked")))
            for k, v in getattr(nets, n).state_dict().items()} for n in PARTS]
    data = dict(densepose=torch.empty((B, 1, H, W), device="meta"),
                attr=torch.zeros((B, 15), dtype=torch.int64, device="meta"),
                segm=torch.zeros((B, H, W), dtype=torch.int64, device="meta"))
    with FlopCounterMode(display=False) as fc:
        loss, _ = TR.train_loss(sds[0], sds[1], sds[2], data, torch.ones((B, 64), device="meta"), P.CLS_NUM,
                                TR.running_stats(sds[1]), TR.running_stats(sds[2]))
        loss.backward()
    return fc.get_total_flops()


def make_inputs(B, H, W):
    nets = ParsingGenNets(OPT)
    sds = [R.fill_state_dict(R.spec_of(getattr(nets, n)), s) for n, s in zip(PARTS, (21, 22, 23))]
    return sds, PT.batch(dict(PT.TRAIN_SEEDS, pose=24, attr=25, labels=26), (B, H, W))


def native(prec, sds, data, dev, steps, warmup):
    ops.set_precision(prec)
    nets = ParsingGenNets(OPT)
    for n, sd in zip(PARTS, sds):
        getattr(nets, n).load_state_dict(sd, strict=True)
    nets = nets.to(dev).eval()
    tr = ParsingGenTrainer(nets.attr_embedder, nets.parsing_encoder, nets.parsing_decoder, lr=OPT["lr"])
    data = {k: v.to(dev) for k, v in data.items()}
    tr.optimize_parameters(data)
    torch.cuda.synchronize()
    l0 = ops.COUNTERS["launches"]
    ms = timed(lambda: tr.optimize_parameters(data), steps, warmup)
    launches = (ops.COUNTERS["launches"] - l0) // (steps + warmup)
    losses = tr.losses()
    ops.profile_tapgemm(True)
    tr.optimize_parameters(data)
    torch.cuda.synchronize()
    recs = ops.profile_records()
    ops.profile_tapgemm(False)
    by_shape = defaultdict(lambda: [0, 0.0, 0.0])
    for algo, _, s0, s1, shape in recs:
        e = by_shape[str(shape)]
        e[0] += 1
        e[1] += s0.elapsed_time(s1)
        e[2] += algo
    top = sorted(by_shape.items(), key=lambda kv: -kv[1][1])[:8]
    del tr, nets
    torch.cuda.empty_cache()
    return dict(ms=ms, launches=launches, losses=losses, gemm_ms_profiled=sum(v[1] for v in by_shape.values()),
                gemm_launches=len(recs),
                top_gemm=[dict(shape=k, n=v[0], ms=round(v[1], 3), tflops=round(v[2] / v[1] / 1e9, 1))
                          for k, v in top])


def reference(tf32, sds, data, dev, steps, warmup):
    from oracle import parsing_gen_ref as PR
    from oracle import ref_loader as RL
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ns = PR.install("reference", wrappers=())
        for sub in ("losses.accuracy", "losses.cross_entropy_loss", "parsing_gen_model"):
            name = "models." + sub
            if name not in sys.modules:
                RL._exec(name, os.path.join(ns.root, "models", *sub.split(".")) + ".py")
        sys.modules["mmcv"].imwrite = getattr(sys.modules["mmcv"], "imwrite", None)
        with contextlib.redirect_stdout(io.StringIO()):
            m = sys.modules["models.parsing_gen_model"].ParsingGenModel(OPT)
        for n, sd in zip(PARTS, sds):
            getattr(m, n).load_state_dict(sd, strict=True)
        m.feed_data(data)
        ms = timed(m.optimize_parameters, steps, warmup)
        loss = float(m.log_dict["loss_total"].detach())
        del m
        torch.cuda.empty_cache()
        return dict(ms=ms, losses=dict(loss_total=loss))
    finally:
        torch.backends.cudnn.allow_tf32 = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["8x256x128", "16x512x256"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    from oracle import ref_loader as RL
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = dict(gpu_info(), workload="parsing generator training step (parsing_gen.yml nets)", shapes={})
    for s in a.shapes:
        B, H, W = (int(v) for v in s.split("x"))
        sds, data = make_inputs(B, H, W)
        flops = algorithmic_flops(B, H, W)
        res = {"algorithmic_gflop_per_step": round(flops / 1e9, 1)}
        arms = [("native_fp32", lambda: native("fp32", sds, data, dev, a.steps, a.warmup)),
                ("native_fp16", lambda: native("fp16", sds, data, dev, a.steps, a.warmup))]
        if RL.available() and not a.no_reference:
            arms += [("eager_fp32", lambda: reference(False, sds, data, dev, a.steps, a.warmup)),
                     ("eager_tf32", lambda: reference(True, sds, data, dev, a.steps, a.warmup))]
        for name, fn in arms:
            r = fn()
            r.update(img_per_s=round(B / r["ms"] * 1e3, 2), tflops=round(flops / r["ms"] / 1e9, 2),
                     ms=round(r["ms"], 3))
            res[name] = r
        ops.set_precision("fp32")
        out["shapes"][s] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
