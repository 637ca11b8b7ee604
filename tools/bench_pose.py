"""Pose -> image generation (configs/sample_from_pose.yml sizes, 512 x 256) timed with CUDA events after a warm-up:

  * parsing generation (pose + shape attributes -> parsing map: ShapeAttrEmbedding -> ShapeUNet -> FCNHead -> argmax)
    per batch size: native (libt2h) in the fp32 (3-product) and fp16 (1-product) modes, and the reference's own
    classes (oracle/_ref, loaded by oracle/parsing_gen_ref.install with ref_loader's mmcv / mmseg stand-ins) in
    stock PyTorch eager, fp32 (TF32 off) and with TF32 convolutions / matmuls;
  * the whole SampleFromPoseModel.generate (parsing map, texture mask, segm tokenizer, diffusion sampler, index
    prediction, decoders) at B = 4 with 256 sampling steps, native fp32, one call after a short warm-up.

Weights are the seeded recipes (tests/parsing_gen_recipes.py): timings do not depend on trained values.  Prints the
GPU's name and power limit read in the same run, the work per image counted by torch's FlopCounterMode over the
reference classes on meta tensors, and one JSON line.
usage: python tools/bench_pose.py [--batches 4 16] [--iters 20] [--warmup 3] [--generate-steps 256]"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
import parsing_gen_recipes as P  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet, generate_parsing_map  # noqa: E402

H, W = 512, 256


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    name, plim, clk = [s.strip() for s in out[0].split(",")] if out else (torch.cuda.get_device_name(0), "?", "?")
    return dict(gpu=name, power_limit=plim, sm_clock_max=clk)


def time_fn(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def reference_nets():
    from oracle import parsing_gen_ref as PG
    if not PG.RL.available():
        return None
    ns = PG.install("reference")
    return (ns.shape_attr_embedding_arch.ShapeAttrEmbedding, ns.unet_arch.ShapeUNet, ns.fcn_arch.FCNHead)


def flops_per_image(classes):
    """FlopCounterMode over the reference classes at B = 1 on meta tensors (no compute)"""
    from torch.utils.flop_counter import FlopCounterMode
    with torch.device("meta"):
        emb, unet, head = (c(**cfg).eval() for c, cfg in zip(classes, (P.REAL_EMBEDDER, P.REAL_SHAPE_UNET,
                                                                        P.REAL_FCN_HEAD)))
        pose = torch.empty(1, 1, H, W)
        attr = torch.zeros(1, len(P.CLS_NUM), dtype=torch.int64)
    fc = FlopCounterMode(display=False)
    with fc, torch.no_grad():
        # F.one_hot needs real values: the embedding is < 0.001 % of the work and is counted from its Linear shapes
        e = torch.empty(1, P.REAL_EMBEDDER["out_dim"], device="meta")
        head(unet(pose, e)).argmax(dim=1)
    D, O, A = P.REAL_EMBEDDER["dim"], P.REAL_EMBEDDER["out_dim"], len(P.CLS_NUM)
    emb_flops = 2 * (A * D * D + A * D * O + O * O)
    return fc.get_total_flops() + emb_flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--generate-steps", type=int, default=256)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pose needs a CUDA device"
    dev = torch.device("cuda:0")
    info = gpu_info()
    ref_classes = None if args.no_reference else reference_nets()
    res = dict(info, flops_per_image=None, parsing={}, generate=None)
    if ref_classes is not None:
        res["flops_per_image"] = flops_per_image(ref_classes)
    print(f"card: {info['gpu']}, power limit {info['power_limit']}, max SM clock {info['sm_clock_max']}", flush=True)
    if res["flops_per_image"]:
        print(f"parsing generator work: {res['flops_per_image'] / 1e9:.1f} GFLOP per image (FlopCounterMode, "
              f"reference classes, {H}x{W})", flush=True)

    mods = ShapeAttrEmbedding(**P.REAL_EMBEDDER), ShapeUNet(**P.REAL_SHAPE_UNET), FCNHead(**P.REAL_FCN_HEAD)
    sds = P.state_dicts(*mods)
    for m, sd in zip(mods, sds):
        m.load_state_dict(sd, strict=True)
    emb, unet, head = (m.to(dev).eval() for m in mods)
    refs = None
    if ref_classes is not None:
        refs = [c(**cfg) for c, cfg in zip(ref_classes, (P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD))]
        for m, sd in zip(refs, sds):
            m.load_state_dict(sd, strict=True)
        refs = [m.to(dev).eval() for m in refs]

    for B in args.batches:
        pose = P.pose(360, B, H, W).to(dev)
        attr = P.shape_attrs(361, B).to(dev)
        row = {}
        for mode in ("fp32", "fp16"):
            ops.set_precision(mode)
            ms = time_fn(lambda: generate_parsing_map(emb, unet, head, pose, attr), args.iters, args.warmup)
            row[f"native_{mode}"] = ms
        ops.set_precision("fp32")
        if refs is not None:
            r_emb, r_unet, r_head = refs

            def ref_fn():
                with torch.no_grad():
                    return r_head(r_unet(pose, r_emb(attr))).argmax(dim=1).unsqueeze(1)
            for arm, tf32 in (("torch_fp32", False), ("torch_tf32", True)):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                torch.backends.cudnn.allow_tf32 = tf32
                row[arm] = time_fn(ref_fn, args.iters, args.warmup)
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        res["parsing"][B] = {k: dict(ms=v, img_s=B * 1e3 / v) for k, v in row.items()}
        line = ", ".join(f"{k} {v:.2f} ms ({B * 1e3 / v:.1f} img/s)" for k, v in row.items())
        print(f"parsing generation B={B}: {line}", flush=True)
        if res["flops_per_image"]:
            for k, v in row.items():
                res["parsing"][B][k]["tflop_s"] = res["flops_per_image"] * B / (v * 1e-3) / 1e12

    if args.generate_steps > 0:
        from test_gpu_parsing_gen import _pose_opt
        from text2human_b200.pipeline import SampleFromPoseModel
        opt = _pose_opt()
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            m = SampleFromPoseModel(opt)
        for sub, seed in ((m.index_pred_guidance_encoder, 53), (m.index_pred_decoder, 54)):
            sub.load_state_dict(R.fill_state_dict(R.spec_of(sub), seed), strict=True)
        for sub, sd in zip((m.shape_attr_embedder, m.shape_parsing_encoder, m.shape_parsing_decoder), sds):
            sub.load_state_dict(sd, strict=True)
        m = m.to(dev).eval()
        B = 4
        pose, attr = P.pose(370, B, H, W), P.shape_attrs(371, B)
        fused = [torch.tensor(v) for v in ([3, 17, 5, 0], [17, 8, 2, 17], [1, 17, 17, 4])]
        g = torch.Generator(device=dev).manual_seed(0)
        m.generate(pose, attr, *fused, sample_steps=4, generator=g)          # warm-up: packing, graph capture
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        img = m.generate(pose, attr, *fused, sample_steps=args.generate_steps, generator=g)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        assert img.shape == (B, 3, H, W) and bool(torch.isfinite(img).all())
        res["generate"] = dict(batch=B, steps=args.generate_steps, wall_s=wall, img_s=B / wall)
        print(f"SampleFromPoseModel.generate B={B}, {args.generate_steps} steps, fp32: {wall:.2f} s wall "
              f"({B / wall:.2f} img/s)", flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
