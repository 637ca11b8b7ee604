"""One training step of the reference's ParsingGenModel.optimize_parameters (unmodified, staged under oracle/_ref/,
built by its own __init__) at configs/parsing_gen.yml's widths (ShapeUNet base 64, FCNHead 64 -> 24 classes), three
ways:

  mirror      the wrapper's code on the text2human_b200 mirrors (ShapeAttrEmbedding, ShapeUNet and FCNHead as
              autograd nodes, NCHW tensors between them)
  reference   the same code on the reference's own arch classes, stock PyTorch eager, fp32 and cuDNN/cuBLAS TF32
  native      text2human_b200.parsing_gen_train.ParsingGenTrainer.optimize_parameters

at each ``--shapes`` entry B,H,W (default: the config's batch 8 at 256 x 128, and 16 at 512 x 256).  Each way runs in
its own process: warm-up steps, then CUDA-event timing over ``--steps`` synchronised steps and the peak allocated
memory over them; the ways alternate ``--repeats`` times and each reports the median time, the range and the peak.
The card name, power limit and maximum SM clock are read in the same run and printed with the numbers (one JSON line).
usage: python tools/bench_parsing_gen_dropin.py [--steps 10] [--warmup 3] [--repeats 3] [--precision fp32|fp16]
                                                [--shapes 8,256,128 16,512,256]"""
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
import parsing_gen_recipes as P  # noqa: E402
import parsing_gen_train_recipes as PT  # noqa: E402
from oracle import ref_loader as RL  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.parsing_gen_train import ParsingGenTrainer  # noqa: E402
from tools.bench_sampler_dropin import gpu_context, timed  # noqa: E402

OPT = dict(is_train=True, embedder_dim=8, embedder_out_dim=128, attr_class_num=P.CLS_NUM, encoder_in_channels=1,
           fc_in_channels=64, fc_in_index=4, fc_channels=64, fc_num_convs=1, fc_concat_input=False,
           fc_dropout_ratio=0.1, fc_num_classes=24, fc_align_corners=False, lr=1e-4, weight_decay=0)
ARMS = ("mirror", "reference_fp32", "reference_tf32", "native")


def build_wrapper(archs):
    """ParsingGenModel(OPT) by its own __init__, finding the mirrors (``archs`` "mirror") or the reference's classes
    under models.archs"""
    RL.install(archs, wrappers=())
    if archs == "mirror":
        from text2human_b200 import parsing_gen_arch as A
        sys.modules["models.archs.unet_arch"].ShapeUNet = A.ShapeUNet
        sys.modules["models.archs.fcn_arch"].FCNHead = A.FCNHead
        sae = types.ModuleType("models.archs.shape_attr_embedding_arch")
        sae.ShapeAttrEmbedding = A.ShapeAttrEmbedding
        sys.modules[sae.__name__] = sae
    sys.modules["mmcv"].imwrite = lambda *a, **k: None
    pg = RL._exec("models.parsing_gen_model", os.path.join(RL.ref_root(), "models", "parsing_gen_model.py"))
    w = pg.ParsingGenModel(OPT)
    nets = (w.attr_embedder, w.parsing_encoder, w.parsing_decoder)
    for m, sd in zip(nets, P.state_dicts(*nets, PT.TRAIN_SEEDS)):
        m.load_state_dict(sd, strict=True)
    return w


def run_arm(arm, shape, a):
    ops.set_precision(a.precision)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = arm == "reference_tf32"
    data = PT.batch(PT.TRAIN_SEEDS, shape)
    w = build_wrapper("reference" if arm.startswith("reference") else "mirror")
    torch.manual_seed(1)
    if arm == "native":
        nets = [m.eval() for m in (w.attr_embedder, w.parsing_encoder, w.parsing_decoder)]
        del w
        tr = ParsingGenTrainer(*nets, lr=OPT["lr"])
        return timed(lambda: tr.optimize_parameters(data), a.steps, a.warmup)
    w.feed_data(data)
    return timed(w.optimize_parameters, a.steps, a.warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=["8,256,128", "16,512,256"])
    ap.add_argument("--arm", choices=ARMS, help="run one way only (the script runs each in its own process)")
    a = ap.parse_args()
    assert torch.cuda.is_available()
    shapes = [tuple(int(v) for v in s.split(",")) for s in a.shapes]
    if a.arm:
        print(json.dumps(run_arm(a.arm, shapes[0], a)))
        return
    res = dict(gpu_context(), precision=a.precision, steps=a.steps, warmup=a.warmup, repeats=a.repeats)
    if not RL.available():
        res["error"] = "reference sources not staged (oracle/make_ref.py)"
        print(json.dumps(res))
        return
    for shape in shapes:
        runs = {arm: [] for arm in ARMS}
        for _ in range(a.repeats):            # the ways alternate, so that a slow spell of a shared host hits them all
            for arm in ARMS:
                out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps",
                                               str(a.steps), "--warmup", str(a.warmup), "--precision", a.precision,
                                               "--shapes", ",".join(map(str, shape))], text=True)
                runs[arm].append(json.loads(out.strip().splitlines()[-1]))
                print(f"B,H,W {shape} {arm}: {runs[arm][-1]}", file=sys.stderr, flush=True)
        key = "B{}_{}x{}".format(*shape)
        res[key] = {}
        for arm, rs in runs.items():
            ms = sorted(r["ms_per_step"] for r in rs)
            res[key][arm] = dict(ms_per_step_median=ms[len(ms) // 2], ms_per_step_range=[ms[0], ms[-1]],
                                 peak_mib=max(r["peak_mib"] for r in rs))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
