"""Index-prediction training step (configs/index_pred_net.yml: UNet 256 -> base 64 with 5 stages, 18 heads of
64 channels -> 512 classes) at 512 x 256 images (32 x 16 latents), timed with CUDA events after a warm-up, at the
config's batch 4 and at batch 16:

  * ground truth: the frozen hierarchy's feed_data (real-size vqvae_top / vqvae_bottom encoders, random weights and
    codebooks), native;
  * the trainable step, native: IndexPredTrainer.optimize_parameters on the ground truth, fp32 (3-product) and fp16
    (1-product) operands, and its launches per step;
  * the trainable step, reference: the reference's own optimize_parameters (unbound, on a stand-in self carrying the
    reference UNet / MultiHeadFCNHead and CrossEntropyLoss) in stock PyTorch eager, fp32 and with cuDNN TF32, when
    oracle/_ref is staged;
  * the routed head cross-entropy (forward + backward of the 18 heads' conv_seg and loss) next to the dense
    MultiHeadFCNHead.forward_logits on the same input (a forward-only floor for the dense alternative).

Prints one JSON line with the GPU's name, power limit and maximum SM clock read in the same run.
usage: python tools/bench_index_pred_train.py [--batches 4 16] [--steps 10] [--warmup 3]"""
import argparse
import contextlib
import io
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_recipes as R  # noqa: E402
from bench_segm_train import gpu_info, timed  # noqa: E402
from test_gpu_modules import HIER_OPT  # noqa: E402
from text2human_b200 import ops  # noqa: E402
from text2human_b200.index_pred_train import IndexPredNets, IndexPredTrainer  # noqa: E402

OPT = dict(encoder_in_channels=256, fc_in_channels=64, fc_in_index=4, fc_channels=64, fc_num_convs=1,
           fc_concat_input=False, fc_dropout_ratio=0.1, fc_num_classes=512, fc_align_corners=False)


def hierarchy(dev):
    from text2human_b200.pipeline import HierarchyVQSpatialTextureAwareModel
    torch.manual_seed(7)
    h = HierarchyVQSpatialTextureAwareModel(HIER_OPT)
    cbt = R.codebooks(8, 18, 1024, 256, "trained")
    cbb = R.codebooks(9, 18, 512, 1024, "trained")
    for k in range(18):
        h.top_quantize.embedding_list[k].weight.data.copy_(cbt[k])
        h.bot_quantize.embedding_list[k].weight.data.copy_(cbb[k])
    return h.to(dev).eval()


def state_dicts():
    nets = IndexPredNets(OPT)
    return (R.fill_state_dict(R.spec_of(nets.guidance_encoder), 31),
            R.fill_state_dict(R.spec_of(nets.index_decoder), 32))


def trainer(sds, dev, hier):
    nets = IndexPredNets(OPT)
    nets.guidance_encoder.load_state_dict(sds[0], strict=True)
    nets.index_decoder.load_state_dict(sds[1], strict=True)
    nets = nets.to(dev)
    return IndexPredTrainer(nets.guidance_encoder, nets.index_decoder, hierarchy=hier)


def native(prec, sds, data, dev, hier, steps, warmup):
    ops.set_precision(prec)
    tr = trainer(sds, dev, hier)
    gt_ms = timed(lambda: tr.feed_data(data), steps, warmup)
    tr.optimize_parameters()
    torch.cuda.synchronize()
    l0 = ops.COUNTERS["launches"]
    ms = timed(tr.optimize_parameters, steps, warmup)
    launches = (ops.COUNTERS["launches"] - l0) // (steps + warmup)
    out = dict(ground_truth_ms=gt_ms, step_ms=ms, launches=launches, losses=tr.losses())
    # the routed loss kernel (3 launches) against the dense 18-head logits of the eval path, same feature map
    B, h, w, _ = tr._gt["feature_t"].shape
    M, G, C, K = B * h * w, tr.n_head, tr.channels, tr.n_classes
    y = torch.relu(torch.randn((M, G * C), device=dev))
    tex, own = tr._gt["tex"].reshape(-1), tr._gt["own"].reshape(-1)
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    out["routed_ce_ms"] = timed(lambda: ops.routed_head_ce(y, tex, own, tr.w_seg, tr.b_seg, loss, tr.gw_seg,
                                                           tr.gb_seg), steps * 5, warmup)
    feat = torch.randn((B, h, w, C), device=dev)
    out["dense_forward_logits_ms"] = timed(lambda: tr.fcn.forward_logits(feat), steps * 5, warmup)
    del tr
    torch.cuda.empty_cache()
    return out


def reference(tf32, sds, feature_t, gt_list, dev, steps, warmup):
    from oracle import ref_loader as RL
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ns = RL.install("reference", wrappers=())
        for sub in ("losses.accuracy", "losses.cross_entropy_loss", "hierarchy_inference_model"):
            name = "models." + sub
            if name not in sys.modules:
                RL._exec(name, os.path.join(ns.root, "models", *sub.split(".")) + ".py")
        Model = sys.modules["models.hierarchy_inference_model"].VQGANTextureAwareSpatialHierarchyInferenceModel
        unet = ns.unet_arch.UNet(in_channels=256)
        fcn = ns.fcn_arch.MultiHeadFCNHead(in_channels=64, in_index=4, channels=64, num_convs=1, concat_input=False,
                                           dropout_ratio=0.1, num_classes=512, align_corners=False, num_head=18)
        unet.load_state_dict(sds[0], strict=True)
        fcn.load_state_dict(sds[1], strict=True)
        fake = types.SimpleNamespace(opt=dict(optimizer="Adam", lr=1e-4, weight_decay=0,
                                              loss_function="cross_entropy"),
                                     device=dev, guidance_encoder=unet.to(dev), index_decoder=fcn.to(dev),
                                     feature_t=feature_t, gt_indices_list=gt_list)
        for name in ("init_training_settings", "optimize_parameters"):
            setattr(fake, name, types.MethodType(getattr(Model, name), fake))
        with contextlib.redirect_stdout(io.StringIO()):
            fake.init_training_settings()
        fake.loss_func = fake.loss_func.to(dev)
        ms = timed(fake.optimize_parameters, steps, warmup)
        loss = float(fake.log_dict["loss_total"].detach())
        del fake, unet, fcn
        torch.cuda.empty_cache()
        return dict(step_ms=ms, losses=dict(loss_total=loss))
    finally:
        torch.backends.cudnn.allow_tf32 = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", nargs="+", type=int, default=[4, 16])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    from oracle import ref_loader as RL
    from oracle.index_pred_train_ref import gt_indices_list
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    hier = hierarchy(dev)
    sds = state_dicts()
    out = dict(gpu_info(), workload="index-prediction training step (index_pred_net.yml nets, 512x256)", batches={})
    for B in a.batches:
        data = dict(image=R.image(41, B, 3, 512, 256).to(dev), texture_mask=R.blocky_mask(42, B, 512, 256, 16).to(dev))
        res = {}
        for prec in ("fp32", "fp16"):
            r = native(prec, sds, data, dev, hier, a.steps, a.warmup)
            res["native_" + prec] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}
        ops.set_precision("fp32")
        if RL.available() and not a.no_reference:
            tr = trainer(sds, dev, hier)
            gt = tr.feed_data(data)
            feature_t = gt["feature_t"].permute(0, 3, 1, 2).contiguous()
            gl = gt_indices_list(torch.where((gt["tex"] >= 0) & (gt["tex"] < 18), gt["own"], -1), gt["tex"])
            del tr
            for name, tf32 in (("eager_fp32", False), ("eager_tf32", True)):
                try:
                    r = reference(tf32, sds, feature_t, gl, dev, a.steps, a.warmup)
                    res[name] = dict(step_ms=round(r["step_ms"], 3), losses=r["losses"])
                except Exception as e:     # the reference arm is optional; report why it did not run
                    res[name] = dict(error=f"{type(e).__name__}: {e}")
        out["batches"][str(B)] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
