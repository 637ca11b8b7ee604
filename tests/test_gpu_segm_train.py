"""GPU: training the parsing tokenizer (VQSegmentationModel, configs/parsing_token.yml) on libt2h.

  * the fused BCE-with-logits kernel (loss, gradient planes, column sums) against fp64 torch;
  * the native SegmTokenizerTrainer against the fixture recorded from the REAL reference training_step +
    loss.backward() + Adam step (oracle/make_golden_segm_train.py), and against autograd of the restatement
    (oracle/segm_train_ref.py) at a second shape; save / load; fp16 vs fp32 mode;
  * the drop-in boundary: the reference's UNMODIFIED VQSegmentationModel.optimize_parameters on the arch mirrors;
  * two-rank data parallel (skipped with fewer than 2 GPUs)."""
import contextlib
import io
import os
import socket

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import segm_recipes as SG
from test_segm_train_oracle import segm_state

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "segm_train.npz")
NETS = ("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv")


def build(cuda, cfg=None):
    from text2human_b200.segm_train import SegmTokenizerModel
    cfg = cfg or SG.TINY_SEGM_TRAIN
    m = SegmTokenizerModel(cfg)
    sd, cb = segm_state(cfg)
    for name in ("encoder", "decoder", "quant_conv", "post_quant_conv"):
        getattr(m, name).load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")},
                                         strict=True)
    m.quantize.embedding.weight.data.copy_(cb)
    return m.to(cuda)


def named_params(m):
    return {f"{n}.{k}": p for n in NETS for k, p in getattr(m, n).named_parameters()}


def fixture_labels(cfg=None):
    cfg = cfg or SG.TINY_SEGM_TRAIN
    return SG.segm_labels(SG.SEGM_TRAIN_SEEDS["labels"], cfg["batch"], cfg["resolution"], cfg["resolution"] // 2)


# ---------------------------------------------------------------------------- 1. the loss kernel
@pytest.mark.parametrize("N,H,W,C", [(3, 37, 19, 24), (2, 13, 29, 20)])
def test_bce_logits_kernel_matches_fp64(cuda, N, H, W, C):
    from text2human_b200 import ops
    g = torch.Generator().manual_seed(N * 1000 + C)
    x = torch.randn((N, H, W, C), generator=g) * 4
    flat = x.view(-1)
    flat[:40], flat[40:80], flat[80:120] = 30.0, -30.0, 0.0
    ids = torch.randint(0, C, (N, 1, H, W), generator=g).float()
    fid = ids.view(-1)
    fid[:7], fid[7:14], fid[14:21], fid[21:28] = float(C), -1.0, 3.5, 1e7     # out of range / non-integer: no class
    valid = (fid == fid.floor()) & (fid >= 0) & (fid < C)
    t = torch.zeros((N * H * W, C), dtype=torch.float64)
    t[valid.nonzero().squeeze(1), fid[valid].long()] = 1.0
    t = t.view(N, H, W, C)
    nel = x.numel()
    gscale = 2.0 ** int(np.floor(np.log2(nel))) / nel
    want_loss = float(F.binary_cross_entropy_with_logits(x.double(), t, reduction="sum"))
    want_g = gscale * (torch.sigmoid(x.double()) - t)
    want_cs = want_g.sum((0, 1, 2))
    for terms in (2, 1):
        acc = torch.zeros(1, dtype=torch.float64, device=cuda)
        cs = torch.zeros(C, dtype=torch.float32, device=cuda)
        p = ops.bce_logits(x.to(cuda), ids.to(cuda), acc, gscale=gscale, colsum_out=cs, terms=terms)
        torch.cuda.synchronize()
        cp = (C + 7) // 8 * 8
        assert p.shape == (terms, N, H, W, cp)
        assert float(p[..., C:].abs().max() if cp > C else 0.0) == 0.0
        got = p.double().sum(0)[..., :C].cpu()
        assert abs(float(acc[0]) - want_loss) <= 1e-6 * abs(want_loss), (float(acc[0]), want_loss)
        gerr = float((got - want_g).abs().max() / want_g.abs().max())
        cerr = float((cs.double().cpu() - want_cs).abs().max() / want_cs.abs().max())
        assert cerr <= 1e-6, cerr
        assert gerr <= (1e-6 if terms == 2 else 1e-3), (terms, gerr)
    # loss only: no planes, no column sums
    acc = torch.zeros(1, dtype=torch.float64, device=cuda)
    assert ops.bce_logits(x.to(cuda), ids.to(cuda), acc, want_grad=False) is None
    assert abs(float(acc[0]) - want_loss) <= 1e-6 * abs(want_loss)


# ---------------------------------------------------------------------------- 2. native step vs the fixture
def test_native_step_matches_reference_fixture(cuda):
    from test_gpu_vqgan_train import _check_grads
    from text2human_b200 import ops
    from text2human_b200.segm_train import SegmTokenizerTrainer
    gold = np.load(GOLD)
    cfg = SG.TINY_SEGM_TRAIN
    ops.set_precision("fp32")
    m = build(cuda)
    tr = SegmTokenizerTrainer(m, lr=cfg["lr"])
    tr.training_step(dict(segm=fixture_labels()))
    torch.cuda.synchronize()
    got = tr.losses()
    for k in ("total_loss", "bce_loss", "quant_loss"):
        assert abs(got[k] - float(gold[k])) <= 2e-4 * abs(float(gold[k])), (k, got[k], float(gold[k]))
    named = named_params(m)
    worst, n = _check_grads(gold, "g", named, tr.loss_scale, 1e-3)
    assert n == len(named) == 243
    gmax = max(float(gold[k]) for k in gold.files if k.startswith("gnorm/"))
    tr.adam_step()
    torch.cuda.synchronize()
    for name, p in named.items():
        want = torch.from_numpy(gold["phead/" + name]).to(cuda)
        g = torch.from_numpy(gold["ghead/" + name]).abs().to(cuda)
        # Adam's first step is ~lr * sign(g): an entry whose gradient is within the comparison's noise (or vanishes
        # in exact arithmetic) may move either way
        small = g <= 1e-2 * max(float(gold["gnorm/" + name]), 1e-6 * gmax)
        tol = torch.where(small, torch.full_like(g, 2.5 * cfg["lr"]), torch.full_like(g, 1e-2 * cfg["lr"]))
        err = (p.detach().reshape(-1)[:8] - want).abs()
        assert bool((err <= tol + 1e-6 * want.abs()).all()), (name, err, g)
    print(f"[segm train fp32] losses {got}; {n} gradient tensors, worst rel err {worst:.2e}")


# ---------------------------------------------------------------------------- 3. second shape, full gradients
def test_native_step_matches_restatement_autograd_full_gradients(cuda):
    from oracle import segm_train_ref as SR
    from text2human_b200 import ops
    from text2human_b200.segm_train import SegmTokenizerTrainer
    ops.set_precision("fp32")
    segm = SG.segm_labels(301, 3, 128, 64, tile=8)
    segm[segm == 7] = 8                                 # class 7 absent from the batch
    assert 7 not in segm.unique().tolist()
    m = build(cuda)
    tr = SegmTokenizerTrainer(m)
    tr.training_step(dict(segm=segm))
    torch.cuda.synchronize()
    got = tr.losses()
    sd, cb = segm_state()
    sd = {k: v.to(cuda).requires_grad_(True) for k, v in sd.items()}
    cb = cb.to(cuda).requires_grad_(True)
    r = SR.segm_training_step(sd, cb, segm.to(cuda))
    r["total_loss"].backward()
    assert torch.equal(tr._out["idx"], r["idx"])
    for k in ("total_loss", "bce_loss", "quant_loss"):
        want = float(r[k].detach())
        assert abs(got[k] - want) <= 2e-4 * abs(want), (k, got[k], want)
    want = dict(sd)
    want["quantize.embedding.weight"] = cb
    named = named_params(m)
    gmax = max(float(p.grad.abs().max()) for p in want.values())
    worst = 0.0
    for name, p in named.items():
        g, gw = p.grad.detach() / tr.loss_scale, want[name].grad
        if float(gw.abs().max()) < 1e-6 * gmax:      # vanishes in exact arithmetic: absolute floor
            assert float((g - gw).abs().max()) < 1e-5 * gmax, name
            continue
        e = float((g - gw).abs().max() / gw.abs().max())
        assert e <= 1e-3, (name, e)
        worst = max(worst, e)
    print(f"[segm train 3x128x64] worst gradient rel err {worst:.2e} over {len(named)} tensors")


# ---------------------------------------------------------------------------- 4. save / load
def test_save_load_resumes_and_feeds_the_sampler_tokenizer(cuda, tmp_path):
    from text2human_b200 import ops
    from text2human_b200.pipeline import SegmTokenizer
    from text2human_b200.segm_train import SegmTokenizerTrainer
    ops.set_precision("fp32")
    cfg = SG.TINY_SEGM_TRAIN
    segm = fixture_labels()
    batches = [dict(segm=SG.segm_labels(400 + i, 2, 64, 32)) for i in range(2)]
    tr = SegmTokenizerTrainer(build(cuda), lr=1e-3)
    tr.optimize_parameters(dict(segm=segm))
    path = os.path.join(tmp_path, "segm_token.pth")
    tr.save(path)
    for b in batches:
        tr.optimize_parameters(b)
    want = tr.space.flat_p.clone()
    tr2 = SegmTokenizerTrainer(build(cuda), lr=1e-3)
    tr2.load(path)
    ck = torch.load(path, map_location=cuda)
    assert set(ck) == set(NETS) | {"optimizer"}
    assert torch.equal(tr2.space.flat_m, ck["optimizer"]["flat_m"]) and tr2.space.step_count == 1
    # the saved encoder / quantize / quant_conv are what the sampling models' segm tokenizer loads (strict=True)
    opt = {"segm_" + k: cfg[k] for k in ("ch", "num_res_blocks", "attn_resolutions", "ch_mult", "in_channels",
                                         "resolution", "z_channels", "double_z", "dropout", "n_embed", "embed_dim",
                                         "num_segm_classes")}
    with contextlib.redirect_stdout(io.StringIO()):
        st = SegmTokenizer(opt)
    st.segm_encoder.load_state_dict(ck["encoder"], strict=True)
    st.segm_quantizer.load_state_dict(ck["quantize"], strict=True)
    st.segm_quant_conv.load_state_dict(ck["quant_conv"], strict=True)
    st = st.to(cuda).eval()
    from text2human_b200.vqgan_arch import conv1x1_nhwc
    m2 = tr2.model
    with torch.no_grad():
        ids = segm.unsqueeze(1).float().to(cuda)
        tokens = st.get_quantized_segm(ids)
        z = conv1x1_nhwc(m2.encoder.forward_planes(ops.onehot_to_planes(ids, 24)), m2.quant_conv)
        own = m2.quantize.forward_nhwc(z)["idx"]
    assert torch.equal(tokens, own)
    for b in batches:
        tr2.optimize_parameters(b)
    # the resumed run continues the uninterrupted one; they differ only where rounding-level gradient noise (atomic
    # accumulation order) flips the sign of Adam's update of a vanishing gradient
    dev_ = (tr2.space.flat_p - want).abs()
    print(f"[segm resume] {100 * float((dev_ == 0).float().mean()):.2f} % of parameters bit-identical, "
          f"max deviation {float(dev_.max()):.2e}")
    assert float(dev_.max()) <= 2 * 2.5 * tr.lr and float((dev_ > 1e-6).float().mean()) < 0.01
    assert tr2.space.step_count == tr.space.step_count == 3


# ---------------------------------------------------------------------------- 5. fp16 mode
def test_fp16_mode_tracks_fp32_mode(cuda):
    from text2human_b200 import ops
    from text2human_b200.segm_train import SegmTokenizerTrainer
    res = {}
    try:
        for mode in ("fp32", "fp16"):
            ops.set_precision(mode)
            tr = SegmTokenizerTrainer(build(cuda))
            tr.training_step(dict(segm=fixture_labels()))
            res[mode] = (tr.losses(), tr.space.flat_g.clone() / tr.loss_scale)
    finally:
        ops.set_precision("fp32")
    (l32, g32), (l16, g16) = res["fp32"], res["fp16"]
    for k in l32:
        assert abs(l16[k] - l32[k]) <= 3e-3 * max(1.0, abs(l32[k])), (k, l16[k], l32[k])
    cos = float(F.cosine_similarity(g16.double(), g32.double(), dim=0))
    print(f"[segm train fp16 vs fp32] losses {l16} vs {l32}; gradient cosine {cos:.5f}")
    assert cos > 0.98


# ---------------------------------------------------------------------------- 6. drop-in boundary
def test_reference_segm_wrapper_trains_unmodified_on_the_mirrors(cuda):
    """VQSegmentationModel.optimize_parameters (vqgan_model.py:86-96) built by its own __init__ on the mirrors vs the
    same code on the reference arch classes.  Before the plain quantizer had a training path the encoder, quant_conv
    and codebook got no gradient at all."""
    from oracle import ref_loader as RL
    from text2human_b200 import ops, vqgan_arch
    if not RL.available():
        pytest.skip("reference sources not staged (run oracle/make_ref.py in the build container)")
    ops.set_precision("fp32")
    opt = dict(SG.TINY_SEGM_TRAIN)
    sd, cb = segm_state()
    data = dict(segm=fixture_labels())
    wrappers = []
    for archs in ("mirror", "reference"):
        ns = RL.install(archs, wrappers=("vqgan_model",))
        with contextlib.redirect_stdout(io.StringIO()):
            w = ns.vqgan_model.VQSegmentationModel(opt)
        for name in ("encoder", "decoder", "quant_conv", "post_quant_conv"):
            getattr(w, name).load_state_dict({k[len(name) + 1:]: v.to(cuda) for k, v in sd.items()
                                              if k.startswith(name + ".")}, strict=True)
        with torch.no_grad():
            w.quantize.embedding.weight.copy_(cb)
        wrappers.append(w)
    wm, wr = wrappers
    assert isinstance(wm.encoder, vqgan_arch.Encoder) and isinstance(wm.quantize, vqgan_arch.VectorQuantizer)
    before = {k: v.detach().clone() for k, v in wm.encoder.state_dict().items()}
    wm.optimize_parameters(data, 0)
    wr.optimize_parameters(data, 0)
    for k in ("total_loss", "bce_loss", "quant_loss"):
        got, want = float(wm.log_dict["train/" + k]), float(wr.log_dict["train/" + k])
        assert abs(got - want) <= 2e-4 * abs(want), (k, got, want)
    pairs = []
    for name in NETS:
        pm, pr = dict(getattr(wm, name).named_parameters()), dict(getattr(wr, name).named_parameters())
        assert pm.keys() == pr.keys()
        for k in pm:
            assert pm[k].grad is not None, f"{name}.{k} got no gradient"
            pairs.append((f"{name}.{k}", pm[k].grad, pr[k].grad))
    gmax = max(float(gr.abs().max()) for _, _, gr in pairs)
    worst = 0.0
    for key, gm, gr in pairs:
        if float(gr.abs().max()) < 1e-6 * gmax:       # vanishes in exact arithmetic: absolute floor
            assert float((gm - gr).abs().max()) < 1e-5 * gmax, key
            continue
        e = float(((gm - gr).abs().max() / gr.abs().max()))
        assert e <= 1e-3, (key, e)
        worst = max(worst, e)
    for key in ("encoder.conv_in.weight", "quant_conv.weight", "quantize.embedding.weight"):
        assert any(k == key and float(g.abs().max()) > 0 for k, g, _ in pairs), key
    print(f"[segm boundary] reference optimize_parameters on the mirrors: worst gradient rel err {worst:.2e}")
    after = wm.encoder.state_dict()
    assert all(not torch.equal(before[k], after[k]) for k in before if k.endswith("conv_in.weight"))


# ---------------------------------------------------------------------------- 7. two-rank data parallel
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_dir):
    import json
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    from text2human_b200 import ops
    from text2human_b200.segm_train import SegmTokenizerTrainer
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    ops.set_precision("fp32")
    segm = SG.segm_labels(501, world, 64, 32)
    out = dict(rank=rank)
    single = None
    if rank == 0:          # the single-process step on both images, before any process group exists
        t1 = SegmTokenizerTrainer(build(dev))
        t1.optimize_parameters(dict(segm=segm))
        single = (t1.space.flat_g.clone(), t1.space.flat_p.clone())
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    dist.init_process_group("nccl", device_id=dev)
    tr = SegmTokenizerTrainer(build(dev), bucket_bytes=256 << 10)      # several buckets even for the reduced net
    tr.training_step(dict(segm=segm[rank:rank + 1]))
    out["n_reduces"], out["n_buckets"] = len(tr._handles), len(tr.space.buckets)
    tr.wait_reduced()
    g = tr.space.flat_g.clone()
    tr.adam_step()
    torch.cuda.synchronize()
    out["psum"] = float(tr.space.flat_p.double().sum())
    if single is not None:
        g1, p1 = single
        out["g_rel"] = float((g - g1).abs().max() / g1.abs().max())
        big = g1.abs() > 1e-3 * g1.abs().max()         # Adam amplifies rounding noise of ~zero gradients
        out["p_dev"] = float((tr.space.flat_p - p1)[big].abs().max())
    with open(os.path.join(out_dir, f"rank{rank}.json"), "w") as f:
        json.dump(out, f)
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
    os._exit(0)


def test_two_rank_step_equals_single_process_step(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    import time
    import torch.multiprocessing as mp
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    files = [os.path.join(str(tmp_path), f"rank{r}.json") for r in range(2)]
    t0 = time.time()
    while (not all(os.path.exists(f) for f in files) and time.time() - t0 < 600
           and all(p.is_alive() or p.exitcode == 0 for p in procs)):
        time.sleep(0.5)
    time.sleep(1.0)
    assert all(os.path.exists(f) for f in files), [p.exitcode for p in procs]
    r0, r1 = (json.load(open(f)) for f in files)
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.kill()
    print(f"[segm ddp] {r0['n_reduces']} bucket all-reduces during backward; gradient rel diff {r0['g_rel']:.2e}; "
          f"parameter deviation after Adam {r0['p_dev']:.2e}")
    assert r0["n_reduces"] == r0["n_buckets"] >= 4
    assert r0["g_rel"] < 1e-4 and r0["p_dev"] < 1e-6
    assert r0["psum"] == r1["psum"]
