"""GPU parity of the parsing generator (pose + shape attributes -> parsing map: ShapeAttrEmbedding -> ShapeUNet ->
FCNHead -> argmax) through libt2h, and of SampleFromPoseModel end to end.  References: the real reference classes
(via oracle/parsing_gen_ref.install, or the fixture from oracle/make_golden_parsing_gen.py) and the fp32
restatement in oracle/parsing_gen_ref.  Tolerance 1e-3 relative on features and logits; parsing maps must be equal
wherever the reference's top-2 logit margin exceeds 2 * tol * max|logit| (a sub-tolerance difference can flip an
argmax)."""
import contextlib
import io
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import parsing_gen_recipes as P

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "parsing_gen.npz")
TOL = 1e-3


def _ops():
    from text2human_b200 import ops
    ops.set_precision("fp32")
    return ops


def _rel(got, ref):
    got = torch.as_tensor(got).double().cpu()
    ref = torch.as_tensor(ref).double().cpu()
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _loader():
    from oracle import parsing_gen_ref as PR
    if not PR.RL.available():
        pytest.skip("reference sources not staged (run oracle/make_ref.py in the build container)")
    return PR


def _mirrors(emb_cfg, unet_cfg, head_cfg, cuda):
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    mods = ShapeAttrEmbedding(**emb_cfg), ShapeUNet(**unet_cfg), FCNHead(**head_cfg)
    sds = P.state_dicts(*mods)
    for m, sd in zip(mods, sds):
        m.load_state_dict(sd, strict=True)
    return [m.to(cuda).eval() for m in mods], sds


def _margin_ok(logits, tol=TOL):
    """[B,n,H,W] reference logits -> [B,1,H,W] bool: where the argmax is decided by more than the tolerance"""
    top2 = logits.topk(2, dim=1).values
    return ((top2[:, 0] - top2[:, 1]) > 2 * tol * logits.abs().max()).unsqueeze(1)


@pytest.mark.parametrize("terms", [2, 1])
@pytest.mark.parametrize("mode", ["plain", "maxpool2"])
@pytest.mark.parametrize("C,Ce", [(1, 128), (64, 128), (512, 128), (1, 5), (64, 5), (512, 5)])
def test_broadcast_conversion_is_bit_exact(cuda, C, Ce, mode, terms):
    """cat([x, e broadcast], 1) (+ max_pool2d) -> hi/lo fp16 planes, zero-padded to a multiple of 8 channels
    (C + Ce = 129, 69, 517 are not); odd H drops the last row under pooling, as nn.MaxPool2d(2)"""
    ops = _ops()
    N, H, W = 2, 9, 6
    x = torch.randn(N, H, W, C, device=cuda)
    e = torch.randn(N, Ce, device=cuda)
    cat = torch.cat([x.permute(0, 3, 1, 2), e.view(N, Ce, 1, 1).expand(N, Ce, H, W)], 1)
    if mode == "maxpool2":
        cat = F.max_pool2d(cat, 2)
    want = cat.permute(0, 2, 3, 1)
    cp = (C + Ce + 7) // 8 * 8
    want = F.pad(want, (0, cp - C - Ce))
    hi = want.half()
    want_planes = torch.stack((hi, (want - hi.float()).half()))[:terms]
    got = ops.f32_to_planes_bcast(x, e, ops.CVT_PLAIN if mode == "plain" else ops.CVT_MAXPOOL2, terms=terms)
    assert got.shape == want_planes.shape and torch.equal(got, want_planes)


def test_embedding_kernel_matches_reference_class(cuda):
    """the real reference ShapeAttrEmbedding (fp32, CPU) on every class of every attribute plus a random batch; an
    out-of-range attribute raises ValueError naming it"""
    _ops()
    PR = _loader()
    ns = PR.install("reference")
    ref = ns.shape_attr_embedding_arch.ShapeAttrEmbedding(**P.REAL_EMBEDDER)
    (emb, _, _), (sd, _, _) = _mirrors(P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD, cuda)
    ref.load_state_dict(sd, strict=True)
    attr = torch.cat([P.every_class_attrs(), P.shape_attrs(310, 37)])
    with torch.no_grad():
        want = ref.eval()(attr)
    got = emb(attr.to(cuda))
    assert got.shape == (attr.shape[0], 128) and _rel(got, want) <= 1e-5
    bad = attr.clone()
    bad[3, 2] = 6                                          # attribute 2 has 6 classes
    with pytest.raises(ValueError, match="shape attribute 2"):
        emb(bad.to(cuda))


def test_tiny_mirrors_match_reference_fixture(cuda):
    _ops()
    from text2human_b200.parsing_gen_arch import generate_parsing_map
    gold = np.load(GOLD)
    (emb, unet, head), _ = _mirrors(P.TINY_EMBEDDER, P.TINY_SHAPE_UNET, P.TINY_FCN_HEAD, cuda)
    pose, attr = torch.from_numpy(gold["pose"]).to(cuda), torch.from_numpy(gold["attr"]).to(cuda)
    e = emb(attr)
    assert _rel(e, gold["embedding"]) < 1e-5
    dec = unet(pose, e)
    assert len(dec) == 5
    for i, d in enumerate(dec):
        assert d.shape == gold[f"dec{i}"].shape and _rel(d, gold[f"dec{i}"]) < TOL, i
    logits = head(dec)
    assert logits.shape == gold["logits"].shape and _rel(logits, gold["logits"]) < TOL
    seg = generate_parsing_map(emb, unet, head, pose, attr).cpu()
    ok = _margin_ok(torch.from_numpy(gold["logits"]))
    assert seg.dtype == torch.float32 and torch.equal(seg[ok], torch.from_numpy(gold["argmax"]).float()[ok])


def _real_inputs(B, seed=320):
    return P.pose(seed, B, 512, 256), P.shape_attrs(seed + 1, B)


def test_real_size_parsing_generator_matches_restatement(cuda):
    """ShapeUNet(in_channels=1) + FCNHead(64, 64, 24 classes) on a blocky part-index pose, B = 2, 512 x 256"""
    _ops()
    from oracle import parsing_gen_ref as PG
    from text2human_b200.parsing_gen_arch import generate_parsing_map
    (emb, unet, head), (sde, sdu, sdh) = _mirrors(P.REAL_EMBEDDER, P.REAL_SHAPE_UNET, P.REAL_FCN_HEAD, cuda)
    pose, attr = _real_inputs(2)
    dev = lambda sd: {k: v.to(cuda) for k, v in sd.items()}   # noqa: E731
    with torch.no_grad():
        want_logits, want_seg = PG.generate_parsing_map(dev(sde), dev(sdu), dev(sdh), pose.to(cuda), attr.to(cuda),
                                                        P.CLS_NUM)
    e = emb(attr.to(cuda))
    logits = head(unet(pose.to(cuda), e))
    assert logits.shape == (2, 24, 512, 256) and _rel(logits, want_logits) < TOL
    seg = generate_parsing_map(emb, unet, head, pose.to(cuda), attr.to(cuda))
    ok = _margin_ok(want_logits)
    assert seg.shape == (2, 1, 512, 256) and torch.equal(seg[ok], want_seg[ok].float())
    frac = float(ok.float().mean())
    print(f"[parsing_gen] real size: logits rel err {_rel(logits, want_logits):.2e}, {100 * frac:.2f} % of pixels "
          f"checked, {100 * float((seg == want_seg.float()).float().mean()):.3f} % equal")
    assert frac > 0.9


def test_reference_generate_parsing_map_runs_unmodified_on_the_mirrors(cuda):
    """SampleFromPoseModel.generate_parsing_map + generate_texture_map (sample_model.py:431-470), bound to a stand-in
    carrying the attributes they read, on the mirrors and on the reference archs (fused attribute 17 = none included)"""
    _ops()
    PR = _loader()
    B = 4
    pose, attr = _real_inputs(B, 330)
    fused = torch.tensor([[17, 3, 17], [5, 17, 2], [0, 11, 17], [17, 17, 17]])   # upper, lower, outer per image
    sds = None
    out = {}
    for archs in ("mirror", "reference"):
        ns = PR.install(archs, wrappers=("sample_model",))
        emb = ns.shape_attr_embedding_arch.ShapeAttrEmbedding(**P.REAL_EMBEDDER)
        unet = ns.unet_arch.ShapeUNet(**P.REAL_SHAPE_UNET)
        head = ns.fcn_arch.FCNHead(**P.REAL_FCN_HEAD)
        sds = sds or P.state_dicts(emb, unet, head)
        for m, sd in zip((emb, unet, head), sds):
            m.load_state_dict(sd, strict=True)
        emb, unet, head = (m.to(cuda).eval() for m in (emb, unet, head))
        fake = types.SimpleNamespace(shape_attr_embedder=emb, shape_parsing_encoder=unet,
                                     shape_parsing_decoder=head, pose=pose.to(cuda),
                                     shape_attr=attr.to(cuda), batch_size=B, upper_fused_attr=fused[:, 0].to(cuda),
                                     lower_fused_attr=fused[:, 1].to(cuda), outer_fused_attr=fused[:, 2].to(cuda))
        PR.RL.bind(ns.sample_model.SampleFromPoseModel, fake, ["generate_parsing_map", "generate_texture_map"])
        fake.generate_parsing_map()
        fake.generate_texture_map()
        with torch.no_grad():
            logits = head(unet(fake.pose, emb(fake.shape_attr)))
        out[archs] = (fake.segm.cpu(), fake.texture_mask.cpu(), logits.cpu())
    (seg, tm, _), (want_seg, want_tm, want_logits) = out["mirror"], out["reference"]
    ok = _margin_ok(want_logits)
    assert seg.shape == want_seg.shape == (B, 1, 512, 256) and torch.equal(seg[ok], want_seg[ok])
    assert float(ok.float().mean()) > 0.9
    same = seg == want_seg
    assert tm.shape == want_tm.shape and torch.equal(tm[same], want_tm[same])
    assert bool((want_tm[3] == 0).all()) and bool((tm[3] == 0).all())          # every group 'none': common codebook


def _pose_opt():
    from test_gpu_indexpred import _sample_opt
    opt = _sample_opt()
    opt.update(shape_embedder_dim=8, shape_embedder_out_dim=128, shape_attr_class_num=P.CLS_NUM,
               shape_encoder_in_channels=1, shape_fc_in_channels=64, shape_fc_in_index=4, shape_fc_channels=64,
               shape_fc_num_convs=1, shape_fc_concat_input=False, shape_fc_dropout_ratio=0.1, shape_fc_num_classes=24,
               shape_fc_align_corners=False, sample_steps=4)
    return opt


def test_sample_from_pose_end_to_end(cuda, tmp_path):
    """pose -> image through every stage of SampleFromPoseModel at 4 sampling steps: shapes, range, reproducibility
    under a seeded generator (to rounding: the fused GroupNorm statistics are accumulated with atomics), a different
    seed changes the result, the chain equals sample_and_refine on its own parsing map and texture mask, and
    inference writes one file per image name"""
    ops = _ops()
    from text2human_b200.pipeline import SampleFromPoseModel
    torch.manual_seed(51)
    with contextlib.redirect_stdout(io.StringIO()):
        m = SampleFromPoseModel(_pose_opt())
    for sub, seed in ((m.index_pred_guidance_encoder, 53), (m.index_pred_decoder, 54)):
        sub.load_state_dict(R.fill_state_dict(R.spec_of(sub), seed), strict=True)
    for sub, sd in zip((m.shape_attr_embedder, m.shape_parsing_encoder, m.shape_parsing_decoder),
                       P.state_dicts(m.shape_attr_embedder, m.shape_parsing_encoder, m.shape_parsing_decoder)):
        sub.load_state_dict(sd, strict=True)
    m = m.to(cuda).eval()
    B = 2
    pose, attr = _real_inputs(B, 340)
    upper, lower, outer = torch.tensor([3, 17]), torch.tensor([17, 8]), torch.tensor([1, 17])
    imgs = []
    for seed in (7, 7, 8):
        g = torch.Generator(device=cuda).manual_seed(seed)
        imgs.append(m.generate(pose, attr, upper, lower, outer, sample_steps=4, generator=g))
    img = imgs[0]
    assert img.shape == (B, 3, 512, 256) and img.dtype == torch.float32
    assert bool(torch.isfinite(img).all()) and float(img.min()) >= 0.0 and float(img.max()) <= 1.0
    assert float((imgs[0] - imgs[1]).abs().max()) < 1e-4
    assert float((imgs[0] - imgs[2]).abs().max()) > 1e-2
    segm = m.generate_parsing_map(pose.to(cuda), attr.to(cuda))
    tm = ops.texture_mask(segm, torch.stack([upper, lower, outer], 1).to(cuda))
    g = torch.Generator(device=cuda).manual_seed(7)
    want = m.sample_and_refine(segm, tm, sample_steps=4, generator=g)
    assert float((img - want).abs().max()) < 1e-4
    names = ["p0.png", "p1.png"]
    loader = [dict(densepose=pose, shape_attr=attr, upper_fused_attr=upper, lower_fused_attr=lower,
                   outer_fused_attr=outer, img_name=names)]
    m.inference(loader, str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == names
