"""CPU: the parsing-generator restatement (oracle/parsing_gen_ref: shape_attr_embedding, shape_unet, fcn_head)
against the fixture made from the real reference ShapeAttrEmbedding / ShapeUNet / FCNHead
(oracle/make_golden_parsing_gen.py), the mirrors' checkpoint ABI (parsing_gen.pth: embedder / encoder / decoder), and what the mirrors accept."""
import os

import numpy as np
import pytest
import torch

import parsing_gen_recipes as P
from oracle import parsing_gen_ref as PG

GOLD = os.path.join(os.path.dirname(__file__), "golden", "parsing_gen.npz")


def _tiny():
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    emb, unet, head = ShapeAttrEmbedding(**P.TINY_EMBEDDER), ShapeUNet(**P.TINY_SHAPE_UNET), FCNHead(**P.TINY_FCN_HEAD)
    return (emb, unet, head), P.state_dicts(emb, unet, head)


def _close(got, want, tol=1e-5):
    want = torch.from_numpy(want)
    return got.shape == want.shape and float((got - want).abs().max()) <= tol * float(want.abs().max())


def test_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    _, (sde, sdu, sdh) = _tiny()
    B, H, W = P.TINY_POSE
    pose, attr = P.pose(P.SEEDS["pose"], B, H, W), P.shape_attrs(P.SEEDS["attr"], B)
    assert np.array_equal(pose.numpy(), gold["pose"]) and np.array_equal(attr.numpy(), gold["attr"])
    with torch.no_grad():
        e = PG.shape_attr_embedding(sde, attr, P.CLS_NUM)
        dec = PG.shape_unet(sdu, pose, e)
        logits = PG.fcn_head(sdh, dec)
    assert _close(e, gold["embedding"])
    assert len(dec) == 5
    for i, d in enumerate(dec):
        assert _close(d, gold[f"dec{i}"]), i
    assert _close(logits, gold["logits"])
    _, seg = PG.generate_parsing_map(sde, sdu, sdh, pose, attr, P.CLS_NUM)
    assert np.array_equal(seg.numpy(), gold["argmax"])


def test_mirrors_keep_the_checkpoint_abi_of_the_real_size_nets():
    from text2human_b200.parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet
    gold = np.load(GOLD)
    for m, key in ((ShapeAttrEmbedding(**P.REAL_EMBEDDER), "embedder_keys"),
                   (ShapeUNet(**P.REAL_SHAPE_UNET), "encoder_keys"), (FCNHead(**P.REAL_FCN_HEAD), "decoder_keys")):
        assert [f"{k}:{tuple(v.shape)}" for k, v in m.state_dict().items()] == list(gold[key]), key


def test_tiny_mirrors_load_the_recipe_state_dicts_strictly():
    mods, sds = _tiny()
    for m, sd in zip(mods, sds):
        m.load_state_dict(sd, strict=True)


def test_out_of_range_attributes_raise_before_any_launch():
    """F.one_hot rejects a class outside 0..n-1; the mirror raises ValueError naming the attribute, from the host
    check that precedes the launch (these CPU tensors would otherwise fail with the no-CPU-path error)"""
    from text2human_b200.parsing_gen_arch import ShapeAttrEmbedding
    emb = ShapeAttrEmbedding(**P.TINY_EMBEDDER).eval()
    sd = emb.state_dict()
    ok = P.every_class_attrs()
    emb.check_attributes(ok)                                 # every class of every attribute is accepted
    for i, bad in ((2, 6), (0, -1), (14, 2)):
        attr = ok.clone()
        attr[1, i] = bad
        with pytest.raises(ValueError, match=f"shape attribute {i} has value {bad}"):
            emb(attr)
        with pytest.raises(RuntimeError):                    # the reference's one_hot refuses it as well
            PG.shape_attr_embedding(sd, attr, P.CLS_NUM)
    with pytest.raises(ValueError):
        emb(ok[:, :14])
    with pytest.raises(ValueError):
        emb(ok.float())


@pytest.mark.parametrize("kw", [dict(strides=(1, 2, 1, 1, 1)), dict(enc_dilations=(1, 2, 1, 1, 1)),
                                dict(dec_dilations=(1, 1, 2, 1)), dict(with_cp=True), dict(dcn=dict(type="DCN")),
                                dict(plugins=[dict()]), dict(downsamples=(True, False, True, True))])
def test_shape_unet_rejects_unsupported_options(kw):
    from text2human_b200.parsing_gen_arch import ShapeUNet
    with pytest.raises(NotImplementedError):
        ShapeUNet(**P.TINY_SHAPE_UNET, **kw)


@pytest.mark.parametrize("kw", [dict(num_convs=2), dict(concat_input=True), dict(kernel_size=1)])
def test_fcn_head_rejects_unsupported_options(kw):
    from text2human_b200.parsing_gen_arch import FCNHead
    with pytest.raises(NotImplementedError):
        FCNHead(**dict(P.TINY_FCN_HEAD, **kw))
