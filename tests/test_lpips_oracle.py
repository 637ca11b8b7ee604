"""CPU checks of the LPIPS restatement (oracle/lpips_ref.py) and of the mirror's parameter layout
(text2human_b200/lpips.py): slice outputs against torchvision's VGG16, state_dict keys and shapes as lpips 0.1.4
names them, loading torchvision / lpips weight files, and the rejected configurations."""
import os

import pytest
import torch

import lpips_recipes as LR
from oracle import lpips_ref
from text2human_b200.lpips import LPIPS


def test_restatement_slices_match_torchvision_features():
    torchvision = pytest.importorskip("torchvision")
    torch.manual_seed(0)
    feats = torchvision.models.vgg16(weights=None).features.double().eval()
    sd = {}
    for i, m in enumerate(feats):
        if isinstance(m, torch.nn.Conv2d):
            key = lpips_ref._slice_key(i)
            sd[key + ".weight"], sd[key + ".bias"] = m.weight.detach(), m.bias.detach()
    x = torch.randn(2, 3, 32, 48, dtype=torch.float64)
    got = lpips_ref.slices(sd, x)
    with torch.no_grad():
        for out, end in zip(got, (4, 9, 16, 23, 30)):
            want = feats[:end](x)
            assert out.shape == want.shape
            assert torch.equal(out, want), end


def _want_keys():
    want = {"scaling_layer.shift": (1, 3, 1, 1), "scaling_layer.scale": (1, 3, 1, 1)}
    for k, convs in enumerate(LR.CONVS):
        for i, cin, cout in convs:
            want[f"net.slice{k + 1}.{i}.weight"] = (cout, cin, 3, 3)
            want[f"net.slice{k + 1}.{i}.bias"] = (cout,)
    for k, c in enumerate(LR.CHNS):
        want[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
        want[f"lins.{k}.model.1.weight"] = (1, c, 1, 1)     # lpips registers its heads under both names
    return want


def test_mirror_state_dict_keys_and_shapes():
    got = {k: tuple(v.shape) for k, v in LPIPS(pretrained=False).state_dict().items()}
    assert got == _want_keys()


def test_pretrained_loads_torchvision_and_lpips_files(tmp_path):
    torchvision = pytest.importorskip("torchvision")
    torch.manual_seed(1)
    tv = torchvision.models.vgg16(weights=None).state_dict()           # features.N.* and classifier.*
    vgg_path = os.path.join(tmp_path, "vgg16-397923af.pth")
    torch.save(tv, vgg_path)
    sd = LR.state_dict()
    lin = {f"lin{k}.model.1.weight": sd[f"lin{k}.model.1.weight"] for k in range(5)}
    model_path = os.path.join(tmp_path, "vgg.pth")
    torch.save(lin, model_path)
    m = LPIPS(pretrained=True, net="vgg", model_path=model_path, vgg_path=vgg_path)
    msd = m.state_dict()
    for k, convs in enumerate(LR.CONVS):
        for i, _, _ in convs:
            assert torch.equal(msd[f"net.slice{k + 1}.{i}.weight"], tv[f"features.{i}.weight"])
            assert torch.equal(msd[f"net.slice{k + 1}.{i}.bias"], tv[f"features.{i}.bias"])
    for k in range(5):
        assert torch.equal(msd[f"lin{k}.model.1.weight"], lin[f"lin{k}.model.1.weight"])
        assert torch.equal(msd[f"lins.{k}.model.1.weight"], lin[f"lin{k}.model.1.weight"])
    # the state dict of a real lpips.LPIPS instance has exactly these keys: it round-trips strictly
    LPIPS(pretrained=False).load_state_dict(msd, strict=True)
    assert not any(p.requires_grad for p in m.parameters())


def test_pretrained_without_files_names_both():
    with pytest.raises(FileNotFoundError) as e:
        LPIPS()
    assert "vgg16-397923af.pth" in str(e.value) and "weights/v0.1/vgg.pth" in str(e.value)


@pytest.mark.parametrize("kw", [dict(net="alex"), dict(net="squeeze"), dict(lpips=False), dict(spatial=True),
                                dict(version="0.0")])
def test_rejected_configurations(kw):
    with pytest.raises(NotImplementedError):
        LPIPS(pretrained=False, **kw)


def test_rejected_inputs_before_any_launch():
    m = LPIPS(pretrained=False)
    x = torch.zeros(2, 3, 32, 16)
    with pytest.raises(NotImplementedError):
        m(x, x, normalize=True)
    with pytest.raises(NotImplementedError):
        m(x.clone().requires_grad_(True), x)
    with pytest.raises(ValueError):
        m(x, torch.zeros(2, 3, 32, 32))
    with pytest.raises(ValueError):
        m(torch.zeros(2, 4, 32, 16), torch.zeros(2, 4, 32, 16))
    with pytest.raises(ValueError):
        m(torch.zeros(2, 3, 24, 16), torch.zeros(2, 3, 24, 16))
    from text2human_b200._lib import T2HError
    with pytest.raises(T2HError):
        m(x, x)


def test_restatement_dead_pixels_give_finite_gradient():
    """relu5_3 zero everywhere: torch's threshold_backward masks the NaN of sqrt's backward at 0"""
    sd = {k: v.double() for k, v in LR.state_dict(dead_slice5=True).items()}
    x0 = torch.rand(1, 3, 32, 16, dtype=torch.float64) * 2 - 1
    x1 = (torch.rand(1, 3, 32, 16, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    v = lpips_ref.lpips(sd, x0, x1)
    v.sum().backward()
    assert torch.isfinite(v).all() and torch.isfinite(x1.grad).all() and x1.grad.abs().max() > 0
