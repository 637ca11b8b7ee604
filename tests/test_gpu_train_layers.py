"""GPU: the training-mode layers shared by the native trainers (text2human_b200/train_layers.py: ConvModuleL,
BasicConvBlockL, UpConvBlockL, UNetL) forward and backward against fp64 autograd of the same torch module in training
mode, with the same parameters: the output, every parameter gradient, the input gradient and the BatchNorm running
statistics.

The fp64 reference is CONDITIONED on the native pass: it takes the ReLU / LeakyReLU masks the native forward used (the
sign of x*scale+shift, restated from the layer's saved pre-activation and batch statistics with the kernel's fp32
scale / shift) and the max-pool argmax positions (from the native stage outputs, first maximum as the kernels route
it).  A rounding-level flip of a kink then cannot make a difference, so what is left is arithmetic and is held to a
bound of its own (TOL below).  Separately, every element whose native mask disagrees with the sign of the fp64
pre-activation is counted, and each must lie within FLIP_ULPS of its kink.

The last test runs the index-prediction fixture step this way.  Its UNet BatchNorm gradients differ from the
reference recording by up to 2.6e-2 because of such flips: conditioned on the native masks they agree with fp64 to
5e-5, and the three elements whose mask differs lie within ~100 rounding units of their kink."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import golden_recipes as R
import index_pred_train_recipes as IT
import parsing_gen_recipes as PG
from oracle import index_pred_train_ref as TR
from test_index_pred_train_oracle import GOLD

pytestmark = pytest.mark.gpu

# Conditioned error bounds, max |native - fp64| / max |fp64| per tensor, measured on an H100 and held with ~5x room.
# A single layer in fp32 mode (hi/lo fp16 planes, three products, fp32 accumulation over K = Cin * taps) lands within
# 1.5e-6: bound 1e-5.  A whole UNet chains 23 ConvModules, and its BatchNorms see few values per channel (4 at the
# bottleneck of a B = 2, 32x16 batch): their backward keeps du*gamma - mean(du*gamma) - xhat*mean(du*gamma*xhat), a
# difference of nearly equal terms, so the fp32 rounding of the forward and backward contractions reaches the weight
# gradients of the coarse stages amplified, 5e-5 .. 1e-3 depending on the widths (bounds per case below).  fp16 mode
# has one product of 11-bit operands: 8e-4 per layer, 4e-2 .. 8e-2 through a UNet (it varies from run to run with
# the order of the statistics kernels' atomic sums).
TOL_LAYER = {"fp32": 1e-5, "fp16": 4e-3}
TOL_UNET_FP16 = 0.25
# A flip is an element whose native ReLU mask differs from the sign of its fp64 pre-activation u.  Its distance from
# the kink, |u|, in units of 2^-24 * (|x * scale| + |shift|) of its channel (the fp32 rounding unit of the terms that
# form u, x the largest conv output of the channel) must stay below this.  Measured: fp32 flips lie within 1.4e3 such
# units, fp16 flips (2^13 units per operand rounding, compounded over the UNet) within 3e5.
FLIP_ULPS = {"fp32": 4096, "fp16": 2 ** 20}

KSP = {"k3": (3, 1, 1), "k1": (1, 1, 0), "k4s2": (4, 2, 1)}
SLOPE = {"relu": 0.0, "lrelu": 0.2}


def _setup(mode="fp32"):
    from text2human_b200 import ops
    ops.set_precision(mode)
    return ops


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


def _values(y):
    """a layer output as fp32 NHWC: fp32 as is, planes as the sum of their terms"""
    return y if y.dtype == torch.float32 else y.float().sum(0)


# ---------------------------------------------------------------------------- native side: a host and a recorder
def _host(device):
    from text2human_b200.train_layers import SingleSpaceTrainer

    class Host(SingleSpaceTrainer):
        """the layers' trainer: one ParamSpace (``space``), set once the layers exist"""
        def _nets(self):
            return {}
    h = Host()
    h.device = device
    return h


def _make_space(host, order, terms):
    from text2human_b200.flat_params import ParamSpace
    host.space = ParamSpace(order, host.device)
    host.space.prepare(terms)


@pytest.fixture
def rec(monkeypatch):
    """every ConvModuleL.fwd call in order: (layer, pre, st, output, drop); the library is unchanged"""
    from text2human_b200.train_layers import ConvModuleL
    log = []
    orig = ConvModuleL.fwd

    def fwd(self, a, out="planes", drop=None):
        y = orig(self, a, out=out, drop=drop)
        _, pre, st, _, _, _ = self.saved[-1]
        log.append(dict(layer=self, pre=pre.clone(), st=st.clone(), y=y, drop=drop))
        return y
    monkeypatch.setattr(ConvModuleL, "fwd", fwd)
    return log


def native_u(r):
    """the native forward's pre-activation x*scale+shift in fp64 (its sign is the mask the kernels used):
    scale = gamma * rstd and shift = beta - mean * scale in fp32 as the apply / backward kernels form them (the
    shift contracted to one fma), the product and sum exact in fp64 (the sign of a correctly rounded fma)"""
    layer, pre, st = r["layer"], r["pre"], r["st"]
    gamma, beta = layer._affine()
    C = pre.shape[-1]
    cnt = pre.numel() // C
    s, q = st[0, :, 0], st[0, :, 1]
    mean = s / cnt
    var = (q / cnt - mean * mean).clamp_min(0)
    rstd = (1.0 / torch.sqrt(var + layer.eps)).float()
    sc = gamma.float() * rstd
    sh = (beta.double() - mean.float().double() * sc.double()).float()
    return pre.double() * sc.double() + sh.double()


def native_masks(log):
    """-> per recorded layer the native mask (bool NCHW); checks it against the layer's own output where that
    output shows it (fp32 outputs exactly; planes except values below fp16's smallest subnormal)"""
    masks = []
    for r in log:
        u = native_u(r)
        m = u > 0
        y = _values(r["y"])
        live = torch.ones_like(m) if r["drop"] is None else \
            (r["drop"] != 0)[:, None, None, :].expand_as(m)
        seen = y > 0               # ReLU and LeakyReLU(0.2) alike, and a positive Dropout2d factor, keep the sign
        tiny = u.abs() < 2.0 ** -24 if r["y"].dtype != torch.float32 else torch.zeros_like(m)
        bad = live & (seen != m) & ~tiny
        assert not bool(bad.any()), ("the restated native mask disagrees with the layer's output", int(bad.sum()))
        masks.append(m.permute(0, 3, 1, 2))
    return masks


def pool_argmax(x):
    """fp32 NHWC stage output -> NCHW argmax [B,C,H/2,W/2] of each 2x2 window (row-major, first maximum)"""
    B, H, W, C = x.shape
    w = x.detach().view(B, H // 2, 2, W // 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H // 2, W // 2, 4)
    return w.argmax(-1)


def pool_at(x, idx):
    B, C, H, W = x.shape
    w = x.view(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)
    return w.gather(-1, idx.unsqueeze(-1)).squeeze(-1)


# ---------------------------------------------------------------------------- the conditioned fp64 reference
class Ref:
    """fp64 autograd of the torch modules, each ConvModule's activation taking the next recorded native mask"""

    def __init__(self, params, masks, device, running0):
        self.P = {id(p): p.detach().to(device).double().requires_grad_(True) for p in params}
        self.masks = iter(masks)
        self.running0 = running0      # id(BatchNorm2d) -> its running statistics before the native pass
        self.running = {}
        self.log = []                 # per ConvModule: (conv output, u, gamma, beta)

    def p(self, t):
        return self.P[id(t)]

    def cm(self, layer, x):
        """ConvModuleL ``layer``'s conv -> BatchNorm (batch statistics, running statistics updated) -> activation"""
        k, s, pad = KSP[layer.kind]
        convs = layer.conv.convs if hasattr(layer.conv, "convs") else (layer.conv,)
        w = torch.cat([self.p(c.weight) for c in convs], 0)
        y = F.conv2d(x, w, None, s, pad)
        gamma = torch.cat([self.p(bn.weight) for bn in layer.bns])
        beta = torch.cat([self.p(bn.bias) for bn in layer.bns])
        if layer not in self.running:
            self.running[layer] = tuple(torch.cat([self.running0[id(bn)][i] for bn in layer.bns]) for i in (0, 1))
        rm, rv = self.running[layer]
        u = F.batch_norm(y, rm, rv, gamma, beta, True, layer.momentum, layer.eps)
        self.log.append((y.detach(), u.detach(), gamma.detach(), beta.detach()))
        return torch.where(next(self.masks), u, SLOPE[layer.act] * u)

    def block(self, blk, x):
        for c in blk.convs:
            x = self.cm(c, x)
        return x

    def unet(self, L, unet, x, e, idx):
        """UNet / ShapeUNet forward (unet_arch.py:460-471 / :657-672) with the native argmax positions ``idx``"""
        enc = []
        for i, stage in enumerate(L.stages):
            a = x if i == 0 else pool_at(enc[-1], idx[i - 1])
            if e is not None:
                a = torch.cat([a, e[:, :, None, None].expand(-1, -1, *a.shape[2:])], 1)
            enc.append(self.block(stage, a))
        y = enc[-1]
        for i in reversed(range(len(L.dec))):
            d = L.dec[i]
            up = self.cm(d.up, F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=False))
            y = self.block(d.block, torch.cat([enc[i], up], 1))
        return y


def running0(*nets):
    """id(BatchNorm2d) -> fp64 copies of (running_mean, running_var): the state the reference starts from"""
    return {id(m): (m.running_mean.double().clone(), m.running_var.double().clone())
            for net in nets for m in net.modules() if isinstance(m, nn.BatchNorm2d)}


def flips(log, ref_log):
    """-> (elements whose native mask differs from the fp64 sign, their largest distance from the kink in ulps)"""
    n, worst = 0, 0.0
    for r, (y, u, gamma, beta) in zip(log, ref_log):
        m = native_u(r).permute(0, 3, 1, 2) > 0
        bad = m != (u > 0)
        if not bool(bad.any()):
            continue
        mean = y.mean((0, 2, 3))
        var = y.var((0, 2, 3), unbiased=False)
        sc = gamma / torch.sqrt(var + r["layer"].eps)
        sh = beta - mean * sc
        unit = 2.0 ** -24 * (sc.abs() * y.abs().amax((0, 2, 3)) + sh.abs())
        ulps = (u.abs() / unit[None, :, None, None])[bad]
        n += int(bad.sum())
        worst = max(worst, float(ulps.max()))
    return n, worst


def compare(tag, mode, pairs, log, ref, bn_layers, tol):
    """pairs: [(name, native, fp64)]; bn_layers: the ConvModuleLs whose running statistics to check"""
    errs = {name: _rel(got, want) for name, got, want in pairs}
    for layer in bn_layers:
        rm, rv = ref.running[layer]
        errs[f"running_mean {id(layer) % 997}"] = _rel(layer.rmean, rm)
        errs[f"running_var {id(layer) % 997}"] = _rel(layer.rvar, rv)
        assert all(int(bn.num_batches_tracked) == 1 for bn in layer.bns)
    n_flip, flip_ulps = flips(log, ref.log)
    name, worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"[train layers {mode} {tag}] worst conditioned error {worst:.2e} ({name}); {len(errs)} tensors; "
          f"mask flips {n_flip}, largest margin {flip_ulps:.1f} ulps")
    assert worst <= tol, sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    assert flip_ulps <= FLIP_ULPS[mode], (n_flip, flip_ulps)


def _grad_pairs(host, ref, params, names):
    return [(names[id(p)] + ".grad", host.space.g(p), ref.P[id(p)].grad) for p in params]


# ---------------------------------------------------------------------------- 1. ConvModuleL
CM_CASES = {
    "k3 relu planes": dict(kind="k3", act="relu", out="planes"),
    "k3 relu f32 drop": dict(kind="k3", act="relu", out="f32", drop=True),
    "k3 relu planes drop B=1": dict(kind="k3", act="relu", out="planes", drop=True, B=1),
    "k1 relu f32": dict(kind="k1", act="relu", out="f32"),
    "k1 relu planes drop": dict(kind="k1", act="relu", out="planes", drop=True),
    "k4s2 lrelu planes": dict(kind="k4s2", act="lrelu", out="planes"),
    "k4s2 lrelu f32 drop": dict(kind="k4s2", act="lrelu", out="f32", drop=True),
    "k3 need_dx=False": dict(kind="k3", act="relu", out="f32", need_dx=False),
    "k3 split": dict(kind="k3", act="relu", out="planes", split=8),
    "k3 want_params=False": dict(kind="k3", act="relu", out="f32", want_params=False),
    "k3 stack of 3, joint BatchNorm": dict(kind="k3", act="relu", out="f32", drop=True, stack=3),
}


@pytest.mark.parametrize("mode", ["fp32", "fp16"])
@pytest.mark.parametrize("case", list(CM_CASES))
def test_conv_module_layer(cuda, rec, case, mode):
    ops = _setup(mode)
    try:
        _conv_module_case(cuda, ops, rec, case, mode, **CM_CASES[case])
    finally:
        ops.set_precision("fp32")


def _conv_module_case(cuda, ops, rec, tag, mode, kind, act, out, drop=False, B=2, need_dx=True, split=None,
                      want_params=True, stack=0):
    from text2human_b200.flat_params import ConvStack
    from text2human_b200.train_layers import ConvModuleL
    k, s, pad = KSP[kind]
    ci, co, H, W = 24, 16, 16, 8
    seed = 700 + sum(map(ord, tag))
    n_conv = stack or 1
    cco = 8 if stack else co
    convs = [nn.Conv2d(ci, cco, k, s, pad, bias=False) for _ in range(n_conv)]
    bns = [nn.BatchNorm2d(cco) for _ in range(n_conv)]
    for m in convs + bns:
        m.load_state_dict(R.fill_state_dict(R.spec_of(m), seed))
        seed += 1
        m.to(cuda)
    host = _host(cuda)
    if stack:
        conv = ConvStack(convs)
        _make_space(host, [tuple(bns), conv], ops.get_terms())
    else:
        conv = convs[0]
        _make_space(host, [bns[0], conv], ops.get_terms())
    layer = ConvModuleL(host, conv, bns, kind, act, need_dx=need_dx)
    params = [c.weight for c in convs] + [p for bn in bns for p in (bn.weight, bn.bias)]
    names = {id(p): n for p, n in zip(params, [f"conv{i}.weight" for i in range(n_conv)] +
                                      [f"bn{i}.{w}" for i in range(n_conv) for w in ("weight", "bias")])}
    g = torch.Generator().manual_seed(seed)
    C = n_conv * cco
    x = torch.randn((B, H, W, ci), generator=g).to(cuda)
    Ho, Wo = (H // 2, W // 2) if s == 2 else (H, W)
    dy = torch.randn((B, Ho, Wo, C), generator=g).to(cuda)
    dmask = (torch.rand((B, C), generator=g) > 0.25).float().to(cuda) if drop else None
    dfac = dmask / 0.9 if drop else None
    a = ops.f32_to_planes(x, ops.CVT_S2D if s == 2 else ops.CVT_PLAIN)
    run0 = running0(*bns)
    y = layer.fwd(a, out=out, drop=dfac)
    dx = layer.bwd(dy, split=split, want_params=want_params)
    torch.cuda.synchronize()
    assert y.dtype == (torch.float32 if out == "f32" else torch.float16)
    ref = Ref(params, native_masks(rec), cuda, run0)
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = ref.cm(layer, x64)
    if drop:
        yr = yr * dfac.double()[:, :, None, None]
    (yr * dy.double().permute(0, 3, 1, 2)).sum().backward()
    pairs = [("output", _values(y), yr.detach().permute(0, 2, 3, 1))]
    gx = x64.grad.permute(0, 2, 3, 1)
    if not need_dx:
        assert dx is None
    elif split is not None:
        assert isinstance(dx, tuple) and len(dx) == 2
        pairs += [("dx[:split]", dx[0], gx[..., :split]), ("dx[split:]", dx[1], gx[..., split:])]
    else:
        pairs.append(("dx", dx, gx))
    if want_params:
        pairs += _grad_pairs(host, ref, params, names)
    else:
        assert float(host.space.flat_g.abs().max()) == 0.0       # no parameter gradient, nothing accumulated
    compare(tag, mode, pairs, rec, ref, [layer], TOL_LAYER[mode])
    if stack:   # the members' running statistics are views of the shared buffer
        for j, bn in enumerate(bns):
            assert bn.running_mean.data_ptr() == layer.rmean.data_ptr() + 4 * j * cco


# ---------------------------------------------------------------------------- 2. BasicConvBlockL, UpConvBlockL
@pytest.mark.parametrize("need_dx", [True, False])
def test_basic_conv_block(cuda, rec, need_dx):
    from text2human_b200.index_pred_arch import BasicConvBlock
    from text2human_b200.train_layers import BasicConvBlockL
    ops = _setup()
    blk = BasicConvBlock(24, 16).to(cuda)
    blk.load_state_dict(R.fill_state_dict(R.spec_of(blk), 811))
    host = _host(cuda)
    L = BasicConvBlockL(host, blk, need_dx=need_dx)
    order = [m for cm in reversed(L.convs) for m in (cm.bns[0], cm.conv)]
    _make_space(host, order, ops.get_terms())
    params = list(blk.parameters())
    names = {id(p): n for n, p in blk.named_parameters()}
    g = torch.Generator().manual_seed(812)
    x = torch.randn((2, 16, 8, 24), generator=g).to(cuda)
    dy = torch.randn((2, 16, 8, 16), generator=g).to(cuda)
    run0 = running0(blk)
    y = L.fwd(ops.f32_to_planes(x))
    dx = L.bwd(dy)
    torch.cuda.synchronize()
    ref = Ref(params, native_masks(rec), cuda, run0)
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = ref.block(L, x64)
    (yr * dy.double().permute(0, 3, 1, 2)).sum().backward()
    pairs = [("output", y, yr.detach().permute(0, 2, 3, 1))] + _grad_pairs(host, ref, params, names)
    if need_dx:
        pairs.append(("dx", dx, x64.grad.permute(0, 2, 3, 1)))
    else:
        assert dx is None
    compare(f"BasicConvBlock need_dx={need_dx}", "fp32", pairs, rec, ref, L.convs, TOL_LAYER["fp32"])


def test_up_conv_block(cuda, rec):
    """bilinear x2 -> 1x1 ConvModule, cat([skip, up]), the conv block; the block's first data gradient split at the
    skip's channels, the coarse input's gradient through the bilinear adjoint"""
    from text2human_b200.index_pred_arch import UpConvBlock
    from text2human_b200.train_layers import UpConvBlockL
    ops = _setup()
    ucb = UpConvBlock(32, 16, 16).to(cuda)
    ucb.load_state_dict(R.fill_state_dict(R.spec_of(ucb), 821))
    host = _host(cuda)
    L = UpConvBlockL(host, ucb)
    order = [m for cm in reversed([L.up] + L.block.convs) for m in (cm.bns[0], cm.conv)]
    _make_space(host, order, ops.get_terms())
    params = list(ucb.parameters())
    names = {id(p): n for n, p in ucb.named_parameters()}
    g = torch.Generator().manual_seed(822)
    skip = torch.randn((2, 16, 8, 16), generator=g).to(cuda)
    x = torch.randn((2, 8, 4, 32), generator=g).to(cuda)
    dy = torch.randn((2, 16, 8, 16), generator=g).to(cuda)
    run0 = running0(ucb)
    y = L.fwd(skip, x)
    d_skip, d_x = L.bwd(dy)
    torch.cuda.synchronize()
    ref = Ref(params, native_masks(rec), cuda, run0)
    s64 = skip.double().permute(0, 3, 1, 2).requires_grad_(True)
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    up = ref.cm(L.up, F.interpolate(x64, scale_factor=2, mode="bilinear", align_corners=False))
    yr = ref.block(L.block, torch.cat([s64, up], 1))
    (yr * dy.double().permute(0, 3, 1, 2)).sum().backward()
    pairs = [("output", y, yr.detach().permute(0, 2, 3, 1)), ("d_skip", d_skip, s64.grad.permute(0, 2, 3, 1)),
             ("d_x", d_x, x64.grad.permute(0, 2, 3, 1))] + _grad_pairs(host, ref, params, names)
    compare("UpConvBlock", "fp32", pairs, rec, ref, [L.up] + L.block.convs, TOL_LAYER["fp32"])


# ---------------------------------------------------------------------------- 3. UNetL
# B = 1 runs at 64x32: at 32x16 its bottleneck BatchNorm sees 2 values per channel, whose normalised values are
# +-1 whatever the input, so the input gradient there is the eps term alone (an fp32 difference of equal terms)
UNET_CASES = {
    "fixture UNet base 8, B=2 32x16": dict(net="unet", cfg=R.TINY_UNET, B=2, hw=(32, 16), tol=5e-4),
    "fixture UNet base 8, B=1 64x32": dict(net="unet", cfg=R.TINY_UNET, B=1, hw=(64, 32), tol=1e-3),
    "fixture UNet base 8, need_dx=False": dict(net="unet", cfg=R.TINY_UNET, B=2, hw=(32, 16), need_dx=False,
                                               tol=1e-3),
    "UNet 256 -> base 64, B=2 32x16": dict(net="unet", cfg=R.REAL_UNET, B=2, hw=(32, 16), need_dx=False, tol=3e-3),
    "ShapeUNet base 8 + e 16, B=2 32x16": dict(net="shape", cfg=PG.TINY_SHAPE_UNET, B=2, hw=(32, 16), tol=1e-3),
    "ShapeUNet base 64 + e 128, B=2 128x64": dict(net="shape", cfg=PG.REAL_SHAPE_UNET, B=2, hw=(128, 64), tol=5e-4),
}


def _unet_case(cuda, rec, tag, mode, net, cfg, B, hw, tol, need_dx=True):
    from text2human_b200.index_pred_arch import UNet
    from text2human_b200.parsing_gen_arch import ShapeUNet
    from text2human_b200.train_layers import UNetL
    ops = _setup(mode)
    unet = (UNet if net == "unet" else ShapeUNet)(**cfg)
    unet.load_state_dict(R.fill_state_dict(R.spec_of(unet), 900 + len(tag)))
    unet = unet.to(cuda).eval()
    host = _host(cuda)
    L = UNetL(host, unet, need_dx=need_dx)
    _make_space(host, L.order(), ops.get_terms())
    params = list(unet.parameters())
    names = {id(p): n for n, p in unet.named_parameters()}
    g = torch.Generator().manual_seed(901 + len(tag))
    H, W = hw
    x = torch.randn((B, H, W, cfg["in_channels"]), generator=g).to(cuda)
    e = torch.randn((B, unet.attr_embedding), generator=g).to(cuda) if net == "shape" else None
    base = unet.decoder[0].conv_block.convs[-1].conv.out_channels
    dy = torch.randn((B, H, W, base), generator=g).to(cuda)
    run0 = running0(unet)
    y = L.fwd(x, e)
    enc = L.saved[-1][1]
    idx = [pool_argmax(t) for t in enc[:-1]]
    de = torch.zeros_like(e) if e is not None else None
    L.bwd(dy, de)
    torch.cuda.synchronize()
    ref = Ref(params, native_masks(rec), cuda, run0)
    x64 = x.double().permute(0, 3, 1, 2)
    e64 = e.double().requires_grad_(True) if e is not None else None
    yr = ref.unet(L, unet, x64, e64, idx)
    (yr * dy.double().permute(0, 3, 1, 2)).sum().backward()
    pairs = [("output", y, yr.detach().permute(0, 2, 3, 1))] + _grad_pairs(host, ref, params, names)
    if e is not None:
        pairs.append(("de", de, e64.grad))
    layers = [c for s in L.stages for c in s.convs] + [c for d in L.dec for c in [d.up] + d.block.convs]
    compare(tag, mode, pairs, rec, ref, layers, tol if mode == "fp32" else TOL_UNET_FP16)


@pytest.mark.parametrize("case", list(UNET_CASES))
def test_unet_layer(cuda, rec, case):
    _unet_case(cuda, rec, case, "fp32", **UNET_CASES[case])


@pytest.mark.parametrize("case", ["fixture UNet base 8, B=2 32x16", "ShapeUNet base 8 + e 16, B=2 32x16"])
def test_unet_layer_fp16(cuda, rec, case):
    try:
        _unet_case(cuda, rec, case, "fp16", **UNET_CASES[case])
    finally:
        _setup("fp32")


# ---------------------------------------------------------------------------- 4. the index-prediction fixture step
def test_index_pred_fixture_step_conditioned(cuda, rec):
    """The whole fixture step of tests/test_gpu_index_pred_train.py (UNet, the 18 stacked head ConvModules with their
    Dropout2d draws, the routed loss) against fp64 autograd conditioned on the native masks and argmax positions:
    every one of the 156 gradients and every running statistic"""
    from test_gpu_index_pred_train import build, named
    _setup()
    gold = np.load(GOLD)
    tr, sds = build(cuda)
    feature, own, tex = IT.batch()
    masks = torch.from_numpy(gold["dropout_mask"])
    enc_box = []
    orig_fwd = tr.unet_l.fwd

    def unet_fwd(x, e=None):
        y = orig_fwd(x, e)
        enc_box.append([t.clone() for t in tr.unet_l.saved[-1][1]])
        return y
    tr.unet_l.fwd = unet_fwd
    run0 = running0(tr.unet, tr.fcn)
    tr.training_step(dropout_mask=masks, feature_t=feature, targets=(own, tex))
    torch.cuda.synchronize()
    params = named(tr)
    ref = Ref(list(params.values()), native_masks(rec), cuda, run0)
    idx = [pool_argmax(t) for t in enc_box[0][:-1]]
    x64 = feature.to(cuda).double()
    y = ref.unet(tr.unet_l, tr.unet, x64, None, idx)
    yh = ref.cm(tr.head, y)
    B, _, h, w = yh.shape
    drop = tr._drop_factor(masks, B).double()
    yh = yh * drop[:, :, None, None]
    C = tr.channels
    loss = 0
    for k, gt in enumerate(TR.gt_indices_list(own.to(cuda), tex.to(cuda))):
        lg = F.conv2d(yh[:, k * C:(k + 1) * C], ref.p(tr.segs[k].weight), ref.p(tr.segs[k].bias))
        loss = loss + F.cross_entropy(lg, gt, reduction="none", ignore_index=-1).mean()
    loss.backward()
    names = {id(p): k for k, p in params.items()}
    pairs = [(names[id(p)], p.grad / tr.loss_scale, ref.P[id(p)].grad) for p in params.values()
             if float(ref.P[id(p)].grad.abs().max()) > 0]
    layers = [c for s in tr.unet_l.stages for c in s.convs] + \
        [c for d in tr.unet_l.dec for c in [d.up] + d.block.convs] + [tr.head]
    compare("index pred fixture step", "fp32", pairs, rec, ref, layers, 2e-4)
