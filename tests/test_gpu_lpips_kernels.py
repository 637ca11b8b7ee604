"""GPU: the LPIPS kernels (csrc/lpips.cu) element by element against fp64, and one whole native LPIPS call stage by
stage and end to end against the fp64 restatement CONDITIONED on the native pass.

Section 1 runs each kernel on synthetic inputs: the ScalingLayer and its adjoint, the fused head (value and gradient
planes) and the ReLU backward, at the shapes and values where they can go wrong (partly empty lanes, grid-stride
loops, several pixels per warp, all-zero and negative pixels, preloaded accumulators, the fp16 range).

Section 2 records one ``LPIPS.run`` (every conv, data gradient, head, ReLU backward, max-pool and scaling call, their
inputs and outputs cloned at call time) and checks every stage on its own recorded inputs against an fp64 statement
of the same operation.  It then runs ``oracle.lpips_ref.lpips_conditioned`` with the native pass's ReLU masks (hi plane
> 0 for a slice's inner convs, the rule of relu_bwd; fp32 > 0 for its last conv, the rule of the head) and max-pool
picks (first maximum of the fp32 window, the rule of maxpool2_bcast_bwd).  With those discrete choices imposed the
gap between native and fp64 is arithmetic.  Every element whose native mask disagrees with the sign of the conditioned
fp64 pre-activation, and every window whose pick differs, is counted, and each must lie within a stated number of
rounding units of its kink or tie.  Those flips are what the unconditioned comparison in test_gpu_lpips.py sees."""
import math
import types

import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R
import lpips_recipes as LR
from oracle import lpips_ref

pytestmark = pytest.mark.gpu

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
SPLIT_MAX = 65519.99609375          # the largest fp32 whose hi/lo fp16 split is finite (csrc/lpips.cu kSplitMax)
# rounding unit of one operand / output per precision mode: fp32 mode carries hi+lo planes (fp32-equivalent), fp16
# mode one fp16 plane
EPS = {"fp32": 2.0 ** -24, "fp16": 2.0 ** -11}

# Bounds, measured on an H100 80GB HBM3 (700 W power limit) and held with 3-5x room.
# The head's value (fp32 per pixel, fp64 sums): within 1.9e-7 relative.  Its planes: within 2.2e-7 of each pixel's
# gradient scale (head_ref), beyond what the planes can represent.
HEAD_VALUE_REL = 1e-6
HEAD_PLANE_REL = 1e-6
# Each stage of a whole call on its own recorded inputs, in rounding units (EPS) of |w| * |x| + |b| (forward convs)
# or |dy| * |w| (data gradients): fp32 mode within 65 (the data gradients of slices 4 and 5, K = 4608 fp32
# accumulations of three fp16 products each, the lo planes of small weights subnormal), fp16 mode within 1.7.
STAGE_UNITS = {"fp32": 256.0, "fp16": 8.0}
# The whole call against lpips_conditioned: fp32 mode value within 2.9e-7 relative, image gradient within 5.2e-6
# (norm) and 6.3e-6 (worst element / largest) at every size; fp16 mode 1.1e-5, 9.0e-4, 1.0e-3.
E2E = {"fp32": dict(value=1e-6, gnorm=2e-5, gmax=3e-5), "fp16": dict(value=5e-5, gnorm=4e-3, gmax=4e-3)}
# Mask and pick flips, in fp32 rounding units 2^-24 (|w| * |x| + |b|) of the element: fp32 mode within 29.4 (mask,
# 74 flips at 3 x 256 x 128) and 5.1 (pick, 16), fp16 mode within 4003 and 1511 (about two fp16 roundings).
FLIP_UNITS = {"fp32": 128.0, "fp16": 2.0 ** 14}


def _ops(mode="fp32"):
    from text2human_b200 import ops
    ops.set_precision(mode)
    return ops


def _bits(t):
    return t.contiguous().view(torch.int16)


def split_ref(v, terms):
    """the kernels' split_f16 in torch: hi = fp16(v), lo = fp16(v - hi) -> [terms, ...]"""
    hi = v.half()
    if terms == 1:
        return hi[None]
    return torch.stack((hi, (v - hi.float()).half()))


def decode(p):
    """planes [T, ...] -> fp64 hi + lo (exact: the two fp16 values span fewer than 53 bits)"""
    return p.double().sum(0)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ============================================================================ 1. kernel by kernel
# ---------------------------------------------------------------------------- ScalingLayer
def check_scale_fwd(x0, x1, shift, scale, out, mode):
    """out [T,2B,H,W,8] of lpips_scale_fwd(x0, x1): in0's images first, bit-exact against the kernel's fp32 recipe
    (x - shift) * (1 / scale) -- a multiplication by the fp32 reciprocal, not a division; channels 3..7 +0 in every
    plane.  -> the worst distance of the planes from the fp64 value, beyond what the planes cannot represent (2^-25,
    half the fp16 subnormal spacing, where the last plane is subnormal, and that plane's rounding: 2^-22 of the value
    for hi + lo, whose lo has 11 bits, 2^-11 for hi alone), in rounding units of (|x| + |shift|) / scale"""
    terms = out.shape[0]
    x = torch.cat([x0, x1]).permute(0, 2, 3, 1).float().cpu()
    s, sc = shift.float().cpu().reshape(3), scale.float().cpu().reshape(3)
    r = torch.tensor(1.0, dtype=torch.float32) / sc                 # IEEE fp32 division, as 1.f / scale[c]
    v = (x - s) * r
    got = out.cpu()
    assert torch.equal(_bits(got[..., :3]), _bits(split_ref(v, terms))), "scale_fwd planes differ from the fp32 recipe"
    assert not bool(_bits(got[..., 3:]).any()), "scale_fwd: padding channels 3..7 not +0"
    v64 = (x.double() - s.double()) / sc.double()
    unit = EPS[mode] * (x.double().abs() + s.double().abs()) / sc.double()
    rep = 2.0 ** -25 + v64.abs() * (2.0 ** -22 if terms == 2 else 2.0 ** -11)
    return float((((decode(got[..., :3]) - v64).abs() - rep).clamp_min(0) / unit).max())


@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("B,H,W", [(1, 32, 16), (3, 48, 80), (4, 512, 256)])
def test_scale_fwd(cuda, terms, B, H, W):
    """(4, 512, 256): 2 B H W = 1 M threads of work, above the grid cap of num_sms * 16 * 256, so the grid-stride loop
    runs more than once"""
    ops = _ops()
    g = _gen(11 + B)
    x0 = (torch.rand((B, 3, H, W), generator=g) * 2.4 - 1.2).to(cuda)
    x1 = (torch.rand((B, 3, H, W), generator=g) * 2.4 - 1.2).to(cuda)
    shift, scale = torch.tensor(SHIFT, device=cuda), torch.tensor(SCALE, device=cuda)
    out = ops.lpips_scale_fwd(x0, x1, shift, scale, terms=terms)
    assert out.shape == (terms, 2 * B, H, W, 8)
    err = check_scale_fwd(x0, x1, shift, scale, out, "fp32" if terms == 2 else "fp16")
    print(f"[lpips scale_fwd T={terms} {B}x{H}x{W}] planes vs fp64 {err:.2f} units (bound 2)")
    assert err <= 2.0, err


def check_scale_bwd(d, scale, alpha, g0, g):
    """g = g0 + alpha * d[..., :3] / scale (NHWC -> NCHW), within 3 fp32 rounding units of |g0| + |alpha d / scale|
    (the rounded alpha / scale, the product and the sum).  -> worst error in units"""
    k = alpha / scale.double().reshape(1, 3, 1, 1)
    dd = d[..., :3].double().permute(0, 3, 1, 2)
    want = g0.double() + k * dd
    unit = EPS["fp32"] * (g0.double().abs() + (k * dd).abs())
    return float(((g.double() - want).abs() / unit).max())


@pytest.mark.parametrize("B,H,W,ld,alpha", [(1, 32, 16, 8, 0.75), (2, 48, 80, 16, 3.0 / 2 ** 19),
                                            (4, 512, 256, 8, 1.0)])
def test_scale_bwd(cuda, B, H, W, ld, alpha):
    """g is preloaded (the kernel adds); channels >= 3 of d hold NaN, which must not be read"""
    ops = _ops()
    gen = _gen(21 + ld)
    d = torch.randn((B, H, W, ld), generator=gen)
    d[..., 3:] = float("nan")
    g0 = torch.randn((B, 3, H, W), generator=gen)
    d, g0 = d.to(cuda), g0.to(cuda)
    scale = torch.tensor(SCALE, device=cuda)
    g = g0.clone()
    ops.lpips_scale_bwd(d, scale, alpha, g)
    err = check_scale_bwd(d, scale, alpha, g0, g)
    print(f"[lpips scale_bwd {B}x{H}x{W} ld {ld}] {err:.2f} units (bound 3)")
    assert err <= 3.0, err


# ---------------------------------------------------------------------------- the head
def head_ref(f0, f1, w, gscale, gin):
    """fp64 head over NHWC features: -> (per-image spatial mean of sum_c w_c (unit(f0) - unit(f1))_c^2 [B],
    planes value (f1 > 0) * (gin + gscale * d(per-pixel d)/df1) [B,h,w,C], each pixel's gradient scale [B,h,w,1]).
    The gradient is torch autograd's; its NaN at an all-zero pixel is masked as torch's threshold_backward masks it.
    The scale is max_c |gin_c| plus the larger of gscale max_c |dd/df1_c| and gscale |2 w (|u| + |v|)| / |f1|: dd/df1
    is gv = -2 w (u - v) made orthogonal to f1, over |f1|, so where u ~ v or gv is nearly parallel to f1 it is a small
    difference of terms of that size, and their fp32 rounding is what the kernel can be held to."""
    x0 = f0.double()
    x = f1.double().requires_grad_(True)
    w64 = w.double().reshape(-1)

    def norm(t):
        return torch.sqrt((t ** 2).sum(-1, keepdim=True))
    dpix = (w64 * (x0 / (norm(x0) + 1e-10) - x / (norm(x) + 1e-10)) ** 2).sum(-1)
    (gd,) = torch.autograd.grad(dpix.sum(), x)
    gd = gscale * gd
    gi = gin.double() if gin is not None else torch.zeros_like(gd)
    pos = x.detach() > 0
    want = torch.where(pos, gi + gd, torch.zeros_like(gd))
    n1 = norm(x.detach())
    gv = 2 * w64 * ((x0 / (norm(x0) + 1e-10)).abs() + (x.detach() / (n1 + 1e-10)).abs())
    terms = torch.where(n1 > 0, gscale * norm(gv) / n1, 0.0)
    scale = gi.abs().amax(-1, keepdim=True) + torch.maximum(gd.nan_to_num(0.0).abs().amax(-1, keepdim=True), terms)
    return dpix.detach().mean((1, 2)), want, scale


def check_head(f0, f1, w, gscale, gin, acc0, acc, planes, sat_ok=False):
    """-> (value error relative, planes error relative to each pixel's gradient scale, saturated elements).  The
    planes are +0 wherever f1 <= 0 (gin there dropped); elements whose fp64 value passes SPLIT_MAX are saturated
    exactly (sat_ok) and elsewhere compared"""
    val, want, scale = head_ref(f0, f1, w, gscale, gin)
    vrel = float(((acc.double() - acc0.double() - val).abs() / val.abs().clamp_min(1e-300)).max())
    if planes is None:
        return vrel, 0.0, 0
    terms = planes.shape[0]
    assert torch.isfinite(planes.float()).all(), "head planes not finite"
    dead = (f1 <= 0)
    assert not bool(_bits(planes[:, dead]).any()), "head planes nonzero where f1 <= 0"
    got = decode(planes)
    sat = want.abs() > SPLIT_MAX
    n_sat = int(sat.sum())
    if n_sat:
        assert sat_ok, n_sat
        assert torch.equal(got[sat], torch.sign(want[sat]) * (65520.0 if terms == 2 else 65504.0))   # hi 65504, lo 16
    # what the planes cannot represent: half the fp16 subnormal spacing (2^-25) where the lo plane (or the one plane)
    # is subnormal, and the rounding of the last plane, 2^-22 (hi + lo) or 2^-11 (hi alone) of the value
    err = ((got - want).abs() - 2.0 ** -25 - want.abs() * (2.0 ** -22 if terms == 2 else 2.0 ** -11)).clamp_min(0)
    prel = float(torch.where(sat, 0, err / scale.clamp_min(1e-300)).max())
    return vrel, prel, n_sat


def head_inputs(seed, B, h, w, C, cuda, with_gin):
    """f0 >= 0 (a ReLU output), f1 = f0 + noise (negative entries), lin weights |N(0,1)| / C; pixels 0 / 1 / 2 of
    image 0 (where present): f1 all zero, f0 all zero, f1 all negative; gin nonzero everywhere"""
    g = _gen(seed)
    f0 = torch.randn((B, h, w, C), generator=g).clamp_min(0)
    f1 = f0 + 0.3 * torch.randn((B, h, w, C), generator=g)
    if h * w >= 3:
        f1.view(B, -1, C)[0, 0] = 0
        f0.view(B, -1, C)[0, 1] = 0
        f1.view(B, -1, C)[0, 2] = -f1.view(B, -1, C)[0, 2].abs() - 0.1
    wl = torch.randn((C,), generator=g).abs() / C
    gin = 0.5 * torch.randn((B, h, w, C), generator=g) if with_gin else None
    to = (lambda t: None if t is None else t.to(cuda))
    return to(f0), to(f1), to(wl), to(gin)


def _gscale(hw):
    return 2.0 ** (math.floor(math.log2(hw)) + 6) / hw


HEAD_HW = [(1, 1), (3, 5), (128, 64), (96, 128)]      # 1, 15 (< one block's 8 warps), 8192, 12288 (> 256 chunks)


@pytest.mark.parametrize("h,w", HEAD_HW)
@pytest.mark.parametrize("C", [4, 60, 64, 132, 512])
def test_head(cuda, C, h, w):
    """value and gradient planes against the fp64 head; B 1 and 5, gin absent and given, terms 1 and 2 (the lo plane
    at offset b hw c), sum_out preloaded (+=); want_grad=False gives the same sums; two calls are bit-identical"""
    ops = _ops()
    gs = _gscale(h * w)
    worst = [0.0, 0.0]
    for B, with_gin, terms in ((1, False, 2), (5, True, 2), (5, True, 1)):
        f0, f1, wl, gin = head_inputs(1000 + C + h * w + B, B, h, w, C, cuda, with_gin)
        acc0 = torch.randn((B,), generator=_gen(C), dtype=torch.float64).to(cuda)
        acc = acc0.clone()
        planes = ops.lpips_head(f0, f1, wl, acc, gscale=gs, gin=gin, want_grad=True, terms=terms)
        assert planes.shape == (terms, B, h, w, C)
        vrel, prel, _ = check_head(f0, f1, wl, gs, gin, acc0, acc, planes)
        worst = [max(worst[0], vrel), max(worst[1], prel)]
        acc2 = acc0.clone()
        planes2 = ops.lpips_head(f0, f1, wl, acc2, gscale=gs, gin=gin, want_grad=True, terms=terms)
        assert torch.equal(acc2, acc) and torch.equal(_bits(planes2), _bits(planes)), "head not deterministic"
        acc3 = acc0.clone()
        assert ops.lpips_head(f0, f1, wl, acc3, gscale=gs, want_grad=False) is None
        assert torch.equal(acc3, acc), "want_grad=False changes the sums"
    print(f"[lpips head C={C} {h}x{w}] value rel {worst[0]:.2e} (bound {HEAD_VALUE_REL:.0e}), planes rel to the "
          f"pixel's gradient scale {worst[1]:.2e} (bound {HEAD_PLANE_REL:.0e})")
    assert worst[0] <= HEAD_VALUE_REL and worst[1] <= HEAD_PLANE_REL, worst


@pytest.mark.parametrize("terms", [2, 1])
def test_head_small_f1_stays_finite(cuda, terms):
    """One pixel's f1 nonzero with its norm swept through the fp16 overflow of the scaled gradient (~ gscale * 2 w
    |u - v| / |f1|, gscale = 64 at slice 1): the planes stay finite, elements whose fp64 value passes fp16's range are
    saturated (hi 65504, lo 16), every other element matches fp64.  Unsaturated, such a split gives hi = +inf,
    lo = -inf, and NaN in every contraction that reads both."""
    ops = _ops()
    B, h, w, C = 2, 128, 64, 64
    gs = _gscale(h * w)
    f0, f1, wl, gin = head_inputs(77, B, h, w, C, cuda, True)
    direction = f1.view(B, -1, C)[1, 100].clamp_min(0).clone()
    direction /= direction.norm()
    sats, worst = [], 0.0
    for s in (1e-2, 1e-3, 1e-4, 1e-5, 1e-6, 1e-7):
        f1.view(B, -1, C)[1, 100] = s * direction
        acc0 = torch.zeros((B,), dtype=torch.float64, device=cuda)
        acc = acc0.clone()
        planes = ops.lpips_head(f0, f1, wl, acc, gscale=gs, gin=gin, terms=terms)
        vrel, prel, n_sat = check_head(f0, f1, wl, gs, gin, acc0, acc, planes, sat_ok=True)
        sats.append(n_sat)
        worst = max(worst, prel)
        assert vrel <= HEAD_VALUE_REL and prel <= HEAD_PLANE_REL, (s, vrel, prel)
    print(f"[lpips head small |f1| T={terms}] saturated elements per |f1| 1e-2 .. 1e-7: {sats}, planes rel to the "
          f"pixel's gradient scale {worst:.2e} (bound {HEAD_PLANE_REL:.0e})")
    assert sats[0] == 0 and sats[-1] > 0


# ---------------------------------------------------------------------------- ReLU backward
def relu_bwd_ref(y_hi, dy, terms):
    v = torch.where(y_hi.float() > 0, dy, torch.zeros_like(dy))
    return split_ref(v.clamp(-SPLIT_MAX, SPLIT_MAX), terms)


@pytest.mark.parametrize("terms", [1, 2])
def test_relu_bwd(cuda, terms):
    """bit-exact against split(dy * (y_hi > 0)) in torch: y in (0, 2^-25] rounds to an fp16 0 and passes nothing,
    y just above 2^-24 (and everything above 2^-25) passes; |dy| beyond fp16's range saturates"""
    ops = _ops()
    g = _gen(31)
    n = 8 * 40000 + 8 * 3
    y = torch.randn((n,), generator=g).clamp_min(0)
    tiny = torch.tensor([2.0 ** -25, 2.0 ** -26, 1e-9, 2.0 ** -25 * 1.0001, 2.0 ** -24, 2.0 ** -24 * 1.001,
                         2.0 ** -23, 0.0])
    y[:8] = tiny
    y_hi = y.half()
    assert (y_hi[:3] == 0).all() and (y_hi[3:7] > 0).all()
    dy = torch.randn((n,), generator=g) * torch.exp(4 * torch.randn((n,), generator=g))
    dy[8:16] = torch.tensor([1e6, -1e6, 65519.0, 65520.0, -65530.0, 1e30, 3e-8, -0.0])
    y[8:16] = 1.0
    y_hi = y.half()
    dy, y_hi = dy.view(-1, 8).to(cuda), y_hi.view(-1, 8).to(cuda)
    out = ops.relu_bwd(y_hi, dy, terms=terms)
    assert out.shape == (terms,) + tuple(dy.shape)
    want = relu_bwd_ref(y_hi, dy, terms)
    assert torch.equal(_bits(out), _bits(want)), int((_bits(out) != _bits(want)).sum())
    assert torch.isfinite(out.float()).all()


# ============================================================================ 2. one native LPIPS call
class Recorder:
    """Every trunk conv, data gradient and LPIPS kernel call of LPIPS.run, in order: (name, args, kwargs, args and
    kwargs after the call, output), tensors cloned at call time (run() frees features and planes as it goes, and
    several calls write into their arguments).  The library itself is unchanged."""

    NAMES = ("f32_to_planes", "lpips_head", "relu_bwd", "maxpool2_bcast_bwd", "lpips_scale_fwd", "lpips_scale_bwd")

    def __init__(self, monkeypatch):
        from text2human_b200 import conv_grad, ops
        from text2human_b200 import lpips as L
        self.ev = []
        ns = types.SimpleNamespace(**{k: getattr(conv_grad, k) for k in dir(conv_grad) if not k.startswith("__")})
        ns.forward = self._wrap("forward", conv_grad.forward)
        ns.dgrad = self._wrap("dgrad", conv_grad.dgrad)
        monkeypatch.setattr(L, "G", ns)
        for name in self.NAMES:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    @staticmethod
    def _clone(x):
        if isinstance(x, torch.Tensor):
            return x.clone()
        if isinstance(x, (tuple, list)):
            return type(x)(Recorder._clone(v) for v in x)
        if isinstance(x, dict):
            return {k: Recorder._clone(v) for k, v in x.items()}
        return x

    def _wrap(self, name, fn):
        def call(*args, **kw):
            before = (self._clone(args), self._clone(kw))
            out = fn(*args, **kw)
            self.ev.append(types.SimpleNamespace(name=name, args=before[0], kw=before[1],
                                                 after=(self._clone(args), self._clone(kw)), out=self._clone(out)))
            return out
        return call

    def of(self, name):
        return [e for e in self.ev if e.name == name]


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _conv_keys():
    """per flat conv index (CONV_IDX order): (state-dict prefix, slice, last conv of its slice?)"""
    out = []
    for k, idxs in enumerate(lpips_ref.CONV_IDX):
        for j, i in enumerate(idxs):
            out.append((lpips_ref._slice_key(i), k, j == len(idxs) - 1))
    return out


def native_choices(rec, B):
    """the native pass's masks (bool NCHW, 2B images, per conv) and max-pool picks (per pool) as lpips_conditioned
    takes them: hi plane > 0 for an inner conv (relu_bwd's rule), fp32 > 0 for a slice's last conv (the head's),
    first maximum of the fp32 window (maxpool2_bcast_bwd's)"""
    masks = []
    for e, (_, _, last) in zip(rec.of("forward"), _conv_keys()):
        y = e.out
        masks.append(_nchw(y > 0 if last else y[0] > 0))
    picks = [lpips_ref.pool_windows(_nchw(e.args[0])).argmax(-1) for e in rec.of("f32_to_planes")]
    return masks, picks


def stage_checks(rec, sd, B, mode):
    """every recorded stage on its own recorded inputs against fp64 -> {stage: worst error in rounding units}"""
    eps = EPS[mode]
    keys = _conv_keys()
    res = {}
    # the ScalingLayer
    e = rec.of("lpips_scale_fwd")[0]
    res["scale_fwd"] = check_scale_fwd(e.args[0], e.args[1], e.args[2], e.args[3], e.out, mode)
    # the forward convs: ReLU(conv(decoded input)) in units of eps * (|w| * |x| + |b|)
    fwd = rec.of("forward")
    for e, (p, k, last) in zip(fwd, keys):
        w64, b64 = sd[p + ".weight"], sd[p + ".bias"]
        x = _nchw(decode(e.args[1]))[:, :w64.shape[1]]
        want = F.relu(F.conv2d(x, w64, b64, padding=1))
        got = _nchw(e.out.double() if last else decode(e.out))
        unit = eps * (F.conv2d(x.abs(), w64.abs(), b64.abs(), padding=1))
        rep = 2.0 ** -25 + want.abs() * (2.0 ** -22 if mode == "fp32" else 2.0 ** -11)
        err = (got - want).abs() if last else ((got - want).abs() - rep).clamp_min(0)
        res[f"fwd {p}"] = float((err / unit).max())
    # the data gradients: conv_transpose of the decoded gradient planes; padded input channels exactly 0
    dg = rec.of("dgrad")
    for e, (p, k, last) in zip(dg, reversed(keys)):
        w64 = sd[p + ".weight"]
        dy = _nchw(decode(e.args[1]))
        want = F.conv_transpose2d(dy, w64, padding=1)
        got = _nchw(e.out.double())
        ci = w64.shape[1]
        assert not bool(got[:, ci:].any()), f"dgrad {p}: padded channels nonzero"
        unit = eps * F.conv_transpose2d(dy.abs(), w64.abs(), padding=1)
        res[f"dgrad {p}"] = float(((got[:, :ci] - want).abs() / unit.clamp_min(1e-300)).max())
    # the heads
    for e in rec.of("lpips_head"):
        f0, f1, wl, acc0 = e.args
        acc = e.after[0][3]
        vrel, prel, n_sat = check_head(f0, f1, wl, e.kw["gscale"], e.kw["gin"], acc0, acc, e.out)
        assert n_sat == 0
        res[f"head C={f1.shape[-1]} value rel"] = vrel
        res[f"head C={f1.shape[-1]} planes rel"] = prel
    # the ReLU backward: bit-exact, and its y is the inner conv's own in1 hi plane
    inner = [e for e, (_, _, last) in zip(fwd, keys) if not last]
    rb = rec.of("relu_bwd")
    assert len(rb) == len(inner)
    for e, f in zip(rb, reversed(inner)):
        y_hi, dy = e.args
        assert torch.equal(_bits(y_hi), _bits(f.out[0, B:])), "relu_bwd mask is not the conv's in1 hi plane"
        assert torch.equal(_bits(e.out), _bits(relu_bwd_ref(y_hi, dy, e.out.shape[0]))), "relu_bwd differs"
    # the max-pool backward: routed to the first maximum of the fp32 window of the forward's own pooled tensor
    pools = rec.of("f32_to_planes")
    for e, pf in zip(rec.of("maxpool2_bcast_bwd"), reversed(pools)):
        d, c = e.args[0], e.args[1]
        x, dx = e.kw["x"], e.after[1]["dx"]
        assert torch.equal(x, pf.args[0][B:]), "max-pool backward does not see the forward's pooled tensor"
        pick = lpips_ref.pool_windows(_nchw(x)).argmax(-1)
        routed = F.one_hot(pick, 4).to(d.dtype) * _nchw(d[..., :c])[..., None]
        Bn, C, h, w, _ = routed.shape
        want = routed.view(Bn, C, h, w, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(Bn, C, 2 * h, 2 * w)
        assert torch.equal(_nchw(dx), want), "max-pool backward routing differs"
    # the ScalingLayer's adjoint
    e = rec.of("lpips_scale_bwd")[0]
    res["scale_bwd"] = check_scale_bwd(e.args[0], e.args[1], e.args[2], e.args[3], e.after[0][3])
    return res


def flips(trace, masks, picks, sd):
    """-> (mask flips, their largest distance from the kink in fp32 rounding units 2^-24 (|w| * |x| + |b|),
    elements with 0 < u <= 2^-25 dropped by design (an inner conv's fp16 hi plane rounds them to 0),
    pick flips, their largest margin in the same units)"""
    convs = [t for t in trace if isinstance(t, tuple)]
    pools = [t for t in trace if not isinstance(t, tuple)]
    keys = _conv_keys()
    units = {}

    def unit(i):
        if i not in units:
            p = keys[i][0]
            x, _ = convs[i]
            units[i] = 2.0 ** -24 * F.conv2d(x.abs(), sd[p + ".weight"].abs(), sd[p + ".bias"].abs(), padding=1)
        return units[i]
    n, worst, n_tiny = 0, 0.0, 0
    for i, ((_, u), msk) in enumerate(zip(convs, masks)):
        bad = msk != (u > 0)
        if not keys[i][2]:
            tiny = bad & ~msk & (u > 0) & (u <= 2.0 ** -25)
            n_tiny += int(tiny.sum())
            bad = bad & ~tiny
        if bool(bad.any()):
            n += int(bad.sum())
            worst = max(worst, float((u.abs() / unit(i))[bad].max()))
    n_pick, worst_pick = 0, 0.0
    last_of = [i for i, (_, _, last) in enumerate(keys) if last]
    for k, (x, pk) in enumerate(zip(pools, picks)):
        win = lpips_ref.pool_windows(x)
        top, p64 = win.max(-1)
        bad = (p64 != pk) & (top > 0)
        if bool(bad.any()):
            n_pick += int(bad.sum())
            gap = top - win.gather(-1, pk.unsqueeze(-1)).squeeze(-1)
            uw = lpips_ref.pool_windows(unit(last_of[k])).amax(-1)
            worst_pick = max(worst_pick, float((gap / uw)[bad].max()))
    return n, worst, n_tiny, n_pick, worst_pick


LPIPS_CASES = {
    "2x64x32 fp32": (2, 64, 32, "fp32"),
    "3x256x128 fp32": (3, 256, 128, "fp32"),
    "1x48x80 fp32": (1, 48, 80, "fp32"),         # hw not a power of two; slice 5 is 3 x 5 = 15 pixels
    "2x64x32 fp16": (2, 64, 32, "fp16"),
}


@pytest.mark.parametrize("case", list(LPIPS_CASES))
def test_lpips_stages_and_conditioned(cuda, monkeypatch, case):
    B, H, W, mode = LPIPS_CASES[case]
    ops = _ops(mode)
    try:
        m = LR.mirror(cuda)
        in0, in1 = R.image(500 + H, B, 3, H, W).to(cuda), R.image(501 + H, B, 3, H, W).to(cuda)
        m._pack()
        rec = Recorder(monkeypatch)
        g = torch.zeros((B, 3, H, W), dtype=torch.float32, device=cuda)
        acc = m.run(in0, in1, g=g, alpha=1.0)
        torch.cuda.synchronize()
    finally:
        ops.set_precision("fp32")
    assert [len(rec.of(n)) for n in ("forward", "dgrad", "lpips_head", "relu_bwd", "f32_to_planes",
                                     "maxpool2_bcast_bwd", "lpips_scale_fwd", "lpips_scale_bwd")] == \
        [13, 13, 5, 8, 4, 4, 1, 1]
    sd = {k: v.double().to(cuda) for k, v in LR.state_dict().items()}
    st = stage_checks(rec, sd, B, mode)
    name, worst = max(((k, v) for k, v in st.items() if "rel" not in k), key=lambda kv: kv[1])
    hv = max(v for k, v in st.items() if "value rel" in k)
    hp = max(v for k, v in st.items() if "planes rel" in k)
    # end to end, conditioned on the native masks and picks
    masks, picks = native_choices(rec, B)
    x1 = in1.double().requires_grad_(True)
    trace = []
    v = lpips_ref.lpips_conditioned(sd, in0.double(), x1, masks, picks, trace)
    v.sum().backward()
    verr = float(((acc - v.detach().reshape(-1)).abs() / v.detach().abs().reshape(-1)).max())
    wg = x1.grad
    gnorm = float((g.double() - wg).norm() / wg.norm())
    gmax = float((g.double() - wg).abs().max() / wg.abs().max())
    n, fu, n_tiny, n_pick, pu = flips(trace, masks, picks, sd)
    top = sorted(((k, round(v, 1)) for k, v in st.items() if "rel" not in k), key=lambda kv: -kv[1])[:4]
    print(f"[lpips {case}] stages: worst {st[name]:.1f} units ({top}; bound {STAGE_UNITS[mode]}), head value rel "
          f"{hv:.2e}, head planes rel {hp:.2e}; conditioned end to end: value rel {verr:.2e}, grad norm rel "
          f"{gnorm:.2e}, worst element / largest {gmax:.2e} (bounds {E2E[mode]}); mask flips {n} within {fu:.1f} "
          f"units, pick flips {n_pick} within {pu:.1f} units (bound {FLIP_UNITS[mode]}); {n_tiny} elements with "
          f"0 < u <= 2^-25 dropped by design")
    assert st[name] <= STAGE_UNITS[mode], sorted(st.items(), key=lambda kv: -kv[1])[:5]
    if mode == "fp32":
        assert hv <= HEAD_VALUE_REL and hp <= HEAD_PLANE_REL, (hv, hp)
    b = E2E[mode]
    assert verr <= b["value"] and gnorm <= b["gnorm"] and gmax <= b["gmax"], (verr, gnorm, gmax)
    assert fu <= FLIP_UNITS[mode] and pu <= FLIP_UNITS[mode], (n, fu, n_pick, pu)


@pytest.mark.parametrize("s", [1e-2, 1e-4, 1e-7])
def test_lpips_small_f1_gradient_stays_finite(cuda, monkeypatch, s):
    """The whole native call with one xrec pixel of relu1_2 (the fp32 output of conv1_2, which both the head and the
    max-pool read) replaced by a nonnegative vector of norm s.  The head's gradient there ~ 64 * 2 w |u - v| / s
    passes fp16's range somewhere between s = 1e-4 and 1e-7 and is saturated: the image gradient and the value stay finite (unsaturated,
    the split's hi + lo is NaN and so is every gradient the trunk's backward derives from it).  At s = 1e-2 nothing
    saturates; test_head_small_f1_stays_finite checks the head's values themselves against fp64."""
    from text2human_b200 import conv_grad
    from text2human_b200 import lpips as L
    ops = _ops()
    m = LR.mirror(cuda)
    m._pack()
    B, H, W = 2, 64, 32
    calls, heads = [], []

    def forward(*args, **kw):
        y = conv_grad.forward(*args, **kw)
        calls.append(1)
        if len(calls) == 2:
            d = y[B + 1, 20, 10].clamp_min(0)
            y[B + 1, 20, 10] = s * d / d.norm()
        return y
    ns = types.SimpleNamespace(**{k: getattr(conv_grad, k) for k in dir(conv_grad) if not k.startswith("__")})
    ns.forward = forward
    monkeypatch.setattr(L, "G", ns)
    head = ops.lpips_head

    def lpips_head(*args, **kw):
        planes = head(*args, **kw)
        heads.append(planes.clone())
        return planes
    monkeypatch.setattr(ops, "lpips_head", lpips_head)
    in0, in1 = R.image(640, B, 3, H, W).to(cuda), R.image(641, B, 3, H, W).to(cuda)
    g = torch.zeros((B, 3, H, W), dtype=torch.float32, device=cuda)
    acc = m.run(in0, in1, g=g, alpha=1.0)
    torch.cuda.synchronize()
    p1 = heads[-1][:, 1, 20, 10]                       # slice 1's gradient planes at the pixel
    n_sat = int((p1[0].float().abs() == 65504).sum())
    print(f"[lpips small |f1| = {s:.0e}] image gradient finite {bool(torch.isfinite(g).all())}, value finite "
          f"{bool(torch.isfinite(acc).all())}, saturated head elements at the pixel {n_sat}, "
          f"largest |image gradient| {float(g.abs().max()):.3e}")
    assert torch.isfinite(g).all() and torch.isfinite(acc).all()
    assert torch.isfinite(p1.float()).all()
    if s >= 1e-2:
        assert n_sat == 0
    if s <= 1e-7:
        assert n_sat > 0
