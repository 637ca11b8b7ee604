"""Every path of the tap-GEMM (t2h_tapgemm) and the GroupNorm statistics kernel, element by element against fp64.

The case table below names the kernel, epilogue, column tile (BN) and spatial tile (TW x TH) each convolution is meant
to run on, through ``route``: a restatement of the selection rule in csrc/gemm_tc.cu (plan_tapgemm, tile shape to
epilogue mode).  It documents intent and does not verify the C code; a change to the routing updates ``route`` in
the same change, and ``test_case_table_covers_every_path`` then says which path or factor level lost its case.

Bounds, shared by every case:
  * the reference is fp64 torch over the values the operand planes hold (hi + lo, or hi alone with one plane);
    products of fp16 values are exact in fp32, so one and two planes have the same bound;
  * element by element, |got - ref| <= 1e-5 B + 1e-6 |ref|, where B is the same operation in fp64 on |x| and |w|
    plus |bias| and |residual| (times max |GELU'| ~ 1.13 behind a GELU): B bounds the magnitude accumulated at that
    element, so a wrong bias, edge pixel or small channel cannot hide under the tensor's largest value;
  * a single fp16 output plane also gets its 11-bit rounding, 2^-11 |ref|;
  * GroupNorm sums are compared per (image, group) through the mean and variance GroupNorm derives from them:
    |dmean| <= 1e-6 (|mean| + std), |dvar| <= 1e-5 var + 1e-6 mean^2.
"""
import collections

import pytest
import torch
import torch.nn.functional as F

from text2human_b200 import _lib

SENTINEL = -7777.0
ACTS = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "lrelu": _lib.ACT_LRELU, "gelu": _lib.ACT_GELU}
GELU_SLOPE = 1.13  # max |GELU'(x)| = 1.1289 at x = +-sqrt(2)


# ------------------------------------------------------------------ the routing rule, restated
def route(*, n_img, H, W, n_out, planes=0, d_plane=0, strides, d_al=True, res=False, res_al=True, bias=False,
          bias_al=True, bias_sn=0, act="none", gn_cpg=0):
    """Kernel, epilogue, BN and spatial tile t2h_tapgemm picks for a spatial conv launch (H > 1, no row tiles, no
    batched or broadcast operands).  planes: output planes (d_terms) or 0 for fp32; strides: (sn, sh, sw, sc) in
    elements; *_al: the pointer is 16-byte aligned."""
    sn, sh, sw, sc = strides
    TW = 16
    while TW > W and TW > 1:
        TW >>= 1
    TH = 128 // TW
    pow2 = gn_cpg >= 1 and gn_cpg & (gn_cpg - 1) == 0
    swap = (n_out % 128 == 0 and not planes and sc == 1 and sw % 4 == 0 and sh % 4 == 0 and sh > 0
            and (n_img == 1 or (sn % 4 == 0 and sn > 0)) and d_al and (not res or res_al)
            and (not gn_cpg or (pow2 and n_out % gn_cpg == 0)))
    swap_direct = (not swap and n_out <= 128 and not planes and sc != 1 and not res and not gn_cpg and act == "none")
    if swap or swap_direct:
        return dict(kernel="swap", epi="direct" if swap_direct else "tma_f32", BN=128, TW=TW, TH=TH)
    BN = 16
    while BN < n_out and BN < 128:
        BN <<= 1
    align = 8 if planes else 4  # elements per 16 bytes
    tma_ok = (sc == 1 and n_out % align == 0 and sw % align == 0 and d_al and BN >= (64 if planes else 32)
              and sh % align == 0 and sh > 0 and (n_img == 1 or (sn % align == 0 and sn > 0)))
    if planes == 2:
        s = sn if n_img > 1 else d_plane
        tma_ok = tma_ok and s > 0 and d_plane % s == 0 and d_plane % align == 0
    if res:
        tma_ok = tma_ok and res_al
    if bias:
        tma_ok = tma_ok and bias_al and bias_sn % 4 == 0
    epi = "direct" if not tma_ok else ("tma_planes" if planes else "tma_f32")
    if epi == "tma_f32" and BN >= 64 and not res and not gn_cpg and act == "none":
        epi = "plain_f32"  # two epilogue warpgroups, alpha and column bias only
    return dict(kernel="generic", epi=epi, BN=BN, TW=TW, TH=TH)


# ------------------------------------------------------------------ the case table
Case = collections.namedtuple("Case", "N H W kind cin cout terms bias alpha act res gn out")
# kind: k3 / k1 (stride 1), down (pad (0,1,0,1) + 3x3 stride 2 on space-to-depth phases), k4s2 / k4s1 (4x4, 16 taps
# in several tap groups), up (nearest x2 + 3x3 folded into four parity launches with a strided destination), dgrad
# (stride-1 data gradient: negated taps on transposed weights).  H, W: the input extents.
# out: nhwc / nchw fp32, or planes1 / planes2 (fp16 output planes).  gn: GroupNorm channels per group (0: none).
CASES = [
    # swapped-operand kernel, TMA epilogue
    Case(2, 21, 40, "k3", 64, 128, 2, "shared", 1.0, "none", True, 4, "nhwc"),
    Case(2, 21, 40, "k3", 64, 256, 1, "image", 0.375, "relu", False, 1, "nhwc"),
    Case(1, 13, 8, "k3", 96, 384, 2, "shared", 1.0, "lrelu", True, 2, "nhwc"),
    Case(3, 9, 5, "k3", 40, 128, 2, "none", 1.0, "gelu", True, 32, "nhwc"),
    Case(1, 17, 3, "k3", 128, 256, 2, "shared", 0.375, "none", False, 64, "nhwc"),
    Case(2, 37, 1, "k3", 64, 128, 2, "shared", 1.0, "none", True, 8, "nhwc"),
    Case(2, 21, 40, "k1", 200, 128, 2, "shared", 1.0, "relu", True, 16, "nhwc"),
    Case(2, 22, 40, "down", 64, 128, 2, "shared", 1.0, "none", True, 128, "nhwc"),
    Case(2, 18, 10, "k4s2", 64, 128, 1, "shared", 1.0, "lrelu", False, 4, "nhwc"),
    Case(2, 7, 6, "up", 128, 128, 2, "shared", 1.0, "none", False, 4, "nhwc"),
    Case(1, 12, 11, "k4s1", 64, 256, 2, "image", 0.375, "relu", False, 0, "nhwc"),
    Case(2, 10, 12, "dgrad", 256, 128, 2, "none", 1.0, "none", False, 0, "nhwc"),
    # swapped-operand kernel, direct (strided NCHW) epilogue
    Case(2, 21, 40, "k3", 64, 3, 2, "shared", 0.375, "none", False, 0, "nchw"),
    Case(1, 13, 8, "k3", 96, 24, 1, "image", 1.0, "none", False, 0, "nchw"),
    Case(3, 9, 5, "k3", 40, 100, 2, "shared", 0.375, "none", False, 0, "nchw"),
    Case(1, 17, 3, "k3", 128, 128, 2, "image", 0.375, "none", False, 0, "nchw"),
    # generic kernel
    Case(2, 21, 40, "k3", 64, 16, 2, "shared", 0.375, "none", False, 0, "nhwc"),
    Case(1, 13, 8, "k3", 96, 64, 2, "shared", 1.0, "none", True, 2, "nhwc"),
    Case(1, 13, 8, "k3", 96, 24, 2, "shared", 1.0, "none", False, 0, "nhwc"),
    Case(3, 9, 5, "k3", 40, 96, 1, "shared", 1.0, "gelu", False, 0, "planes1"),
    Case(1, 17, 3, "k3", 128, 200, 2, "image", 1.0, "lrelu", False, 0, "planes2"),
    Case(2, 37, 1, "k3", 64, 64, 2, "none", 1.0, "none", False, 0, "nhwc"),
    Case(2, 21, 40, "k3", 64, 256, 1, "shared", 1.0, "relu", False, 0, "planes2"),
    Case(2, 18, 10, "k4s2", 64, 64, 1, "shared", 1.0, "lrelu", False, 0, "nhwc"),
    Case(2, 21, 40, "k3", 64, 96, 2, "shared", 0.375, "none", True, 0, "nhwc"),
]


def _case_id(c):
    return (f"{c.kind}-n{c.N}x{c.H}x{c.W}-{c.cin}to{c.cout}-t{c.terms}-b{c.bias}-a{c.alpha:g}-{c.act}"
            f"{'-res' if c.res else ''}{f'-gn{c.gn}' if c.gn else ''}-{c.out}")


def _out_hw(c):
    if c.kind in ("k3", "k1", "dgrad"):
        return c.H, c.W
    if c.kind in ("down", "k4s2"):
        return c.H // 2, c.W // 2
    if c.kind == "k4s1":
        return c.H - 1, c.W - 1
    return 2 * c.H, 2 * c.W  # up


def _layouts(c):
    """route() arguments of each launch of a case, for destinations allocated fresh (16-byte aligned)"""
    Ho, Wo = _out_hw(c)
    Co = c.cout
    planes = int(c.out[-1]) if c.out.startswith("planes") else 0
    common = dict(n_out=Co, planes=planes, res=c.res, bias=c.bias != "none", bias_sn=Co if c.bias == "image" else 0,
                  act=c.act, gn_cpg=c.gn)
    if c.kind == "up":  # four parity launches over the low-resolution grid, each writing every other pixel
        return [dict(common, n_img=c.N, H=c.H, W=c.W, strides=(Ho * Wo * Co, 2 * Wo * Co, 2 * Co, 1),
                     d_al=((pa * Wo + pb) * Co) % 4 == 0) for pa in (0, 1) for pb in (0, 1)]
    if c.out == "nchw":
        strides = (Co * Ho * Wo, Wo, 1, Ho * Wo)
    else:
        strides = (Ho * Wo * Co, Wo * Co, Co, 1)
    return [dict(common, n_img=c.N, H=Ho, W=Wo, strides=strides, d_plane=c.N * Ho * Wo * Co)]


def _label(c):
    r = route(**_layouts(c)[0])
    Ho, Wo = (c.H, c.W) if c.kind == "up" else _out_hw(c)
    r["ragged"] = Ho % r["TH"] != 0 or Wo % r["TW"] != 0
    return r


def test_case_table_covers_every_path():
    """every kernel path, epilogue, tile size and epilogue feature the case table is meant to reach has a case; the
    swapped kernel's features each run once on a ragged tile and once at TW < 16"""
    labels = [(c, _label(c)) for c in CASES]
    for c, r in labels:  # the launches of one case share a path
        assert all(route(**lay) == {k: v for k, v in r.items() if k != "ragged"} for lay in _layouts(c)), c
    swap = [(c, r) for c, r in labels if r["kernel"] == "swap" and r["epi"] == "tma_f32"]
    sdir = [(c, r) for c, r in labels if r["kernel"] == "swap" and r["epi"] == "direct"]
    gen = [(c, r) for c, r in labels if r["kernel"] == "generic"]

    def levels(rows, f):
        return {f(c, r) for c, r in rows}

    assert levels(swap, lambda c, r: r["TW"]) >= {16, 8, 4, 2, 1}
    assert all(any(r["ragged"] and r["TW"] == tw for c, r in swap) for tw in (16, 8, 4, 2, 1))
    assert levels(swap, lambda c, r: c.N) >= {1, 3}
    assert levels(swap, lambda c, r: c.cout) >= {128, 256, 384}
    assert levels(swap, lambda c, r: c.kind) >= {"k3", "k1", "down", "k4s2", "k4s1", "up", "dgrad"}
    assert levels(swap, lambda c, r: c.bias) >= {"none", "shared", "image"}
    assert levels(swap, lambda c, r: c.alpha) >= {1.0, 0.375}
    assert levels(swap, lambda c, r: c.act) >= set(ACTS)
    assert levels(swap, lambda c, r: c.gn) >= {1, 2, 4, 8, 16, 32, 64, 128}
    assert any(c.kind in ("down", "k4s2", "k4s1") and (c.res or c.gn) for c, r in swap)
    features = {"shared bias": lambda c: c.bias == "shared", "per-image bias": lambda c: c.bias == "image",
                "alpha": lambda c: c.alpha != 1.0, "relu": lambda c: c.act == "relu",
                "lrelu": lambda c: c.act == "lrelu", "gelu": lambda c: c.act == "gelu",
                "residual": lambda c: c.res, "gn sums": lambda c: c.gn > 0}
    for name, f in features.items():
        assert any(f(c) and r["ragged"] for c, r in swap), f"no ragged swapped-kernel case with {name}"
        assert any(f(c) and r["TW"] < 16 for c, r in swap), f"no swapped-kernel case with {name} at TW < 16"
    assert levels(sdir, lambda c, r: c.cout) >= {3, 24, 100, 128}
    assert all(c.bias != "none" for c, r in sdir) and any(c.alpha != 1.0 for c, r in sdir)
    assert levels(gen, lambda c, r: c.cout) >= {16, 64, 96, 200}
    assert levels(gen, lambda c, r: r["BN"]) >= {16, 32, 64, 128}
    assert levels(gen, lambda c, r: r["epi"]) >= {"direct", "tma_f32", "plain_f32", "tma_planes"}
    assert levels(gen, lambda c, r: r["TW"]) >= {16, 8, 4, 2, 1}
    assert levels(gen, lambda c, r: c.out) >= {"nhwc", "planes1", "planes2"}
    assert any(c.res for c, r in gen) and any(c.gn == 2 for c, r in gen)
    assert any(r["epi"] == "direct" and c.alpha != 1.0 and c.bias != "none" for c, r in gen)
    # one conv runs on both kernels with the same operands: the generic one because its output is planes
    operands = lambda c: (c.N, c.H, c.W, c.kind, c.cin, c.cout, c.terms)  # noqa: E731
    assert any(c.cout == 256 and c.out.startswith("planes") and operands(c) in levels(swap, lambda s, r: operands(s))
               for c, r in gen)


# ------------------------------------------------------------------ fp64 references
def _pv(p):
    """values the planes hold, fp64"""
    return p.double().sum(0)


def _uns2d(v):
    """space-to-depth values [4, N, h, w, C] -> [N, C, 2h, 2w]"""
    _, N, h, w, C = v.shape
    return v.view(2, 2, N, h, w, C).permute(2, 5, 3, 0, 4, 1).reshape(N, C, 2 * h, 2 * w)


def _upsample_fold_ref(x, w16):
    """out[2i+a, 2j+b] = sum_{r,s} W_ab[r, s] . x[i + a + r - 1, j + b + s - 1] (pack_upsample_conv_weight);
    x [N, C, H, W], w16 [16, Cout, C] -> [N, Cout, 2H, 2W]"""
    N, C, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros((N, w16.shape[1], 2 * H, 2 * W))
    for a in (0, 1):
        for b in (0, 1):
            for r in (0, 1):
                for s in (0, 1):
                    wt = w16[((a * 2 + b) * 2 + r) * 2 + s]
                    win = xp[:, :, a + r:a + r + H, b + s:b + s + W]
                    out[:, :, a::2, b::2] += torch.einsum("oc,nchw->nohw", wt, win)
    return out


def _conv_ref(c, xv, wv):
    """the case's convolution on fp64 operand values -> NCHW.  xv: NCHW input (full resolution for the stride-2
    kinds); wv: [taps, Cout, Cin] weight values (dgrad: [9, Cx, Cy] transposed planes)"""
    if c.kind == "up":
        return _upsample_fold_ref(xv, wv)
    if c.kind == "dgrad":
        wf = wv.reshape(3, 3, wv.shape[1], wv.shape[2]).permute(3, 2, 0, 1)  # forward weight [Cy, Cx, 3, 3]
        return F.conv_transpose2d(xv, wf, padding=1)
    k = {"k3": 3, "k1": 1, "down": 3, "k4s2": 4, "k4s1": 4}[c.kind]
    w = wv.reshape(k, k, wv.shape[1], wv.shape[2]).permute(2, 3, 0, 1)
    if c.kind == "down":
        return F.conv2d(F.pad(xv, (0, 1, 0, 1)), w, stride=2)
    return F.conv2d(xv, w, stride=2 if c.kind == "k4s2" else 1, padding=0 if c.kind == "k1" else 1)


def _act_ref(y, act):
    if act == "relu":
        return y.clamp_min(0)
    if act == "lrelu":
        return torch.where(y > 0, y, 0.2 * y)
    if act == "gelu":
        return F.gelu(y)
    return y


def _check(got, ref, B, what, rel=1e-6, tol=1e-5):
    """|got - ref| <= tol B + rel |ref| element by element; prints the worst err / B"""
    err = (got.double() - ref).abs()
    worst = (err / B.clamp_min(1e-30)).max().item()
    print(f"{what}: worst err/B = {worst:.3g}")
    bad = err > tol * B + rel * ref.abs()
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound, first at "
                           f"{tuple(bad.nonzero()[0].tolist())}, worst err/B {worst:.3g}")
    return worst


def _check_gn(stats, out_nhwc, cpg, what):
    """stats [N, G, 2] (sum, sumsq) against fp64 sums of out [N, H, W, C], per (image, group)"""
    N, H, W, C = out_nhwc.shape
    o = out_nhwc.double().reshape(N, H * W, C // cpg, cpg)
    _check_moments(stats, o.sum((1, 3)), (o * o).sum((1, 3)), H * W * cpg, what)


def _check_moments(stats, s_ref, q_ref, cnt, what):
    mean, var = stats[..., 0] / cnt, stats[..., 1] / cnt - (stats[..., 0] / cnt) ** 2
    mref = s_ref / cnt
    vref = (q_ref / cnt - mref ** 2).clamp_min(0)
    dm, dv = (mean - mref).abs(), (var - vref).abs()
    bm, bv = 1e-6 * (mref.abs() + vref.sqrt()), 1e-5 * vref + 1e-6 * mref ** 2
    print(f"{what}: worst |dmean|/bound = {(dm / bm.clamp_min(1e-300)).max().item():.3g}, "
          f"|dvar|/bound = {(dv / bv.clamp_min(1e-300)).max().item():.3g}")
    assert (dm <= bm).all(), f"{what}: group mean off in {int((dm > bm).sum())} (image, group) slots"
    assert (dv <= bv).all(), f"{what}: group variance off in {int((dv > bv).sum())} (image, group) slots"


# ------------------------------------------------------------------ launching
def _launch(a, w, taps, *, n, out_hw, d, d_strides, planes=0, d_plane=0, bias=None, bias_sn=0, alpha=1.0,
            act="none", residual=None, stats=None, cpg=0, tap_w=None):
    """one t2h_tapgemm launch as ops.tap_conv makes it, with every epilogue option open; returns route()'s view of it
    from the real pointers"""
    from text2human_b200 import ops
    T = a.shape[0]
    aH, aW, Cc = a.shape[-3:]
    a_imgs = a.numel() // (aH * aW * Cc)
    H, W = out_hw
    slots = w.shape[1] if tap_w is None else max(tap_w) + 1
    b_term_g = w.stride(0) // w.stride(1) if w.shape[0] > 1 else slots
    ops._tapgemm(a=a, a_term_imgs=a_imgs // T, a_imgs=a_imgs, a_bcast=0, n_img=n, H=H, W=W, a_H=aH, a_W=aW, Cc=Cc,
                 a_sw=Cc, a_sh=aW * Cc, a_sn=aH * aW * Cc,
                 b=w, b_term_g=b_term_g, b_groups=(w.shape[0] - 1) * b_term_g + slots, b_batched=0, n_out=w.shape[2],
                 b_sn=Cc, b_sg=w.stride(1), taps=taps, d=d, d_mode=_lib.OUT_PLANES if planes else _lib.OUT_F32,
                 d_strides=d_strides, d_plane=d_plane, bias=bias, bias_mode=_lib.BIAS_COL, bias_sn=bias_sn,
                 act=ACTS[act], alpha=alpha, residual=residual, gn_stats=stats, gn_cpg=cpg, tap_w=tap_w)
    al = lambda t: t is None or t.data_ptr() % 16 == 0  # noqa: E731
    return route(n_img=n, H=H, W=W, n_out=w.shape[2], planes=planes, d_plane=d_plane, strides=d_strides,
                 d_al=al(d), res=residual is not None, res_al=al(residual), bias=bias is not None, bias_al=al(bias),
                 bias_sn=bias_sn, act=act, gn_cpg=cpg if stats is not None else 0)


def _operands(c, dev):
    """(planes a, weight planes w, input values NCHW fp64, weight values [taps, Cout, Cin] fp64, taps)"""
    from text2human_b200 import conv_grad, ops
    g = torch.Generator().manual_seed(c.N * 1000 + c.H * 100 + c.W + c.cin * 7 + c.cout * 13 + c.terms)
    x = torch.randn(c.N, c.H, c.W, c.cin, generator=g).to(dev)
    if c.kind == "up":
        w = torch.randn(c.cout, c.cin, 3, 3, generator=g).to(dev) / (9 * c.cin) ** 0.5
        wp = ops.pack_upsample_conv_weight(w, c.terms)
        a = ops.f32_to_planes(x, ops.CVT_PLAIN, c.terms)
        return a, wp, _pv(a).permute(0, 3, 1, 2), _pv(wp), None
    k = {"k3": 3, "k1": 1, "down": 3, "k4s2": 4, "k4s1": 4, "dgrad": 3}[c.kind]
    w = torch.randn(k * k, c.cout, c.cin, generator=g).to(dev) / (k * k * c.cin) ** 0.5
    wp = ops.split_planes(w, c.terms)
    if c.kind in ("down", "k4s2"):
        a = ops.f32_to_planes(x, ops.CVT_S2D, c.terms)
        xv = _uns2d(_pv(a))
    else:
        a = ops.f32_to_planes(x, ops.CVT_PLAIN, c.terms)
        xv = _pv(a).permute(0, 3, 1, 2)
    if c.kind == "dgrad":
        taps = tuple((-ty, -tx, 0) for ty, tx, _ in conv_grad.fwd_taps("k3", c.N))
    elif c.kind == "k1":
        taps = ((0, 0, 0),)
    else:
        taps = conv_grad.fwd_taps(c.kind, c.N)
    return a, wp, xv, _pv(wp), taps


def _run_case(c, a, wp, taps, bias, res, dev):
    Ho, Wo = _out_hw(c)
    N, Co = c.N, c.cout
    planes = int(c.out[-1]) if c.out.startswith("planes") else 0
    if planes:
        d = torch.full((planes, N, Ho, Wo, Co), SENTINEL, dtype=torch.float16, device=dev)
    elif c.out == "nchw":
        d = torch.full((N, Co, Ho, Wo), SENTINEL, device=dev)
    else:
        d = torch.full((N, Ho, Wo, Co), SENTINEL, device=dev)
    stats = None
    if c.gn:  # guard slots after the n_img x groups x 2 sums
        stats_buf = torch.zeros(N * (Co // c.gn) * 2 + 64, dtype=torch.float64, device=dev)
        stats_buf[-64:] = SENTINEL
        stats = stats_buf[:-64]
    kw = dict(n=N, bias=bias, bias_sn=Co if c.bias == "image" else 0, alpha=c.alpha, act=c.act, residual=res,
              stats=stats, cpg=c.gn)
    routes = []
    if c.kind == "up":
        for pa in (0, 1):
            for pb in (0, 1):
                par = pa * 2 + pb
                ptaps = tuple((pa + r - 1, pb + s - 1, 0) for r in (0, 1) for s in (0, 1))
                routes.append(_launch(a, wp[:, par * 4:(par + 1) * 4], ptaps, out_hw=(c.H, c.W),
                                      d=d[:, pa::2, pb::2, :], d_strides=(Ho * Wo * Co, 2 * Wo * Co, 2 * Co, 1), **kw))
    else:
        strides = (Co * Ho * Wo, Wo, 1, Ho * Wo) if c.out == "nchw" else (Ho * Wo * Co, Wo * Co, Co, 1)
        routes.append(_launch(a, wp, taps, out_hw=(Ho, Wo), d=d, d_strides=strides, planes=planes,
                              d_plane=N * Ho * Wo * Co, **kw))
    if stats is not None:
        assert (stats_buf[-64:] == SENTINEL).all(), "GroupNorm sums written past n_img x groups x 2"
    return d, stats, routes


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=_case_id)
def test_tapgemm_path_matches_fp64(cuda, c):
    """one conv of the case table against fp64 torch on the planes' values, element by element"""
    dev = cuda
    g = torch.Generator().manual_seed(c.cout * 31 + c.N)
    a, wp, xv, wv, taps = _operands(c, dev)
    Ho, Wo = _out_hw(c)
    N, Co = c.N, c.cout
    bias = None
    if c.bias == "shared":
        bias = torch.randn(Co, generator=g).to(dev)
    elif c.bias == "image":
        bias = torch.randn(N, Co, generator=g).to(dev)
    res = torch.randn(N, Ho, Wo, Co, generator=g).to(dev) if c.res else None
    d, stats, routes = _run_case(c, a, wp, taps, bias, res, dev)
    label = _label(c)
    assert all(r == {k: v for k, v in label.items() if k != "ragged"} for r in routes), (routes, label)

    conv = _conv_ref(c, xv, wv)
    cabs = _conv_ref(c, xv.abs(), wv.abs())
    pre, pre_b = c.alpha * conv, abs(c.alpha) * cabs
    if bias is not None:  # shared [Co] or per image [N, Co]
        bv = bias.double().view(-1, Co, 1, 1)
        pre, pre_b = pre + bv, pre_b + bv.abs()
    ref = _act_ref(pre, c.act)
    B = pre_b * (GELU_SLOPE if c.act == "gelu" else 1.0)
    if res is not None:
        rv = res.double().permute(0, 3, 1, 2)
        ref, B = ref + rv, B + rv.abs()
    if c.out == "nchw":
        got = d
    elif c.out.startswith("planes"):
        got = _pv(d).permute(0, 3, 1, 2)
    else:
        got = d.permute(0, 3, 1, 2)
    rel = 1e-6
    if c.out == "planes1":  # one fp16 plane: 11-bit rounding (and fp16 subnormal spacing near zero)
        rel, B = 2.0 ** -11, B + 2.0 ** -24 / 1e-5
    label_s = f"{label['kernel']}/{label['epi']} BN{label['BN']} TW{label['TW']} {_case_id(c)}"
    _check(got, ref, B, label_s, rel)
    if stats is not None:
        _check_gn(stats.view(N, Co // c.gn, 2), d, c.gn, label_s + " gn sums")
    if label["kernel"] == "swap":  # same launch again: bit-identical output (the sums' fp64 atomic order may vary)
        d2, _, _ = _run_case(c, a, wp, taps, bias, res, dev)
        assert torch.equal(d, d2), "swapped kernel is not run-to-run reproducible"


# ------------------------------------------------------------------ which elements a launch writes
@pytest.mark.gpu
@pytest.mark.parametrize("c0", [32, 1], ids=["aligned-swap", "unaligned-generic-direct"])
def test_channel_slice_launch_writes_only_its_slice(cuda, c0):
    """a Cout = 128 conv into channels [c0, c0 + 128) of a 224-channel NHWC buffer with a guard image before and after
    and a guard tile of rows and columns: everything outside the slice keeps the sentinel bit for bit"""
    from text2human_b200 import ops
    dev = cuda
    N, H, W, Ci, Co, Ct = 2, 21, 40, 64, 128, 224
    g = torch.Generator().manual_seed(c0)
    x = torch.randn(N, H, W, Ci, generator=g).to(dev)
    w = (torch.randn(9, Co, Ci, generator=g) / (9 * Ci) ** 0.5).to(dev)
    bias = torch.randn(Co, generator=g).to(dev)
    a, wp = ops.f32_to_planes(x, ops.CVT_PLAIN, 2), ops.split_planes(w, 2)
    TH, TW = 8, 16
    buf = torch.full((N + 2, H + TH, W + TW, Ct), SENTINEL, device=dev)
    rbuf = torch.randn(buf.shape, generator=g).to(dev)  # the residual has the destination's layout
    view = buf[1:N + 1, :H, :W, c0:c0 + Co]
    rview = rbuf[1:N + 1, :H, :W, c0:c0 + Co]
    s = buf.stride()
    r = _launch(a, wp, ops._TAPS_3x3, n=N, out_hw=(H, W), d=view, d_strides=s, bias=bias, alpha=0.375,
                residual=rview)
    assert (r["kernel"], r["epi"]) == (("swap", "tma_f32") if c0 % 4 == 0 else ("generic", "direct")), r
    c = Case(N, H, W, "k3", Ci, Co, 2, "shared", 0.375, "none", True, 0, "nhwc")
    xv, wv = _pv(a).permute(0, 3, 1, 2), _pv(wp)
    rv = rview.double().permute(0, 3, 1, 2)
    ref = 0.375 * _conv_ref(c, xv, wv) + bias.double().view(1, Co, 1, 1) + rv
    B = 0.375 * _conv_ref(c, xv.abs(), wv.abs()) + bias.double().abs().view(1, Co, 1, 1) + rv.abs()
    _check(view.permute(0, 3, 1, 2), ref, B, f"channel slice at {c0} ({r['kernel']}/{r['epi']})")
    outside = torch.ones(buf.shape, dtype=torch.bool, device=dev)
    outside[1:N + 1, :H, :W, c0:c0 + Co] = False
    assert (buf[outside] == SENTINEL).all(), f"{int((buf[outside] != SENTINEL).sum())} stray writes"


@pytest.mark.gpu
@pytest.mark.parametrize("Co", [128, 64], ids=["swap", "generic"])
@pytest.mark.parametrize("kind", ["upsample-fold", "dgrad-s2"])
def test_single_parity_launch_writes_only_its_parity(cuda, kind, Co):
    """one of the four parity launches of the upsample fold / the stride-2 data gradient, alone in a sentinel buffer
    with a guard image before and after: only its parity's elements change, and they match fp64"""
    from text2human_b200 import conv_grad, ops
    dev = cuda
    N, h, w, Ci = 2, 7, 6, 128
    H, W = 2 * h, 2 * w
    pa, pb = 1, 0
    g = torch.Generator().manual_seed(Co + len(kind))
    buf = torch.full((N + 2, H, W, Co), SENTINEL, device=dev)
    sn, sh, sw, sc = buf.stride()
    x = torch.randn(N, h, w, Ci, generator=g).to(dev)
    a = ops.f32_to_planes(x, ops.CVT_PLAIN, 2)
    xv = _pv(a).permute(0, 3, 1, 2)
    bias = torch.randn(Co, generator=g).to(dev)
    start = buf[1:N + 1].storage_offset() + pa * sh + pb * sw
    dview = buf.view(-1)[start:]
    if kind == "upsample-fold":
        w3 = torch.randn(Co, Ci, 3, 3, generator=g).to(dev) / (9 * Ci) ** 0.5
        wp = ops.pack_upsample_conv_weight(w3, 2)
        par = pa * 2 + pb
        taps = tuple((pa + r - 1, pb + s - 1, 0) for r in (0, 1) for s in (0, 1))
        rt = _launch(a, wp[:, par * 4:(par + 1) * 4], taps, n=N, out_hw=(h, w), d=dview,
                     d_strides=(sn, 2 * sh, 2 * sw, sc), bias=bias)
        full = _upsample_fold_ref(xv, _pv(wp))
        babs = _upsample_fold_ref(xv.abs(), _pv(wp).abs())
    else:  # the 4x4 stride-2 conv's data gradient: taps that reach input parity (pa, pb), weight slots via tap_w
        wt = ops.split_planes(torch.randn(16, Co, Ci, generator=g).to(dev) / (16 * Ci) ** 0.5, 2)  # [T,16,Cx,Cy]
        taps, slots = conv_grad.dgrad_parity_taps("k4s2", pa, pb)
        rt = _launch(a, wt, taps, n=N, out_hw=(h, w), d=dview, d_strides=(sn, 2 * sh, 2 * sw, sc), bias=bias,
                     tap_w=slots)
        wf = _pv(wt).reshape(4, 4, Co, Ci).permute(3, 2, 0, 1)  # forward weight [Cy, Cx, 4, 4]
        full = F.conv_transpose2d(xv, wf, stride=2, padding=1)
        babs = F.conv_transpose2d(xv.abs(), wf.abs(), stride=2, padding=1)
    assert rt["kernel"] == ("swap" if Co == 128 else "generic"), rt
    bv = bias.double().view(1, Co, 1, 1)
    got = buf[1:N + 1, pa::2, pb::2].permute(0, 3, 1, 2)
    _check(got, full[:, :, pa::2, pb::2] + bv, babs[:, :, pa::2, pb::2] + bv.abs(),
           f"{kind} parity ({pa},{pb}) {rt['kernel']}/{rt['epi']}")
    outside = torch.ones(buf.shape, dtype=torch.bool, device=dev)
    outside[1:N + 1, pa::2, pb::2] = False
    assert (buf[outside] == SENTINEL).all(), f"{int((buf[outside] != SENTINEL).sum())} stray writes"


# ------------------------------------------------------------------ GroupNorm statistics at every channels-per-group
GN_SHAPES = [(64, 64), (64, 32), (96, 32), (128, 32), (40, 8), (192, 32), (320, 32), (384, 32), (512, 32), (256, 8),
             (512, 1)]  # (C, groups): cpg 1 (BatchNorm mode), 2, 3, 4, 5, 6, 10, 12, 16, 32, 512
GN_CASES = [(C, G, n, hw) for C, G in GN_SHAPES for n in (1, 3) for hw in (1, 7, 2048)]
GN_CASES += [(40, 8, 1, 131072), (192, 32, 1, 131072), (512, 32, 1, 131072)]  # one 512 x 256 image


@pytest.mark.gpu
@pytest.mark.parametrize("C,groups,n,hw", GN_CASES, ids=lambda v: str(v))
def test_group_norm_statistics_per_group(cuda, C, groups, n, hw):
    """t2h_gn_stats per (image, group) against fp64, and norm_apply / group_norm against F.group_norm in fp64; every
    channel has its own offset, so a channel summed into the wrong group moves that group's mean"""
    from text2human_b200 import ops
    dev = cuda
    g = torch.Generator().manual_seed(C * 7 + groups + n * 3 + hw)
    offset = torch.rand(C, generator=g) * 20
    x = (torch.randn(n, hw, 1, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + offset).to(dev)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev)
    eps = 1e-6
    bn = groups == C  # BatchNorm mode: the whole batch is one normalisation domain
    nn_ = 1 if bn else n
    stats = ops.norm_stats(x, groups, n=1 if bn else None)
    xd = x.double().reshape(nn_, -1, groups, C // groups)
    cnt = xd.shape[1] * xd.shape[3]
    _check_moments(stats, xd.sum((1, 3)), (xd * xd).sum((1, 3)), cnt, f"gn_stats C={C} groups={groups}")

    if cnt > 1:
        xr = x.double().reshape(nn_, -1, C).permute(0, 2, 1).unsqueeze(-1)  # [n, C, pixels, 1]
        ref = F.group_norm(xr, groups, gamma.double(), beta.double(), eps=eps).squeeze(-1).permute(0, 2, 1)
        ref = ref.reshape(n, hw, 1, C)
    else:  # one value per group (F.group_norm refuses it): x - mean = 0
        ref = beta.double().view(1, 1, 1, C).expand(n, hw, 1, C)
    # what the statistics bounds above allow, carried through (x - mean) * rstd * gamma + beta, plus the fp32
    # scale / shift arithmetic at 1e-6 of its terms
    xs = xd.reshape(nn_, -1, C)
    mean = xd.mean((1, 3), keepdim=True).expand_as(xd).reshape(nn_, -1, C)
    var = xd.var((1, 3), unbiased=False, keepdim=True).expand_as(xd).reshape(nn_, -1, C)
    ga = gamma.double().abs() / (var + eps).sqrt()
    dmean, dvar = 1e-6 * (mean.abs() + var.sqrt()), 1e-5 * var + 1e-6 * mean ** 2
    bound = ga * (dmean + (xs - mean).abs() * dvar / (2 * (var + eps))) + 1e-6 * (ga * (xs.abs() + mean.abs()))
    bound = bound.reshape(n, hw, 1, C) + 1e-6 * beta.double().abs().view(1, 1, 1, C)
    out = ops.norm_apply(x, stats, gamma, beta, act=None, groups=groups, eps=eps, n=1 if bn else None, terms=2)
    _check(_pv(out), ref, bound, f"norm_apply C={C} groups={groups}", tol=1.0)
    if not bn:
        out = ops.group_norm(x, gamma, beta, swish=False, groups=groups, eps=eps, terms=2)
        _check(_pv(out), ref, bound, f"group_norm C={C} groups={groups}", tol=1.0)
