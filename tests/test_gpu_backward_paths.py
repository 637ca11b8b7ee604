"""The norm backward (t2h_norm_bwd), its pass 1 fused into the data-gradient conv (t2h_tapgemm_params.nb_sums) and
the conv weight gradient (t2h_conv_wgrad), path by path and element by element against fp64.

``norm_bwd_route`` and ``wgrad_route`` restate the launch choices of t2h_norm_bwd (csrc/gan.cu) and t2h_conv_wgrad
(csrc/gemm_tc.cu); a comment next to each rule points here.  They document intent and do not verify the C code: a
change to a rule updates its restatement in the same change, and the CPU coverage tests then say which level lost
its case.  Levels that depend on the SM count are labelled for the 132 SMs of an H100 SXM.

Bounds:
  * norm backward, reference in fp64 from the mean and variance derived from the same ``stats`` buffer the kernel
    reads (so the backward is isolated from the statistics kernel):
      dx = rstd (g - mean_g(g) - xhat mean_g(g xhat)) + add,  g = dy act'(u) gamma,  u = xhat gamma + beta;
    element by element |err| <= 1e-5 B + 1e-6 |ref| with B = rstd (|g| + mean_g|g| + |xhat| mean_g|g xhat|) + |add|.
    Pass 1's sums (sum du, sum du xhat per image and channel), dgamma, dbeta and the column sums of dx are checked
    per channel at 1e-5 of the sum of their terms' magnitudes (plus |start value|: they accumulate).  Swish: the
    kernels evaluate the sigmoid with a fast exp, whose absolute error on act' reaches ~1e-7 where act' ~ 0 (u near
    -1.28); every bound therefore takes |du| + 0.1 |dy| as the magnitude of du, 1e-6 |dy| at k = 1e-5.  LeakyReLU's
    branch is taken from the kernel's own fp32 pre-activation, fma((x - mean) rstd, gamma, beta) -- its sign is exact
    in fp64 -- so an element at u ~ 0 cannot take different sides in the kernel and the reference;
  * planes: hi == fp16(dx) and lo == fp16(dx - hi) bit for bit, and a planes-only launch on the same pass-1 sums
    writes the same planes bit for bit;
  * nb_sums: the same per-channel bound, 1e-5 of sum |du| (sum |du| (|xhat| + rstd |mean|) for the du xhat sums),
    with the same swish allowance; the epilogue's swish derivative also uses an approximate reciprocal (relative
    error ~1e-6), which the allowance covers;
  * weight gradient: dw = alpha sum dy shift_tap(x) in fp64 over the values the planes hold, |err| <= 1e-5 B +
    1e-6 |ref| with B = |alpha| sum |dy| |shift_tap(x)| + |dw0|.  Split-K reduce-adds in any order, so the bound is
    the only check.
"""
import collections

import pytest
import torch
import torch.nn.functional as F

from text2human_b200 import _lib

SENTINEL = -7777.0
EPS = 1e-6
K_TOL, K_REL = 1e-5, 1e-6
SWISH_ALLOW = 0.1  # swish: |du| + 0.1 |dy| in every magnitude, i.e. 1e-6 |dy| of absolute error on du at K_TOL
H100_SMS = 132


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------ the launch rules, restated
def norm_bwd_route(n, hw, c, sms=H100_SMS):
    """t2h_norm_bwd's launch shapes: reduce block, pixel lanes and pixels per block of pass 1, pixels per block and
    the column-sum branch of the apply pass"""
    c4 = c // 4
    block = 256
    if c4 > block:
        block = (c4 + 31) // 32 * 32
    block = block // c4 * c4
    lanes = block // c4
    bx = _cdiv(sms * 4, n)
    ppb = max(_cdiv(hw, bx), lanes * 8)
    bx2 = _cdiv(sms * 8, n)
    ppb2 = max(_cdiv(hw, bx2), 16)
    return dict(block=block, lanes=lanes, ppb=ppb, blocks=_cdiv(hw, ppb), short_last=hw % ppb != 0, ppb2=ppb2,
                blocks2=_cdiv(hw, ppb2), short_last2=hw % ppb2 != 0, fixed_cols=256 % c4 == 0)


def wgrad_route(H, W, n, cin, cout, ntaps, k_split, sms=H100_SMS):
    """t2h_conv_wgrad's launch shape: the 64-pixel patch (PW x PH), the cin tile BN, the output tiles and split-K"""
    PW = 16
    while PW > 1 and PW // 2 >= W:
        PW //= 2
    PH = 64 // PW
    chunks = n * _cdiv(W, PW) * _cdiv(H, PH)
    BN = 64 if cin <= 64 else 128
    tiles = ntaps * _cdiv(cout, 128) * _cdiv(cin, BN)
    ks = k_split if k_split > 0 else sms // tiles
    ks = min(max(ks, 1), chunks)
    kper = _cdiv(chunks, ks)
    return dict(PW=PW, PH=PH, chunks=chunks, BN=BN, col_tiles=_cdiv(cin, BN), row_tiles=_cdiv(cout, 128), ks=ks,
                kper=kper, ksplit=_cdiv(chunks, kper), ragged_h=H % PH != 0, ragged_w=W % PW != 0)


# ------------------------------------------------------------------ shared fp64 helpers
def _check(got, ref, B, what, tol=K_TOL, rel=K_REL):
    """|got - ref| <= tol B + rel |ref| element by element; returns the worst err / B"""
    err = (got.double() - ref).abs()
    worst = (err / B.clamp_min(1e-300)).max().item()
    print(f"{what}: worst err/B = {worst:.3g}")
    bad = err > tol * B + rel * ref.abs()
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound, first at "
                           f"{tuple(bad.nonzero()[0].tolist())}, worst err/B {worst:.3g}")
    return worst


def _f32(v):
    """an fp32 scalar as the kernel holds it, in fp64"""
    return float(torch.tensor(v, dtype=torch.float32).double())


def _moments(stats, cnt, eps):
    """mean, rstd per (image, group) in fp64 from a (sum, sumsq) buffer [n, groups, 2], as the kernels derive them;
    and the fp32-rounded pair the kernels compute with"""
    mean = stats[..., 0] / cnt
    var = (stats[..., 1] / cnt - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + _f32(eps))
    return mean, rstd, mean.float(), rstd.float()


def _act_grad(u, act, u_sign=None):
    """act'(u) in fp64; LeakyReLU's branch from ``u_sign`` (the kernel's fp32 pre-activation) when given"""
    if act == "swish":
        s = torch.sigmoid(u)
        return s * (1 + u * (1 - s))
    if act == "lrelu":
        return torch.where((u if u_sign is None else u_sign) > 0, 1.0, 0.2).double()
    return torch.ones_like(u)


def _norm_bwd_ref(x, stats, gamma, beta, dy, add, *, groups, act, eps):
    """fp64 backward of act(norm(x) gamma + beta).  x, dy, add: [n, hw, C]; stats [n, groups, 2].
    -> dict(dx, B, du, xh, rstd, mean per element)"""
    n, hw, Cc = x.shape
    cpg = Cc // groups
    mean, rstd, mean32, rstd32 = _moments(stats.double(), hw * cpg, eps)
    per_c = lambda t: t.repeat_interleave(cpg, dim=1).view(n, 1, Cc)  # noqa: E731  [n, groups] -> [n, 1, C]
    xd, ga, be = x.double(), gamma.double().view(1, 1, Cc), beta.double().view(1, 1, Cc)
    xh = (xd - per_c(mean)) * per_c(rstd)
    u = xh * ga + be
    xh32 = (x - per_c(mean32)) * per_c(rstd32)  # the kernel's fp32 xhat; fma(xh32, gamma, beta) has this sign
    du = dy.double() * _act_grad(u, act, xh32.double() * ga + be)
    dum = du.abs() + (SWISH_ALLOW * dy.double().abs() if act == "swish" else 0)  # the magnitude bounds use for du
    g = du * ga
    gm = dum * ga.abs()
    gsum = lambda t: t.view(n, hw, groups, cpg).sum((1, 3))  # noqa: E731
    cnt = hw * cpg
    m1, m2 = per_c(gsum(g) / cnt), per_c(gsum(g * xh) / cnt)
    a1, a2 = per_c(gsum(gm) / cnt), per_c(gsum(gm * xh.abs()) / cnt)
    r = per_c(rstd)
    dx = r * (g - m1 - xh * m2)
    B = r * (gm + a1 + xh.abs() * a2)
    if add is not None:
        dx, B = dx + add.double(), B + add.double().abs()
    return dict(dx=dx, B=B, du=du, dum=dum, xh=xh, mrstd=per_c(mean).abs() * r)


def _sums_check(sums, ref, what):
    """pass 1's (sum du, sum du xhat) [n, C, 2] against the fp64 reference's du and xhat"""
    du, dum, xh = ref["du"], ref["dum"], ref["xh"]
    w = []
    w.append(_check(sums[..., 0], du.sum(1), dum.sum(1), f"{what} sum du", rel=0))
    w.append(_check(sums[..., 1], (du * xh).sum(1), (dum * (xh.abs() + ref["mrstd"])).sum(1),
                    f"{what} sum du*xhat", rel=0))
    return max(w)


# ------------------------------------------------------------------ section 1: t2h_norm_bwd, case table
NB = collections.namedtuple("NB", "C groups n hw act add colsum params terms")
# n = 1 with groups = C is BatchNorm mode (the whole batch is one normalisation domain); params: which of dgamma /
# dbeta the first launch accumulates; terms: the planes of the dx-and-planes launch and the planes-only launch
NORM_CASES = [
    NB(64, 64, 1, 3 * 37 * 29, "lrelu", True, True, "both", 2),      # BatchNorm, cpg 1
    NB(96, 96, 1, 3 * 37 * 29, "swish", False, True, "gamma", 1),    # BatchNorm, atomic column sums
    NB(64, 32, 3, 1000, "swish", False, True, "both", 2),            # cpg 2
    NB(96, 32, 3, 7, "lrelu", True, True, "beta", 2),                # cpg 3
    NB(128, 32, 9, 1, "none", True, True, "both", 1),                # cpg 4, one pixel
    NB(40, 8, 3, 1000, "swish", True, True, "none", 2),              # cpg 5
    NB(192, 32, 1, 4096, "lrelu", False, True, "both", 2),           # cpg 6
    NB(192, 32, 9, 1, "swish", True, True, "gamma", 2),              # cpg 6, one pixel
    NB(640, 64, 3, 7, "swish", False, True, "beta", 1),              # cpg 10
    NB(24, 2, 9, 1000, "none", True, True, "both", 2),               # cpg 12
    NB(24, 24, 3, 7, "lrelu", False, False, "both", 2),              # cpg 1 per image
    NB(512, 16, 3, 1000, "lrelu", False, False, "both", 2),          # cpg 32
    NB(128, 32, 1, 16384, "swish", True, False, "gamma", 2),         # cpg 4, large
    NB(512, 1, 3, 1000, "lrelu", True, True, "both", 2),             # groups = 1
    NB(1024, 32, 1, 2048, "swish", False, True, "both", 2),          # cpg 32, reduce block = C/4
    NB(1032, 8, 3, 1000, "swish", True, True, "beta", 2),            # cpg 129, reduce block = C/4
    NB(1536, 32, 1, 1024, "lrelu", False, True, "both", 1),          # cpg 48
    NB(2048, 32, 3, 7, "none", True, True, "both", 2),               # cpg 64, largest C
    NB(2048, 2048, 1, 3 * 7 * 11, "swish", False, True, "gamma", 2),  # BatchNorm at the largest C
]


def _nb_id(c):
    return (f"C{c.C}-g{c.groups}-n{c.n}-hw{c.hw}-{c.act}{'-add' if c.add else ''}{'-colsum' if c.colsum else ''}"
            f"-{c.params}-t{c.terms}")


def test_norm_bwd_case_table_covers_every_path():
    """every channels-per-group, channel-count class, launch-shape level and output combination of t2h_norm_bwd that
    the case table is meant to reach has a case"""
    rows = [(c, norm_bwd_route(c.n, c.hw, c.C)) for c in NORM_CASES]
    levels = lambda f: {f(c, r) for c, r in rows}  # noqa: E731
    bn = lambda c: c.n == 1 and c.groups == c.C  # noqa: E731
    assert any(bn(c) and c.hw % 8 and c.hw > 1000 for c, r in rows), "no BatchNorm case at a non-round N*H*W"
    assert levels(lambda c, r: c.C // c.groups if not bn(c) else 0) >= {1, 2, 3, 4, 5, 6, 10, 12, 32}
    assert any(c.groups == 1 for c, r in rows)
    atomic = {c.C for c, r in rows if not r["fixed_cols"]}
    register = {c.C for c, r in rows if r["fixed_cols"]}
    assert atomic >= {24, 40, 96, 192, 640} and register >= {64, 128, 512, 1024}
    assert {c.C for c, r in rows if r["lanes"] == 1 and r["block"] == c.C // 4 and c.C > 1024} >= {1032, 1536, 2048}
    assert levels(lambda c, r: r["lanes"] > 1) == {True, False}
    assert any(r["short_last"] and r["blocks"] > 1 for c, r in rows), "no short last reduce block"
    assert any(r["short_last2"] and r["blocks2"] > 1 for c, r in rows), "no short last apply block"
    assert levels(lambda c, r: c.n) >= {1, 3, 9}
    assert {1, 7} <= levels(lambda c, r: c.hw) and max(c.hw for c in NORM_CASES) >= 16384
    assert levels(lambda c, r: c.act) == {"none", "swish", "lrelu"}
    assert levels(lambda c, r: c.params) == {"both", "gamma", "beta", "none"}
    assert levels(lambda c, r: (c.add, c.colsum)) == {(a, b) for a in (True, False) for b in (True, False)}
    assert levels(lambda c, r: c.terms) == {1, 2}
    for C_ in (96, 192):  # the atomic column-sum branch under its column sums
        assert any(c.C == C_ and c.colsum for c, r in rows)
    assert any(not r["fixed_cols"] and c.colsum and c.C > 1024 for c, r in rows)


def _norm_inputs(c, dev):
    g = torch.Generator().manual_seed(c.C * 31 + c.groups * 7 + c.n * 3 + c.hw)
    Cc = c.C
    x = torch.randn(c.n, c.hw, Cc, generator=g) * (0.5 + torch.rand(Cc, generator=g)) + 2 * torch.randn(Cc, generator=g)
    gamma = (0.5 + torch.rand(Cc, generator=g)) * torch.where(torch.rand(Cc, generator=g) < 0.3, -1.0, 1.0)
    beta = 0.5 * torch.randn(Cc, generator=g)
    dy = torch.randn(c.n, c.hw, Cc, generator=g)
    add = torch.randn(c.n, c.hw, Cc, generator=g) if c.add else None
    xd = x.double().view(c.n, c.hw, c.groups, Cc // c.groups)
    stats = torch.stack((xd.sum((1, 3)), (xd * xd).sum((1, 3))), -1)  # the buffer both the kernel and fp64 read
    to = lambda t: None if t is None else t.to(dev)  # noqa: E731
    return to(x), to(stats), to(gamma), to(beta), to(dy), to(add)


def _guarded(numel, dtype, dev, fill=SENTINEL):
    buf = torch.full((numel + 64,), fill, dtype=dtype, device=dev)
    return buf, buf[:numel]


def _norm_bwd(x, stats, gamma, beta, dy, *, add, dx, planes, terms, dgamma, dbeta, ws, n, hw, c, groups, act,
              colsum, sums_ready, eps=EPS):
    """t2h_norm_bwd with every pointer open; returns the status code"""
    from text2human_b200 import ops
    p = ops._ptr
    return _lib.load().t2h_norm_bwd(p(x), p(stats), p(gamma), p(beta), p(dy), p(add), p(dx), p(planes), terms,
                                    p(dgamma), p(dbeta), p(ws), n, hw, c, groups, eps, ops.ACT_CODE[act], p(colsum),
                                    sums_ready, ops._stream())


def _check_planes(planes, dx, terms, what):
    hi = planes[0]
    assert torch.equal(hi, dx.half()), f"{what}: hi plane is not fp16(dx)"
    if terms == 2:
        assert torch.equal(planes[1], (dx - hi.float()).half()), f"{what}: lo plane is not fp16(dx - hi)"


@pytest.mark.gpu
@pytest.mark.parametrize("c", NORM_CASES, ids=_nb_id)
def test_norm_bwd_matches_fp64(cuda, c):
    """three launches on one input: dx + planes (pass 1 included), planes only on the same pass-1 sums
    (sums_ready), fp32 dx only; every output against fp64, guard elements after each output untouched"""
    dev = cuda
    x, stats, gamma, beta, dy, add = _norm_inputs(c, dev)
    n, hw, Cc, T = c.n, c.hw, c.C, c.terms
    numel = n * hw * Cc
    ref = _norm_bwd_ref(x, stats, gamma, beta, dy, add, groups=c.groups, act=c.act, eps=EPS)
    kw = dict(n=n, hw=hw, c=Cc, groups=c.groups, act=c.act)
    h16 = torch.tensor(SENTINEL).half().item()
    colsum0 = torch.linspace(-1, 1, Cc, device=dev) if c.colsum else None
    par0 = torch.linspace(0.5, 2, Cc, device=dev)
    dg_buf, dgamma = _guarded(Cc, torch.float32, dev)
    db_buf, dbeta = _guarded(Cc, torch.float32, dev)
    dgamma.copy_(par0)
    dbeta.copy_(-par0)
    use_g, use_b = c.params in ("both", "gamma"), c.params in ("both", "beta")
    worst = 0.0

    # 1: fp32 dx and planes, pass 1 included
    dx_buf, dx = _guarded(numel, torch.float32, dev)
    pl_buf, planes = _guarded(T * numel, torch.float16, dev)
    ws = torch.full((n * Cc * 2,), SENTINEL, dtype=torch.float64, device=dev)
    cs = colsum0.clone() if c.colsum else None
    rc = _norm_bwd(x, stats, gamma, beta, dy, add=add, dx=dx, planes=planes, terms=T, dgamma=dgamma if use_g else None,
                   dbeta=dbeta if use_b else None, ws=ws, colsum=cs, sums_ready=0, **kw)
    assert rc == 0, _lib.load().t2h_last_error()
    torch.cuda.synchronize()
    what = _nb_id(c)
    worst = max(worst, _check(dx.view(n, hw, Cc), ref["dx"], ref["B"], f"{what} dx"))
    worst = max(worst, _sums_check(ws.view(n, Cc, 2), ref, f"{what} pass 1"))
    planes = planes.view(T, numel)
    _check_planes(planes, dx, T, what)
    assert (dx_buf[numel:] == SENTINEL).all() and (pl_buf[T * numel:] == h16).all(), "writes past dx / planes"
    du, dum, xh = ref["du"], ref["dum"], ref["xh"]
    if use_g:
        worst = max(worst, _check(dgamma, par0.double() + (du * xh).sum((0, 1)),
                                  (dum * (xh.abs() + ref["mrstd"])).sum((0, 1)) + par0.double().abs(),
                                  f"{what} dgamma", rel=0))
    else:
        assert torch.equal(dgamma, par0), "dgamma written although NULL was passed"
    if use_b:
        worst = max(worst, _check(dbeta, -par0.double() + du.sum((0, 1)), dum.sum((0, 1)) + par0.double().abs(),
                                  f"{what} dbeta", rel=0))
    else:
        assert torch.equal(dbeta, -par0), "dbeta written although NULL was passed"
    assert (dg_buf[Cc:] == SENTINEL).all() and (db_buf[Cc:] == SENTINEL).all(), "writes past dgamma / dbeta"
    colsum_B = (ref["dx"].abs() + ref["B"]).sum((0, 1))
    if c.colsum:
        worst = max(worst, _check(cs, colsum0.double() + ref["dx"].sum((0, 1)), colsum_B + colsum0.double().abs(),
                                  f"{what} dx column sums", rel=0))

    # 2: planes only, on the pass-1 sums launch 1 left in ws
    dgamma_before, dbeta_before = dgamma.clone(), dbeta.clone()
    pl2_buf, planes2 = _guarded(T * numel, torch.float16, dev)
    cs2 = colsum0.clone() if c.colsum else None
    rc = _norm_bwd(x, stats, gamma, beta, dy, add=add, dx=None, planes=planes2, terms=T, dgamma=None, dbeta=None, ws=ws,
                   colsum=cs2, sums_ready=1, **kw)
    assert rc == 0, _lib.load().t2h_last_error()
    torch.cuda.synchronize()
    assert torch.equal(planes2.view(T, numel), planes), "planes-only launch differs from the dx-and-planes launch"
    assert (pl2_buf[T * numel:] == h16).all(), "writes past the planes"
    assert torch.equal(dgamma, dgamma_before) and torch.equal(dbeta, dbeta_before)
    if c.colsum:
        _check(cs2, colsum0.double() + ref["dx"].sum((0, 1)), colsum_B + colsum0.double().abs(),
               f"{what} planes-only column sums", rel=0)

    # 3: fp32 dx only, its own pass 1
    dx3_buf, dx3 = _guarded(numel, torch.float32, dev)
    ws3 = torch.full((n * Cc * 2,), SENTINEL, dtype=torch.float64, device=dev)
    rc = _norm_bwd(x, stats, gamma, beta, dy, add=add, dx=dx3, planes=None, terms=T, dgamma=None, dbeta=None, ws=ws3,
                   colsum=None, sums_ready=0, **kw)
    assert rc == 0, _lib.load().t2h_last_error()
    torch.cuda.synchronize()
    worst = max(worst, _check(dx3.view(n, hw, Cc), ref["dx"], ref["B"], f"{what} dx only"))
    assert (dx3_buf[numel:] == SENTINEL).all(), "writes past dx"
    print(f"{what}: worst err/B over every output = {worst:.3g}")


@pytest.mark.gpu
def test_norm_bwd_through_ops_at_the_largest_channel_count(cuda):
    """ops.norm_bwd at C = 2048 (more than the default 48 KB of dynamic shared memory) with dgamma alone"""
    from text2human_b200 import ops
    c = NB(2048, 32, 2, 48, "swish", False, False, "gamma", 2)
    x, stats, gamma, beta, dy, _ = _norm_inputs(c, cuda)
    ref = _norm_bwd_ref(x, stats, gamma, beta, dy, None, groups=32, act="swish", eps=EPS)
    dgamma = torch.zeros(2048, device=cuda)
    dx, planes = ops.norm_bwd(x.view(2, 6, 8, 2048), stats, gamma, beta, dy.view(2, 6, 8, 2048), act="swish",
                              groups=32, eps=EPS, dgamma=dgamma, want_planes=True, terms=2)
    _check(dx.view(2, 48, 2048), ref["dx"], ref["B"], "ops.norm_bwd C=2048 dx")
    _check_planes(planes.view(2, -1), dx.view(-1), 2, "ops.norm_bwd C=2048")
    du, dum, xh = ref["du"], ref["dum"], ref["xh"]
    _check(dgamma, (du * xh).sum((0, 1)), (dum * (xh.abs() + ref["mrstd"])).sum((0, 1)), "dgamma alone", rel=0)


# ------------------------------------------------------------------ section 2: pass 1 in the data-gradient conv
NBS = collections.namedtuple("NBS", "N H W C groups act")
NB_SUMS_CASES = [
    NBS(5, 13, 40, 128, 32, "swish"),   # TW 16, ragged in H and W, tiles of several images per CTA
    NBS(2, 21, 9, 256, 8, "lrelu"),     # TW 8
    NBS(3, 37, 5, 384, 32, "none"),     # TW 4, cpg 12
    NBS(2, 70, 3, 128, 128, "swish"),   # TW 2, groups = C
    NBS(5, 150, 1, 256, 1, "lrelu"),    # TW 1, groups = 1
    NBS(1, 2, 40, 384, 8, "none"),      # the smallest height the fused path takes
    NBS(2, 16, 32, 256, 32, "lrelu"),   # interior tiles only
]


def _nbs_id(c):
    return f"n{c.N}x{c.H}x{c.W}-C{c.C}-g{c.groups}-{c.act}"


def _tile(W):
    TW = 16
    while TW > W and TW > 1:
        TW >>= 1
    return TW, 128 // TW


def test_nb_sums_case_table_covers_every_path():
    """the fused pass 1 runs at every spatial tile width, ragged in H at each, at several channel and group counts
    and every activation"""
    tiles = [(c, *_tile(c.W)) for c in NB_SUMS_CASES]
    assert {tw for c, tw, th in tiles} >= {16, 8, 4, 2, 1}
    assert all(any(tw == t and c.H % th for c, tw, th in tiles) for t in (16, 8, 4, 2, 1)), "a TW without ragged H"
    assert any(c.W % tw for c, tw, th in tiles) and any(c.H % th == 0 and c.W % tw == 0 for c, tw, th in tiles)
    assert any(c.N == 5 for c in NB_SUMS_CASES)
    assert {c.C for c in NB_SUMS_CASES} >= {128, 256, 384}
    assert {c.groups for c in NB_SUMS_CASES if c.groups != c.C} >= {1, 8, 32} and any(c.groups == c.C
                                                                                     for c in NB_SUMS_CASES)
    assert any(c.C == 384 and c.groups == 32 for c in NB_SUMS_CASES)
    assert {c.act for c in NB_SUMS_CASES} == {"none", "swish", "lrelu"}


@pytest.mark.gpu
@pytest.mark.parametrize("c", NB_SUMS_CASES, ids=_nbs_id)
def test_nb_sums_in_the_data_gradient_conv_match_fp64(cuda, c):
    """pass 1 of the norm backward accumulated in the epilogue of a stride-1 3x3 data-gradient conv: the sums per
    (image, channel) against fp64, the conv's output bit-identical with and without them, and the apply pass on
    them within the dx bound"""
    from text2human_b200 import conv_grad as G
    from text2human_b200 import ops
    dev = cuda
    N, H, W, Cc, Co = c.N, c.H, c.W, c.C, 64
    g = torch.Generator().manual_seed(N * 1000 + H * 10 + W + Cc)
    x = (torch.randn(N, H, W, Cc, generator=g) * (0.5 + torch.rand(Cc, generator=g)) + torch.randn(Cc, generator=g))
    x = x.to(dev)
    gamma = ((0.5 + torch.rand(Cc, generator=g)) * torch.where(torch.rand(Cc, generator=g) < 0.3, -1.0, 1.0)).to(dev)
    beta = (0.5 * torch.randn(Cc, generator=g)).to(dev)
    w = (torch.randn(Co, Cc, 3, 3, generator=g) / (9 * Cc) ** 0.5).to(dev)  # the conv that consumed act(norm(x))
    gy = torch.randn(N, H, W, Co, generator=g).to(dev)
    xd = x.double().view(N, H * W, c.groups, Cc // c.groups)
    stats = torch.stack((xd.sum((1, 3)), (xd * xd).sum((1, 3))), -1).contiguous()
    _, wt = G.weight_planes(G.oihw_to_master(w), 2)
    gyp = ops.split_planes(gy, 2)
    nb = ops.nb_context(x, stats, gamma, beta, act=c.act, groups=c.groups, eps=EPS)
    assert nb is not None
    da_f = G.dgrad("k3", gyp, wt, n=N, in_hw=(H, W), nb=nb)
    da_p = G.dgrad("k3", gyp, wt, n=N, in_hw=(H, W))
    torch.cuda.synchronize()
    assert torch.equal(da_f, da_p), "the norm-backward sums changed the conv's output"
    flat = lambda t: t.reshape(N, H * W, Cc)  # noqa: E731
    ref = _norm_bwd_ref(flat(x), stats, gamma, beta, flat(da_p), None, groups=c.groups, act=c.act, eps=EPS)
    w1 = _sums_check(nb["sums"].view(N, Cc, 2), ref, f"nb {_nbs_id(c)}")
    dx = ops.norm_bwd(x, stats, gamma, beta, da_f, act=c.act, groups=c.groups, eps=EPS, sums=nb["sums"])
    w2 = _check(flat(dx), ref["dx"], ref["B"], f"nb {_nbs_id(c)} dx on the fused sums")
    print(f"nb {_nbs_id(c)}: worst err/B {max(w1, w2):.3g}")


@pytest.mark.gpu
def test_nb_sums_refused_off_the_swapped_kernel(cuda):
    """a data-gradient conv with 96 output channels cannot run on the swapped-operand kernel: asking it for the
    norm-backward sums is an error (T2H_EINVAL), not a silently skipped pass 1"""
    from text2human_b200 import conv_grad as G
    from text2human_b200 import ops
    dev = cuda
    N, H, W, Cc, Co = 2, 8, 16, 96, 64
    g = torch.Generator().manual_seed(96)
    x = torch.randn(N, H, W, Cc, generator=g).to(dev)
    w = (torch.randn(Co, Cc, 3, 3, generator=g) / (9 * Cc) ** 0.5).to(dev)
    gyp = ops.split_planes(torch.randn(N, H, W, Co, generator=g).to(dev), 2)
    _, wt = G.weight_planes(G.oihw_to_master(w), 2)
    stats = ops.norm_stats(x, 32)
    assert ops.nb_context(x, stats, torch.ones(Cc, device=dev), torch.zeros(Cc, device=dev), act="swish", groups=32,
                          eps=EPS) is None
    sums = torch.zeros(N * Cc * 2, dtype=torch.float64, device=dev)
    nb = dict(x=x, stats=stats, gamma=torch.ones(Cc, device=dev), beta=torch.zeros(Cc, device=dev), act="swish",
              groups=32, eps=EPS, sums=sums)
    with pytest.raises(_lib.T2HError, match=r"libt2h error -1\b"):
        G.dgrad("k3", gyp, wt, n=N, in_hw=(H, W), nb=nb)
    torch.cuda.synchronize()
    assert not sums.any()


# ------------------------------------------------------------------ section 3: t2h_conv_wgrad
WG = collections.namedtuple("WG", "kind N H W cin cout terms k_split alpha accumulate")
# H, W: dY's extents (the forward conv's output); cin 8 is 3 real channels padded to 8; k_split 0 is the automatic
# split, 1000 exceeds every case's chunk count
WGRAD_CASES = [
    WG("k3", 2, 13, 40, 64, 128, 2, 0, 1.0, True),
    WG("k1", 5, 7, 9, 200, 136, 2, 3, 0.375, True),
    WG("down", 2, 11, 8, 64, 128, 2, 2, 1.0, False),
    WG("k4s2", 2, 9, 5, 72, 24, 1, 1, 1.0, True),
    WG("k4s1", 1, 19, 3, 8, 8, 2, 0, 0.375, False),
    WG("k3", 2, 37, 2, 64, 136, 2, 1000, 1.0, True),
    WG("k3", 3, 70, 1, 72, 128, 1, 3, 1.0, False),
    WG("down", 1, 6, 5, 200, 24, 1, 0, 0.375, True),
    WG("k4s2", 2, 5, 3, 64, 136, 2, 3, 1.0, True),
    WG("k1", 1, 9, 2, 8, 24, 2, 2, 1.0, True),
]
_S = {"k3": 1, "k1": 1, "k4s1": 1, "down": 2, "k4s2": 2}


def _wg_id(c):
    return (f"{c.kind}-n{c.N}x{c.H}x{c.W}-{c.cin}to{c.cout}-t{c.terms}-ks{c.k_split}-a{c.alpha:g}"
            f"{'-acc' if c.accumulate else ''}")


def _wg_route(c):
    from text2human_b200 import conv_grad as G
    return wgrad_route(c.H, c.W, c.N, c.cin, c.cout, G.KSIZE[c.kind] ** 2, c.k_split)


def test_wgrad_case_table_covers_every_path():
    """every patch shape (ragged in H at each), tap set, cin tile, output row tile and split-K level of t2h_conv_wgrad
    has a case"""
    rows = [(c, _wg_route(c)) for c in WGRAD_CASES]
    assert {r["PW"] for c, r in rows} >= {16, 8, 4, 2, 1}
    assert all(any(r["PW"] == pw and r["ragged_h"] for c, r in rows) for pw in (16, 8, 4, 2, 1))
    assert {c.W for c, r in rows} >= {40, 9, 8, 5, 3, 2, 1}
    assert {c.kind for c, r in rows} == {"k3", "k1", "down", "k4s2", "k4s1"}
    assert {c.cin for c, r in rows} >= {8, 64, 72, 200} and {c.cout for c, r in rows} >= {8, 24, 128, 136}
    assert {r["BN"] for c, r in rows} == {64, 128}
    assert any(r["BN"] == 128 and c.cin % 128 and r["col_tiles"] > 1 for c, r in rows), "no half-empty last cin tile"
    assert any(r["row_tiles"] > 1 and c.cout % 128 for c, r in rows), "no half-empty last cout tile"
    assert {c.k_split for c, r in rows} >= {0, 1, 2, 3}
    assert any(c.k_split == 3 and r["chunks"] % r["kper"] for c, r in rows), "no uneven last split-K slice"
    assert any(c.k_split > r["chunks"] and r["kper"] == 1 for c, r in rows), "no k_split beyond the chunk count"
    assert any(c.k_split == 0 and r["ksplit"] > 1 for c, r in rows)
    assert {c.terms for c, r in rows} == {1, 2}
    assert any(c.alpha != 1.0 for c, r in rows) and {c.accumulate for c, r in rows} == {True, False}
    assert any(c.kind in ("down", "k4s2") and c.terms == 2 for c, r in rows)


def _wg_operands(c, dev):
    """(dy planes [T,N,H,W,Co], x planes as the forward conv consumed them, x values [imgs, xh, xw, cin] fp64,
    dy values fp64, taps)"""
    from text2human_b200 import conv_grad as G
    from text2human_b200 import ops
    g = torch.Generator().manual_seed(c.N * 1000 + c.H * 37 + c.W + c.cin * 7 + c.cout)
    if c.kind == "k4s1":
        xH, xW = c.H + 1, c.W + 1
    else:
        xH, xW = c.H * _S[c.kind], c.W * _S[c.kind]
    real = 3 if c.cin == 8 else c.cin
    x = torch.zeros(c.N, xH, xW, c.cin)
    x[..., :real] = torch.randn(c.N, xH, xW, real, generator=g)
    dy = torch.randn(c.N, c.H, c.W, c.cout, generator=g)
    if _S[c.kind] == 2:  # space-to-depth phases [4, N, h, w, C], phase = 2 * row parity + column parity
        x = x.view(c.N, c.H, 2, c.W, 2, c.cin).permute(2, 4, 0, 1, 3, 5).reshape(4, c.N, c.H, c.W, c.cin)
    xp = ops.split_planes(x.to(dev), c.terms)
    dyp = ops.split_planes(dy.to(dev), c.terms)
    xv = xp.double().sum(0)
    xv = xv.reshape(-1, *xv.shape[-3:])
    taps = G.fwd_taps(c.kind, c.N) if c.kind != "k1" else ((0, 0, 0),)
    return dyp, xp, xv, dyp.double().sum(0), taps


def _wg_ref(xv, dyv, taps, alpha):
    """dw[t] = alpha sum_{n,h,w} dy[n,h,w,:]^T x[n + off_t, h + dy_t, w + dx_t, :] (zero outside the image), and the
    same on magnitudes"""
    N, H, W, _ = dyv.shape
    P = 2
    xpad = F.pad(xv, (0, 0, P, P + W, P, P + H))  # room for every shift
    ref, B = [], []
    for ty, tx, off in taps:
        s = xpad[off:off + N, P + ty:P + ty + H, P + tx:P + tx + W]
        ref.append(alpha * torch.einsum("nhwo,nhwi->oi", dyv, s))
        B.append(abs(alpha) * torch.einsum("nhwo,nhwi->oi", dyv.abs(), s.abs()))
    return torch.stack(ref), torch.stack(B)


@pytest.mark.gpu
@pytest.mark.parametrize("c", WGRAD_CASES, ids=_wg_id)
def test_conv_wgrad_matches_fp64(cuda, c):
    """one weight gradient into a [taps, cout, cin] view of a larger buffer (rows cin + 4 long, a spare output row per
    tap and a spare tap slot, all holding a sentinel) against fp64; nothing outside the view changes"""
    from text2human_b200 import ops
    dev = cuda
    dyp, xp, xv, dyv, taps = _wg_operands(c, dev)
    nt = len(taps)
    buf = torch.full((nt + 1, c.cout + 1, c.cin + 4), SENTINEL, device=dev)
    dw = buf[:nt, :c.cout, :c.cin]
    g = torch.Generator().manual_seed(c.cout)
    dw0 = torch.randn(nt, c.cout, c.cin, generator=g) if c.accumulate else torch.zeros(nt, c.cout, c.cin)
    dw0 = dw0.to(dev)
    dw.copy_(dw0)
    ops.conv_wgrad(dyp, xp, taps, dw, n=c.N, alpha=c.alpha, k_split=c.k_split)
    torch.cuda.synchronize()
    ref, B = _wg_ref(xv, dyv, taps, c.alpha)
    r = _wg_route(c)
    _check(dw, ref + dw0.double(), B + dw0.double().abs(),
           f"wgrad {_wg_id(c)} PW{r['PW']}xPH{r['PH']} BN{r['BN']} ks{r['ks']} kper{r['kper']}")
    outside = torch.ones(buf.shape, dtype=torch.bool, device=dev)
    outside[:nt, :c.cout, :c.cin] = False
    assert (buf[outside] == SENTINEL).all(), f"{int((buf[outside] != SENTINEL).sum())} stray writes"
