"""The transformer's row kernels, the fused attention and the sampler's token draw, route by route and element by
element against fp64: LayerNorm forward / scatter / split-K reduce + LayerNorm and the embedding sum
(csrc/elementwise.cu), softmax forward and backward, LayerNorm backward, GELU, the multi-head cross-entropy, the
embedding backward, column sums and Adam (csrc/train.cu), t2h_attn_fwd (csrc/attn_fused.cuh) and t2h_sample_step
(csrc/gan.cu).  Every kernel is called through the C ABI, so column placements, strides, row maps and unaligned
views that ``ops`` never passes are reachable.

The ``*_route`` functions restate the launch choices; a comment next to each rule in the C source points here.  They
document intent and do not verify the C code: a change to a rule updates its restatement in the same change, and the
CPU coverage tests then say which level lost its case.

Every reference is fp64 over the values the kernel reads (fp32 inputs, or fp16 planes summed in fp64).  Checks are
element by element, |err| <= k B + r |ref| + a, and print the worst err / B.  u = 2^-24 is fp32's unit roundoff.
Planes: where the fp32 value is also an output, hi == fp16(v) and lo == fp16(v - hi) bit for bit; where it is not,
hi must be an fp16 nearest to hi + lo (|lo| at most half of hi's spacing in lo's direction) and every element is
finite, with one allowance: a kernel that splits a product p = a b may be compiled with a b - hi contracted into
one fma, so that hi = fp16(fp32(p)) but lo = fp16(p - hi), and hi is then nearest to hi + lo only within one fp32
rounding.  The attention's o / sum does this: on an H100 build, 13 to 442 elements per two-plane case (up to ~1e-3 of
them).  Reading a value through its planes adds the planes' own rounding: lo is exact to 2^-23 |v| + 2^-25 (half a
subnormal step), hi alone to 2^-11 |v| + 2^-25; those terms are the r and a of the value checks.  Every output buffer
is a view into a sentinel-filled buffer, and every element outside the written region must keep its sentinel.

Bounds:
  * LayerNorm (forward, scatter, split-K reduce + LN): B = |gamma| (X + 1) + |beta|, k = 1e-5, with
    X = |xhat| + rstd mean|x| n u / k and n = ceil(C / 32) + 8.  The issue-level estimate was
    B = |xhat| |gamma| + |beta| + |gamma|; the extra term covers the fp32 row mean, whose terms each pass through at
    most n roundings (ceil(C / 32) lane adds, 2 pair adds in the float4 kernel, 5 butterfly levels, the division), so
    that the mean carries up to n u mean|x| of error and moves every xhat by rstd times that.  It matters only for rows
    with a large mean (mean 1e2, std 1 here), and there it is needed: without it the H100 measured err/B up to 8.2e-6
    on those rows (C = 513), against k = 1e-5 and a worst case near 2e-4.  Every case runs with one and two planes.
    Rows of one repeated dyadic value sum exactly, so their output is beta bit for bit.  Split-K: x_out must equal the fp32 sum residual + bias + slab 0 + slab 1 + ... bit for bit, and the
    vector and scalar routes must give the same x_out bits.
  * softmax forward: B = p (1 + |s scale - max|), k = 1e-5: the exp's argument carries u |s scale - max| of its own
    rounding plus u (|s scale| + |max|) <= 60 u from the product, and the row sum at most 69 roundings; both sit
    inside k.  Rows sum to 1 within (cols + 4) 2^-23: cols 2^-23 for the planes, 4 for the reciprocal, the final
    add, the expf ulp and the product's rounding.
  * softmax backward: B = |scale| p (|dp| + sum |dp| p), k = 1e-5 (the dot product rounds at most 69 times).  The
    planes launch with a power-of-two out_scale writes split(ds out_scale) of the fp32 launch's ds bit for bit.
  * LayerNorm backward: dx = rstd (g - mean g - xhat mean(g xhat)) + dx0, g = dy gamma, with the closed-form bound
    of test_gpu_backward_paths.py, B = rstd (|g| + mean|g| + X mean(|g| X)) + |dx0|, k = 1e-5, r = 1e-6; dgamma,
    dbeta and the dx column sums at 1e-5 of sum |terms| + |start value| (they accumulate, atomics in any order).
  * GELU forward: 4.2e-7 absolute (the gelu_erf comment's measurement over [-8, 8]) + 2^-22 |ref|: past |x| = 8 the
    result's own rounding (one product, ~1 ulp of up to 12) dominates.  Backward: B = |dg| (Phi + |x| phi (1 + x^2/2)
    + 1/2), k = 1e-6: the cdf carries ~4 u absolute (erff, 1 + erf), the exp's argument u x^2 / 2 relative.
  * ce_heads: loss |err| <= 1e-5 (|lse| + |x_t|); dlogits B = |w| (p (1 + |x - lse| + |lse|) + onehot), k = 1e-5.  The
    issue-level estimate was |w| (p + onehot); with logits up to +-80 the exp's argument x - lse reaches 160 and
    carries u (|x - lse| + |lse|) of rounding, which is relative error in p; and p below fp32's normal range
    (2^-126, reached at x - lse < -87) is held to |w| 2^-126 absolute.  Every other head of the row and every
    ignored row must be exactly 0 (the buffer starts at a sentinel).
  * embed_sum: torch fp32 ((tok + pos) + segm) + tex bit for bit.  embed_bwd and colsum: 1e-6 of
    sum |terms| + |start value| per output (fp32 atomics in any order).
  * Adam: one step from the state the kernel read, against an fp64 restatement of torch.optim.Adam: m and v at 1e-6
    of b1 |m| + (1 - b1) |g| and b2 v + (1 - b2) g^2, p at 1e-6 of |p'| + lr / bc1 (B_m + |m'|) / denom.  Elements
    whose scaled gradient is +-inf or NaN keep p, m and v bit for bit.
  * attention: B = sum_j p_j |v_j| (1 + |scale| max_j sum_i |q_i k_ji|), k = 2e-5 with two planes, 3e-4 with one: there the
    probabilities enter the p v product as one fp16 plane, rounded by up to 2^-12 = 2.4e-4 of p.
  * sample_step: the kernel's Philox4x32-10 with counter (class group c0, row lo, row hi, step) and key (seed lo,
    seed hi) is restated in numpy and checked against the Random123 known-answer vectors.  Each revealed row's token
    must be a class whose fp64 value logit inv_temp - log(-log uu) can be the row's maximum given the kernel's
    error, bounded per class from __logf's documented accuracy (2^-21.41 absolute on [0.5, 2], else 3 ulp) and fp32
    rounding; at least 95 % of rows must have exactly one such class.  The kernel's uu = ((r >> 8) + 0.5) 2^-24 rounds
    to 1.0 in fp32 when r >> 8 = 2^24 - 1, which gives that class a Gumbel value of +inf (probability 2^-24 per class
    and row); the restatement reproduces this.  The row-hi counter word is 0 for every row
    below 2^32, which no test can allocate: that word is left unverified.
"""
import collections
import ctypes

import numpy as np
import pytest
import torch

from text2human_b200 import _lib

SENTINEL = -7777.0
H16 = float(torch.tensor(SENTINEL).half())  # the sentinel as an fp16 plane holds it
U = 2.0 ** -24
EINVAL = -1
LN_EPS = 1e-5
H100_SMS = 132
K_LN = 1e-5
K_SM = 1e-5
K_TOL, K_REL = 1e-5, 1e-6
K_SUM = 1e-6
GELU_ABS, GELU_REL, K_GELU_BWD = 4.2e-7, 2.0 ** -22, 1e-6
K_ADAM = 1e-6
K_ATTN = {2: 2e-5, 1: 3e-4}
PLANE_R = {2: 2.0 ** -23, 1: 2.0 ** -11}  # the planes' own rounding, relative ...
PLANE_A = 2.0 ** -25                      # ... and absolute


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------ the launch rules, restated
def layernorm_route(c):
    """PER_LANE of layernorm_kernel (t2h_layernorm and t2h_layernorm_scatter)"""
    return 16 if c <= 512 else 32


def softmax_rows_route(cols):
    """PER_LANE of softmax_rows_kernel"""
    return 16 if cols <= 512 else 64


def softmax_bwd_route(cols):
    """PAIRS of softmax_bwd_kernel (t2h_softmax_bwd and t2h_softmax_bwd_planes)"""
    return 8 if cols <= 512 else 32


def layernorm_bwd_route(rows, c):
    """PER_LANE of layernorm_bwd_kernel and its grid: 8 warps per block, 2 rows per warp"""
    grid = max(_cdiv(rows, 16), 1)
    return dict(per_lane=16 if c <= 512 else 32, grid=grid, rows_per_warp=_cdiv(rows, grid * 8))


def splitk_route(c, slab, addrs, ln_addr, plane):
    """t2h_splitk_reduce_ln's kernel: the float4 kernel when C, the slab stride and every fp32 pointer (partials,
    x_out, residual, bias, gamma, beta; NULL counts as aligned) allow 16-byte accesses and ln_out / the ln plane allow
    8-byte ones, else the scalar kernel; VEC 4 / PER_LANE 16 up to C = 512"""
    aligned = (c % 4 == 0 and slab % 4 == 0 and all(a % 16 == 0 for a in addrs) and ln_addr % 8 == 0
               and plane % 4 == 0)
    if aligned:
        return "vec4" if c <= 512 else "vec8"
    return "scalar16" if c <= 512 else "scalar32"


def attn_route(batch, tokens, heads):
    """t2h_attn_fwd's grid: one CTA per (sequence, head, 128-query block), 64-key chunks"""
    qblocks = tokens // 128
    return dict(qblocks=qblocks, nchunks=tokens // 64, grid=batch * heads * qblocks)


def colsum_route(rows, c):
    """t2h_colsum: 128 columns per block, 64 rows per block until grid.y would pass 16384"""
    rpb = 64
    if _cdiv(rows, rpb) > 16384:
        rpb = _cdiv(rows, 16384)
    return dict(rpb=rpb, grid_x=_cdiv(c, 128), grid_y=_cdiv(rows, rpb))


# ------------------------------------------------------------------ shared helpers
def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ok(rc):
    assert rc == 0, _lib.load().t2h_last_error().decode()


def _f32(v):
    """an fp32 scalar as the kernel holds it, in fp64"""
    return float(np.float32(v))


def _check(got, ref, B, what, k, r=0.0, a=0.0):
    """|got - ref| <= k B + r |ref| + a element by element (NaN fails); returns the worst err / B, the error net of
    the r |ref| + a allowance (the planes' own rounding) so that it measures the kernel"""
    err = (got.double() - ref).abs()
    net = (err - r * ref.abs() - a).clamp_min(0)
    worst = (net / B.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    print(f"{what}: worst err/B = {worst:.3g}")
    bad = ~(err <= k * B + r * ref.abs() + a)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound, first at "
                           f"{tuple(bad.nonzero()[0].tolist())}, worst err/B {worst:.3g}")
    return worst


def _guarded(numel, dtype, dev, fill=SENTINEL):
    buf = torch.full((numel + 64,), fill, dtype=dtype, device=dev)
    return buf, buf[:numel]


def _split_of(planes, v, terms, what):
    """planes == split(v) bit for bit"""
    hi = v.half()
    assert torch.equal(planes[0], hi), f"{what}: hi plane is not fp16(v)"
    if terms == 2:
        assert torch.equal(planes[1], (v - hi.float()).half()), f"{what}: lo plane is not fp16(v - hi)"


def _nearest(planes, terms, what):
    """finite planes, and hi an fp16 nearest to hi + lo, within one fp32 rounding: a kernel that splits a product
    p = a b may, once nvcc contracts a b - hi into an fma, store hi = fp16(fp32(p)) and lo = fp16(p - hi), and
    fp32(p) and p can lie on either side of a midpoint between fp16 values"""
    assert torch.isfinite(planes).all(), f"{what}: non-finite planes"
    if terms == 1:
        return
    hi, lo = planes[0].double(), planes[1].double()
    m, e = torch.frexp(hi.abs())  # |hi| = m 2^e, m in [0.5, 1): spacing 2^(e - 11) in hi's binade
    normal = hi.abs() >= 2.0 ** -14
    up = torch.where(normal, torch.pow(2.0, (e - 11).double()), torch.full_like(hi, 2.0 ** -24))
    down = torch.where(normal & (m == 0.5) & (hi.abs() > 2.0 ** -14), up / 2, up)
    half = torch.where((lo * hi > 0) | (hi == 0), up, down) / 2
    exact = lo.abs() <= half
    bad = lo.abs() > half * (1 + 2.0 ** -10) + 2.0 ** -23 * hi.abs() + PLANE_A
    print(f"{what}: {int((~exact).sum())} of {exact.numel()} hi planes are nearest only within one fp32 rounding")
    assert not bad.any(), f"{what}: {int(bad.sum())} hi planes are not the nearest fp16 of hi + lo"


def _pval(planes, terms):
    return planes[0].double() + (planes[1].double() if terms == 2 else 0)


def _gamma_beta(C, g):
    gamma = (0.5 + torch.rand(C, generator=g)) * torch.where(torch.rand(C, generator=g) < 0.3, -1.0, 1.0)
    return gamma, 0.5 * torch.randn(C, generator=g)


def _mean_roundings(C):
    """roundings any term of a LayerNorm row mean passes through: ceil(C / 32) adds in its lane, 2 more in the
    float4 kernel's pair adds, 5 butterfly levels and the division"""
    return _cdiv(C, 32) + 8


def _ln_ref(x, gamma, beta, eps=LN_EPS):
    """fp64 LayerNorm of fp32 rows [rows, C] -> (y, B, X)"""
    xd = x.double()
    mean = xd.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mean) ** 2).mean(1, keepdim=True) + _f32(eps))
    xh = (xd - mean) * rstd
    X = xh.abs() + rstd * xd.abs().mean(1, keepdim=True) * _mean_roundings(x.shape[1]) * U / K_LN
    ga, be = gamma.double(), beta.double()
    return xh * ga + be, ga.abs() * (X + 1) + be.abs(), X, rstd


def _ln_rows(rows, C, g):
    """random rows of varied scale and offset; row 0 mean 1e2 with std 1, row 1 one repeated dyadic value"""
    x = torch.randn(rows, C, generator=g) * (0.5 + torch.rand(rows, 1, generator=g)) + 0.5 * torch.randn(rows, 1,
                                                                                                      generator=g)
    x[0] = 100 + torch.randn(C, generator=g)
    if rows > 1:
        x[1] = -2.75
    return x


def _check_ln_planes(planes, x, gamma, beta, terms, what):
    """LayerNorm output planes [terms, rows, C] of fp32 rows x against fp64"""
    _nearest(planes, terms, what)
    y, B, X, rstd = _ln_ref(x, gamma, beta)
    got = _pval(planes, terms)
    xh = X - rstd * x.double().abs().mean(1, keepdim=True) * _mean_roundings(x.shape[1]) * U / K_LN
    B0 = gamma.double().abs() * (xh + 1) + beta.double().abs()  # without the mean term, reported only
    net = ((got - y).abs() - PLANE_R[terms] * y.abs() - PLANE_A).clamp_min(0)
    print(f"{what}: worst err/B0 without the mean term = {(net / B0).max().item():.3g}, "
          f"on the mean-1e2 row {(net[0] / B0[0]).max().item():.3g}")
    w = _check(got, y, B, what, K_LN, PLANE_R[terms], PLANE_A)
    if x.shape[0] > 1 and bool((x[1] == x[1, 0]).all()):  # the constant row: exactly beta
        _split_of(planes[:, 1], beta, terms, f"{what} constant row")
    return w


# ------------------------------------------------------------------ section 1: LayerNorm forward and scatter
LN = collections.namedtuple("LN", "C rows")
# every case runs with one and with two planes
LN_CASES = [LN(1, 5), LN(31, 37), LN(32, 6), LN(33, 130), LN(96, 7), LN(511, 9), LN(512, 66), LN(513, 3), LN(640, 21),
            LN(1000, 10), LN(1024, 35)]


def test_layernorm_case_table_covers_every_route():
    """both PER_LANE levels, C at and just past each boundary, rows never a multiple of the 4 warps per block"""
    assert {layernorm_route(c.C) for c in LN_CASES} == {16, 32}
    assert {c.C for c in LN_CASES} >= {1, 31, 32, 33, 96, 511, 512, 513, 640, 1000, 1024}
    assert all(c.rows % 4 for c in LN_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("c", LN_CASES, ids=lambda c: f"C{c.C}-r{c.rows}")
def test_layernorm_and_scatter_match_fp64(cuda, c, terms):
    """t2h_layernorm into a guarded planes buffer, and t2h_layernorm_scatter of the same rows through a permutation
    into a larger buffer whose unmapped rows keep their sentinel in both planes"""
    dev, C, rows, T = cuda, c.C, c.rows, terms
    g = torch.Generator().manual_seed(C * 7 + rows)
    x = _ln_rows(rows, C, g)
    gamma, beta = _gamma_beta(C, g)
    out_rows = rows + 5 + rows // 2
    row_map = torch.randperm(out_rows, generator=g)[:rows]
    xd, gd, bd, rmd = x.to(dev), gamma.to(dev), beta.to(dev), row_map.to(dev)
    what = f"layernorm C{C} PER_LANE {layernorm_route(C)} t{T}"

    buf, out = _guarded(T * rows * C, torch.float16, dev)
    _ok(_lib.load().t2h_layernorm(_p(xd), _p(gd), _p(bd), _p(out), rows, C, LN_EPS, T, _st()))
    torch.cuda.synchronize()
    assert (buf[T * rows * C:] == H16).all(), f"{what}: writes past the planes"
    _check_ln_planes(out.view(T, rows, C).cpu(), x, gamma, beta, T, what)

    sbuf, sout = _guarded(T * out_rows * C, torch.float16, dev)
    _ok(_lib.load().t2h_layernorm_scatter(_p(xd), _p(gd), _p(bd), _p(sout), rows, C, LN_EPS, T, _p(rmd), out_rows, _st()))
    torch.cuda.synchronize()
    assert (sbuf[T * out_rows * C:] == H16).all(), f"{what} scatter: writes past the planes"
    sp = sout.view(T, out_rows, C).cpu()
    assert torch.equal(sp[:, row_map], out.view(T, rows, C).cpu()), f"{what}: scatter differs from the plain launch"
    untouched = torch.ones(out_rows, dtype=torch.bool)
    untouched[row_map] = False
    assert (sp[:, untouched] == H16).all(), f"{what} scatter: an unmapped row lost its sentinel"


# ------------------------------------------------------------------ section 2: split-K reduce + LayerNorm
SK = collections.namedtuple("SK", "C rows n_slabs bias residual alias ln off slab_pad row_map terms")
# off: the partials view starts `off` floats into its buffer; slab_pad: slab = rows * C + slab_pad (NaN in the gap)
SK_CASES = [
    SK(96, 6, 1, True, True, False, True, 0, 4, False, 2),
    SK(512, 9, 3, True, True, True, True, 0, 0, True, 1),
    SK(1000, 5, 2, False, True, False, True, 0, 8, False, 2),
    SK(1024, 7, 5, True, True, True, True, 0, 4, True, 2),
    SK(516, 3, 4, True, False, False, False, 0, 0, False, 1),
    SK(512, 6, 2, True, False, False, True, 1, 4, False, 2),
    SK(33, 10, 4, True, True, True, True, 0, 0, False, 1),
    SK(1, 5, 1, False, False, False, True, 0, 0, False, 2),
    SK(640, 6, 2, True, True, False, False, 1, 0, False, 1),
    SK(1023, 3, 5, False, True, True, True, 0, 0, True, 2),
    SK(768, 5, 3, True, True, False, True, 0, 1, False, 2),
    SK(96, 7, 2, True, True, False, True, 0, 3, False, 1),
]


def _sk_id(c):
    return (f"C{c.C}-r{c.rows}-s{c.n_slabs}{'-bias' if c.bias else ''}{'-res' if c.residual else ''}"
            f"{'-alias' if c.alias else ''}{'-ln' if c.ln else ''}-off{c.off}-pad{c.slab_pad}"
            f"{'-map' if c.row_map else ''}-t{c.terms}")


def _sk_table_route(c):
    """the route a case takes with torch's 256-byte aligned allocations"""
    return splitk_route(c.C, c.rows * c.C + c.slab_pad, [4 * c.off], 0, (c.rows + 3 if c.row_map else c.rows) * c.C)


def test_splitk_case_table_covers_every_route():
    """all four kernels, each misalignment cause (pointer, C % 4, slab), n_slabs 1 to 5, bias / residual absent,
    x_out aliasing the residual, no LayerNorm, a row map, both plane counts"""
    rows = [(c, _sk_table_route(c)) for c in SK_CASES]
    assert {r for c, r in rows} == {"vec4", "vec8", "scalar16", "scalar32"}
    assert any(c.off for c, r in rows) and any(c.C % 4 for c, r in rows) and any(c.slab_pad % 4 for c, r in rows)
    assert {c.n_slabs for c in SK_CASES} == {1, 2, 3, 4, 5}
    assert any(r.startswith("vec") and c.n_slabs >= 2 for c, r in rows)
    assert any(r == "vec8" and 512 < c.C < 1024 for c, r in rows)
    for key in ("bias", "residual", "alias", "ln", "row_map"):
        assert {getattr(c, key) for c in SK_CASES} == {True, False}, key
    assert any(c.alias and r.startswith("vec") for c, r in rows) and any(c.alias and r.startswith("scalar")
                                                                          for c, r in rows)
    assert {(r, c.terms) for c, r in rows if c.ln} >= {("vec4", 2), ("vec8", 2), ("scalar16", 1), ("scalar32", 2)}


def _splitk_run(c, dev, part_src, bias, res0, gamma, beta, row_map, off):
    """one launch; returns (x_out, ln planes or None, route)"""
    C, rows, T = c.C, c.rows, c.terms
    slab = rows * C + c.slab_pad
    pbuf = torch.full((off + c.n_slabs * slab + 64,), float("nan"), device=dev)
    for s in range(c.n_slabs):
        pbuf[off + s * slab:off + s * slab + rows * C] = part_src[s].reshape(-1)
    part = pbuf[off:]
    xbuf, x_out = _guarded(rows * C, torch.float32, dev)
    residual = None
    if c.residual:
        if c.alias:
            x_out.copy_(res0.reshape(-1))
            residual = x_out
        else:
            residual = res0.reshape(-1).clone()
    ln_rows = rows + 3 if c.row_map else rows
    lbuf, ln_out = _guarded(T * ln_rows * C, torch.float16, dev) if c.ln else (None, None)
    g_, b_ = (gamma, beta) if c.ln else (None, None)
    rm = row_map if c.row_map else None
    route = splitk_route(C, slab, [t.data_ptr() if t is not None else 0 for t in (part, x_out, residual, bias, g_, b_)],
                         ln_out.data_ptr() if c.ln else 0, ln_rows * C)
    _ok(_lib.load().t2h_splitk_reduce_ln(_p(part), c.n_slabs, slab, _p(bias), _p(residual), _p(x_out), _p(g_), _p(b_),
                                     LN_EPS, _p(ln_out), T, _p(rm), ln_rows, rows, C, _st()))
    torch.cuda.synchronize()
    assert (xbuf[rows * C:] == SENTINEL).all(), "writes past x_out"
    planes = None
    if c.ln:
        assert (lbuf[T * ln_rows * C:] == H16).all(), "writes past ln_out"
        planes = ln_out.view(T, ln_rows, C)
        if c.row_map:
            untouched = torch.ones(ln_rows, dtype=torch.bool, device=dev)
            untouched[row_map] = False
            assert (planes[:, untouched] == H16).all(), "an unmapped ln row lost its sentinel"
            planes = planes[:, row_map]
    return x_out.view(rows, C), planes, route


@pytest.mark.gpu
@pytest.mark.parametrize("c", SK_CASES, ids=_sk_id)
def test_splitk_reduce_ln_matches_fp64(cuda, c):
    """x_out == the fp32 sum in slab order bit for bit, LayerNorm of it against fp64; an aligned case also runs on
    a partials view one float off (the scalar kernel), which must give the same x_out bits"""
    dev, C, rows, T = cuda, c.C, c.rows, c.terms
    g = torch.Generator().manual_seed(C * 13 + rows * 5 + c.n_slabs)
    part_src = torch.randn(c.n_slabs, rows, C, generator=g).to(dev)
    bias = torch.randn(C, generator=g).to(dev) if c.bias else None
    res0 = torch.randn(rows, C, generator=g)
    res0[0] += 100  # a row with mean 1e2 and std ~1.4 once the slabs are added
    res0 = res0.to(dev)
    gamma, beta = (t.to(dev) for t in _gamma_beta(C, g))
    row_map = torch.randperm(rows + 3, generator=g)[:rows].to(dev)
    x_out, planes, route = _splitk_run(c, dev, part_src, bias, res0, gamma, beta, row_map, c.off)
    assert route == _sk_table_route(c)
    what = f"splitk {_sk_id(c)} {route}"
    want = res0.clone() if c.residual else torch.zeros(rows, C, device=dev)
    if c.bias:
        want = want + bias
    for s in range(c.n_slabs):
        want = want + part_src[s]
    assert torch.equal(x_out, want), f"{what}: x_out is not the fp32 sum in slab order"
    if c.ln:
        _check_ln_planes(planes.cpu(), x_out.cpu(), gamma.cpu(), beta.cpu(), T, what)
    if route.startswith("vec"):
        x2, planes2, route2 = _splitk_run(c, dev, part_src, bias, res0, gamma, beta, row_map, 1)
        assert route2.startswith("scalar")
        assert torch.equal(x2, x_out), f"{what}: the scalar kernel's x_out differs from the vector kernel's"
        if c.ln:
            _check_ln_planes(planes2.cpu(), x2.cpu(), gamma.cpu(), beta.cpu(), T, f"{what} on the scalar kernel")


# ------------------------------------------------------------------ section 3: softmax forward and backward
SM = collections.namedtuple("SM", "cols rows scale spread terms")
# spread: max - min of s * scale over a row, so the smallest probabilities reach e^-spread (~1e-26 at 60)
SM_CASES = [SM(1, 5, 0.125, 4, 2), SM(2, 7, -1.0, 10, 1), SM(31, 9, 0.5, 60, 2), SM(33, 3, -0.25, 60, 1),
            SM(512, 6, 1.0, 60, 2), SM(513, 5, -2.0, 60, 2), SM(1000, 11, 0.125, 30, 1), SM(2048, 7, -1.0, 60, 2)]


def test_softmax_case_table_covers_every_route():
    assert {(softmax_rows_route(c.cols), c.terms) for c in SM_CASES} == {(r, t) for r in (16, 64) for t in (1, 2)}
    assert {c.cols for c in SM_CASES} >= {1, 2, 31, 33, 512, 513, 1000, 2048}
    assert any(c.scale < 0 for c in SM_CASES) and max(c.spread for c in SM_CASES) >= 60
    assert all(c.rows % 4 for c in SM_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("c", SM_CASES, ids=lambda c: f"cols{c.cols}-r{c.rows}-s{c.scale:g}-w{c.spread}-t{c.terms}")
def test_softmax_rows_matches_fp64(cuda, c):
    dev, cols, rows, T = cuda, c.cols, c.rows, c.terms
    g = torch.Generator().manual_seed(cols * 3 + rows)
    s = (torch.rand(rows, cols, generator=g) - 0.5) * (c.spread / abs(c.scale))
    buf, out = _guarded(T * rows * cols, torch.float16, dev)
    sd = s.to(dev)
    _ok(_lib.load().t2h_softmax_rows(_p(sd), _p(out), rows, cols, c.scale, T, _st()))
    torch.cuda.synchronize()
    what = f"softmax cols {cols} PER_LANE {softmax_rows_route(cols)} t{T}"
    assert (buf[T * rows * cols:] == H16).all(), f"{what}: writes past the planes"
    planes = out.view(T, rows, cols).cpu()
    _nearest(planes, T, what)
    z = s.double() * _f32(c.scale)
    arg = z - z.max(1, keepdim=True).values
    p = torch.softmax(z, 1)
    got = _pval(planes, T)
    _check(got, p, p * (1 + arg.abs()), what, K_SM, PLANE_R[T], PLANE_A)
    if T == 2:
        dev1 = (got.sum(1) - 1).abs().max().item()
        print(f"{what}: worst |row sum - 1| = {dev1:.3g}")
        assert dev1 <= (cols + 4) * 2.0 ** -23


SB = collections.namedtuple("SB", "cols rows scale")
SB_CASES = [SB(2, 5, 0.125), SB(64, 6, -0.7), SB(510, 7, 0.125), SB(512, 9, 1.0), SB(514, 5, -0.7), SB(1024, 6, 0.125),
            SB(2048, 3, 0.125)]


def test_softmax_bwd_case_table_covers_every_route():
    assert {softmax_bwd_route(c.cols) for c in SB_CASES} == {8, 32}  # every case runs with one and two planes
    assert {c.cols for c in SB_CASES} >= {2, 64, 510, 512, 514, 1024, 2048}
    assert any(c.scale < 0 for c in SB_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("c", SB_CASES, ids=lambda c: f"cols{c.cols}-r{c.rows}-s{c.scale:g}")
def test_softmax_bwd_matches_fp64(cuda, c, terms):
    """fp32 ds against fp64 over the probabilities the planes hold; the planes launch writes split(ds out_scale)
    of the fp32 launch's ds bit for bit"""
    dev, cols, rows, T = cuda, c.cols, c.rows, terms
    g = torch.Generator().manual_seed(cols + rows * 11)
    prob = torch.softmax(torch.randn(rows, cols, generator=g) * 3, 1)
    hi = prob.half()
    pl = torch.stack((hi, (prob - hi.float()).half()))[:T].contiguous()
    dp = torch.randn(rows, cols, generator=g)
    pld, dpd = pl.to(dev), dp.to(dev)
    buf, ds = _guarded(rows * cols, torch.float32, dev)
    _ok(_lib.load().t2h_softmax_bwd(_p(pld), _p(dpd), _p(ds), rows, cols, c.scale, T, _st()))
    out_scale = 2.0 ** 6
    pbuf, dsp = _guarded(T * rows * cols, torch.float16, dev)
    _ok(_lib.load().t2h_softmax_bwd_planes(_p(pld), _p(dpd), _p(dsp), rows, cols, c.scale, T, out_scale, _st()))
    torch.cuda.synchronize()
    what = f"softmax_bwd cols {cols} PAIRS {softmax_bwd_route(cols)} t{T}"
    assert (buf[rows * cols:] == SENTINEL).all() and (pbuf[T * rows * cols:] == H16).all(), f"{what}: writes past"
    pv = _pval(pl, T)
    dpv = dp.double()
    sc = _f32(c.scale)
    ref = sc * pv * (dpv - (pv * dpv).sum(1, keepdim=True))
    B = abs(sc) * pv * (dpv.abs() + (pv * dpv.abs()).sum(1, keepdim=True))
    _check(ds.view(rows, cols).cpu(), ref, B, what, K_SM)
    _split_of(dsp.view(T, rows, cols), ds.view(rows, cols) * out_scale, T, f"{what} planes")


# ------------------------------------------------------------------ section 4: LayerNorm backward
LB = collections.namedtuple("LB", "C rows accumulate terms colsum")
LB_CASES = [LB(1, 17, True, 2, True), LB(33, 1, False, 1, True), LB(96, 15, True, 2, False), LB(512, 16, False, 2, True),
            LB(512, 2048, True, 1, True), LB(513, 17, False, 2, True), LB(1024, 5000, True, 2, True),
            LB(33, 5000, False, 2, False), LB(1024, 1, True, 1, False), LB(96, 2048, False, 2, True),
            LB(513, 15, True, 1, True)]


def _lb_id(c):
    return f"C{c.C}-r{c.rows}{'-acc' if c.accumulate else ''}-t{c.terms}{'-colsum' if c.colsum else ''}"


def test_layernorm_bwd_case_table_covers_every_route():
    rows = [(c, layernorm_bwd_route(c.rows, c.C)) for c in LB_CASES]
    assert {(r["per_lane"], c.accumulate) for c, r in rows} == {(p, a) for p in (16, 32) for a in (True, False)}
    assert {r["rows_per_warp"] for c, r in rows} == {1, 2}
    assert any(r["grid"] > 1 and c.rows % 16 for c, r in rows), "no partial last block"
    assert {c.C for c in LB_CASES} >= {1, 33, 96, 512, 513, 1024}
    assert {c.rows for c in LB_CASES} >= {1, 15, 16, 17, 2048, 5000}
    assert {c.terms for c in LB_CASES} == {1, 2} and {c.colsum for c in LB_CASES} == {True, False}


@pytest.mark.gpu
@pytest.mark.parametrize("c", LB_CASES, ids=_lb_id)
def test_layernorm_bwd_fused_matches_fp64(cuda, c):
    """dx (overwritten or accumulated), its planes, dgamma, dbeta and the dx column sums, all starting non-zero"""
    dev, C, rows, T = cuda, c.C, c.rows, c.terms
    g = torch.Generator().manual_seed(C * 17 + rows)
    x = torch.randn(rows, C, generator=g) * (0.5 + torch.rand(rows, 1, generator=g)) + 0.5 * torch.randn(rows, 1,
                                                                                                      generator=g)
    dy = torch.randn(rows, C, generator=g)
    gamma, _ = _gamma_beta(C, g)
    dx0 = torch.randn(rows, C, generator=g)
    start = torch.linspace(-1, 2, C)
    dxbuf, dx = _guarded(rows * C, torch.float32, dev)
    dx.copy_(dx0.view(-1))
    plbuf, planes = _guarded(T * rows * C, torch.float16, dev)
    bufs = [_guarded(C, torch.float32, dev) for _ in range(3)]
    (dgb, dgam), (dbb, dbet), (csb, cs) = bufs
    dgam.copy_(start)
    dbet.copy_(-start)
    cs.copy_(0.5 * start)
    dyd, xd_, gd = dy.to(dev), x.to(dev), gamma.to(dev)
    _ok(_lib.load().t2h_layernorm_bwd_fused(_p(dyd), _p(xd_), _p(gd), _p(dx), _p(dgam), _p(dbet),
                                        rows, C, LN_EPS, int(c.accumulate), _p(planes), T,
                                        _p(cs if c.colsum else None), _st()))
    torch.cuda.synchronize()
    r = layernorm_bwd_route(rows, C)
    what = f"layernorm_bwd {_lb_id(c)} PER_LANE {r['per_lane']} grid {r['grid']}"
    assert (dxbuf[rows * C:] == SENTINEL).all() and (plbuf[T * rows * C:] == H16).all(), f"{what}: writes past"
    assert all((b[C:] == SENTINEL).all() for b, _ in bufs), f"{what}: writes past a per-channel output"
    _, _, X, rstd = _ln_ref(x, gamma, torch.zeros(C))
    xd = x.double()
    xh = (xd - xd.mean(1, keepdim=True)) * rstd
    ga = gamma.double()
    gg = dy.double() * ga
    gm = dy.double().abs() * ga.abs()
    ref = rstd * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    B = rstd * (gm + gm.mean(1, keepdim=True) + X * (gm * X).mean(1, keepdim=True))
    if c.accumulate:
        ref, B = ref + dx0.double(), B + dx0.double().abs()
    dxc = dx.view(rows, C).cpu()
    worst = _check(dxc, ref, B, f"{what} dx", K_TOL, K_REL)
    _split_of(planes.view(T, rows, C).cpu(), dxc, T, f"{what} dx planes")
    s0 = start.double()
    dya = dy.double().abs()
    worst = max(worst, _check(dgam.cpu(), s0 + (dy.double() * xh).sum(0), (dya * X).sum(0) + s0.abs(),
                              f"{what} dgamma", K_TOL))
    worst = max(worst, _check(dbet.cpu(), -s0 + dy.double().sum(0), dya.sum(0) + s0.abs(), f"{what} dbeta", K_TOL))
    if c.colsum:
        worst = max(worst, _check(cs.cpu(), 0.5 * s0 + ref.sum(0), (ref.abs() + B).sum(0) + 0.5 * s0.abs(),
                                  f"{what} dx column sums", K_TOL))
    else:
        assert torch.equal(cs.cpu(), 0.5 * start), f"{what}: column sums written although NULL was passed"
    print(f"{what}: worst err/B over every output = {worst:.3g}")


# ------------------------------------------------------------------ section 5: GELU
def _gelu_sweep():
    return torch.cat((torch.linspace(-12, 12, 240001), torch.tensor([0.0, 1e-30, -1e-30])))


@pytest.mark.gpu
def test_gelu_fwd_matches_fp64(cuda):
    """a dense sweep of [-12, 12] plus 0 and +-1e-30: two planes against fp64, one plane == the same hi"""
    a = _gelu_sweep()
    n = a.numel()
    ad = a.to(cuda)
    b2, o2 = _guarded(2 * n, torch.float16, cuda)
    b1, o1 = _guarded(n, torch.float16, cuda)
    _ok(_lib.load().t2h_gelu_fwd(_p(ad), _p(o2), n, 2, _st()))
    _ok(_lib.load().t2h_gelu_fwd(_p(ad), _p(o1), n, 1, _st()))
    torch.cuda.synchronize()
    assert (b2[2 * n:] == H16).all() and (b1[n:] == H16).all(), "gelu_fwd: writes past the planes"
    planes = o2.view(2, n).cpu()
    _nearest(planes, 2, "gelu_fwd")
    assert torch.equal(o1.cpu(), planes[0]), "gelu_fwd: one-plane hi differs from the two-plane hi"
    xd = a.double()
    ref = 0.5 * xd * (1 + torch.erf(xd / 2 ** 0.5))
    got = _pval(planes, 2)
    net = ((got - ref).abs() - PLANE_R[2] * ref.abs() - PLANE_A).clamp_min(0)  # beyond the planes' own rounding
    print(f"gelu_fwd: worst absolute error beyond the planes' rounding {net.max().item():.3g} "
          f"(|x| <= 8: {net[xd.abs() <= 8].max().item():.3g})")
    _check(got, ref, torch.full_like(ref, GELU_ABS), "gelu_fwd", 1.0, GELU_REL + PLANE_R[2], PLANE_A)


@pytest.mark.gpu
def test_gelu_bwd_matches_fp64(cuda):
    a = _gelu_sweep()
    n = a.numel()
    dg = torch.randn(n, generator=torch.Generator().manual_seed(3))
    db, da = _guarded(n, torch.float32, cuda)
    pb, dap = _guarded(2 * n, torch.float16, cuda)
    ad, dgd = a.to(cuda), dg.to(cuda)
    _ok(_lib.load().t2h_gelu_bwd(_p(ad), _p(dgd), _p(da), _p(dap), n, 2, _st()))
    torch.cuda.synchronize()
    assert (db[n:] == SENTINEL).all() and (pb[2 * n:] == H16).all(), "gelu_bwd: writes past"
    xd = a.double()
    cdf = 0.5 * (1 + torch.erf(xd / 2 ** 0.5))
    pdf = torch.exp(-0.5 * xd * xd) / (2 * torch.pi) ** 0.5
    ref = dg.double() * (cdf + xd * pdf)
    B = dg.double().abs() * (cdf + xd.abs() * pdf * (1 + xd * xd / 2) + 0.5)
    dac = da.cpu()
    _check(dac, ref, B, "gelu_bwd", K_GELU_BWD)
    _split_of(dap.view(2, n).cpu(), dac, 2, "gelu_bwd planes")


# ------------------------------------------------------------------ section 6: masked multi-head cross-entropy
CE = collections.namedtuple("CE", "ncls nh rows")
CE_CASES = [CE(1, 18, 7), CE(7, 1, 9), CE(31, 18, 7), CE(256, 1, 8), CE(257, 18, 8), CE(1024, 18, 7), CE(2000, 1, 7),
            CE(2000, 18, 8)]


def test_ce_heads_case_table():
    assert {c.ncls for c in CE_CASES} >= {1, 7, 31, 256, 257, 1024, 2000} and {c.nh for c in CE_CASES} == {1, 18}
    assert all(c.rows >= 7 for c in CE_CASES)  # rows 0..6 carry the edge cases below
    assert {(c.ncls > 256, c.nh) for c in CE_CASES} == {(a, b) for a in (True, False) for b in (1, 18)}


@pytest.mark.gpu
@pytest.mark.parametrize("c", CE_CASES, ids=lambda c: f"ncls{c.ncls}-nh{c.nh}-r{c.rows}")
def test_ce_heads_matches_fp64(cuda, c):
    """rows 0 / 1: target 0 / ncls - 1, row 2: ignored target, rows 3 / 4: head -1 / nh, row 5: logits up to +-80,
    row 6: a three-way tie at the maximum, on the target; dlogits starts at a sentinel everywhere"""
    dev, ncls, nh, rows = cuda, c.ncls, c.nh, c.rows
    g = torch.Generator().manual_seed(ncls * 19 + nh)
    logits = torch.randn(rows, nh, ncls, generator=g) * 3
    target = torch.randint(0, ncls, (rows,), generator=g)
    head = torch.randint(0, nh, (rows,), generator=g)
    target[0], target[1], target[2] = 0, ncls - 1, -1
    head[3], head[4] = -1, nh
    logits[5] = (torch.rand(nh, ncls, generator=g) * 2 - 1) * 80
    top = logits[6, head[6]].max() + 1
    tied = torch.tensor([0, ncls // 2, ncls - 1])
    logits[6, head[6], tied] = top
    target[6] = ncls // 2
    w = 0.5 + torch.rand(rows, generator=g)
    lbuf, loss = _guarded(rows, torch.float32, dev)
    dbuf, dlog = _guarded(rows * nh * ncls, torch.float32, dev)
    ld_, td, hd, wd_ = logits.to(dev), target.to(dev), head.to(dev), w.to(dev)
    _ok(_lib.load().t2h_ce_heads(_p(ld_), _p(td), _p(hd), _p(wd_), _p(loss),
                             _p(dlog), rows, nh, ncls, _st()))
    torch.cuda.synchronize()
    what = f"ce_heads ncls {ncls} nh {nh}"
    assert (lbuf[rows:] == SENTINEL).all() and (dbuf[rows * nh * ncls:] == SENTINEL).all(), f"{what}: writes past"
    loss, dlog = loss.cpu(), dlog.view(rows, nh, ncls).cpu()
    valid = (target >= 0) & (head >= 0) & (head < nh)
    own = torch.zeros(rows, nh, dtype=torch.bool)
    for m in range(rows):
        if valid[m]:
            own[m, head[m]] = True
    assert (dlog[~own] == 0).all(), f"{what}: {int((dlog[~own] != 0).sum())} elements outside the own head are not 0"
    assert (loss[~valid] == 0).all(), f"{what}: an ignored row has a non-zero loss"
    vm = valid.nonzero().flatten()
    lr = logits[vm, head[vm]].double()
    lse = torch.logsumexp(lr, 1)
    xt = lr[torch.arange(len(vm)), target[vm]]
    w1 = _check(loss[vm], lse - xt, lse.abs() + xt.abs(), f"{what} loss", K_TOL)
    p = torch.exp(lr - lse[:, None])
    onehot = torch.nn.functional.one_hot(target[vm], ncls).double()
    wd = w[vm].double()[:, None]
    w2 = _check(dlog[vm, head[vm]], wd * (p - onehot),
                wd.abs() * (p * (1 + (lr - lse[:, None]).abs() + lse.abs()[:, None]) + onehot), f"{what} dlogits",
                K_TOL, a=wd.abs() * 2.0 ** -126)
    print(f"{what}: worst err/B {max(w1, w2):.3g}")


# ------------------------------------------------------------------ section 7: embeddings and column sums
ES = collections.namedtuple("ES", "C b t")
ES_CASES = [ES(4, 2, 7), ES(508, 3, 37), ES(512, 1, 5), ES(516, 2, 3), ES(2052, 2, 13)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", ES_CASES, ids=lambda c: f"C{c.C}-b{c.b}-t{c.t}")
def test_embed_sum_is_the_fp32_sum_bit_for_bit(cuda, c):
    """x = ((tok[idx] + pos[t]) + segm[s]) + tex[x] in fp32, with indices at both ends of every table"""
    dev, C, b, t = cuda, c.C, c.b, c.t
    g = torch.Generator().manual_seed(C + t)
    V, S, X = 11, 6, 4
    tabs = [torch.randn(n, C, generator=g) * sc for n, sc in ((V, 1.0), (t, 0.3), (S, 2.0), (X, 0.7))]
    rows = b * t
    idx = torch.randint(0, V, (rows,), generator=g)
    seg = torch.randint(0, S, (rows,), generator=g)
    tex = torch.randint(0, X, (rows,), generator=g)
    for ix, n in ((idx, V), (seg, S), (tex, X)):
        ix[0], ix[-1] = 0, n - 1
    tok, pos, sg, tx = (tb.to(dev) for tb in tabs)
    buf, x = _guarded(rows * C, torch.float32, dev)
    idd, sgd, txd = idx.to(dev), seg.to(dev), tex.to(dev)
    _ok(_lib.load().t2h_embed_sum(_p(idd), _p(sgd), _p(txd), _p(tok), _p(pos), _p(sg), _p(tx), _p(x), b, t, C, _st()))
    torch.cuda.synchronize()
    assert (buf[rows * C:] == SENTINEL).all(), "embed_sum: writes past x"
    tpos = torch.arange(rows, device=dev) % t
    want = ((tok[idd] + pos[tpos]) + sg[sgd]) + tx[txd]
    assert torch.equal(x.view(rows, C), want), "embed_sum differs from ((tok + pos) + segm) + tex in fp32"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["one_index", "spread", "positional"])
def test_embed_bwd_matches_fp64(cuda, mode):
    """every row on one index; indices at both table ends; the positional table with rows % t_mod != 0"""
    dev = cuda
    g = torch.Generator().manual_seed(len(mode))
    rows, C, V, t_mod = (300, 129, 5, 0) if mode == "one_index" else ((64, 130, 9, 0) if mode == "spread"
                                                                       else (25, 64, 7, 7))
    dx = torch.randn(rows, C, generator=g)
    idx = None
    if mode == "one_index":
        idx = torch.full((rows,), 3)
    elif mode == "spread":
        idx = torch.randint(0, V, (rows,), generator=g)
        idx[0], idx[-1] = 0, V - 1
    e0 = torch.randn(V, C, generator=g)
    buf, de = _guarded(V * C, torch.float32, dev)
    de.copy_(e0.view(-1))
    dxd, idd = dx.to(dev), None if idx is None else idx.to(dev)
    _ok(_lib.load().t2h_embed_bwd(_p(dxd), _p(idd), _p(de), rows, C, t_mod, _st()))
    torch.cuda.synchronize()
    assert (buf[V * C:] == SENTINEL).all(), "embed_bwd: writes past the table"
    e = idx if idx is not None else torch.arange(rows) % t_mod
    ref = e0.double().index_add(0, e, dx.double())
    B = e0.double().abs().index_add(0, e, dx.double().abs())
    got = de.view(V, C).cpu()
    _check(got, ref, B, f"embed_bwd {mode}", K_SUM)
    hit = torch.zeros(V, dtype=torch.bool)
    hit[e] = True
    assert torch.equal(got[~hit], e0[~hit]), "embed_bwd: a table row no index names changed"


CS = collections.namedtuple("CS", "rows C")
CS_CASES = [CS(1, 1), CS(63, 127), CS(64, 129), CS(65, 1), CS(1048577, 129)]


def test_colsum_case_table_covers_every_route():
    rows = [(c, colsum_route(c.rows, c.C)) for c in CS_CASES]
    assert {r["rpb"] == 64 for c, r in rows} == {True, False}, "both rows-per-block rules"
    assert any(r["rpb"] > 64 and r["grid_x"] > 1 and c.C % 128 for c, r in rows)
    assert {c.rows for c in CS_CASES} >= {1, 63, 64, 65, 1048577} and {c.C for c in CS_CASES} >= {1, 127, 129}


@pytest.mark.gpu
@pytest.mark.parametrize("c", CS_CASES, ids=lambda c: f"r{c.rows}-C{c.C}")
def test_colsum_matches_fp64(cuda, c):
    dev = cuda
    gen = torch.Generator(device=dev).manual_seed(c.rows + c.C)
    x = torch.randn(c.rows, c.C, device=dev, generator=gen)
    start = torch.linspace(-3, 3, c.C, device=dev)
    buf, out = _guarded(c.C, torch.float32, dev)
    out.copy_(start)
    _ok(_lib.load().t2h_colsum(_p(x), _p(out), c.rows, c.C, _st()))
    torch.cuda.synchronize()
    assert (buf[c.C:] == SENTINEL).all(), "colsum: writes past out"
    xd = x.double()
    r = colsum_route(c.rows, c.C)
    _check(out, start.double() + xd.sum(0), xd.abs().sum(0) + start.double().abs(),
           f"colsum rows {c.rows} C {c.C} rpb {r['rpb']} grid {r['grid_x']}x{r['grid_y']}", K_SUM)


# ------------------------------------------------------------------ section 8: Adam
LR, B1, B2, ADAM_EPS = 2e-3, 0.9, 0.999, 1e-8


def _adam_ref(p, g, m, v, step, gs):
    """one torch.optim.Adam step (weight_decay 0, amsgrad off) in fp64 from the fp32 state and the kernel's fp32
    hyper-parameters -> (p, m, v, Bp, Bm, Bv)"""
    b1, b2, lr, eps = _f32(B1), _f32(B2), _f32(LR), _f32(ADAM_EPS)
    gi = g.double() * _f32(gs)
    md, vd = m.double(), v.double()
    m1 = b1 * md + (1 - b1) * gi
    v1 = b2 * vd + (1 - b2) * gi * gi
    bc1, bc2s = 1 - b1 ** step, (1 - b2 ** step) ** 0.5
    denom = v1.sqrt() / bc2s + eps
    p1 = p.double() - (lr / bc1) * (m1 / denom)
    Bm = b1 * md.abs() + (1 - b1) * gi.abs()
    return p1, m1, v1, p1.abs() + (lr / bc1) * (Bm + m1.abs()) / denom, Bm, v1


def _adam_launch(p, g, m, v, step, gs):
    _ok(_lib.load().t2h_adam(_p(p), _p(g), _p(m), _p(v), p.numel(), LR, B1, B2, ADAM_EPS, step, gs, _st()))
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, H100_SMS * 16 * 256 + 4099])
def test_adam_matches_fp64(cuda, n):
    """steps 1, 2, 3 and 1000 from the state the previous step left, grad_scale != 1; the larger n runs the
    grid-stride loop (the grid is capped at 16 blocks of 256 per SM)"""
    dev = cuda
    gen = torch.Generator(device=dev).manual_seed(n)
    p = torch.randn(n, device=dev, generator=gen)
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    worst = 0.0
    for step, gs in ((1, 0.5), (2, 0.25), (3, 0.5), (1000, 0.125)):
        g = torch.randn(n, device=dev, generator=gen) * 3
        ref = _adam_ref(p, g, m, v, step, gs)
        _adam_launch(p, g, m, v, step, gs)
        for got, want, B, name in ((p, ref[0], ref[3], "p"), (m, ref[1], ref[4], "m"), (v, ref[2], ref[5], "v")):
            worst = max(worst, _check(got, want, B, f"adam n {n} step {step} {name}", K_ADAM))
    print(f"adam n {n}: worst err/B {worst:.3g}")


@pytest.mark.gpu
def test_adam_leaves_non_finite_gradients_untouched(cuda):
    """elements whose gradient is +inf, -inf or NaN keep p, m and v bit for bit; every other element, their
    neighbours included, takes the step"""
    dev = cuda
    n = 4099
    g0 = torch.Generator().manual_seed(9)
    p, m = torch.randn(n, generator=g0).to(dev), torch.randn(n, generator=g0).to(dev) * 0.1
    v = (torch.rand(n, generator=g0) * 0.01).to(dev)
    g = torch.randn(n, generator=g0)
    bad = torch.tensor([0, 5, 6, 7, 100, 2048, 4097, 4098])
    g[bad] = torch.tensor([float("inf"), float("-inf"), float("nan"), float("inf"), float("nan"), float("-inf"),
                           float("nan"), float("inf")])
    g = g.to(dev)
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    ref = _adam_ref(p0, torch.where(g.isfinite(), g, 0.0), m0, v0, 4, 0.5)
    _adam_launch(p, g, m, v, 4, 0.5)
    bm = torch.zeros(n, dtype=torch.bool, device=dev)
    bm[bad] = True
    for got, before, want, B, name in ((p, p0, ref[0], ref[3], "p"), (m, m0, ref[1], ref[4], "m"),
                                       (v, v0, ref[2], ref[5], "v")):
        assert torch.equal(got[bm].view(torch.int32), before[bm].view(torch.int32)), f"adam: {name} changed at a " \
                                                                                      "non-finite gradient"
        _check(got[~bm], want[~bm], B[~bm], f"adam non-finite neighbours {name}", K_ADAM)
        assert (got[~bm] != before[~bm]).all(), f"adam: a finite-gradient element kept its {name}"


# ------------------------------------------------------------------ section 9: the fused attention through the ABI
AT = collections.namedtuple("AT", "tokens heads batch terms spread")
AT_CASES = [AT(128, 1, 1, 2, 1.0), AT(256, 3, 5, 1, 4.0), AT(384, 8, 2, 2, 4.0), AT(512, 16, 1, 2, 2.0),
            AT(512, 3, 3, 1, 1.0), AT(128, 16, 4, 1, 2.0), AT(384, 1, 5, 1, 0.5), AT(256, 8, 2, 2, 4.0)]


def _at_id(c):
    return f"T{c.tokens}-h{c.heads}-b{c.batch}-t{c.terms}-w{c.spread:g}"


def test_attn_case_table_covers_every_route():
    rows = [(c, attn_route(c.batch, c.tokens, c.heads)) for c in AT_CASES]
    assert {(r["qblocks"], c.terms) for c, r in rows} == {(q, t) for q in (1, 2, 3, 4) for t in (1, 2)}
    assert {r["nchunks"] for c, r in rows} == {2, 4, 6, 8}
    assert {c.heads for c in AT_CASES} >= {1, 3, 8, 16} and {1, 5} <= {c.batch for c in AT_CASES}
    assert max(c.spread for c in AT_CASES) >= 4


def _attn_layout(c, idx):
    """q / k / v column blocks of C = 64 heads columns, permuted per case, 8 columns apart inside ld = 3C + 64"""
    C = 64 * c.heads
    order = [(0, 1, 2), (2, 0, 1), (1, 2, 0), (2, 1, 0)][idx % 4]
    cols = [8 + order[i] * (C + 16) for i in range(3)]
    return C, cols, 3 * C + 64


@pytest.mark.gpu
@pytest.mark.parametrize("ci", range(len(AT_CASES)), ids=lambda i: _at_id(AT_CASES[i]))
def test_attn_fwd_matches_fp64(cuda, ci):
    """q, k, v in permuted column blocks of a padded projection with NaN everywhere the kernel must not read (the
    padding columns, the gaps, spare trailing rows, the gap between the planes); the output into a column window of
    a wider sentinel buffer with ld_out > C and a plane stride that is not rows * ld_out"""
    c = AT_CASES[ci]
    dev, T, Tn, nh, Bt = cuda, c.terms, c.tokens, c.heads, c.batch
    C, (qc, kc, vc), ld = _attn_layout(c, ci)
    BT = Bt * Tn
    rows = BT + 37
    plane = rows * ld + 24
    g = torch.Generator().manual_seed(ci * 101 + Tn)
    sig = c.spread ** 0.5  # scores q.k / 8 then have standard deviation `spread`
    q, k = (torch.randn(BT, C, generator=g) * sig for _ in range(2))
    v = torch.randn(BT, C, generator=g)
    qkv = torch.full((T * plane + 64,), float("nan"), dtype=torch.float16, device=dev)
    for t in range(T):
        pv = qkv[t * plane:t * plane + rows * ld].view(rows, ld)
        for col, val in ((qc, q), (kc, k), (vc, v)):
            hi = val.half()
            pv[:BT, col:col + C] = (hi if t == 0 else (val - hi.float()).half()).to(dev)
    ld_out, col0 = C + 48, 16
    out_plane = rows * ld_out + 40
    obuf = torch.full((T * out_plane + 64,), H16, dtype=torch.float16, device=dev)
    out_ptr = ctypes.c_void_p(obuf.data_ptr() + 2 * col0)
    scale = 0.125
    _ok(_lib.load().t2h_attn_fwd(_p(qkv), T, plane, ld, rows, qc, kc, vc, Bt, Tn, nh, 64, scale, out_ptr, out_plane, ld_out,
                             _st()))
    torch.cuda.synchronize()
    r = attn_route(Bt, Tn, nh)
    what = f"attn {_at_id(c)} qblocks {r['qblocks']} nchunks {r['nchunks']}"
    window = torch.zeros(obuf.numel(), dtype=torch.bool, device=dev)
    for t in range(T):
        window[t * out_plane:t * out_plane + rows * ld_out].view(rows, ld_out)[:BT, col0:col0 + C] = True
    assert (obuf[~window] == H16).all(), f"{what}: {int((obuf[~window] != H16).sum())} writes outside the window"
    got = torch.stack([obuf[t * out_plane:t * out_plane + rows * ld_out].view(rows, ld_out)[:BT, col0:col0 + C]
                       for t in range(T)])
    _nearest(got, T, what)

    def heads(val):  # the fp64 values the planes hold -> [B, nh, T, 64]
        hi = val.half()
        d = hi.double() + ((val - hi.float()).half().double() if T == 2 else 0)
        return d.view(Bt, Tn, nh, 64).permute(0, 2, 1, 3).to(dev)

    qd, kd, vd = heads(q), heads(k), heads(v)
    sc = _f32(scale)
    P = torch.softmax(qd @ kd.transpose(-1, -2) * sc, -1)
    ref = P @ vd
    B = (P @ vd.abs()) * (1 + abs(sc) * (qd.abs() @ kd.abs().transpose(-1, -2)).max(-1, keepdim=True).values)
    flat = lambda t4: t4.permute(0, 2, 1, 3).reshape(BT, C)  # noqa: E731
    _check(_pval(got, T), flat(ref), flat(B), what, K_ATTN[T], PLANE_R[T], PLANE_A)


@pytest.mark.gpu
def test_attn_fwd_refuses_bad_arguments(cuda):
    """one call per argument check, each with a single bad argument: T2H_EINVAL, and the output keeps every bit.
    These checks are on the host; the buffers are nevertheless sized for anything a launch of these shapes could
    touch (640 tokens, three planes, ld_out down to 120), and the misaligned output is 8 bytes off, so a store
    through it would still be aligned"""
    dev = cuda
    heads, C = 2, 128
    rows_alloc, ld, ld_out = 640, 3 * C + 8, C + 8
    plane = rows_alloc * ld
    qkv = torch.zeros(3 * plane, dtype=torch.float16, device=dev)
    obuf = torch.full((3 * rows_alloc * ld_out + 256,), H16, dtype=torch.float16, device=dev)
    base = dict(terms=2, plane=plane, ld=ld, rows=rows_alloc, q_col=0, k_col=C, v_col=2 * C, batch=1, tokens=128,
                heads=heads, head_dim=64, out=obuf.data_ptr(), out_plane=rows_alloc * ld_out, ld_out=ld_out)
    bad = [("tokens", 64), ("tokens", 200), ("tokens", 640), ("head_dim", 32), ("q_col", 4), ("v_col", 2 * C + 16),
           ("ld_out", 64 * heads - 8), ("out", obuf.data_ptr() + 8), ("rows", 127), ("terms", 3)]
    for key, val in bad:
        a = dict(base, **{key: val})
        rc = _lib.load().t2h_attn_fwd(_p(qkv), a["terms"], a["plane"], a["ld"], a["rows"], a["q_col"], a["k_col"],
                                  a["v_col"], a["batch"], a["tokens"], a["heads"], a["head_dim"], 0.125,
                                  ctypes.c_void_p(a["out"]), a["out_plane"], a["ld_out"], _st())
        torch.cuda.synchronize()
        assert rc == EINVAL, f"attn_fwd {key}={val}: returned {rc}, not T2H_EINVAL"
        assert b"attn_fwd" in _lib.load().t2h_last_error()
        assert (obuf == H16).all(), f"attn_fwd {key}={val}: the output changed"
    _ok(_lib.load().t2h_attn_fwd(_p(qkv), 2, plane, ld, rows_alloc, 0, C, 2 * C, 1, 128, heads, 64, 0.125, _p(obuf),
                             rows_alloc * ld_out, ld_out, _st()))  # the base arguments are valid
    torch.cuda.synchronize()


# ------------------------------------------------------------------ section 10: the sampler's token draw
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on uint32 arrays, as sample_step_kernel computes it"""
    c = [np.asarray(x, dtype=np.uint64) & _M32 for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & _M32, np.uint64(k1) & _M32
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return [x.astype(np.uint32) for x in c]


def test_philox_restatement_matches_known_answers():
    """the Random123 known-answer vectors of philox4x32-10"""
    kat = [((0, 0, 0, 0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 6, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for args, want in kat:
        assert tuple(int(x) for x in philox4x32_10(*args)) == want


def sample_uniforms(rows, ncls, seed, step):
    """uu[row, class] as the kernel forms it: class group c0 = 4 (c // 4) keys counter (c0, row lo, row hi, step) and
    key (seed lo, seed hi); word c % 4, top 24 bits, ((float)(r >> 8) + 0.5f) / 2^24 in fp32 (which rounds to 1.0 at
    r >> 8 = 2^24 - 1)"""
    c0 = np.arange(0, ncls, 4, dtype=np.uint64)[None, :]
    m = np.arange(rows, dtype=np.uint64)[:, None]
    words = philox4x32_10(np.broadcast_to(c0, (rows, c0.shape[1])), m & _M32, m >> np.uint64(32),
                          np.full((rows, c0.shape[1]), step, dtype=np.uint64), seed & 0xFFFFFFFF, seed >> 32)
    r = np.stack(words, -1).reshape(rows, -1)[:, :ncls]
    return (np.float32(r >> 8) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


def _gumbel_candidates(logits, inv_temp, uu):
    """per row: the classes whose fp64 value logit inv_temp - log(-log uu) can be the kernel's maximum, and the fp64
    argmax.  The kernel's error per class: u (|x inv_temp| + |v|) for its two fp32 roundings, the outer __logf's
    2^-21.41 absolute on [0.5, 2] or 3 ulp, and the inner __logf's error dL (2^-21.41 absolute for uu in [0.5, 1),
    else 3 ulp) carried through log as dL / (L - dL); doubled"""
    x = logits.astype(np.float64) * float(inv_temp)
    u64 = uu.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        L = -np.log(u64)
        gum = -np.log(L)
        v = x + gum
        dL = np.where(u64 >= 0.5, 2.0 ** -21.41, 3 * 2.0 ** -23 * L)
        prop = np.where(L > dL, dL / (L - dL), np.inf)
        e = 2 * (U * (np.abs(x) + np.abs(v)) + 2.0 ** -21.41 + 3 * 2.0 ** -23 * np.abs(gum) + prop)
    one = u64 == 1.0  # -log(-log 1) = +inf in the kernel and here
    v = np.where(one, np.inf, v)
    e = np.where(one, 0.0, e)
    lower = np.max(np.where(np.isinf(e), -np.inf, v - e), 1, keepdims=True)
    return (v + e >= lower) | one, np.argmax(v, 1)


SS = collections.namedtuple("SS", "ncls rows")
SS_CASES = [SS(1, 300), SS(127, 2000), SS(128, 2000), SS(129, 2000), SS(1024, 600)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", SS_CASES, ids=lambda c: f"ncls{c.ncls}-r{c.rows}")
def test_sample_step_draws_the_keyed_gumbel_max(cuda, c):
    """each revealed row's token is the argmax of logit inv_temp + Gumbel noise from the restated Philox stream;
    rows already unmasked and rows not revealed keep x_t, rows with a texture outside 0..17 are unmasked without a
    token"""
    dev, ncls, rows = cuda, c.ncls, c.rows
    g = torch.Generator().manual_seed(ncls * 7 + rows)
    logits = torch.randn(rows, ncls, generator=g) * 2
    u = torch.rand(rows, generator=g)
    tex = torch.randint(0, 18, (rows,), generator=g)
    tex[3::50], tex[4::50] = -1, 18
    unm0 = torch.zeros(rows, dtype=torch.uint8)
    unm0[::7] = 1
    x0 = torch.full((rows,), -5, dtype=torch.long)
    seed, step, inv_t, inv_temp, cont = 0x9E3779B97F4A7C15 ^ ncls, 77 + ncls, 0.5, _f32(1 / 0.8), 1024
    x_t, unm = x0.to(dev), unm0.to(dev)
    ld_, ud, txd = logits.to(dev), u.to(dev), tex.to(dev)
    _ok(_lib.load().t2h_sample_step(_p(ld_), _p(ud), _p(txd), _p(x_t), _p(unm), rows, ncls, 18,
                                inv_t, inv_temp, seed, step, cont, _st()))
    torch.cuda.synchronize()
    x_t, unm = x_t.cpu(), unm.cpu()
    rev = (u < inv_t) & (unm0 == 0)
    assert torch.equal(unm.bool(), rev | unm0.bool()), "sample_step: wrong rows unmasked"
    valid = (tex >= 0) & (tex < 18)
    assert torch.equal(x_t[~(rev & valid)], x0[~(rev & valid)]), "sample_step: x_t written where it must not be"
    sel = (rev & valid).nonzero().flatten()
    assert sel.numel() > rows // 4
    tok = (x_t[sel] - cont * tex[sel]).numpy()
    assert tok.min() >= 0 and tok.max() < ncls
    uu = sample_uniforms(rows, ncls, seed, step)[sel.numpy()]
    cand, best = _gumbel_candidates(logits[sel].numpy(), inv_temp, uu)
    ok = cand[np.arange(len(sel)), tok]
    single = cand.sum(1) == 1
    print(f"sample_step ncls {ncls}: {len(sel)} rows drawn, {int(single.sum())} unambiguous, "
          f"{int((tok == best).sum())} equal to the fp64 argmax")
    assert ok.all(), (f"sample_step ncls {ncls}: {int((~ok).sum())} tokens no keyed draw allows, first at row "
                      f"{int(sel[np.nonzero(~ok)[0][0]])}")
    assert single.mean() >= 0.95, "too few unambiguous rows: the check says little"
