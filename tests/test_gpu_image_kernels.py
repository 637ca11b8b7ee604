"""The image-side kernels, route by route and element by element against fp64: the plane producers and layout
kernels of csrc/elementwise.cu (NCHW / NHWC transposes, t2h_f32_to_planes in every mode, GroupNorm / BatchNorm
apply with swish / LeakyReLU, one-hot, uint8 in and out, the per-head argmax, the nearest id resize, the in-place
add), the GAN training step's kernels of csrc/gan.cu (L1, hinge, BCE-with-logits, quantizer backward, sum-pool,
space-to-depth planes, LeakyReLU backward, DiffAugment forward and backward, adaptive weight, axpy, BatchNorm
running statistics) and the quantizer's edges (csrc/vq.cu) against oracle/vq_oracle.c.  Every kernel is called
through the C ABI, so NULL optional outputs, misaligned views and sizes that ``ops`` never passes are reachable.

The ``*_route`` functions restate the launch choices; a comment next to each rule in the C source points here.  They
document intent and do not verify the C code: a change to a rule updates its restatement in the same change, and the
CPU coverage tests then say which level lost its case.  num_sms() is 132 on an H100 SXM.

Every reference is fp64 over the values the kernel reads.  Checks are element by element, |err| <= k B + r |ref| + a,
and print the worst err / B.  u = 2^-24 is fp32's unit roundoff.  Planes: where the fp32 value is an output or an
exact input, hi == fp16_rn(v) and lo == fp16_rn(v - hi) bit for bit (a split that truncated hi fails this), and pad
channels are 0 in both planes.  Where the fp32 value is not observable, reading a value through its planes adds the
planes' own rounding: 2^-23 |v| + 2^-25 with two planes, 2^-11 |v| + 2^-25 with one; those are the r and a of the
value checks.  Every output buffer is a view into a sentinel-filled buffer, and everything outside the written region
must keep its sentinel.

Bounds:
  * transposes, PLAIN / UP2X / S2D / MAXPOOL2 planes, sum-pool, space-to-depth, one-hot, add_inplace, lrelu_bwd,
    l1 / hinge gradients: bit for bit (copies, max, fixed-order fp32 adds, sign rules).
  * BILINEAR2X: B = the same interpolation of |x|, k = 4u (1 + 2^-20): each neighbour's term passes through at most
    four roundings (inner product and add, outer product and add, or fewer once contracted into fmas), and the
    weights 0, 1/4, 3/4, 1 are exact; the factor covers the second-order remainder.
  * gn_apply, pre-activation y: B = |gamma| rstd (|x| + |mean|) + |beta| + |y|, k = 5u: rstd, gamma rstd and the
    product put 3u on x scale, the mean's own rounding a fourth on mean scale, the shift's subtraction and the
    final add u each.  swish = 2 (LeakyReLU, slope fp32(0.2)): the same B (slope <= 1) plus u |out| for the
    product.  swish = 1: B scaled by max |silu'| = 1.1, plus a relative (2 + floor(1.16 |y|)) 2^-23 for __expf's
    documented error (y / (1 + E) moves by at most E's relative error) and 2u for the add and the division.
  * l1 / hinge sums: B = sum |term|, k = u + n 2^-53: one fp32 rounding per term (the difference), fp64 accumulation.
    A start value in the accumulator is part of the reference.
  * bce_logits: loss within 1e-6 of sum (max(x, 0) + |x| t + log1p(e^-|x|)) (expf, log1pf, two adds and the
    8-term fp32 partial sum, about 12u); gradient planes within 8u |g| (expf's 2 ulp, the add, the division, the
    product with e^-|x|, gscale) plus the planes' rounding.  A target logit above about 17 has g = -gscale
    sigmoid(-x), which is checked relatively down to 2^-25 (the case with gscale 2^14 keeps it in fp16's range
    up to x ~ 22; beyond that only the absolute 2^-25 applies).  colsum: 1e-6 sum |g| + G u (|start| + sum |g|),
    G the grid: every block adds its sums with one fp32 atomic, which rounds relative to the running value, and that
    value is dominated by the start value.  The issue-level estimate, 1e-6 (sum |g| + |start|), held on the H100 only
    by a factor 1.16 (8.6e-7 with 528 blocks) and has no derivation behind it, so the bound counts the atomics.
  * vq_bwd: dz B = |dzq| + |coef_z| |z - e|, k = 3u (difference, product, add).  dcodebook: 1e-6 sum |terms| +
    m u (|start| + sum |terms|), m the rows on that code: each of the m fp32 atomic adds rounds relative to the
    running value, which the start value dominates.  The issue-level estimate, 1e-6 (|start| + sum |terms|), failed
    on the H100 (err / B 1.5e-6 on codes with 333 and 700 rows: about sqrt(m) u, as rounding errors of random sign
    add up).  With one row on a code the bound is little more than that add's own half ulp, so err / B near 1 (0.94
    measured) is expected there.
  * DiffAugment forward: B = (1 + c (1 + s)) (max_k |x_k + b| + |M|), k = 10u: the brightness add, the channel mean
    (two adds and the rounded 1/3), and each of the five operations of ((v - m) s + m - M) c + M contributes at most
    u of its operands.  Backward: B = (1 + s + |1 - s|) (c max_k |dz_k| + (c + |1 - c|) mean |dz|), k = 10u, the
    same count over c dz + mterm and s dy + (1 - s) mean_k dy.  The reference is fp64 autograd of the forward
    written with the sample mean taken over y, not the kernel's algebra.
  * adaptive_weight: one fp32 rounding of the fp64 value, 2u |ref|.  axpy_dev: B = |a + w b| + |w b|, k = u, one
    rounding with an fma, two without.  bn_update_running: B = (1 - m) |r| + m |batch stat|, k = 3u.
  * u8_to_planes: torch fp32 x / 127.5 - 1 bit for bit; pack_u8: torchvision's mul(255).add_(0.5).clamp_(0, 255)
    .to(uint8) in fp32 bit for bit.
  * argmax_heads: the lowest index of the maximum over the non-NaN values (the kernel skips NaN; torch.argmax would
    return the first NaN); rows with no such value, all -inf or all NaN, give 0, heads outside [0, G) give -1.
  * mask_to_ids: floor(dst fp32(in / out)) in fp32, clamped to the source, which is torch's nearest rule
    (F.interpolate mode="nearest").  It differs from the exact floor(dst in / out) at many enlarging ratios
    (for example in 2, out 82, dst 41: fp32 gives 0, exact gives 1); the test counts and prints those positions.
  * lrelu_bwd reads the slope from y's hi plane: 0 < y <= 2^-25 rounds to an fp16 0 and gets slope 0.2 where
    autograd uses 1.  Planes alone cannot tell those y from 0, the effect is 0.8 |dy| on values below 2^-25, and the
    test pins this rule on both sides of 2^-25.
  * quantizer: bit for bit against oracle/vq_oracle.c; a row with a NaN gets index 0 (the oracle used to return the
    kernel's sentinel there and index the codebook with it).
"""
import collections
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from text2human_b200 import _lib

SENTINEL = -7777.0
H16 = float(torch.tensor(SENTINEL).half())  # the sentinel as an fp16 plane holds it
U = 2.0 ** -24
EINVAL = -1
H100_SMS = 132
PLANE_R = {2: 2.0 ** -23, 1: 2.0 ** -11}  # the planes' own rounding, relative ...
PLANE_A = 2.0 ** -25                      # ... and absolute
K_BIL = 4 * U * (1 + 2.0 ** -20)
K_GN = 5 * U
K_BCE_LOSS, K_BCE_G, K_SUM = 1e-6, 8 * U, 1e-6
K_VQ_DZ = 3 * U
K_DA = 10 * U
CVT_PLAIN, CVT_UP2X, CVT_S2D, CVT_MAXPOOL2, CVT_BILINEAR2X = (_lib.CVT_PLAIN, _lib.CVT_UP2X, _lib.CVT_S2D,
                                                               _lib.CVT_MAXPOOL2, _lib.CVT_BILINEAR2X)
MODE_NAMES = {CVT_PLAIN: "plain", CVT_UP2X: "up2x", CVT_S2D: "s2d", CVT_MAXPOOL2: "maxpool2",
              CVT_BILINEAR2X: "bilinear2x"}


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------ the launch rules, restated
def grid_route(work, block=256, per_sm=16):
    """grid_cap (gan.cu) and grid_for (elementwise.cu): one thread per work item up to per_sm blocks per SM, then
    grid-stride sweeps"""
    grid = min(max(_cdiv(work, block), 1), H100_SMS * per_sm)
    return dict(grid=grid, sweeps=_cdiv(work, grid * block))


def f32_to_planes_route(mode, n, h, w, c):
    """t2h_f32_to_planes: one thread per 8 output channels, grid_for over them"""
    out = n * h * w * c
    if mode in (CVT_UP2X, CVT_BILINEAR2X):
        out *= 4
    if mode == CVT_MAXPOOL2:
        out = n * (h // 2) * (w // 2) * c
    return grid_route(out // 8)


def gn_apply_route(n, hw, c):
    """t2h_gn_apply: ceil(8 SMs / n) blocks per image, at least 16 pixels each, 256 threads over ppb * C / 8 items"""
    blocks = _cdiv(H100_SMS * 8, n)
    ppb = max(_cdiv(hw, blocks), 16)
    return dict(ppb=ppb, blocks=_cdiv(hw, ppb), partial=hw % ppb != 0, sweeps=_cdiv(ppb * (c // 8), 256))


def bce_route(c_pad, npix):
    """t2h_bce_logits: c8 = c_pad / 8 threads per pixel; block 32 c8 (8 / c8) below c8 = 8, else 32 c8; grid_cap
    at 4 blocks per SM over the pixels"""
    c8 = c_pad // 8
    block = 32 * c8 * (8 // c8 if c8 < 8 else 1)
    lanes = block // c8
    return dict(branch="c8<8" if c8 < 8 else "c8>=8", block=block, lanes=lanes,
                **grid_route(npix, lanes, per_sm=4))


def loss_route(n):
    """t2h_l1_loss and t2h_hinge_loss: grid_cap at 4 blocks per SM"""
    return grid_route(n, 256, per_sm=4)


def diffaug_route(h, w):
    """t2h_diffaug_fwd / _bwd: the per-sample sum over 3 h w values on at most 64 blocks, the apply (and the
    backward's sum) over h w pixels on at most 128, both from grid_cap at 2 blocks per SM"""
    gx = min(grid_route(3 * h * w, 256, 2)["grid"], 64)
    gy = min(grid_route(h * w, 256, 2)["grid"], 128)
    return dict(gx=gx, gy=gy, sum_sweeps=_cdiv(3 * h * w, gx * 256), apply_sweeps=_cdiv(h * w, gy * 256))


def adaptive_weight_route(n):
    """t2h_adaptive_weight: one block of 1024 threads"""
    return _cdiv(n, 1024)


def add_inplace_route(numel):
    """t2h_add_inplace: float4 items on grid_for, the numel % 4 tail on block 0"""
    n4 = numel // 4
    return dict(tail=numel % 4, **grid_route(max(n4, 1)))


def vq_bin_route(book_ids, n_books):
    """vq_bin_kernel: one block of 1024 threads bins every row; 32-row tiles per bin, ids outside [0, n_books) in
    the unselected bin n_books"""
    ids = np.where((book_ids >= 0) & (book_ids < n_books), book_ids, n_books)
    cnt = np.bincount(ids.ravel(), minlength=n_books + 1)
    return dict(bin_sweeps=_cdiv(ids.size, 1024), counts=cnt, partial_multi=any(c > 32 and c % 32 for c in cnt))


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
    the r |ref| + a allowance"""
    got, ref = got.double(), ref.double()
    B = torch.as_tensor(B, dtype=torch.float64, device=ref.device).expand_as(ref)
    r = torch.as_tensor(r, dtype=torch.float64, device=ref.device)
    err = (got - ref).abs()
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


def _untouched(buf, numel, what, fill=SENTINEL):
    assert (buf[numel:] == fill).all(), f"{what}: writes past the output"


def _split_of(hi, lo, v, what):
    """planes == split(v) bit for bit; lo may be None (one plane)"""
    h = v.half()
    assert torch.equal(hi, h), f"{what}: hi plane is not fp16_rn(v) at {int((hi != h).sum())} elements"
    if lo is not None:
        lv = (v - h.float()).half()
        assert torch.equal(lo, lv), f"{what}: lo plane is not fp16_rn(v - hi) at {int((lo != lv).sum())} elements"


def _planes_of(out, T, *shape):
    pl = out.view(T, *shape)
    return pl[0], (pl[1] if T == 2 else None)


def _pval(hi, lo):
    return hi.double() + (lo.double() if lo is not None else 0)


def _varied(shape, g, spread=2.0):
    """normal values whose magnitudes spread over several binades, so that lo planes are non-trivial"""
    return torch.randn(*shape, generator=g) * torch.exp(spread * torch.randn(*shape, generator=g))


# ------------------------------------------------------------------ section 1: transposes and plane producers
NP = collections.namedtuple("NP", "N C H W c_pad terms")
NP_CASES = [NP(2, 3, 9, 5, 8, 2), NP(1, 8, 7, 11, 16, 1), NP(2, 37, 9, 5, 40, 2), NP(1, 64, 33, 3, 64, 1),
            NP(1, 64, 5, 13, 72, 2), NP(1, 513, 6, 7, 520, 2)]


def test_transpose_case_table():
    assert {c.C for c in NP_CASES} >= {3, 8, 37, 64, 513} and {c.terms for c in NP_CASES} == {1, 2}
    assert all((c.H * c.W) % 32 for c in NP_CASES) and sum(c.c_pad > c.C for c in NP_CASES) >= 4


@pytest.mark.gpu
@pytest.mark.parametrize("c", NP_CASES, ids=lambda c: f"N{c.N}-C{c.C}-{c.H}x{c.W}-pad{c.c_pad}-t{c.terms}")
def test_nchw_transposes_and_planes_bit_exact(cuda, c):
    dev, N, C, HW, P, T = cuda, c.N, c.C, c.H * c.W, c.c_pad, c.terms
    g = torch.Generator().manual_seed(C * 31 + HW)
    x = _varied((N, C, c.H, c.W), g).to(dev)
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    what = f"nchw_to_planes {c}"
    buf, out = _guarded(T * N * HW * P, torch.float16, dev)
    _ok(_lib.load().t2h_nchw_to_planes(_p(x), _p(out), N, C, c.H, c.W, P, T, _st()))
    b1, o1 = _guarded(N * HW * C, torch.float32, dev)
    _ok(_lib.load().t2h_nchw_to_nhwc(_p(x), _p(o1), N, C, c.H, c.W, _st()))
    b2, o2 = _guarded(N * HW * C, torch.float32, dev)
    _ok(_lib.load().t2h_nhwc_to_nchw(_p(nhwc), _p(o2), N, C, c.H, c.W, _st()))
    torch.cuda.synchronize()
    _untouched(buf, T * N * HW * P, what, H16)
    _untouched(b1, N * HW * C, "nchw_to_nhwc")
    _untouched(b2, N * HW * C, "nhwc_to_nchw")
    hi, lo = _planes_of(out, T, N, HW, P)
    _split_of(hi[..., :C], None if lo is None else lo[..., :C], nhwc.view(N, HW, C), what)
    assert (hi[..., C:] == 0).all() and (lo is None or (lo[..., C:] == 0).all()), f"{what}: pad channels not 0"
    assert torch.equal(o1.view(N, c.H, c.W, C), nhwc), "nchw_to_nhwc is not the permutation"
    assert torch.equal(o2.view(N, C, c.H, c.W), x), "nhwc_to_nchw is not the permutation"


F2P = collections.namedtuple("F2P", "mode N H W C terms")
F2P_CASES = [F2P(CVT_PLAIN, 2, 256, 128, 128, 2), F2P(CVT_PLAIN, 1, 3, 5, 8, 1),
             F2P(CVT_UP2X, 2, 128, 64, 128, 2), F2P(CVT_UP2X, 1, 3, 5, 16, 1),
             F2P(CVT_S2D, 2, 256, 128, 128, 1), F2P(CVT_S2D, 1, 4, 6, 8, 2),
             F2P(CVT_MAXPOOL2, 2, 513, 257, 128, 2), F2P(CVT_MAXPOOL2, 1, 2, 2, 8, 1), F2P(CVT_MAXPOOL2, 3, 5, 7, 16, 2),
             F2P(CVT_BILINEAR2X, 2, 128, 64, 128, 2), F2P(CVT_BILINEAR2X, 1, 1, 6, 8, 1),
             F2P(CVT_BILINEAR2X, 2, 5, 1, 16, 2), F2P(CVT_BILINEAR2X, 1, 3, 4, 24, 1)]


def _f2p_id(c):
    return f"{MODE_NAMES[c.mode]}-N{c.N}-{c.H}x{c.W}-C{c.C}-t{c.terms}"


def test_f32_to_planes_case_table_covers_every_route():
    """every mode with one sweep and with several, both plane counts, odd and 2x2 max-pool inputs, bilinear with a
    single row or column"""
    for mode in MODE_NAMES:
        sw = {f32_to_planes_route(c.mode, c.N, c.H, c.W, c.C)["sweeps"] > 1 for c in F2P_CASES if c.mode == mode}
        assert sw == {True, False}, MODE_NAMES[mode]
    assert {(c.mode, c.terms) for c in F2P_CASES} == {(m, t) for m in MODE_NAMES for t in (1, 2)}
    mp = [c for c in F2P_CASES if c.mode == CVT_MAXPOOL2]
    assert any(c.H % 2 and c.W % 2 for c in mp) and any(c.H == c.W == 2 for c in mp)
    assert any(c.H == 1 for c in F2P_CASES if c.mode == CVT_BILINEAR2X)
    assert any(c.W == 1 for c in F2P_CASES if c.mode == CVT_BILINEAR2X)


def _f2p_ref(mode, x):
    """the fp32 values a mode writes (NHWC), or for BILINEAR2X the fp64 value and its bound"""
    N, H, W, C = x.shape
    if mode == CVT_PLAIN:
        return x
    if mode == CVT_UP2X:
        return x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    if mode == CVT_S2D:
        return torch.stack([x[:, a::2, b::2] for a, b in ((0, 0), (0, 1), (1, 0), (1, 1))])
    if mode == CVT_MAXPOOL2:
        return x[:, :H // 2 * 2, :W // 2 * 2].reshape(N, H // 2, 2, W // 2, 2, C).amax((2, 4))

    def up(t):
        return F.interpolate(t.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                             align_corners=False).permute(0, 2, 3, 1)
    xd = x.double()
    return up(xd), up(xd.abs())


@pytest.mark.gpu
@pytest.mark.parametrize("c", F2P_CASES, ids=_f2p_id)
def test_f32_to_planes_every_mode(cuda, c):
    dev, T = cuda, c.terms
    g = torch.Generator().manual_seed(c.mode * 101 + c.H * 7 + c.W)
    x = _varied((c.N, c.H, c.W, c.C), g).to(dev)
    r = f32_to_planes_route(c.mode, c.N, c.H, c.W, c.C)
    what = f"f32_to_planes {_f2p_id(c)} sweeps {r['sweeps']}"
    ref = _f2p_ref(c.mode, x)
    numel = (ref[0] if c.mode == CVT_BILINEAR2X else ref).numel()
    buf, out = _guarded(T * numel, torch.float16, dev)
    _ok(_lib.load().t2h_f32_to_planes(_p(x), _p(out), c.N, c.H, c.W, c.C, c.mode, T, _st()))
    torch.cuda.synchronize()
    _untouched(buf, T * numel, what, H16)
    hi, lo = _planes_of(out, T, numel)
    if c.mode != CVT_BILINEAR2X:
        _split_of(hi, lo, ref.reshape(-1), what)
        return
    val, B = (t.reshape(-1) for t in ref)
    _check(_pval(hi, lo), val, B, what, K_BIL, PLANE_R[T], PLANE_A)


GA = collections.namedtuple("GA", "N H W C G swish terms")
GA_CASES = [GA(2, 7, 9, 64, 32, 1, 2), GA(1, 13, 11, 128, 32, 0, 1), GA(2, 5, 19, 192, 32, 1, 1),
            GA(1, 256, 128, 128, 32, 1, 2), GA(1, 31, 17, 192, 32, 0, 2), GA(3, 9, 7, 64, 64, 2, 1),
            GA(2, 11, 13, 512, 512, 2, 2), GA(1, 64, 33, 64, 64, 2, 2)]
GN_EPS = {True: 1e-5, False: 1e-6}  # BatchNorm (groups = C), GroupNorm


def _ga_id(c):
    return f"N{c.N}-{c.H}x{c.W}-C{c.C}-G{c.G}-swish{c.swish}-t{c.terms}"


def test_gn_apply_case_table_covers_every_route():
    rows = [(c, gn_apply_route(c.N, c.H * c.W, c.C)) for c in GA_CASES]
    assert {(c.swish, c.terms) for c in GA_CASES} == {(s, t) for s in (0, 1, 2) for t in (1, 2)}
    assert {c.C // c.G for c in GA_CASES if c.G < c.C} == {2, 4, 6}
    assert {c.C for c in GA_CASES if c.G == c.C} == {64, 512}
    assert any(r["partial"] for c, r in rows) and any(r["sweeps"] > 1 for c, r in rows)
    assert any(r["sweeps"] == 1 for c, r in rows)


@pytest.mark.gpu
@pytest.mark.parametrize("c", GA_CASES, ids=_ga_id)
def test_gn_apply_matches_fp64(cuda, c):
    """per-channel offsets (a channel normalised with another group's statistics moves its output), statistics
    given as the fp64 sums of the input"""
    dev, N, HW, C, G, T = cuda, c.N, c.H * c.W, c.C, c.G, c.terms
    g = torch.Generator().manual_seed(C * 3 + HW + c.swish)
    offset = torch.rand(C, generator=g) * 20 - 10
    x = torch.randn(N, HW, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + offset
    gamma = (0.5 + torch.rand(C, generator=g)) * torch.where(torch.rand(C, generator=g) < 0.3, -1.0, 1.0)
    beta = torch.randn(C, generator=g)
    xg = x.double().view(N, HW, G, C // G)
    stats = torch.stack((xg.sum((1, 3)), (xg * xg).sum((1, 3))), -1).contiguous()  # [N][G][2]
    eps = GN_EPS[G == C]
    buf, out = _guarded(T * N * HW * C, torch.float16, dev)
    xd, sd, gd, bd = x.to(dev), stats.to(dev), gamma.to(dev), beta.to(dev)
    _ok(_lib.load().t2h_gn_apply(_p(xd), _p(sd), _p(gd), _p(bd), _p(out), N, HW, C, G, eps, c.swish, T, _st()))
    torch.cuda.synchronize()
    r = gn_apply_route(N, HW, C)
    what = f"gn_apply {_ga_id(c)} ppb {r['ppb']} sweeps {r['sweeps']}"
    _untouched(buf, T * N * HW * C, what, H16)
    hi, lo = _planes_of(out.cpu(), T, N, HW, C)
    cnt = HW * (C // G)
    mean = (stats[..., 0] / cnt).repeat_interleave(C // G, 1)[:, None, :]
    var = (stats[..., 1] / cnt).repeat_interleave(C // G, 1)[:, None, :] - mean * mean
    rstd = 1.0 / torch.sqrt(var + _f32(eps))
    ga, be = gamma.double(), beta.double()
    y = (x.double() - mean) * rstd * ga + be
    B = ga.abs() * rstd * (x.double().abs() + mean.abs()) + be.abs() + y.abs()
    r_extra = torch.zeros_like(y)
    if c.swish == 1:
        sig = torch.sigmoid(y)
        ref = y * sig
        B = 1.1 * B
        r_extra = (2 + torch.floor(1.16 * y.abs())) * 2.0 ** -23 + 2 * U
    elif c.swish == 2:
        ref = torch.where(y > 0, y, _f32(0.2) * y)
        r_extra = torch.full_like(y, U)
    else:
        ref = y
    _check(_pval(hi, lo), ref, B, what, K_GN, PLANE_R[T] + r_extra, PLANE_A)


OH = collections.namedtuple("OH", "n_classes c_pad B H W terms")
OH_CASES = [OH(24, 24, 2, 16, 8, 2), OH(20, 24, 1, 5, 7, 1), OH(1, 8, 1, 3, 3, 2), OH(19, 24, 2, 512, 256, 2)]


def test_onehot_case_table():
    assert {c.c_pad == c.n_classes for c in OH_CASES} == {True, False}
    assert any(grid_route(c.B * c.H * c.W * c.c_pad // 8)["sweeps"] > 1 for c in OH_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("c", OH_CASES, ids=lambda c: f"n{c.n_classes}-pad{c.c_pad}-B{c.B}-{c.H}x{c.W}-t{c.terms}")
def test_onehot_to_planes_bit_exact(cuda, c):
    """integer ids in range, non-integer, negative and >= n_classes ids (all-zero rows); lo is exactly 0"""
    dev, T, P = cuda, c.terms, c.c_pad
    npix = c.B * c.H * c.W
    g = torch.Generator().manual_seed(npix + c.n_classes)
    ids = torch.randint(0, c.n_classes, (npix,), generator=g).float()
    edge = torch.tensor([0.0, c.n_classes - 1, 2.5, -1.0, -3.0, c.n_classes, c.n_classes + 7, 0.25, -0.0])
    ids[:len(edge)] = edge
    buf, out = _guarded(T * npix * P, torch.float16, dev)
    idd = ids.to(dev)
    _ok(_lib.load().t2h_onehot_to_planes(_p(idd), _p(out), c.B, c.H, c.W, c.n_classes, P, T, _st()))
    torch.cuda.synchronize()
    what = f"onehot_to_planes {c}"
    _untouched(buf, T * npix * P, what, H16)
    valid = (ids == ids.floor()) & (ids >= 0) & (ids < c.n_classes)
    want = torch.zeros(npix, P)
    want[valid.nonzero().flatten(), ids[valid].long()] = 1.0
    hi, lo = _planes_of(out.cpu(), T, npix, P)
    assert torch.equal(hi.float(), want), f"{what}: hi plane differs from the one-hot"
    assert (hi[~valid] == 0).all(), f"{what}: an id without a class has a non-zero row"
    if lo is not None:
        assert (lo == 0).all() and not torch.signbit(lo).any(), f"{what}: lo plane is not exactly 0"


@pytest.mark.gpu
@pytest.mark.parametrize("C,c_pad,terms,nchw", [(3, 8, 2, True), (8, 16, 1, False), (1, 8, 2, True)])
def test_u8_to_planes_every_byte(cuda, C, c_pad, terms, nchw):
    """all 256 byte values in every channel: x / 127.5 - 1 in fp32 bit for bit, NCHW output and planes"""
    dev, T = cuda, terms
    B, H, W = 2, 16, 16
    x = ((torch.arange(B * H * W)[:, None] * 7 + torch.arange(C) * 13) % 256).to(torch.uint8).view(B, H, W, C)
    for ch in range(C):
        assert len(torch.unique(x[..., ch])) == 256
    npix = B * H * W
    buf, out = _guarded(T * npix * c_pad, torch.float16, dev)
    nbuf, nout = _guarded(B * C * H * W, torch.float32, dev) if nchw else (None, None)
    xd = x.to(dev)
    _ok(_lib.load().t2h_u8_to_planes(_p(xd), _p(out), _p(nout), B, H, W, C, c_pad, 127.5, -1.0, T, _st()))
    torch.cuda.synchronize()
    what = f"u8_to_planes C{C} pad{c_pad} t{T}"
    _untouched(buf, T * npix * c_pad, what, H16)
    want = x.float().div(127.5).sub(1.0)
    npw = torch.from_numpy(x.numpy().astype(np.float32) / np.float32(127.5) - np.float32(1.0))
    assert torch.equal(want, npw), "torch and IEEE fp32 disagree on x / 127.5 - 1"
    if nchw:
        _untouched(nbuf, B * C * H * W, what)
        assert torch.equal(nout.view(B, C, H, W).cpu(), want.permute(0, 3, 1, 2)), f"{what}: NCHW output differs"
    hi, lo = _planes_of(out.cpu(), T, npix, c_pad)
    _split_of(hi[:, :C], None if lo is None else lo[:, :C], want.view(npix, C), what)
    assert (hi[:, C:] == 0).all() and (lo is None or (lo[:, C:] == 0).all()), f"{what}: pad channels not 0"


def _pack_values():
    """every k/255 rounding boundary (m - 0.5) / 255 in fp32 with its two neighbours on each side, and values
    below 0, above 1 and +-inf"""
    b = np.float32((np.arange(1, 256) - 0.5) / 255)
    vals = [b]
    for s in (1, 2):
        vals.append(np.nextafter(b, np.float32(np.inf) if s == 1 else np.float32(-np.inf)))
    vals.append(np.nextafter(vals[1], np.float32(np.inf)))
    vals.append(np.nextafter(vals[2], np.float32(-np.inf)))
    extra = np.array([0, 1, -0.0, -1e-30, -0.3, 1.0000001, 1.7, 255, np.inf, -np.inf, 1e30], np.float32)
    return torch.from_numpy(np.concatenate(vals + [extra]).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 4])
def test_pack_u8_matches_torchvision(cuda, C):
    dev = cuda
    v = _pack_values()
    N, H = 2, 7
    W = _cdiv(v.numel(), N * C * H)
    x = v.repeat(_cdiv(N * C * H * W, v.numel()))[:N * C * H * W]
    x = x[torch.randperm(x.numel(), generator=torch.Generator().manual_seed(C))].view(N, C, H, W)
    xd = x.to(dev)
    buf, out = _guarded(N * H * W * C, torch.uint8, dev, fill=77)
    _ok(_lib.load().t2h_pack_u8(_p(xd), _p(out), N, C, H, W, 1.0, 0.0, _st()))
    torch.cuda.synchronize()
    _untouched(buf, N * H * W * C, f"pack_u8 C{C}", 77)
    want = x.mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    got = out.view(N, H, W, C).cpu()
    assert torch.equal(got, want), f"pack_u8 C{C}: {int((got != want).sum())} bytes differ from torchvision's"


AM = collections.namedtuple("AM", "G M ncls")
AM_CASES = [AM(3, 40, 1), AM(18, 37, 31), AM(2, 50, 33), AM(18, 45, 100), AM(1, 33, 257)]


def test_argmax_case_table():
    assert any(c.ncls % 32 for c in AM_CASES) and any(c.ncls > 64 for c in AM_CASES) and min(c.ncls for c in
                                                                                           AM_CASES) == 1
    assert all(c.M >= 8 for c in AM_CASES) and all(c.M % 8 for c in AM_CASES if c.M > 40)


@pytest.mark.gpu
@pytest.mark.parametrize("c", AM_CASES, ids=lambda c: f"G{c.G}-M{c.M}-ncls{c.ncls}")
def test_argmax_heads_rule(cuda, c):
    """row 0: a three-way tie at the maximum, row 1: all -inf, rows 2 / 3: head -1 / G, row 4: a NaN ahead of the
    maximum, row 5: all NaN, row 6: NaN and -inf around one finite value, row 7: a -0 / +0 tie"""
    dev, G, M, ncls = cuda, c.G, c.M, c.ncls
    g = torch.Generator().manual_seed(G * 7 + ncls)
    logits = torch.randn(G, M, ncls, generator=g) * 3
    head = torch.randint(0, G, (M,), generator=g)
    head[2], head[3] = -1, G
    h = head.tolist()
    tied = sorted({0, ncls // 2, ncls - 1})
    logits[h[0], 0, tied] = logits[h[0], 0].max() + 1
    logits[h[1], 1] = -math.inf
    mx = ncls - 1 if ncls > 1 else 0
    logits[h[4], 4, mx] = logits[h[4], 4].max() + 5
    logits[h[4], 4, 0] = math.nan
    logits[h[5], 5] = math.nan
    logits[h[6], 6] = torch.where(torch.arange(ncls) % 2 == 0, -math.inf, math.nan)
    logits[h[6], 6, ncls - 1] = -50.0
    logits[h[7], 7] = -1.0
    logits[h[7], 7, ncls - 1] = -0.0
    logits[h[7], 7, ncls // 3] = 0.0
    buf, out = _guarded(M, torch.int64, dev, fill=-7777)
    ld, hd = logits.to(dev), head.to(dev)
    _ok(_lib.load().t2h_argmax_heads(_p(ld), _p(hd), _p(out), M, G, ncls, _st()))
    torch.cuda.synchronize()
    _untouched(buf, M, f"argmax_heads {c}", -7777)
    want = torch.full((M,), -1, dtype=torch.int64)
    for m in range(M):
        if 0 <= head[m] < G:
            row = logits[head[m], m]
            want[m] = torch.where(torch.isnan(row), -math.inf, row).argmax()  # first index of the maximum
    got = out.cpu()
    assert got[0] == tied[0] and got[1] == 0 and got[2] == -1 and got[3] == -1 and got[5] == 0
    assert got[4] == mx and got[6] == ncls - 1
    assert torch.equal(got, want), f"argmax_heads {c}: rows {(got != want).nonzero().flatten().tolist()} differ"


MI = collections.namedtuple("MI", "B Hs Ws Ht Wt")
MI_CASES = [MI(2, 512, 256, 32, 16), MI(1, 2, 2, 82, 94), MI(2, 512, 256, 37, 23), MI(1, 3, 7, 300, 211),
            MI(3, 100, 60, 64, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", MI_CASES, ids=lambda c: f"B{c.B}-{c.Hs}x{c.Ws}-to-{c.Ht}x{c.Wt}")
def test_mask_to_ids_nearest_rule(cuda, c):
    """the fp32 nearest rule (torch's), against F.interpolate and the fp64 floor; id values: integers, -1, -2,
    non-integers, 999999 and 1e6"""
    dev = cuda
    g = torch.Generator().manual_seed(c.Hs + c.Ht)
    mask = torch.randint(0, 24, (c.B, 1, c.Hs, c.Ws), generator=g).float()
    edge = torch.tensor([-1.0, -2.0, 2.5, 999999.0, 1e6, 0.5, 23.0, -0.0])
    flat = mask.view(-1)
    pos = torch.randperm(flat.numel(), generator=g)[:min(flat.numel(), 64)]
    flat[pos] = edge.repeat(8)[:len(pos)]
    md = mask.to(dev)
    buf, out = _guarded(c.B * c.Ht * c.Wt, torch.int32, dev, fill=-7777)
    _ok(_lib.load().t2h_mask_to_ids(_p(md), _p(out), c.B, c.Hs, c.Ws, c.Ht, c.Wt, _st()))
    torch.cuda.synchronize()
    _untouched(buf, c.B * c.Ht * c.Wt, "mask_to_ids", -7777)

    def src(n_in, n_out, exact):
        d = np.arange(n_out)
        if exact:
            s = (d * n_in) // n_out
        else:
            s = np.floor(d.astype(np.float32) * (np.float32(n_in) / np.float32(n_out))).astype(np.int64)
        return np.minimum(s, n_in - 1)
    sy, sx = src(c.Hs, c.Ht, False), src(c.Ws, c.Wt, False)
    v = mask[:, 0][:, sy][:, :, sx]
    ok = (v == v.floor()) & (v >= -1) & (v < 1e6)
    want = torch.where(ok, v, torch.full_like(v, -1)).to(torch.int32)
    got = out.view(c.B, c.Ht, c.Wt).cpu()
    assert torch.equal(got, want), f"mask_to_ids {c}: {int((got != want).sum())} ids differ from the fp32 rule"
    torch_ids = F.interpolate(mask, size=(c.Ht, c.Wt), mode="nearest")[:, 0]
    assert torch.equal(torch.where(ok, torch_ids, torch.full_like(torch_ids, -1)).to(torch.int32), want)
    ey, ex = src(c.Hs, c.Ht, True), src(c.Ws, c.Wt, True)
    print(f"mask_to_ids {c}: fp32 rule differs from the exact floor at {int((ey != sy).sum())} of {c.Ht} rows and "
          f"{int((ex != sx).sum())} of {c.Wt} columns")


@pytest.mark.gpu
@pytest.mark.parametrize("numel", [4, 5, 4099, 4096 * 7 + 1, 2 * H100_SMS * 16 * 256 * 4 + 4 * 1001 + 3,
                                   H100_SMS * 16 * 256 * 4 + 20001])
def test_add_inplace_bit_exact(cuda, numel):
    dev = cuda
    r = add_inplace_route(numel)
    g = torch.Generator(device=dev).manual_seed(numel % 1000)
    a0 = torch.randn(numel, device=dev, generator=g)
    b = torch.randn(numel, device=dev, generator=g) * 3
    buf, x = _guarded(numel, torch.float32, dev)
    x.copy_(a0)
    _ok(_lib.load().t2h_add_inplace(_p(x), _p(b), numel, _st()))
    torch.cuda.synchronize()
    _untouched(buf, numel, f"add_inplace {numel}")
    assert torch.equal(x, a0 + b), f"add_inplace numel {numel} (tail {r['tail']}, sweeps {r['sweeps']})"


def test_add_inplace_sizes_cover_every_route():
    sizes = [4, 5, 4099, 4096 * 7 + 1, 2 * H100_SMS * 16 * 256 * 4 + 4 * 1001 + 3, H100_SMS * 16 * 256 * 4 + 20001]
    rows = [add_inplace_route(n) for n in sizes]
    assert {r["tail"] for r in rows} >= {0, 1, 3} and any(r["sweeps"] > 1 and r["tail"] for r in rows)


# ------------------------------------------------------------------ section 2: the GAN step's kernels
LOSS_SIZES = [1, 257, 135169, 16 * 3 * 512 * 256]


def test_loss_sizes_cover_every_route():
    assert {loss_route(n)["sweeps"] > 1 for n in LOSS_SIZES} == {True, False}
    assert any(loss_route(n)["sweeps"] == 2 for n in LOSS_SIZES)


@pytest.mark.gpu
@pytest.mark.parametrize("with_grad", [True, False])
@pytest.mark.parametrize("n", LOSS_SIZES)
def test_l1_loss_matches_fp64(cuda, n, with_grad):
    """equal pairs (d = +0) and a +0 / -0 pair (d = -0) give gradient 0; the sum adds onto a start value"""
    dev = cuda
    g = torch.Generator(device=dev).manual_seed(n)
    x = torch.randn(n, device=dev, generator=g)
    xr = x + torch.randn(n, device=dev, generator=g) * 0.3
    xr[::7] = x[::7]
    if n > 3:
        x[1], xr[1] = 0.0, -0.0
    gs = 1.0 / n
    sbuf = torch.tensor([0.75, SENTINEL], dtype=torch.float64, device=dev)
    gbuf, grad = _guarded(n, torch.float32, dev) if with_grad else (None, None)
    _ok(_lib.load().t2h_l1_loss(_p(x), _p(xr), _p(grad), _p(sbuf), n, gs, _st()))
    torch.cuda.synchronize()
    r = loss_route(n)
    what = f"l1_loss n {n} sweeps {r['sweeps']}"
    assert sbuf[1] == SENTINEL, f"{what}: writes past the sum"
    term = (xr.double() - x.double()).abs()
    _check(sbuf[:1] - 0.75, term.sum()[None], term.sum()[None], f"{what} sum", U + n * 2.0 ** -53)
    if with_grad:
        _untouched(gbuf, n, what)
        want = torch.sign(xr - x) * np.float32(gs)
        assert torch.equal(grad, want), f"{what}: gradient differs from gscale sign(xrec - x)"
        assert (grad[::7] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("sgn", [1.0, -1.0, 0.0])
@pytest.mark.parametrize("n", LOSS_SIZES)
def test_hinge_loss_matches_fp64(cuda, n, sgn):
    """logits exactly at the margin (l = sgn) give term 0 and gradient 0; a NULL gradient on the largest size"""
    dev = cuda
    g = torch.Generator(device=dev).manual_seed(n + 3)
    l = torch.randn(n, device=dev, generator=g) * 2
    if sgn:
        l[::5] = sgn
    gs = 0.5 / n
    with_grad = n != LOSS_SIZES[-1] or sgn != 1.0
    sbuf = torch.tensor([-1.5, SENTINEL], dtype=torch.float64, device=dev)
    gbuf, grad = _guarded(n, torch.float32, dev) if with_grad else (None, None)
    _ok(_lib.load().t2h_hinge_loss(_p(l), _p(grad), _p(sbuf), n, sgn, gs, _st()))
    torch.cuda.synchronize()
    what = f"hinge_loss n {n} sgn {sgn:g} sweeps {loss_route(n)['sweeps']}"
    assert sbuf[1] == SENTINEL, f"{what}: writes past the sum"
    ld = l.double()
    term = ld if sgn == 0 else (1 - sgn * ld).clamp_min(0)
    _check(sbuf[:1] + 1.5, term.sum()[None], term.abs().sum()[None], f"{what} sum", U + n * 2.0 ** -53)
    if with_grad:
        _untouched(gbuf, n, what)
        gsf = np.float32(gs)
        if sgn == 0:
            want = torch.full_like(l, float(gsf))
        else:
            want = torch.where(1.0 - sgn * l > 0, torch.full_like(l, float(-sgn * gsf)), torch.zeros_like(l))
            assert (grad[::5] == 0).all(), f"{what}: a logit at the margin has a gradient"
        assert torch.equal(grad, want), f"{what}: gradient differs"


BC = collections.namedtuple("BC", "c_pad C n h w terms gscale")
BC_CASES = [BC(8, 8, 2, 9, 7, 2, None), BC(8, 4, 1, 5, 13, 1, None), BC(24, 24, 2, 16, 8, 2, None),
            BC(24, 20, 2, 160, 128, 2, None), BC(40, 40, 1, 9, 11, 1, None), BC(40, 36, 1, 9, 11, 0, None),
            BC(64, 64, 1, 7, 9, 1, None), BC(64, 60, 2, 3, 5, 2, None), BC(72, 72, 1, 5, 5, 0, None),
            BC(72, 68, 2, 5, 5, 2, None), BC(256, 256, 1, 4, 6, 2, None), BC(256, 252, 1, 3, 3, 0, None),
            BC(24, 24, 1, 8, 8, 2, 2.0 ** 14)]


def _bc_id(c):
    return f"pad{c.c_pad}-C{c.C}-{c.n}x{c.h}x{c.w}-t{c.terms}{'-g2^14' if c.gscale else ''}"


def test_bce_case_table_covers_every_route():
    rows = [(c, bce_route(c.c_pad, c.n * c.h * c.w)) for c in BC_CASES]
    assert {r["branch"] for c, r in rows} == {"c8<8", "c8>=8"}
    assert {(c.c_pad, c.c_pad - c.C) for c in BC_CASES} == {(p, d) for p in (8, 24, 40, 64, 72, 256) for d in (0, 4)}
    assert {c.terms for c in BC_CASES} == {0, 1, 2}
    assert any(r["sweeps"] > 1 for c, r in rows)
    assert {r["block"] for c, r in rows} >= {256, 192, 160, 288, 1024}


@pytest.mark.gpu
@pytest.mark.parametrize("c", BC_CASES, ids=_bc_id)
def test_bce_logits_matches_fp64(cuda, c):
    """logits up to +-100 (and 17..30 on targets), ids non-integer / negative / >= C (no target), the loss and the
    column sums accumulating onto start values; terms 0 passes NULL planes"""
    dev, C, P, T = cuda, c.C, c.c_pad, c.terms
    npix = c.n * c.h * c.w
    g = torch.Generator().manual_seed(P * 13 + C + npix)
    x = torch.randn(npix, C, generator=g) * 4
    ids = torch.randint(0, C, (npix,), generator=g).float()
    ids[:6] = torch.tensor([2.5, -1.0, float(C), float(C + 3), float(P - 1), 0.0])
    big = torch.rand(npix, C, generator=g) < 0.05
    x[big] = (torch.rand(int(big.sum()), generator=g) * 2 - 1) * 100
    tgt = (ids == ids.floor()) & (ids >= 0) & (ids < C)
    tp = tgt.nonzero().flatten()
    x[tp, ids[tp].long()] = torch.where(torch.arange(len(tp)) % 3 == 0, 17 + 13 * torch.rand(len(tp), generator=g),
                                        x[tp, ids[tp].long()])
    gs = c.gscale if c.gscale else 1.0 / (npix * C)
    lbuf = torch.tensor([2.25, SENTINEL], dtype=torch.float64, device=dev)
    start = torch.linspace(-1, 1, C)
    cbuf, cs = _guarded(C, torch.float32, dev)
    cs.copy_(start)
    pbuf, planes = _guarded(max(T, 1) * npix * P, torch.float16, dev) if T else (None, None)
    xd, idd = x.to(dev), ids.to(dev)
    _ok(_lib.load().t2h_bce_logits(_p(xd), _p(idd), c.n, c.h, c.w, C, P, gs, _p(lbuf), _p(planes), T, _p(cs), _st()))
    torch.cuda.synchronize()
    r = bce_route(P, npix)
    what = f"bce_logits {_bc_id(c)} block {r['block']} sweeps {r['sweeps']}"
    assert lbuf[1] == SENTINEL, f"{what}: writes past the loss"
    _untouched(cbuf, C, what)
    xd64 = x.double()
    t = torch.zeros(npix, C, dtype=torch.float64)
    t[tp, ids[tp].long()] = 1.0
    sp = torch.nn.functional.softplus(-xd64.abs())
    term = xd64.clamp_min(0) - xd64 * t + sp
    Bl = xd64.clamp_min(0) + xd64.abs() * t + sp
    w1 = _check(lbuf[:1].cpu() - 2.25, term.sum()[None], Bl.sum()[None], f"{what} loss", K_BCE_LOSS)
    gref = _f32(gs) * (torch.sigmoid(xd64) - t)
    gsum = gref.abs().sum(0)
    w2 = _check(cs.cpu(), start.double() + gref.sum(0), K_SUM * gsum + r["grid"] * U * (gsum + start.double().abs()),
                f"{what} colsum", 1.0)
    if T:
        _untouched(pbuf, T * npix * P, what, H16)
        hi, lo = _planes_of(planes.cpu(), T, npix, P)
        assert (hi[:, C:] == 0).all() and (lo is None or (lo[:, C:] == 0).all()), f"{what}: pad channels not 0"
        w3 = _check(_pval(hi[:, :C], None if lo is None else lo[:, :C]), gref, gref.abs(), f"{what} gradient",
                    K_BCE_G, PLANE_R[T], PLANE_A)
        sat = (t > 0) & (xd64 > 17) & (gref.abs() > 2.0 ** -20)
        if sat.any():
            got = _pval(hi[:, :C], None if lo is None else lo[:, :C])[sat]
            rel = ((got - gref[sat]).abs() / gref[sat].abs()).max().item()
            print(f"{what}: {int(sat.sum())} saturated targets, worst relative gradient error {rel:.3g}")
            assert (got < 0).all(), f"{what}: a saturated target's gradient is not -gscale sigmoid(-x)"
        w1 = max(w1, w3)
    print(f"{what}: worst err/B {max(w1, w2):.3g}")


VB = collections.namedtuple("VB", "rows D n_books n_e book dzq")
VB_CASES = [VB(300, 4, 3, 5, True, True), VB(2000, 36, 2, 3, True, False), VB(129, 256, 1, 16, False, True),
            VB(64, 36, 18, 7, True, True), VB(700, 256, 1, 2, False, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", VB_CASES, ids=lambda c: f"r{c.rows}-D{c.D}-b{c.n_books}-e{c.n_e}"
                         f"{'-book' if c.book else '-nobook'}{'-dzq' if c.dzq else ''}")
def test_vq_bwd_matches_fp64(cuda, c):
    """rows with book or idx out of range (e = 0, no codebook update), many rows on few codes (contended fp32
    atomics), book_id NULL (the segmentation tokenizer), dzq NULL"""
    dev, rows, D, nb, ne = cuda, c.rows, c.D, c.n_books, c.n_e
    g = torch.Generator().manual_seed(rows + D * 3 + ne)
    cb = torch.randn(nb, ne, D, generator=g)
    idx = torch.randint(0, ne, (rows,), generator=g)
    book = torch.randint(0, nb, (rows,), generator=g, dtype=torch.int32) if c.book else None
    idx[:3] = torch.tensor([-1, ne, 10 ** 9])
    if book is not None:
        book[3:6] = torch.tensor([-1, nb, 1000], dtype=torch.int32)
    sel = (idx >= 0) & (idx < ne)
    bk = book.long() if book is not None else torch.zeros(rows, dtype=torch.long)
    sel &= (bk >= 0) & (bk < nb)
    e = torch.zeros(rows, D)
    e[sel] = cb[bk[sel], idx[sel]]
    z = e + 0.3 * torch.randn(rows, D, generator=g)
    dzq = torch.randn(rows, D, generator=g) if c.dzq else None
    coef_z, coef_e = 2.5 / (rows * D), -1.75 / (rows * D)
    start = torch.randn(nb * ne * D, generator=g)
    dbuf, dz = _guarded(rows * D, torch.float32, dev)
    cbuf, dcb = _guarded(nb * ne * D, torch.float32, dev)
    dcb.copy_(start)
    zd, cbd, idd = z.to(dev), cb.to(dev), idx.to(dev)
    bd = book.to(dev) if book is not None else None
    dqd = dzq.to(dev) if dzq is not None else None
    _ok(_lib.load().t2h_vq_bwd(_p(zd), _p(cbd), _p(idd), _p(bd), _p(dqd), _p(dz), _p(dcb), rows, D, nb, ne, coef_z,
                               coef_e, _st()))
    torch.cuda.synchronize()
    what = f"vq_bwd {c}"
    _untouched(dbuf, rows * D, what)
    _untouched(cbuf, nb * ne * D, what)
    cz, ce = _f32(coef_z), _f32(coef_e)
    diff = z.double() - e.double()
    dq = dzq.double() if dzq is not None else torch.zeros(rows, D, dtype=torch.float64)
    w1 = _check(dz.view(rows, D).cpu(), dq + cz * diff, dq.abs() + abs(cz) * diff.abs(), f"{what} dz", K_VQ_DZ)
    code = bk * ne + idx
    ref = start.double().view(nb * ne, D).index_add(0, code[sel], -ce * diff[sel])
    tsum = torch.zeros(nb * ne, D, dtype=torch.float64).index_add(0, code[sel], abs(ce) * diff[sel].abs())
    m = torch.zeros(nb * ne, dtype=torch.float64).index_add(0, code[sel], torch.ones(int(sel.sum()),
                                                                                   dtype=torch.float64))
    B = K_SUM * tsum + m[:, None] * U * (tsum + start.double().abs().view(nb * ne, D))
    got = dcb.view(nb * ne, D).cpu()
    w2 = _check(got, ref, B, f"{what} dcodebook", 1.0)
    hit = torch.zeros(nb * ne, dtype=torch.bool)
    hit[code[sel]] = True
    assert torch.equal(got[~hit], start.view(nb * ne, D)[~hit]), f"{what}: a code no row selects changed"
    print(f"{what}: worst err/B {max(w1, w2):.3g}, {int(sel.sum())} of {rows} rows on {int(hit.sum())} codes")


def test_vq_bwd_case_table():
    assert {c.D for c in VB_CASES} >= {4, 36, 256} and {c.book for c in VB_CASES} == {True, False}
    assert {c.dzq for c in VB_CASES} == {True, False} and max(c.rows / (c.n_books * c.n_e) for c in VB_CASES) > 300


SP = collections.namedtuple("SP", "N H W C")
SP_CASES = [SP(1, 256, 128, 128), SP(2, 5, 3, 4), SP(1, 7, 9, 8)]  # H, W: the output (x is 2H x 2W)


def test_sumpool_case_table():
    assert any(grid_route(c.N * c.H * c.W * c.C // 4)["sweeps"] > 1 for c in SP_CASES)
    assert {4, 128} <= {c.C for c in SP_CASES}


@pytest.mark.gpu
@pytest.mark.parametrize("c", SP_CASES, ids=lambda c: f"N{c.N}-{c.H}x{c.W}-C{c.C}")
def test_sumpool2_bit_exact(cuda, c):
    """(a0 + a1) + (a2 + a3) over each 2x2 block, a0 a1 the top row"""
    dev = cuda
    g = torch.Generator(device=dev).manual_seed(c.H * c.C)
    x = torch.randn(c.N, 2 * c.H, 2 * c.W, c.C, device=dev, generator=g) * torch.exp(
        3 * torch.randn(c.N, 2 * c.H, 2 * c.W, c.C, device=dev, generator=g))
    n = c.N * c.H * c.W * c.C
    buf, out = _guarded(n, torch.float32, dev)
    _ok(_lib.load().t2h_sumpool2(_p(x), _p(out), c.N, c.H, c.W, c.C, _st()))
    torch.cuda.synchronize()
    what = f"sumpool2 {c} sweeps {grid_route(n // 4)['sweeps']}"
    _untouched(buf, n, what)
    want = (x[:, 0::2, 0::2] + x[:, 0::2, 1::2]) + (x[:, 1::2, 0::2] + x[:, 1::2, 1::2])
    assert torch.equal(out.view_as(want), want), f"{what}: differs from (a0 + a1) + (a2 + a3)"


S2 = collections.namedtuple("S2", "T N H W C")
S2_CASES = [S2(2, 2, 256, 128, 128), S2(1, 1, 6, 10, 8), S2(2, 3, 4, 2, 16)]


def test_planes_s2d_case_table():
    assert any(grid_route(c.T * c.N * c.H * c.W * c.C // 8)["sweeps"] > 1 for c in S2_CASES)
    assert 8 in {c.C for c in S2_CASES} and {c.T for c in S2_CASES} == {1, 2}


@pytest.mark.gpu
@pytest.mark.parametrize("c", S2_CASES, ids=lambda c: f"T{c.T}-N{c.N}-{c.H}x{c.W}-C{c.C}")
def test_planes_s2d_bit_exact(cuda, c):
    dev = cuda
    g = torch.Generator(device=dev).manual_seed(c.W * c.C)
    x = torch.randn(c.T, c.N, c.H, c.W, c.C, device=dev, generator=g).half()
    n = x.numel()
    buf, out = _guarded(n, torch.float16, dev)
    _ok(_lib.load().t2h_planes_s2d(_p(x), _p(out), c.T, c.N, c.H, c.W, c.C, _st()))
    torch.cuda.synchronize()
    _untouched(buf, n, f"planes_s2d {c}", H16)
    want = torch.stack([x[:, :, a::2, b::2] for a, b in ((0, 0), (0, 1), (1, 0), (1, 1))], 1)
    assert torch.equal(out.view_as(want), want), f"planes_s2d {c}: differs from the 4-phase space-to-depth"


LR = collections.namedtuple("LR", "n terms planes")
LR_CASES = [LR(1000, 2, True), LR(2 * H100_SMS * 16 * 256 + 5, 1, True), LR(1000, 2, False), LR(3001, 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", LR_CASES, ids=lambda c: f"n{c.n}-t{c.terms}{'' if c.planes else '-noplanes'}")
def test_lrelu_bwd_bit_exact(cuda, c):
    """dpre = dy (hi(y) > 0 ? 1 : fp32(0.2)); y's planes hold split(y), and y includes values on both sides of 2^-25,
    where hi rounds to 0 (slope 0.2) or to 2^-24 (slope 1)"""
    dev, n, T = cuda, c.n, c.terms
    g = torch.Generator(device=dev).manual_seed(n)
    y = torch.randn(n, device=dev, generator=g)
    edge = torch.tensor([2.0 ** -25, 1e-9, 2.0 ** -25 * (1 + 2.0 ** -20), 2.0 ** -24, 0.0, -0.0, -2.0 ** -25, 3e-8],
                        device=dev)
    y[:len(edge)] = edge
    hi = y.half()
    yp = torch.cat((hi, (y - hi.float()).half()))[:T * n].contiguous()
    dy = torch.randn(n, device=dev, generator=g)
    buf, dpre = _guarded(n, torch.float32, dev)
    pbuf, planes = _guarded(T * n, torch.float16, dev) if c.planes else (None, None)
    _ok(_lib.load().t2h_lrelu_bwd(_p(yp), _p(dy), _p(dpre), _p(planes), T, n, _st()))
    torch.cuda.synchronize()
    what = f"lrelu_bwd {c} sweeps {grid_route(n)['sweeps']}"
    _untouched(buf, n, what)
    want = torch.where(hi.float() > 0, dy, dy * 0.2)
    assert torch.equal(dpre, want), f"{what}: dpre differs from dy (hi(y) > 0 ? 1 : 0.2)"
    slope = [1.0 if v else 0.2 for v in (hi[:len(edge)].float() > 0).tolist()]
    assert slope == [0.2, 0.2, 1.0, 1.0, 0.2, 0.2, 0.2, 1.0], slope  # the pinned rule around 2^-25
    if c.planes:
        _untouched(pbuf, T * n, what, H16)
        p = planes.view(T, n)
        _split_of(p[0], p[1] if T == 2 else None, dpre, f"{what} planes")


DA = collections.namedtuple("DA", "B H W")
DA_CASES = [DA(4, 512, 256), DA(4, 16, 8), DA(5, 33, 17)]


def test_diffaug_case_table_covers_every_route():
    rows = [diffaug_route(c.H, c.W) for c in DA_CASES]
    assert any(r["gx"] == 64 and r["sum_sweeps"] > 1 for r in rows)
    assert any(r["gy"] == 128 and r["apply_sweeps"] > 1 for r in rows)
    assert any(r["apply_sweeps"] == 1 and r["gy"] < 128 for r in rows)


def _diffaug_draws(c, g):
    """r at 0 and just below 1 on samples 0 and 1; translations +-sx, +-sy and 0 on different samples"""
    r = torch.rand(c.B, 3, generator=g)
    r[0] = 0.0
    r[1] = 1 - 2.0 ** -24
    sx, sy = int(c.H * 0.125 + 0.5), int(c.W * 0.125 + 0.5)
    t = torch.tensor([[sx, -sy], [-sx, sy], [0, 0], [sx, 0], [-sx, -sy]][:c.B], dtype=torch.int32)
    return r, t


def _diffaug_ref64(x, r, t):
    """DiffAugment color + translation (brightness, saturation, contrast with the sample mean of the saturated
    image, then a zero-padded shift) in fp64"""
    Bn, _, H, W = x.shape
    rd = r.double()
    b, s, c = rd[:, 0] - 0.5, rd[:, 1] * 2, rd[:, 2] + 0.5
    v = x + b.view(-1, 1, 1, 1)
    m = v.mean(1, keepdim=True)
    y = (v - m) * s.view(-1, 1, 1, 1) + m
    M = y.mean((1, 2, 3), keepdim=True)
    z = (y - M) * c.view(-1, 1, 1, 1) + M
    out = torch.zeros_like(z)
    for i in range(Bn):
        tx, ty = int(t[i, 0]), int(t[i, 1])
        hs, ws = slice(max(0, -tx), min(H, H - tx)), slice(max(0, -ty), min(W, W - ty))
        hz, wz = slice(max(0, tx), min(H, H + tx)), slice(max(0, ty), min(W, W + ty))
        out[i, :, hs, ws] = z[i, :, hz, wz]
    return out, v, M, (b, s, c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", DA_CASES, ids=lambda c: f"B{c.B}-{c.H}x{c.W}")
def test_diffaug_fwd_bwd_match_fp64(cuda, c):
    dev, Bn, H, W = cuda, c.B, c.H, c.W
    g = torch.Generator().manual_seed(H * W + Bn)
    x = torch.randn(Bn, 3, H, W, generator=g) * 0.6 + 0.2
    r, t = _diffaug_draws(c, g)
    dout = torch.randn(Bn, 3, H, W, generator=g) + 0.5  # a non-zero mean, so the contrast term's weight matters
    xd, rd, td, dd = x.to(dev), r.to(dev), t.to(dev), dout.to(dev)
    n = Bn * 3 * H * W
    ws = torch.full((Bn + 8,), SENTINEL, dtype=torch.float64, device=dev)
    obuf, out = _guarded(n, torch.float32, dev)
    _ok(_lib.load().t2h_diffaug_fwd(_p(xd), _p(rd), _p(td), _p(ws), _p(out), Bn, H, W, _st()))
    xbuf, dx = _guarded(n, torch.float32, dev)
    _ok(_lib.load().t2h_diffaug_bwd(_p(dd), _p(rd), _p(td), _p(ws), _p(dx), Bn, H, W, _st()))
    torch.cuda.synchronize()
    rt = diffaug_route(H, W)
    what = f"diffaug {c} grids {rt['gx']} / {rt['gy']} sweeps {rt['sum_sweeps']} / {rt['apply_sweeps']}"
    _untouched(obuf, n, what)
    _untouched(xbuf, n, what)
    assert (ws[Bn:] == SENTINEL).all(), f"{what}: writes past the per-sample sums"
    x64 = x.double().requires_grad_(True)
    ref, v, M, (b, s, cc) = _diffaug_ref64(x64, r, t)
    ref.backward(dout.double())
    got = out.view(Bn, 3, H, W).cpu()
    shifted = torch.zeros(Bn, 3, H, W, dtype=torch.bool)
    for i in range(Bn):
        tx, ty = int(t[i, 0]), int(t[i, 1])
        shifted[i, :, max(0, -tx):min(H, H - tx), max(0, -ty):min(W, W - ty)] = True
    assert (got[~shifted] == 0).all(), f"{what}: a pixel shifted in from outside is not 0"
    vmax = v.detach().abs().amax(1, keepdim=True)
    Bv = (1 + cc.view(-1, 1, 1, 1) * (1 + s.view(-1, 1, 1, 1))) * (vmax + M.detach().abs())
    Bf = torch.zeros_like(ref)
    for i in range(Bn):
        tx, ty = int(t[i, 0]), int(t[i, 1])
        Bf[i, :, max(0, -tx):min(H, H - tx), max(0, -ty):min(W, W - ty)] = Bv[i, :, max(0, tx):min(H, H + tx),
                                                                               max(0, ty):min(W, W + ty)]
    w1 = _check(got, ref.detach(), Bf, f"{what} forward", K_DA)
    # backward bound: dz is dout moved back by t (0 where no output read the pixel)
    dz = torch.zeros(Bn, 3, H, W, dtype=torch.float64)
    for i in range(Bn):
        tx, ty = int(t[i, 0]), int(t[i, 1])
        dz[i, :, max(0, tx):min(H, H + tx), max(0, ty):min(W, W + ty)] = dout.double()[
            i, :, max(0, -tx):min(H, H - tx), max(0, -ty):min(W, W - ty)]
    c4, s4 = cc.view(-1, 1, 1, 1), s.view(-1, 1, 1, 1)
    Bdy = c4 * dz.abs().amax(1, keepdim=True) + (c4 + (1 - c4).abs()) * dz.abs().mean((1, 2, 3), keepdim=True)
    Bb = (1 + s4 + (1 - s4).abs()) * Bdy
    w2 = _check(dx.view(Bn, 3, H, W).cpu(), x64.grad, Bb.expand_as(dz), f"{what} backward", K_DA)
    print(f"{what}: worst err/B {max(w1, w2):.3g}")


AW = collections.namedtuple("AW", "n rg gg enable wmax")
# rg, gg: the gradients' root-sum-square before the loss scale; gg 0 gives |rg| / 1e-4
AW_CASES = [AW(1, 0.3, 0.7, 1.0, 1e4), AW(1023, 2.0, 0.5, 1.0, 1e4), AW(1025, 5.0, 1e-7, 1.0, 1e4),
            AW(3456, 1.5, 0.25, 0.0, 1e4), AW(3456, 0.05, 0.0, 1.0, 1e4), AW(3456, 3.0, 0.0, 1.0, 1e4),
            AW(1025, 0.8, 0.1, 1.0, 2.0)]


def test_adaptive_weight_case_table():
    assert {c.n for c in AW_CASES} == {1, 1023, 1025, 3456}
    assert {adaptive_weight_route(c.n) for c in AW_CASES} == {1, 2, 4}
    assert any(c.gg == 0 for c in AW_CASES) and any(c.enable == 0 for c in AW_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("c", AW_CASES, ids=lambda c: f"n{c.n}-rg{c.rg:g}-gg{c.gg:g}-en{c.enable:g}-max{c.wmax:g}")
def test_adaptive_weight_matches_fp64(cuda, c):
    dev = cuda
    g = torch.Generator().manual_seed(c.n)
    inv_scale = 2.0 ** -10
    rg = torch.randn(c.n, generator=g)
    gg = torch.randn(c.n, generator=g)
    rg = (rg * (c.rg / rg.double().norm()) / inv_scale).float()
    gg = (gg * (c.gg / gg.double().norm().clamp_min(1e-30)) / inv_scale).float()
    buf = torch.full((2,), SENTINEL, device=dev)
    rgd, ggd = rg.to(dev), gg.to(dev)
    _ok(_lib.load().t2h_adaptive_weight(_p(rgd), _p(ggd), c.n, inv_scale, c.wmax, c.enable, _p(buf), _st()))
    torch.cuda.synchronize()
    what = f"adaptive_weight {c} sweeps {adaptive_weight_route(c.n)}"
    assert buf[1] == SENTINEL, f"{what}: writes past the output"
    w = (rg.double() * inv_scale).norm() / ((gg.double() * inv_scale).norm() + 1e-4)
    ref = w.clamp(0, _f32(c.wmax)) * c.enable
    got = buf[0].double().cpu()
    if c.enable == 0:
        assert got == 0
    _check(got[None], ref[None], ref.abs()[None], what, 2 * U)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [5, 2 * H100_SMS * 16 * 256 + 3])
def test_axpy_dev_matches_fp64(cuda, n):
    dev = cuda
    gen = torch.Generator(device=dev).manual_seed(n)
    a = torch.randn(n, device=dev, generator=gen)
    b = torch.randn(n, device=dev, generator=gen) * 1e3
    w = torch.tensor([0.37], device=dev)
    buf, out = _guarded(n, torch.float32, dev)
    _ok(_lib.load().t2h_axpy_dev(_p(a), _p(b), _p(w), _p(out), n, _st()))
    torch.cuda.synchronize()
    what = f"axpy_dev n {n} sweeps {grid_route(n)['sweeps']}"
    _untouched(buf, n, what)
    wb = _f32(0.37) * b.double()
    ref = a.double() + wb
    _check(out, ref, ref.abs() + wb.abs(), what, U)


@pytest.mark.gpu
@pytest.mark.parametrize("count,C", [(1, 64), (2, 7), (4096, 64), (100000, 16)])
def test_bn_update_running_matches_fp64(cuda, count, C):
    """the momentum update of torch.batch_norm (unbiased variance); a single value per channel keeps the biased
    variance 0 (torch refuses that batch)"""
    dev = cuda
    g = torch.Generator().manual_seed(count + C)
    x = torch.randn(count, C, generator=g) * (0.5 + torch.rand(C, generator=g)) + torch.rand(C, generator=g) * 10
    xd64 = x.double()
    stats = torch.stack((xd64.sum(0), (xd64 * xd64).sum(0)), 1).contiguous()
    rm0, rv0 = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    mom = 0.1
    bm, rm = _guarded(C, torch.float32, dev)
    bv, rv = _guarded(C, torch.float32, dev)
    rm.copy_(rm0)
    rv.copy_(rv0)
    sd = stats.to(dev)
    _ok(_lib.load().t2h_bn_update_running(_p(sd), _p(rm), _p(rv), count, mom, C, _st()))
    torch.cuda.synchronize()
    what = f"bn_update_running count {count} C {C}"
    _untouched(bm, C, what)
    _untouched(bv, C, what)
    m = _f32(mom)
    wm, wv = rm0.double().clone(), rv0.double().clone()
    if count > 1:
        F.batch_norm(xd64, wm, wv, training=True, momentum=m)
        var = xd64.var(0, unbiased=True)
    else:
        var = torch.zeros(C, dtype=torch.float64)
        wm, wv = (1 - m) * wm + m * xd64[0], (1 - m) * wv
    mean = xd64.mean(0)
    _check(rm.cpu(), wm, (1 - m) * rm0.double().abs() + m * mean.abs(), f"{what} running mean", 3 * U)
    _check(rv.cpu(), wv, (1 - m) * rv0.double().abs() + m * var.abs(), f"{what} running var", 3 * U)


# ------------------------------------------------------------------ section 3: quantizer edges against the C oracle
VQ = collections.namedtuple("VQ", "B Hz Wz Cz ps n_books n_e nan")
VQ_CASES = [VQ(1, 12, 10, 4, 1, 3, 100, False), VQ(2, 32, 24, 20, 1, 63, 1, True), VQ(1, 16, 12, 36, 1, 18, 1000, True),
            VQ(2, 32, 24, 9, 2, 5, 130, False)]


def _vq_id(c):
    return f"B{c.B}-{c.Hz}x{c.Wz}-Cz{c.Cz}-ps{c.ps}-books{c.n_books}-ne{c.n_e}{'-nan' if c.nan else ''}"


def _vq_books(c, g):
    """a bin of 33 rows and one of 65, ids -1, n_books and 1000 mixed in, the rest uniform"""
    rows = c.B * (c.Hz // c.ps) * (c.Wz // c.ps)
    nb = c.n_books
    fixed = [min(1, nb - 1)] * 33 + [min(2, nb - 1)] * 65 + [-1] * 5 + [nb] * 4 + [1000] * 3
    lo, hi = (3, nb) if nb > 3 else (0, 1)  # the rest stays out of the two fixed bins
    rest = torch.randint(lo, hi, (rows - len(fixed),), generator=g).tolist()
    ids = torch.tensor(fixed + rest, dtype=torch.int32)
    return ids[torch.randperm(rows, generator=g)].view(c.B, c.Hz // c.ps, c.Wz // c.ps)


def test_vq_case_table_covers_every_route():
    g = torch.Generator().manual_seed(0)
    routes = [vq_bin_route(_vq_books(c, g).numpy(), c.n_books) for c in VQ_CASES]
    assert any(r["bin_sweeps"] > 1 for r in routes) and all(r["partial_multi"] for r in routes)
    assert all(33 in r["counts"][:-1] and 65 in r["counts"][:-1] for r in routes)
    assert {c.Cz * c.ps ** 2 for c in VQ_CASES} >= {4, 20, 36} and {c.n_e for c in VQ_CASES} >= {1, 100, 1000}
    assert max(c.n_books for c in VQ_CASES) == 63 and any(c.nan for c in VQ_CASES)
    assert any(c.ps == 2 for c in VQ_CASES)


def _vq_search(c, z, cb, books, dev, ws_bytes=None, cb_view=None):
    rows = c.B * (c.Hz // c.ps) * (c.Wz // c.ps)
    lib = _lib.load()
    need = lib.t2h_vq_workspace_bytes(rows, c.n_books, c.n_e)
    ws = torch.zeros(need + 256, dtype=torch.uint8, device=dev)
    outs = dict(idx=_guarded(rows, torch.int64, dev, -7777), idx_cont=_guarded(rows, torch.int64, dev, -7777),
                idx_list=_guarded(c.n_books * rows, torch.int64, dev, -7777),
                zq_nhwc=_guarded(z.numel(), torch.float32, dev), zq_nchw=_guarded(z.numel(), torch.float32, dev))
    sq = torch.tensor([0.0, SENTINEL], dtype=torch.float64, device=dev)
    o = {k: v[1] for k, v in outs.items()}
    cbv = cb if cb_view is None else cb_view
    rc = lib.t2h_vq_search(_p(z), _p(cbv), _p(books), c.B, c.Hz, c.Wz, c.Cz, c.ps, c.n_books, c.n_e, 4096,
                           _p(o["idx"]), _p(o["idx_cont"]), _p(o["idx_list"]), _p(o["zq_nhwc"]), _p(o["zq_nchw"]),
                           _p(sq), _p(ws), need if ws_bytes is None else ws_bytes, _st())
    return rc, outs, sq


@pytest.mark.gpu
@pytest.mark.parametrize("c", VQ_CASES, ids=_vq_id)
def test_quantizer_edges_bit_exact_vs_oracle(cuda, c):
    from oracle import vq_oracle
    dev = cuda
    g = torch.Generator().manual_seed(c.n_e + c.Cz * 7 + c.n_books)
    D = c.Cz * c.ps ** 2
    cb = torch.randn(c.n_books, c.n_e, D, generator=g) * 0.5
    z = torch.randn(c.B, c.Hz, c.Wz, c.Cz, generator=g) * 0.5
    books = _vq_books(c, g)
    if c.nan:  # a NaN in the first row of the 65-row bin
        r = int((books.view(-1) == min(2, c.n_books - 1)).nonzero()[0])
        Wp, Hp = c.Wz // c.ps, c.Hz // c.ps
        b, ph, pw = r // (Hp * Wp), (r // Wp) % Hp, r % Wp
        z[b, ph * c.ps, pw * c.ps, 0] = math.nan
    zd, cbd, bd = z.to(dev), cb.to(dev), books.to(dev)
    rc, outs, sq = _vq_search(c, zd, cbd, bd, dev)
    _ok(rc)
    torch.cuda.synchronize()
    want = vq_oracle.search(z.numpy(), cb.numpy(), books.numpy(), ps=c.ps, cont_stride=4096)
    what = f"vq_search {_vq_id(c)}"
    for k, (buf, o) in outs.items():
        _untouched(buf, o.numel(), f"{what} {k}", -7777 if o.dtype == torch.int64 else SENTINEL)
    assert sq[1] == SENTINEL, f"{what}: writes past sqerr"
    rows = books.numel()
    for k in ("idx", "idx_cont", "idx_list"):
        got = outs[k][1].cpu().numpy()
        assert np.array_equal(got, want[k].reshape(-1)), f"{what}: {k} differs from the oracle"
    zq = outs["zq_nhwc"][1].view(z.shape).cpu().numpy()
    assert np.array_equal(zq, want["zq_nhwc"], equal_nan=True), f"{what}: zq differs from the oracle"
    assert np.array_equal(outs["zq_nchw"][1].view(c.B, c.Cz, c.Hz, c.Wz).cpu().numpy(),
                          np.transpose(want["zq_nhwc"], (0, 3, 1, 2)), equal_nan=True)
    if c.nan:
        assert math.isnan(sq[0].item()) and math.isnan(want["sqerr"])
        assert outs["idx"][1][r].item() == 0, f"{what}: a NaN row did not get index 0"
    else:
        assert abs(sq[0].item() - want["sqerr"]) <= 1e-9 * abs(want["sqerr"]) + 1e-12
    idx = outs["idx"][1].cpu()
    sel = (books.view(-1) >= 0) & (books.view(-1) < c.n_books)
    assert (idx[~sel] == -1).all() and (idx[sel] >= 0).all() and (idx[sel] < c.n_e).all()
    print(f"{what}: bin counts {vq_bin_route(books.numpy(), c.n_books)['counts'].tolist()}, {rows} rows bit-exact")

    # gather with out-of-range indices: zeros
    gi = idx.clone()
    gi[:4] = torch.tensor([-1, c.n_e, 10 ** 9, -(10 ** 9)])
    gid = gi.to(dev)
    gb1, g1 = _guarded(z.numel(), torch.float32, dev)
    gb2, g2 = _guarded(z.numel(), torch.float32, dev)
    _ok(_lib.load().t2h_vq_gather(_p(cbd), _p(gid), _p(bd), c.B, c.Hz, c.Wz, c.Cz, c.ps, c.n_books, c.n_e, _p(g1),
                                  _p(g2), _st()))
    torch.cuda.synchronize()
    _untouched(gb1, z.numel(), "vq_gather nhwc")
    _untouched(gb2, z.numel(), "vq_gather nchw")
    wg = vq_oracle.gather(cb.numpy(), gi.numpy(), books.numpy(), c.B, c.Hz, c.Wz, c.Cz, c.ps)
    assert np.array_equal(g1.view(z.shape).cpu().numpy(), wg), f"{what}: gather differs from the oracle"
    assert np.array_equal(g2.view(c.B, c.Cz, c.Hz, c.Wz).cpu().numpy(), np.transpose(wg, (0, 3, 1, 2)))
    bv = books.view(-1)
    for rr in range(4):
        if 0 <= bv[rr] < c.n_books:
            Wp, Hp = c.Wz // c.ps, c.Hz // c.ps
            b, ph, pw = rr // (Hp * Wp), (rr // Wp) % Hp, rr % Wp
            blk = g1.view(z.shape)[b, ph * c.ps:(ph + 1) * c.ps, pw * c.ps:(pw + 1) * c.ps]
            assert (blk == 0).all(), f"{what}: gather of an out-of-range index is not 0"


@pytest.mark.gpu
def test_quantizer_refusals(cuda):
    """a workspace one byte short and a codebook off 16-byte alignment are refused before any launch"""
    dev = cuda
    c = VQ(1, 4, 4, 8, 1, 2, 16, False)
    cbuf = torch.zeros(c.n_books * c.n_e * 8 + 4, device=dev)
    z = torch.zeros(1, 4, 4, 8, device=dev)
    books = torch.zeros(1, 4, 4, dtype=torch.int32, device=dev)
    rows = 16
    need = _lib.load().t2h_vq_workspace_bytes(rows, c.n_books, c.n_e)
    rc, outs, _ = _vq_search(c, z, cbuf[:-4], books, dev, ws_bytes=need - 1)
    assert rc == EINVAL and "workspace" in _lib.load().t2h_last_error().decode()
    rc, outs, _ = _vq_search(c, z, cbuf[:-4], books, dev, cb_view=cbuf[1:])
    assert rc == EINVAL and "aligned" in _lib.load().t2h_last_error().decode()
    torch.cuda.synchronize()
    assert (outs["idx"][0] == -7777).all(), "a refused launch wrote its output"
