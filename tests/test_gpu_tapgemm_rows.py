"""The row-GEMM mode of the tap-GEMM (t2h_tapgemm with H == 1 or tile_rows: a 128-row tile is 128 consecutive rows of
a matrix) element by element against fp64: nn.Linear forward and backward, MN-major operands, batched, broadcast and
multi-head products, split-K (reduce-add and stored slabs) and gradient accumulation; and the operand conversions
these GEMMs consume, t2h_f32_to_planes_t and t2h_planes_transpose, bit for bit.

``rows_route`` restates, for row-mode launches, plan_tapgemm's column tile BN and epilogue and t2h_tapgemm's
k_partials / k_split / accumulate rules (csrc/gemm_tc.cu; a comment next to each rule points here).  It documents
intent and does not verify the C code: a change to a rule updates it in the same change, and
``test_row_case_table_covers_every_path`` then says which level lost its case.  The GPU tests compare rows_route's
view of every launch they make with the case's label, so a case cannot drift off the path it is listed for.

Cases come in two kinds.  ABI cases (``Spec``) call ops._tapgemm with operands laid out by hand: padded row strides
(the padding holds 999, which no correct launch reads), MN-major storage, broadcast and batched B, and destinations
that are views into sentinel-filled buffers with a guard image (or guard slab), a guard row, guard rows past the last
GEMM row and guard columns on both sides.  Production cases call the ops wrappers with the flag combinations the
models use; outputs the wrapper allocates are launched a second time from the captured arguments into a
sentinel-filled buffer with guards before and after.  Every element outside the written region must keep its
sentinel bit for bit.  A launch that stores writes the same bits when run again; a reduce-add launch starts from
random D0 and must give D0 + P after one launch and D0 + 2 P after two, P = alpha A.B (+ column bias), so the bias
is added once per launch, by the first k-slice only.  Each k_partials slab s is checked against fp64 over its own
contraction range [s kper 64, min(K, (s + 1) kper 64)), and the slab after the last one must stay untouched.

Bounds, element by element, |got - ref| <= 1e-5 B + 1e-6 |ref|:
  * ref is fp64 over the values the operand planes hold: hi + lo with the 3-product split (two planes on both
    operands), hi alone otherwise -- including the mixed fallback of a 2-plane A with a 1-plane B, which must be
    hi.hi exactly (a lo.hi term would move it by 2^-11 of the product, 200 times the bound);
  * B = |alpha| (|A|.|B|) + |bias| + |residual| in fp64, times max |GELU'| = 1.13 behind a GELU; for reduce-add B
    also includes |D0| (|D0| + 2 (...) after the second launch).  Products of fp16 values are exact in fp32; the
    3-product split omits lo.lo, at most 2^-22 of each product, inside k = 1e-5;
  * reduce-add: a k-slice's partial sum carries the same accumulation error as a whole tile, and each of at most
    132 slices (ops.wgrad_k_split never asks for more than the H100's 132 SMs) adds one fp32 rounding of at most
    2^-24 of the running sum, which B bounds: 132 2^-24 = 7.9e-6 < 1e-5;
  * long contractions (K >= 4096, the token contractions of wgrad): the worst-case fp32 accumulation bound, K 2^-24
    of B, exceeds 1e-5 B there, but rounding errors of random-signed terms do not line up: K = 4160 measured
    err/B = 1.5e-6 on an H100 80GB HBM3 at its 700 W power limit, so the same k holds;
  * a single fp16 output plane adds its 11-bit rounding, 2^-11 |ref|, and the fp16 subnormal spacing 2^-24;
  * two output planes must be a nearest split: hi an fp16 nearest to hi + lo (_nearest of test_gpu_row_kernels.py).

Refusals: launches the host code must refuse return T2H_EINVAL and leave D unchanged.  They are all argument or
tensor-map checks on the host; nothing is launched.
"""
import collections
import ctypes
import types
import zlib

import pytest
import torch

from text2human_b200 import _lib, ops

SENTINEL = -7777.0
EINVAL = -1
K_TOL, K_REL = 1e-5, 1e-6
GELU_SLOPE = 1.13  # max |GELU'(x)| = 1.1289 at x = +-sqrt(2)
ACTS = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "lrelu": _lib.ACT_LRELU, "gelu": _lib.ACT_GELU}
ACT_NAMES = {v: k for k, v in ACTS.items()}


def _cdiv(a, b):
    return -(-a // b)


def _up(a, b):
    return _cdiv(a, b) * b


# ------------------------------------------------------------------ the launch rules, restated
def k_slices(K, ks):
    """set_k_slices: (contraction chunks per slice, slices) for a request of ks slices"""
    kchunks = _cdiv(K, 64)
    ks = min(max(ks, 1), kchunks)
    kper = _cdiv(kchunks, ks)
    return kper, _cdiv(kchunks, kper)


def rows_route(*, n_img, H, W, K, n_out, planes=0, d_plane=0, strides, d_al=True, a_mn=0, b_mn=0, b_bh=0,
               tile_rows=0, res=False, res_al=True, bias="none", bias_al=True, bias_sn=0, act="none", k_split=0,
               accumulate=False, k_partials=0, d_slab=0, a_str=(8, 8, 8), a_al=True, b_str=(8, 8, 8), b_al=True):
    """BN, epilogue, store form and k-slices of a t2h_tapgemm row-mode launch, or the reason it is refused.
    planes: output planes (d_terms) or 0 for fp32; strides: D's (sn, sh, sw, sc) in elements; *_al: the pointer is
    16-byte aligned; a_str / b_str: the fp16 operands' element strides their tensor maps encode"""
    if not (H == 1 or tile_rows):
        if a_mn or b_mn or b_bh:
            return dict(refused="MN-major operands and b_batched_h need row tiles")
        return dict(spatial=True)
    if any(s % 8 for s in tuple(a_str) + tuple(b_str)) or not (a_al and b_al):
        return dict(refused="operand tensor map: strides and base must be 16-byte multiples")
    sn, sh, sw, sc = strides
    BN = 16
    while BN < n_out and BN < 128:
        BN <<= 1
    if b_mn and BN < 64:
        BN = 64  # an MN-major B tile is made of whole 64-column boxes
    align = 8 if planes else 4  # elements per 16 bytes
    tma_ok = sc == 1 and n_out % align == 0 and sw % align == 0 and d_al and BN >= (64 if planes else 32)
    if H > 1:
        tma_ok = tma_ok and sh % align == 0 and sh > 0
    if n_img > 1:
        tma_ok = tma_ok and sn % align == 0 and sn > 0
    if planes == 2:
        s = sn if n_img > 1 else d_plane
        tma_ok = tma_ok and s > 0 and d_plane % s == 0 and d_plane % align == 0
    if res:
        tma_ok = tma_ok and res_al
    if bias in ("col", "img"):
        tma_ok = tma_ok and bias_al and bias_sn % 4 == 0
    epi = "direct" if not tma_ok else ("tma_planes" if planes else "tma_f32")
    if epi == "tma_f32" and BN >= 64 and not res and act == "none" and bias != "row":
        epi = "plain_f32"  # two epilogue warpgroups: alpha and column bias only
    f32_tma = epi in ("tma_f32", "plain_f32")
    reducible = f32_tma and not res and bias != "row" and act == "none"
    if k_partials > 1:
        if not (f32_tma and not res and bias == "none" and act == "none" and n_img == 1 and k_split <= 1
                and d_slab > 0 and d_slab % 4 == 0):
            return dict(refused="k_partials needs a plain single-image fp32 output and an aligned slab stride")
        store, (kper, slices) = "slabs", k_slices(K, k_partials)
    elif k_split > 1:
        if not reducible:
            return dict(refused="k_split needs an aligned fp32 output and no row bias / act / residual")
        store, (kper, slices) = "reduce", k_slices(K, k_split)
    else:
        store, (kper, slices) = "store", k_slices(K, 1)
    if accumulate:
        if not reducible:
            return dict(refused="accumulate needs an aligned fp32 output and no row bias / act / residual")
        if store == "store":
            store = "reduce"
    return dict(BN=BN, epi=epi, store=store, kper=kper, slices=slices)


def _al(t):
    return t is None or t.data_ptr() % 16 == 0


def _route_of(kw):
    """rows_route's view of one ops._tapgemm launch, from its arguments and real pointers"""
    d = kw["d"]
    planes = d.shape[0] if kw["d_mode"] == _lib.OUT_PLANES else 0
    bias = kw.get("bias")
    bm = kw.get("bias_mode", _lib.BIAS_NONE) if bias is not None else _lib.BIAS_NONE
    bias_kind = {_lib.BIAS_NONE: "none", _lib.BIAS_ROW: "row"}.get(bm, "img" if kw.get("bias_sn", 0) else "col")
    g2 = kw.get("b_groups2", 1)
    return rows_route(n_img=kw["n_img"], H=kw["H"], W=kw["W"], K=kw["Cc"], n_out=kw["n_out"], planes=planes,
                      d_plane=kw.get("d_plane", 0), strides=kw["d_strides"], d_al=_al(d), a_mn=kw.get("a_mn", 0),
                      b_mn=kw.get("b_mn", 0), b_bh=kw.get("b_batched_h", 0), tile_rows=kw.get("tile_rows", 0),
                      res=kw.get("residual") is not None, res_al=_al(kw.get("residual")), bias=bias_kind,
                      bias_al=_al(bias), bias_sn=kw.get("bias_sn", 0), act=ACT_NAMES[kw.get("act", _lib.ACT_NONE)],
                      k_split=kw.get("k_split", 0), accumulate=kw.get("accumulate", False),
                      k_partials=kw.get("k_partials", 0), d_slab=kw.get("d_slab", 0),
                      a_str=(kw["a_sw"], kw["a_sh"], kw["a_sn"]), a_al=_al(kw["a"]),
                      b_str=(kw["b_sn"], kw["b_sg"], kw.get("b_sg2", 0) if g2 > 1 else kw["b_sg"]), b_al=_al(kw["b"]))


def _features(kw):
    """the factor levels of one launch that the coverage test counts"""
    bias = kw.get("bias")
    bm = kw.get("bias_mode", _lib.BIAS_NONE) if bias is not None else _lib.BIAS_NONE
    f = dict(_route_of(kw))
    f.update(out="f32" if kw["d_mode"] == _lib.OUT_F32 else f"p{kw['d'].shape[0]}", n=kw["n_img"], H=kw["H"],
             M=kw["W"], K=kw["Cc"], N=kw["n_out"], a_mn=kw.get("a_mn", 0), b_mn=kw.get("b_mn", 0),
             a_bcast=kw.get("a_bcast", 0), b_batched=kw.get("b_batched", 0), b_bh=kw.get("b_batched_h", 0),
             planes=(kw["a"].shape[0], kw["b"].shape[0]),
             bias={_lib.BIAS_NONE: "none", _lib.BIAS_ROW: "row"}.get(bm, "img" if kw.get("bias_sn", 0) else "col"),
             act=ACT_NAMES[kw.get("act", _lib.ACT_NONE)], res=kw.get("residual") is not None,
             alpha=kw.get("alpha", 1.0), ks=kw.get("k_split", 0), acc=bool(kw.get("accumulate", False)),
             kp=kw.get("k_partials", 0), tile_rows=kw.get("tile_rows", 0))
    return f


# ------------------------------------------------------------------ the case table: launches laid out by hand
Spec = collections.namedtuple(
    "Spec", "name n H W K N at bt a_mn b_mn a_bcast b_batched b_bh tile_rows out c0 bias b_off act res alpha ks acc "
            "kp slab_skew lda",
    defaults=(1, 1, 128, 64, 64, 2, 2, 0, 0, 0, 0, 0, None, "f32", 0, "none", 0, "none", False, 1.0, 0, False, 0, 0,
              None))
# n images x H x W GEMM rows (W = M), contraction K, N output columns; at / bt: planes of A / B; out: f32, p1, p2
# (fp16 output planes); c0: first destination column inside the wider buffer; bias: none, col (shared), img (one
# vector per image, bias_sn), row (bias[h W + w]); b_off: the bias pointer's offset in elements (1: misaligned)
CASES = [
    # column tiles and epilogues
    Spec("bn16-direct-gelu-alpha", W=200, K=200, N=16, bias="col", act="gelu", alpha=0.375),
    Spec("bn32-tma-gelu", W=256, K=96, N=24, bias="col", act="gelu"),
    Spec("bn64-plain-img-bias", n=3, W=40, K=64, N=48, b_batched=1, bias="img", alpha=0.375),
    Spec("bn128-plain-m1-k8", W=1, K=8, N=200, bias="col"),
    Spec("bn64-forced-by-bmn", W=130, K=64, N=24, b_mn=1, out="p2"),
    Spec("direct-planes-n20-relu", n=2, W=150, K=128, N=20, b_batched=1, out="p2", act="relu", bias="col"),
    Spec("direct-f32-n30-lrelu-res", W=128, K=256, N=30, bias="col", act="lrelu", res=True),
    Spec("direct-misaligned-slice", W=96, K=64, N=64, c0=1, bias="col"),
    Spec("direct-misaligned-img-bias-bcast", n=2, W=96, K=64, N=64, a_bcast=1, b_batched=1, bias="img", b_off=1),
    Spec("planes1-n1-gelu", W=200, K=128, N=128, at=1, bt=1, out="p1", bias="col", act="gelu"),
    Spec("planes1-n3", n=3, W=64, K=64, N=64, b_batched=1, out="p1", bias="img"),
    Spec("planes2-n2-lrelu-slice", n=2, W=200, K=96, N=128, b_batched=1, out="p2", bias="col", act="lrelu", c0=8),
    # operand forms
    Spec("a-mn", W=256, K=200, N=96, a_mn=1, bias="col"),
    Spec("a-mn-b-mn-long-k", W=96, K=4160, N=80, a_mn=1, b_mn=1, alpha=0.125),
    Spec("b-mn-res-relu", W=200, K=128, N=96, b_mn=1, res=True, act="relu", alpha=0.375),
    Spec("mixed-fallback-hi-hi", W=128, K=128, N=64, at=2, bt=1, bias="col"),
    Spec("single-plane", W=70, K=192, N=64, at=1, bt=1),
    # row bias
    Spec("row-bias-h1", W=100, K=64, N=64, bias="row"),
    Spec("row-bias-tile-rows-b-batched-h", n=2, H=3, W=70, K=64, N=48, b_batched=1, b_bh=1, bias="row"),
    # split-K, accumulation and stored slabs
    Spec("ksplit-even", W=128, K=1024, N=128, ks=4, bias="col"),
    Spec("ksplit-uneven-img-bias", n=2, W=200, K=1024, N=64, b_batched=1, ks=6, bias="img", alpha=0.5),
    Spec("ksplit-beyond-kchunks", W=64, K=200, N=32, ks=16, bias="col"),
    Spec("accumulate", W=96, K=128, N=64, acc=True, bias="col"),
    Spec("accumulate-ksplit-mn", W=128, K=512, N=128, a_mn=1, b_mn=1, ks=3, acc=True),
    Spec("kpartials-fewer-slabs", W=128, K=320, N=96, kp=4),
    Spec("kpartials-even", W=64, K=512, N=64, kp=4, alpha=0.375),
]

REFUSED = [
    Spec("refuse-ksplit-residual", W=64, K=512, N=64, ks=4, res=True),
    Spec("refuse-ksplit-row-bias", W=64, K=512, N=64, ks=4, bias="row"),
    Spec("refuse-ksplit-act", W=64, K=512, N=64, ks=4, act="gelu"),
    Spec("refuse-accumulate-act", W=64, K=128, N=64, acc=True, act="relu"),
    Spec("refuse-kpartials-bias", W=64, K=512, N=64, kp=4, bias="col"),
    Spec("refuse-kpartials-n-img", n=2, W=64, K=512, N=64, b_batched=1, kp=4),
    Spec("refuse-kpartials-misaligned-slab", W=64, K=512, N=64, kp=4, slab_skew=-2),
    Spec("refuse-a-mn-spatial", H=4, W=16, K=64, N=64, a_mn=1, tile_rows=0),
    Spec("refuse-b-batched-h-spatial", n=2, H=4, W=16, K=64, N=64, b_bh=1, tile_rows=0),
    Spec("refuse-operand-row-stride", W=64, K=60, N=64, lda=60),
]


def _vals(planes, nterms):
    """fp64 values the planes hold as the kernel reads them: hi + lo with the 3-product split, hi alone otherwise"""
    return planes.double().sum(0) if nterms == 3 else planes[0].double()


def _build(s, dev):
    """operands, destination and ops._tapgemm arguments of an ABI case"""
    gen = torch.Generator().manual_seed(zlib.crc32(s.name.encode()))
    rnd = lambda *shape: torch.randn(*shape, generator=gen)  # noqa: E731
    n, H, W, K, N = s.n, s.H, s.W, s.K, s.N
    na = 1 if s.a_bcast else n
    # rows of different magnitudes: a row's small elements cannot hide under another row's large ones
    x = rnd(na, H, W, K) * 2.0 ** torch.randint(-4, 5, (na, H, W, 1), generator=gen).float()
    ap = ops.split_planes(x, s.at)  # [at, na, H, W, K]
    nbi, nbh = (n if s.b_batched else 1), (H if s.b_bh else 1)
    bp = ops.split_planes(rnd(nbi, nbh, N, K) / K ** 0.5, s.bt)  # [bt, nbi, nbh, N, K]
    kld = s.lda if s.lda is not None else _up(K, 8) + 8
    f16 = dict(dtype=torch.float16)
    if s.a_mn:  # [k][row] storage: a_sw = distance between consecutive k
        wld = _up(W, 8) + 8
        abuf = torch.full((s.at, na, H, K, wld), 999.0, **f16)
        abuf[..., :W] = ap.transpose(-1, -2)
        a_str = (wld, K * wld, H * K * wld)
    else:
        abuf = torch.full((s.at, na, H, W, kld), 999.0, **f16)
        abuf[..., :K] = ap
        a_str = (kld, W * kld, H * W * kld)
    bpt = bp.transpose(0, 1)  # the image index g2 is B's outermost dim: [nbi, bt, nbh, ...]
    if s.b_mn:  # [k][column] storage: b_sn = distance between consecutive k
        nld = _up(N, 8) + 8
        bst = torch.full((nbi, s.bt, nbh, K, nld), 999.0, **f16)
        bst[..., :N] = bpt.transpose(-1, -2)
        b_sn, b_sg = nld, K * nld
    else:
        bst = torch.full((nbi, s.bt, nbh, N, kld), 999.0, **f16)
        bst[..., :K] = bpt
        b_sn, b_sg = kld, N * kld
    nt = 3 if s.at == 2 and s.bt == 2 else 1
    av = _vals(ap, nt).expand(n, H, W, K)
    bv = _vals(bp, nt).expand(n, H, N, K)

    planes = int(s.out[1]) if s.out != "f32" else 0
    lead = s.kp + 1 if s.kp else n + 1  # a guard image (or slab) after the last one
    shape = (lead, H + 1, W + 3, s.c0 + _up(N, 8) + 8)  # a guard row, 3 guard GEMM rows, guard columns
    region = (slice(0, n), slice(0, H), slice(0, W), slice(s.c0, s.c0 + N))
    if planes:
        dbuf = torch.full((planes + 1,) + shape, SENTINEL, **f16)  # and a guard plane
        d = dbuf[(slice(0, planes),) + region]
        strides, d_plane = dbuf.stride()[1:], dbuf.stride(0)
    else:
        dbuf = torch.full(shape, SENTINEL)
        d = dbuf[region]
        strides, d_plane = dbuf.stride(), 0
    rbuf = rnd(*shape) if s.res else None
    d0 = None
    if s.ks > 1 or s.acc:
        d0 = rnd(n, H, W, N)
        dbuf[region] = d0
    bbuf, bias_sn, bvals = None, 0, None  # the bias starts b_off elements into bbuf
    if s.bias == "col":
        bbuf = rnd(s.b_off + N + 4)
        bvals = bbuf[s.b_off:s.b_off + N].double().view(1, 1, 1, N)
    elif s.bias == "img":
        bias_sn = _up(N, 4) + 4
        bbuf = rnd(s.b_off + n * bias_sn)
        bvals = bbuf[s.b_off:].double().view(n, bias_sn)[:, :N].reshape(n, 1, 1, N)
    elif s.bias == "row":
        bbuf = rnd(s.b_off + H * W)
        bvals = bbuf[s.b_off:].double().view(1, H, W, 1)
    mv = lambda t: None if t is None else t.to(dev)  # noqa: E731
    abuf, bst, dbuf, rbuf, bbuf = mv(abuf), mv(bst), mv(dbuf), mv(rbuf), mv(bbuf)
    bias = bbuf[s.b_off:] if bbuf is not None else None  # sliced on the device: the offset survives
    d = dbuf[(slice(0, planes),) + region] if planes else dbuf[region]
    residual = rbuf[region] if rbuf is not None else None
    kw = dict(a=abuf, a_term_imgs=na, a_imgs=s.at * na, a_bcast=s.a_bcast, n_img=n, H=H, W=W, a_H=H, a_W=W, Cc=K,
              a_sw=a_str[0], a_sh=a_str[1], a_sn=a_str[2],
              b=bst.transpose(0, 1), b_term_g=nbh, b_groups=s.bt * nbh, b_batched=s.b_batched, n_out=N, b_sn=b_sn,
              b_sg=b_sg, b_groups2=nbi, b_sg2=bst.stride(0), b_batched_h=s.b_bh,
              taps=ops._TAPS_1, d=d, d_mode=_lib.OUT_PLANES if planes else _lib.OUT_F32, d_strides=tuple(strides),
              d_plane=d_plane, bias=bias, bias_mode=_lib.BIAS_ROW if s.bias == "row" else _lib.BIAS_COL,
              bias_sn=bias_sn, act=ACTS[s.act], alpha=s.alpha, residual=residual,
              tile_rows=s.tile_rows if s.tile_rows is not None else int(H > 1),
              k_split=s.ks, accumulate=s.acc, a_mn=s.a_mn, b_mn=s.b_mn, k_partials=s.kp,
              d_slab=dbuf.stride(0) + s.slab_skew if s.kp else 0)
    return types.SimpleNamespace(kw=kw, av=av, bv=bv, bvals=bvals, dbuf=dbuf, region=region, planes=planes, d0=d0,
                                 rv=residual.double() if residual is not None else None)


def _label(s):
    return _route_of(_build(s, "cpu").kw)


# ------------------------------------------------------------------ production flag combinations, through ops
class _DryRun(Exception):
    pass


class _Capture:
    """replaces ops._tapgemm: records every launch's arguments, and launches them unless dry (CPU: the argument
    construction of the wrappers only)"""

    def __init__(self, dry):
        self.dry, self.kws = dry, []

    def __enter__(self):
        self._real, self._need = ops._tapgemm, ops._need_cuda
        ops._tapgemm = self._call
        if self.dry:
            ops._need_cuda = lambda *ts: None
        return self

    def _call(self, **kw):
        self.kws.append(kw)
        if not self.dry:
            self._real(**kw)

    def __exit__(self, *exc):
        ops._tapgemm, ops._need_cuda = self._real, self._need


def _planes(gen, shape, terms=2, scale=1.0):
    return ops.split_planes(torch.randn(*shape, generator=gen) * scale, terms)


def _prod_linear_residual(dev, run):
    gen = torch.Generator().manual_seed(1)
    M, K, N = 200, 96, 96
    a, w = _planes(gen, (M, K)), ops.pack_linear_weight(torch.randn(N, K, generator=gen) / K ** 0.5, 2)
    bias = torch.randn(N, generator=gen)
    dbuf = torch.full((M + 2, N + 16), SENTINEL)
    rbuf = torch.randn(M + 2, N + 16, generator=gen)
    a, w, bias, dbuf, rbuf = (t.to(dev) for t in (a, w, bias, dbuf, rbuf))
    out, res = dbuf[:M, 8:8 + N], rbuf[:M, 8:8 + N]
    kws = run(lambda: ops.linear(a, w, bias, residual=res, out=out))
    pre, pb = _mm(_vals(a, 3), _vals(w[:, 0], 3), 1.0, bias)
    return kws, [dict(buf=dbuf, region=(slice(0, M), slice(8, 8 + N)), ref=pre + res.double(),
                      B=pb + res.double().abs(), planes=0)]


def _mm(av, bv, alpha, bias=None, bias_row=None):
    """alpha a @ b^T (+ column bias / row bias) in fp64 and its magnitude bound"""
    pre = alpha * av @ bv.transpose(-1, -2)
    pb = abs(alpha) * av.abs() @ bv.abs().transpose(-1, -2)
    if bias is not None:
        pre, pb = pre + bias.double(), pb + bias.double().abs()
    if bias_row is not None:
        pre, pb = pre + bias_row.double().unsqueeze(-1), pb + bias_row.double().abs().unsqueeze(-1)
    return pre, pb


def _prod_linear_planes_gelu(dev, run):
    gen = torch.Generator().manual_seed(2)
    M, K, N = 130, 200, 256
    a, w = _planes(gen, (M, K)), ops.pack_linear_weight(torch.randn(N, K, generator=gen) / K ** 0.5, 2)
    bias = torch.randn(N, generator=gen)
    dbuf = torch.full((3, M + 2, N + 16), SENTINEL, dtype=torch.float16)
    a, w, bias, dbuf = (t.to(dev) for t in (a, w, bias, dbuf))
    out = dbuf[:2, :M, 8:8 + N]
    kws = run(lambda: ops.linear(a, w, bias, planes_out=True, act=ops.ACT_GELU, out=out))
    pre, pb = _mm(_vals(a, 3), _vals(w[:, 0], 3), 1.0, bias)
    return kws, [dict(buf=dbuf, region=(slice(0, 2), slice(0, M), slice(8, 8 + N)),
                      ref=torch.nn.functional.gelu(pre), B=GELU_SLOPE * pb, planes=2)]


def _prod_linear_w_kn(dev, run):
    """the data gradient dX = dY W with W as stored [out, in]: B consumed MN-major, planes out (d_y of attn.proj)"""
    gen = torch.Generator().manual_seed(3)
    M, K, N = 70, 128, 48
    a, w = _planes(gen, (M, K)), ops.split_planes((torch.randn(K, N, generator=gen) / K ** 0.5).unsqueeze(0), 2)
    a, w = a.to(dev), w.to(dev)
    kws = run(lambda: ops.linear(a, w, w_kn=True, planes_out=True))
    pre, pb = _mm(_vals(a, 3), _vals(w[:, 0], 3).t(), 1.0)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=2)]


def _prod_linear_ksplit_residual_stream(dev, run):
    """x += proj(y) + bias at small batch: k_split reduce-adds into the residual stream itself"""
    gen = torch.Generator().manual_seed(4)
    M, K, N = 64, 1024, 128
    a, w = _planes(gen, (M, K)), ops.pack_linear_weight(torch.randn(N, K, generator=gen) / K ** 0.5, 2)
    bias = torch.randn(N, generator=gen)
    dbuf = torch.full((M + 2, N + 16), SENTINEL)
    d0 = torch.randn(M, N, generator=gen)
    dbuf[:M, 8:8 + N] = d0
    a, w, bias, dbuf, d0 = (t.to(dev) for t in (a, w, bias, dbuf, d0))
    out = dbuf[:M, 8:8 + N]
    kws = run(lambda: ops.linear(a, w, bias, out=out, k_split=6))
    pre, pb = _mm(_vals(a, 3), _vals(w[:, 0], 3), 1.0, bias)
    return kws, [dict(buf=dbuf, region=(slice(0, M), slice(8, 8 + N)), ref=pre, B=pb, planes=0, d0=d0.double())]


def _prod_linear_partials(dev, run):
    gen = torch.Generator().manual_seed(5)
    M, K, N = 64, 712, 96
    a, w = _planes(gen, (M, K)), ops.pack_linear_weight(torch.randn(N, K, generator=gen) / K ** 0.5, 2)
    a, w = a.to(dev), w.to(dev)
    kws = run(lambda: ops.linear_partials(a, w, 4, alpha=0.5))
    av, wv = _vals(a, 3), _vals(w[:, 0], 3)
    kper, S = k_slices(K, 4)
    refs, bs = [], []
    for sl in range(S):
        k0, k1 = sl * kper * 64, min(K, (sl + 1) * kper * 64)
        r, b = _mm(av[:, k0:k1], wv[:, k0:k1], 0.5)
        refs.append(r)
        bs.append(b)
    return kws, [dict(out=run.outputs[-1], ref=torch.stack(refs), B=torch.stack(bs), planes=0)]


def _prod_wgrad(dev, run):
    """dW += alpha dY^T X over 4160 tokens: both operands MN-major, k_split + accumulate into a gradient buffer"""
    gen = torch.Generator().manual_seed(6)
    M, No, Ni = 4160, 96, 80
    dy, x = _planes(gen, (M, No)), _planes(gen, (M, Ni))
    dbuf = torch.full((No + 2, Ni + 16), SENTINEL)
    d0 = torch.randn(No, Ni, generator=gen)
    dbuf[:No, 8:8 + Ni] = d0
    dy, x, dbuf, d0 = (t.to(dev) for t in (dy, x, dbuf, d0))
    out = dbuf[:No, 8:8 + Ni]
    ks = ops.wgrad_k_split(No, Ni, M)
    kws = run(lambda: ops.wgrad(dy, x, out, k_split=ks, alpha=0.125, accumulate=True))
    pre, pb = _mm(_vals(dy, 3).t(), _vals(x, 3).t(), 0.125)
    return kws, [dict(buf=dbuf, region=(slice(0, No), slice(8, 8 + Ni)), ref=pre, B=pb, planes=0, d0=d0.double())]


def _prod_bmm_attnblock_v(dev, run):
    """AttnBlock v^T[b] = Wv hn[b]^T + bias per row: broadcast A, row bias, planes out"""
    gen = torch.Generator().manual_seed(7)
    N, HW, C = 2, 80, 64
    wv = ops.pack_linear_weight(torch.randn(C, C, generator=gen) / C ** 0.5, 2)  # [2, 1, C, C]
    hn, bias = _planes(gen, (N, HW, C)), torch.randn(C, generator=gen)
    wv, hn, bias = wv.to(dev), hn.to(dev), bias.to(dev)
    kws = run(lambda: ops.bmm_nt(wv, hn, planes_out=True, bias_row=bias, a_bcast=True))
    pre, pb = _mm(_vals(wv, 3), _vals(hn, 3), 1.0, bias_row=bias)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=2)]


def _prod_bmm_qk_views(dev, run):
    """AttnBlock q k^T with q and k column views of the fused qk projection"""
    gen = torch.Generator().manual_seed(8)
    N, HW, C = 2, 80, 64
    qk = _planes(gen, (N, HW, 2 * C)).to(dev)
    q, k = qk[..., :C], qk[..., C:]
    kws = run(lambda: ops.bmm_nt(q, k))
    pre, pb = _mm(_vals(q, 3), _vals(k, 3), 1.0)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=0)]


def _prod_bmm_pv(dev, run):
    gen = torch.Generator().manual_seed(9)
    N, HW, C = 2, 80, 64
    p, vt = _planes(gen, (N, HW, HW), scale=0.1).to(dev), _planes(gen, (N, C, HW)).to(dev)
    kws = run(lambda: ops.bmm_nt(p, vt, planes_out=True))
    pre, pb = _mm(_vals(p, 3), _vals(vt, 3), 1.0)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=2)]


def _prod_bmm_index_pred(dev, run):
    """index-prediction heads: A is the permuted [T, G, M, ch] view of [T, M, G*ch] (group stride ch < row stride
    G ch), a bias vector per group; 18 classes take the direct epilogue"""
    gen = torch.Generator().manual_seed(10)
    G, M, ch, ncls = 3, 150, 32, 18
    y = _planes(gen, (M, G * ch)).to(dev)
    a = y.view(2, M, G, ch).permute(0, 2, 1, 3)
    w1 = _planes(gen, (G, ncls, ch)).to(dev)
    b1 = torch.randn(G, ncls, generator=gen).to(dev)
    kws = run(lambda: ops.bmm_nt(a, w1, bias_col=b1))
    pre, pb = _mm(_vals(a, 3), _vals(w1, 3), 1.0)
    pre, pb = pre + b1.double().unsqueeze(1), pb + b1.double().abs().unsqueeze(1)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=0)]


def _prod_bmm_heads(dev, run):
    """the sampler's per-head logits: hf grouped by head [T, nh, rows, C] against each head's weight"""
    gen = torch.Generator().manual_seed(11)
    nh, rows, C, ncls = 3, 70, 64, 40
    hf = _planes(gen, (nh * rows, C)).to(dev)
    w = _planes(gen, (nh, ncls, C), scale=C ** -0.5).to(dev)
    kws = run(lambda: ops.bmm_nt(hf.view(2, nh, rows, C), w))
    pre, pb = _mm(_vals(hf, 3).view(nh, rows, C), _vals(w, 3), 1.0)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=0)]


def _heads(x, B, Tn, nh):
    """[B Tn, C] -> [B, nh, Tn, hs]"""
    return x.reshape(B, Tn, nh, -1).permute(0, 2, 1, 3)


def _prod_mha_scores(dev, run):
    gen = torch.Generator().manual_seed(12)
    B, Tn, nh, C = 2, 96, 2, 64
    qkv = _planes(gen, (B * Tn, 3 * C)).to(dev)
    kws = run(lambda: ops.mha_scores(qkv[:, :, :C], B, Tn, nh, alpha=0.125, k=qkv[:, :, C:2 * C]))
    v = _vals(qkv, 3)
    pre, pb = _mm(_heads(v[:, :C], B, Tn, nh), _heads(v[:, C:2 * C], B, Tn, nh), 0.125)
    return kws, [dict(out=run.outputs[-1], ref=pre, B=pb, planes=0)]


def _pv_ref(p, v, B, Tn, nh, alpha, p_mn):
    """y[b Tn + i, h hs + d] = alpha sum_j p[b, h, i, j] v[b Tn + j, h hs + d] (p^T with p_mn)"""
    pv = p.transpose(-1, -2) if p_mn else p
    vh = _heads(v, B, Tn, nh)
    y, yb = alpha * pv @ vh, abs(alpha) * pv.abs() @ vh.abs()
    back = lambda t: t.permute(0, 2, 1, 3).reshape(B * Tn, -1)  # noqa: E731
    return back(y), back(yb)


def _prod_mha_pv_vtok(dev, run):
    """att v with v a column view of qkv, token-major (MN-major B); hs = 16 forces BN 64"""
    gen = torch.Generator().manual_seed(13)
    B, Tn, nh, C = 2, 96, 4, 64
    p = _planes(gen, (B, nh, Tn, Tn), scale=0.1).to(dev)
    qkv = _planes(gen, (B * Tn, 3 * C)).to(dev)
    kws = run(lambda: ops.mha_pv(p, qkv[:, :, 2 * C:], B, Tn, nh, v_tok=True))
    ref, bb = _pv_ref(_vals(p, 3), _vals(qkv, 3)[:, 2 * C:], B, Tn, nh, 1.0, False)
    return kws, [dict(out=run.outputs[-1], ref=ref, B=bb, planes=2)]


def _prod_mha_pv_backward(dev, run):
    """the attention backward's three products into column slices of d_qkv: dV = P^T dY (p_mn), dQ = dS K / DS and
    dK = dS^T Q / DS (p_mn), K and Q column views of qkv"""
    gen = torch.Generator().manual_seed(14)
    B, Tn, nh, C, DS = 2, 96, 2, 64, 1024.0
    p = _planes(gen, (B, nh, Tn, Tn), scale=0.1).to(dev)
    dsp = _planes(gen, (B, nh, Tn, Tn), scale=30.0).to(dev)
    dy = _planes(gen, (B * Tn, C)).to(dev)
    qkv = _planes(gen, (B * Tn, 3 * C)).to(dev)
    dbuf = torch.full((B * Tn + 2, 3 * C + 16), SENTINEL, device=dev)
    d_qkv = dbuf[:B * Tn, 8:8 + 3 * C]
    q, k = qkv[:, :, :C], qkv[:, :, C:2 * C]

    def go():
        ops.mha_pv(p, dy, B, Tn, nh, planes_out=False, out=d_qkv[:, 2 * C:], p_mn=True, v_tok=True)
        ops.mha_pv(dsp, k, B, Tn, nh, planes_out=False, out=d_qkv[:, :C], alpha=1.0 / DS, v_tok=True)
        ops.mha_pv(dsp, q, B, Tn, nh, planes_out=False, out=d_qkv[:, C:2 * C], alpha=1.0 / DS, p_mn=True,
                   v_tok=True)

    kws = run(go)
    qv = _vals(qkv, 3)
    rv, bv = _pv_ref(_vals(p, 3), _vals(dy, 3), B, Tn, nh, 1.0, True)
    rq, bq = _pv_ref(_vals(dsp, 3), qv[:, C:2 * C], B, Tn, nh, 1.0 / DS, False)
    rk, bk = _pv_ref(_vals(dsp, 3), qv[:, :C], B, Tn, nh, 1.0 / DS, True)
    return kws, [dict(buf=dbuf, region=(slice(0, B * Tn), slice(8, 8 + 3 * C)), ref=torch.cat((rq, rk, rv), 1),
                      B=torch.cat((bq, bk, bv), 1), planes=0)]


PROD = {
    "linear-residual": _prod_linear_residual,
    "linear-planes-gelu": _prod_linear_planes_gelu,
    "linear-w-kn": _prod_linear_w_kn,
    "linear-ksplit-residual-stream": _prod_linear_ksplit_residual_stream,
    "linear-partials": _prod_linear_partials,
    "wgrad-ksplit-accumulate": _prod_wgrad,
    "bmm-attnblock-v": _prod_bmm_attnblock_v,
    "bmm-qk-column-views": _prod_bmm_qk_views,
    "bmm-pv": _prod_bmm_pv,
    "bmm-index-pred-bias-col": _prod_bmm_index_pred,
    "bmm-heads": _prod_bmm_heads,
    "mha-scores-qk-views": _prod_mha_scores,
    "mha-pv-v-tok": _prod_mha_pv_vtok,
    "mha-pv-backward-slices": _prod_mha_pv_backward,
}


class _Runner:
    """run(fn): the wrapper call(s) of a production case under _Capture; keeps fn's return value in outputs"""

    def __init__(self, dry):
        self.dry, self.outputs = dry, []

    def __call__(self, fn):
        with _Capture(self.dry) as cap:
            self.outputs.append(fn())
            if self.dry:
                self.kws = cap.kws
                raise _DryRun
        return cap.kws


def _prod_kws_cpu(name):
    run = _Runner(dry=True)
    with pytest.raises(_DryRun):
        PROD[name]("cpu", run)
    return run.kws


# ------------------------------------------------------------------ coverage of the case table (CPU)
def test_row_case_table_covers_every_path():
    """every column tile, epilogue, output form, operand form, bias, activation, product count, ragged shape,
    split-K form and production flag combination has a case, and every refusal case is refused by the rules"""
    abi = [(s, _features(_build(s, "cpu").kw)) for s in CASES]
    prod = [(name, f) for name in PROD for f in map(_features, _prod_kws_cpu(name))]
    rows = [f for _, f in abi] + [f for _, f in prod]
    assert all("refused" not in f and "spatial" not in f for f in rows), [f for f in rows if "BN" not in f]
    has = lambda pred: any(pred(f) for f in rows)  # noqa: E731
    lv = lambda key, src=rows: {f[key] for f in src}  # noqa: E731
    # column tiles, incl. BN 64 forced by an MN-major B at n_out <= 32 (the hs = 16 mha_pv(v_tok=True) launch)
    assert lv("BN") >= {16, 32, 64, 128}
    assert has(lambda f: f["BN"] == 64 and f["b_mn"] and f["N"] <= 32)
    assert any(f["BN"] == 64 and f["N"] == 16 and f["b_mn"] for _, f in prod)
    # epilogues; the direct one for fp32 n_out % 4, planes n_out % 8, a misaligned slice and a misaligned bias
    assert lv("epi") >= {"direct", "tma_f32", "plain_f32", "tma_planes"}
    direct = [(s, f) for s, f in abi if f["epi"] == "direct"]
    assert any(f["out"] == "f32" and f["N"] % 4 for _, f in direct)
    assert any(f["out"] != "f32" and f["N"] % 8 for _, f in direct)
    assert any(s.c0 % 4 for s, _ in direct) and any(s.b_off % 4 for s, _ in direct)
    # output planes
    for out in ("p1", "p2"):
        assert has(lambda f: f["out"] == out and f["n"] == 1) and has(lambda f: f["out"] == out and f["n"] > 1), out
    # operand forms
    for am in (0, 1):
        for bm in (0, 1):
            assert has(lambda f: (f["a_mn"], f["b_mn"]) == (am, bm)), (am, bm)
    assert has(lambda f: f["a_bcast"] and f["n"] > 1) and has(lambda f: f["b_batched"] and f["n"] > 1)
    assert has(lambda f: f["b_bh"] and f["n"] > 1 and f["H"] > 1)
    # bias
    assert lv("bias") >= {"none", "col", "img", "row"}
    assert has(lambda f: f["bias"] == "img" and f["epi"] == "plain_f32")
    assert has(lambda f: f["bias"] == "img" and f["epi"] == "direct")
    assert has(lambda f: f["bias"] == "row" and f["H"] == 1) and has(lambda f: f["bias"] == "row" and f["H"] > 1
                                                                      and f["tile_rows"])
    # activations on a TMA epilogue and on the direct one; residual; alpha
    for act in ("none", "gelu", "relu", "lrelu"):
        assert has(lambda f: f["act"] == act and f["epi"] in ("tma_f32", "tma_planes")), act
        assert has(lambda f: f["act"] == act and f["epi"] == "direct"), act
    assert has(lambda f: f["res"]) and has(lambda f: f["alpha"] != 1.0)
    assert has(lambda f: f["alpha"] != 1.0 and f["epi"] == "direct")
    # products: 1 and 3, and the mixed fallback (2-plane A, 1-plane B: hi.hi)
    assert lv("planes") >= {(1, 1), (2, 2), (2, 1)}
    # ragged shapes
    assert has(lambda f: f["M"] % 128 == 0) and has(lambda f: f["M"] % 128 and f["M"] > 128)
    assert has(lambda f: f["M"] < 64) and has(lambda f: f["M"] == 1)
    assert has(lambda f: f["N"] % f["BN"])
    assert has(lambda f: f["K"] == 8) and has(lambda f: f["K"] % 64) and has(lambda f: f["K"] >= 4096)
    # split-K: even, uneven (last slice shorter), beyond kchunks; accumulate alone and with k_split; fewer slabs
    red = [f for f in rows if f["store"] == "reduce"]
    kch = lambda f: _cdiv(f["K"], 64)  # noqa: E731
    assert any(f["ks"] > 1 and kch(f) % f["kper"] == 0 for f in red)
    assert any(f["ks"] > 1 and kch(f) % f["kper"] for f in red)
    assert any(f["ks"] > kch(f) for f in red)
    assert any(f["acc"] and f["ks"] < 2 for f in red) and any(f["acc"] and f["ks"] > 1 for f in red)
    assert any(f["store"] == "slabs" and f["slices"] < f["kp"] for f in rows)
    assert any(f["store"] == "slabs" for _, f in prod)
    # bias with split-K on both fp32 TMA epilogues (the first k-slice carries it)
    assert any(f["bias"] in ("col", "img") and f["ks"] > 1 and f["epi"] == "plain_f32" for f in red)
    assert any(f["bias"] == "col" and f["ks"] > 1 and f["epi"] == "tma_f32" for f in red)
    assert any(f["bias"] == "img" and f["ks"] > 1 for f in red)
    # production combinations: every flag combination the wrappers use has a case
    assert set(PROD) >= {"linear-residual", "linear-planes-gelu", "linear-w-kn", "linear-ksplit-residual-stream",
                         "linear-partials", "wgrad-ksplit-accumulate", "bmm-attnblock-v", "bmm-qk-column-views",
                         "bmm-pv", "bmm-index-pred-bias-col", "bmm-heads", "mha-scores-qk-views", "mha-pv-v-tok",
                         "mha-pv-backward-slices"}
    pf = dict(prod)
    assert pf["linear-residual"]["res"] and pf["linear-planes-gelu"]["act"] == "gelu"
    assert pf["linear-w-kn"]["b_mn"] and pf["linear-ksplit-residual-stream"]["store"] == "reduce"
    assert pf["wgrad-ksplit-accumulate"]["acc"] and pf["wgrad-ksplit-accumulate"]["ks"] > 1
    assert pf["bmm-attnblock-v"]["a_bcast"] and pf["bmm-attnblock-v"]["bias"] == "row"
    assert pf["bmm-index-pred-bias-col"]["bias"] == "img"
    bwd = [f for n, f in prod if n == "mha-pv-backward-slices"]
    assert {(f["a_mn"], f["alpha"] != 1.0) for f in bwd} == {(1, False), (0, True), (1, True)}
    # refusals
    for s in REFUSED:
        assert "refused" in _label(s), (s.name, _label(s))


# ------------------------------------------------------------------ checks shared by the GPU tests
def _check(got, ref, B, what, rel=K_REL, tol=K_TOL):
    """|got - ref| <= tol B + rel |ref| element by element (NaN fails); prints and returns the worst err / B"""
    err = (got.double() - ref).abs()
    worst = (err / B.clamp_min(1e-30)).max().item() if err.numel() else 0.0
    print(f"{what}: worst err/B = {worst:.3g}")
    bad = ~(err <= tol * B + rel * ref.abs())
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound, first at "
                           f"{tuple(bad.nonzero()[0].tolist())}, worst err/B {worst:.3g}")
    return worst


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _sentinel_kept(buf, inside, what):
    sent = torch.full((), SENTINEL, dtype=buf.dtype, device=buf.device)
    stray = _bits(buf)[~inside] != _bits(sent)
    assert not stray.any(), f"{what}: {int(stray.sum())} stray writes outside the destination"


def _check_out(got, ref, B, planes, what):
    """fp32, one fp16 plane or two (a nearest split) against ref"""
    if planes == 0:
        return _check(got, ref, B, what)
    from test_gpu_row_kernels import _nearest
    assert torch.isfinite(got).all(), f"{what}: non-finite planes"
    if planes == 2:
        _nearest(got, 2, what)
        return _check(got.double().sum(0), ref, B, what)
    # one plane: its 11-bit rounding and the fp16 subnormal spacing
    return _check(got[0], ref, B + 2.0 ** -24 / K_TOL, what, rel=2.0 ** -11)


def _launch_rc(kw):
    """t2h_tapgemm's return code for ops._tapgemm arguments (no exception on refusal)"""
    rcs = []
    real = ops._launch
    ops._launch = lambda fn, p, algo, shape: rcs.append(fn(ctypes.byref(p), ops._stream()))
    try:
        ops._tapgemm(**kw)
    finally:
        ops._launch = real
    return rcs[0]


# ------------------------------------------------------------------ GPU: ABI cases
def _abi_ref(c, s, k0=0, k1=None):
    """alpha A.B over contractions [k0, k1) plus the column / row bias, and its magnitude bound"""
    av, bv = c.av[..., k0:k1].to(c.dbuf.device), c.bv[..., k0:k1].to(c.dbuf.device)
    pre = s.alpha * torch.einsum("ihwk,ihnk->ihwn", av, bv)
    pb = abs(s.alpha) * torch.einsum("ihwk,ihnk->ihwn", av.abs(), bv.abs())
    if c.bvals is not None:
        bvals = c.bvals.to(pre.device)
        pre, pb = pre + bvals, pb + bvals.abs()
    return pre, pb


@pytest.mark.gpu
@pytest.mark.parametrize("s", CASES, ids=lambda s: s.name)
def test_row_gemm_case_matches_fp64(cuda, s):
    """one row-mode launch of the case table against fp64 on the planes' values, element by element; nothing
    outside the destination changes; a stored launch repeats bit for bit, a reduce-add launch adds once per launch"""
    c = _build(s, cuda)
    route = _route_of(c.kw)
    assert route == _label(s), (route, _label(s))
    what = f"{s.name} [BN{route['BN']} {route['epi']} {route['store']} x{route['slices']}]"
    inside = torch.zeros(c.dbuf.shape, dtype=torch.bool, device=cuda)
    pl = (slice(0, c.planes),) if c.planes else ()
    if route["store"] == "slabs":
        ops._tapgemm(**c.kw)
        kper, S = route["kper"], route["slices"]
        inside[(slice(0, S),) + c.region[1:]] = True
        for sl in range(S):
            pre, pb = _abi_ref(c, s, sl * kper * 64, min(s.K, (sl + 1) * kper * 64))
            _check(c.dbuf[(slice(sl, sl + 1),) + c.region[1:]], pre, pb, f"{what} slab {sl}")
        _sentinel_kept(c.dbuf, inside, what)  # incl. the guard slab after the last one
        return
    inside[pl + c.region] = True
    pre, pb = _abi_ref(c, s)
    ref, B = _act(pre, s.act), pb * (GELU_SLOPE if s.act == "gelu" else 1.0)
    if c.rv is not None:
        ref, B = ref + c.rv, B + c.rv.abs()
    ops._tapgemm(**c.kw)
    got = c.dbuf[pl + c.region]
    if route["store"] == "reduce":
        d0 = c.d0.to(cuda).double()
        _check_out(got, d0 + ref, B + d0.abs(), c.planes, what)
        ops._tapgemm(**c.kw)  # the second launch adds P again, column bias included
        _check_out(got, d0 + 2 * ref, 2 * B + d0.abs(), c.planes, what + " twice")
    else:
        _check_out(got, ref, B, c.planes, what)
        first = c.dbuf.clone()
        ops._tapgemm(**c.kw)
        assert torch.equal(_bits(c.dbuf), _bits(first)), f"{what}: a second launch wrote different bits"
    _sentinel_kept(c.dbuf, inside, what)


def _act(y, act):
    if act == "relu":
        return y.clamp_min(0)
    if act == "lrelu":
        return torch.where(y > 0, y, 0.2 * y)
    if act == "gelu":
        return torch.nn.functional.gelu(y)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("s", REFUSED, ids=lambda s: s.name)
def test_row_gemm_refusal_leaves_d_unchanged(cuda, s):
    """argument and tensor-map checks on the host: T2H_EINVAL, nothing launched, D keeps its contents"""
    c = _build(s, cuda)
    assert "refused" in _route_of(c.kw)
    before = c.dbuf.clone()
    rc = _launch_rc(c.kw)
    torch.cuda.synchronize()
    assert rc == EINVAL, (rc, _lib.load().t2h_last_error().decode())
    assert torch.equal(_bits(c.dbuf), _bits(before)), f"{s.name}: refused launch changed D"


# ------------------------------------------------------------------ GPU: production combinations
def _guarded_relaunch(kw, what):
    """the captured launch again, its wrapper-allocated (contiguous) output replaced by the same shape inside a
    sentinel-filled buffer with guards before and after: the guards keep their bits, the output repeats bit for bit"""
    d = kw["d"]
    assert d.is_contiguous()
    n = d.numel()
    gbuf = torch.full((3 * n,), SENTINEL, dtype=d.dtype, device=d.device)
    d2 = gbuf[n:2 * n].view(d.shape)
    ops._tapgemm(**dict(kw, d=d2))
    inside = torch.zeros_like(gbuf, dtype=torch.bool)
    inside[n:2 * n] = True
    _sentinel_kept(gbuf, inside, what + " (relaunch)")
    assert torch.equal(_bits(d2), _bits(d)), f"{what}: the relaunch wrote different bits"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PROD))
def test_row_gemm_production_matches_fp64(cuda, name):
    """the wrappers' production flag combinations against fp64 of what they compute, launch by launch on the
    paths the CPU coverage test counted them on"""
    run = _Runner(dry=False)
    kws, checks = PROD[name](cuda, run)
    routes = [_route_of(kw) for kw in kws]
    assert routes == [_route_of(kw) for kw in _prod_kws_cpu(name)], routes
    what = f"{name} [" + "; ".join(f"BN{r['BN']} {r['epi']} {r['store']} x{r['slices']}" for r in routes) + "]"
    for ck in checks:
        if "out" in ck:  # allocated by the wrapper
            got, d0 = ck["out"], None
        else:
            got, d0 = ck["buf"][ck["region"]], ck.get("d0")
        if d0 is not None:
            _check_out(got, d0 + ck["ref"], ck["B"] + d0.abs(), ck["planes"], what)
        else:
            _check_out(got, ck["ref"], ck["B"], ck["planes"], what)
        if "buf" in ck:
            inside = torch.zeros(ck["buf"].shape, dtype=torch.bool, device=cuda)
            inside[ck["region"]] = True
            _sentinel_kept(ck["buf"], inside, what)
    for kw, r in zip(kws, routes):
        if "out" in checks[0] and r["store"] != "reduce":
            _guarded_relaunch(kw, what)


# ------------------------------------------------------------------ the operands these GEMMs consume
def _split_ref(x, scale, terms):
    """hi = fp16_rn(fl32(scale x)), lo = fp16_rn(v - hi) (the subtraction exact in fp32)"""
    v = x * scale
    hi = v.half()
    lo = (v - hi.float()).half()
    return torch.stack((hi, lo))[:terms]


F2P_CASES = [  # (G, R, C, terms, scale, outputs)
    (1, 67, 45, 2, 1.0, "both"),
    (3, 64, 128, 2, 2.0 ** 10, "both"),
    (2, 33, 64, 1, 2.0 ** -3, "t"),
    (1, 128, 63, 2, 4.0, "n"),
    (2, 65, 130, 2, 2.0 ** 12, "t"),
    (1, 1, 7, 2, 1.0, "both"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("G,R,C,terms,scale,outs", F2P_CASES, ids=lambda v: str(v))
def test_f32_to_planes_t_bit_exact(cuda, G, R, C, terms, scale, outs):
    """t2h_f32_to_planes_t: hi == fp16_rn(fl32(scale x)) and lo == fp16_rn(v - hi) bit for bit, untransposed and
    transposed, on the vector and the scalar tail paths (odd R / C); the guard elements after each output stay"""
    gen = torch.Generator().manual_seed(G * 1000 + R * 10 + C)
    # magnitudes from 2^-24 (fp16 subnormals) to 2^4 after scaling: power-of-two scales keep v = scale x exact
    x = torch.randn(G, R, C, generator=gen) * 2.0 ** torch.randint(-24, 4, (G, R, C), generator=gen).float() / scale
    x[0, 0, :min(C, 3)] = torch.tensor([0.0, -0.0, 1.0 / 3.0])[:min(C, 3)] / scale
    want = _split_ref(x, scale, terms)  # [terms, G, R, C]
    n = terms * G * R * C
    guard = 64
    buf_t = torch.full((n + guard,), SENTINEL, dtype=torch.float16, device=cuda)
    buf_n = torch.full((n + guard,), SENTINEL, dtype=torch.float16, device=cuda)
    out_t = buf_t[:n] if outs in ("t", "both") else None
    out_n = buf_n[:n] if outs in ("n", "both") else None
    xd = x.to(cuda)
    p = lambda t: ctypes.c_void_p(0 if t is None else t.data_ptr())  # noqa: E731
    rc = _lib.load().t2h_f32_to_planes_t(p(xd), p(out_t), p(out_n), G, R, C, terms, scale, ops._stream())
    assert rc == 0, _lib.load().t2h_last_error().decode()
    wb = _bits(want).to(cuda)
    sent = _bits(torch.full((guard,), SENTINEL, dtype=torch.float16, device=cuda))
    for buf, used, ref in ((buf_n, out_n, wb), (buf_t, out_t, wb.transpose(-1, -2))):
        if used is None:
            assert torch.equal(_bits(buf), _bits(torch.full_like(buf, SENTINEL))), "unrequested output written"
            continue
        got = _bits(buf[:n]).view(terms, G, *ref.shape[-2:])
        bad = got != ref
        assert not bad.any(), f"{int(bad.sum())} planes elements differ, first at {tuple(bad.nonzero()[0].tolist())}"
        assert torch.equal(_bits(buf[n:]), sent), "guard elements after the planes were written"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["odd-ld-column-views", "into-wider-buffer"])
def test_planes_transpose_views(cuda, kind):
    """t2h_planes_transpose from and into column-sliced views: an odd ld turns the 4-byte path off; an output in the
    middle of a wider buffer keeps every element outside its slice"""
    gen = torch.Generator().manual_seed(len(kind))
    T, G, R, C = 2, 3, 130, 70
    src = torch.randn(T, G, R, C, generator=gen).half().to(cuda)
    if kind == "odd-ld-column-views":
        xbuf = torch.full((T, G, R, C + 7), SENTINEL, dtype=torch.float16, device=cuda)  # ld 77
        xbuf[..., 3:3 + C] = src
        x = xbuf[..., 3:3 + C]
        obuf = torch.full((T, G, C, R + 5), SENTINEL, dtype=torch.float16, device=cuda)  # ld 135
        out = obuf[..., 1:1 + R]
        region = (Ellipsis, slice(1, 1 + R))
    else:
        x = src
        obuf = torch.full((T, G, C + 4, R + 16), SENTINEL, dtype=torch.float16, device=cuda)
        out = obuf[:, :, 2:2 + C, 8:8 + R]
        region = (slice(None), slice(None), slice(2, 2 + C), slice(8, 8 + R))
    xb = _bits(x).clone()
    ops.planes_transpose(x, out=out)
    assert torch.equal(_bits(out), _bits(src.transpose(-1, -2))), f"{kind}: transposed planes differ"
    assert torch.equal(_bits(x), xb)
    inside = torch.zeros(obuf.shape, dtype=torch.bool, device=cuda)
    inside[region] = True
    _sentinel_kept(obuf, inside, kind)
