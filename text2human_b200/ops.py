"""Thin torch-tensor wrappers over the libt2h C ABI.

PyTorch is only plumbing here: device memory (``torch.empty``) and the current
CUDA stream.  Every numerical operation is a libt2h kernel; a missing library
or a non-CUDA tensor raises instead of falling back.

"planes" tensors are ``torch.float16`` tensors whose leading dim is the number
of split terms T (1 = TF32-like fast mode, 2 = hi/lo pair for fp32-equivalent
3-product contractions); the remaining dims are the logical NHWC / matrix dims.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_GELU, ACT_LRELU, ACT_NONE, ACT_RELU, CVT_BILINEAR2X, CVT_MAXPOOL2, BIAS_COL, BIAS_NONE, BIAS_ROW, CVT_PLAIN, CVT_S2D, CVT_UP2X,
                   OUT_F32, OUT_PLANES, TapGemmParams)

# ----------------------------------------------------------------------------
# precision policy
# ----------------------------------------------------------------------------
_PRECISION = {"terms": 2, "mixed": False}


def set_precision(mode):
    """"fp32" : hi/lo fp16 planes, 3 tensor-core products per contraction
    (fp32-equivalent; the parity mode).  "fp16": single fp16 plane, one product
    (10-bit mantissa operands like TF32, fp32 accumulate; the fast mode).
    "mixed": as "fp32", except that the layers the per-layer precision map clears (tools/precision_map.py: the six
    128-channel 3x3 convs of the decoder's full-resolution level, 30 % of all conv FLOPs) run single-product --
    decoder pixels stay within 1e-3 of the fp32 reference (tests/test_gpu_baseline_configs.py), the encoder and
    therefore the codebook indices are untouched."""
    _PRECISION["mixed"] = False
    if mode in ("fp32", "fp16x3", "exact"):
        _PRECISION["terms"] = 2
    elif mode in ("fp16", "fast", "tf32"):
        _PRECISION["terms"] = 1
    elif mode == "mixed":
        _PRECISION["terms"] = 2
        _PRECISION["mixed"] = True
    else:
        raise ValueError(f"unknown precision mode {mode!r}")


def layer_terms(mod):
    """planes per operand for one conv module: 1 where the mixed map marks the layer single-product"""
    if _PRECISION["mixed"] and getattr(mod, "_t2h_single", False):
        return 1
    return _PRECISION["terms"]


def get_terms():
    return _PRECISION["terms"]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ----------------------------------------------------------------------------
# launch accounting (bench.py reads these; not used for control flow)
# ----------------------------------------------------------------------------
COUNTERS = {"launches": 0}
_PROFILE = {"on": False, "records": []}


def _count(n=1):
    COUNTERS["launches"] += n


def profile_tapgemm(on):
    """When on, every t2h_tapgemm launch is bracketed by CUDA events on the launching stream and
    recorded as (algorithmic_flops, issued_flops, start_event, end_event, (n_img, H, W, n_out, K))."""
    _PROFILE["on"] = bool(on)
    _PROFILE["records"] = []


def profile_records():
    return _PROFILE["records"]


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.T2HError("text2human_b200 kernels need CUDA tensors; there is no CPU path")


def _f32c(t):
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


# ----------------------------------------------------------------------------
# the tensor-core contraction
# ----------------------------------------------------------------------------
_TAPS_1 = ((0, 0, 0),)
_TAPS_3x3 = tuple((kh - 1, kw - 1, 0) for kh in range(3) for kw in range(3))


def _tapgemm(*, a, a_term_imgs, a_imgs, a_bcast, n_img, H, W, a_H, a_W, Cc, a_sw, a_sh, a_sn,
             b, b_term_g, b_groups, b_batched, n_out, b_sn, b_sg, taps, d, d_mode, d_strides,
             d_plane=0, bias=None, bias_mode=BIAS_NONE, act=ACT_NONE, alpha=1.0, residual=None,
             tile_rows=0, b_groups2=1, b_sg2=0, b_batched_h=0, gn_stats=None, gn_cpg=0, k_split=0, bias_sn=0, a_mn=0, b_mn=0,
             tap_w=None, accumulate=False, k_partials=0, d_slab=0, nb=None):
    lib = _lib.load()
    Tb = b.shape[0]
    p = TapGemmParams()
    T = a.shape[0]
    p.a = a.data_ptr(); p.a_terms = T; p.a_term_imgs = a_term_imgs; p.a_imgs = a_imgs
    p.a_bcast = a_bcast
    p.n_img, p.H, p.W, p.a_H, p.a_W, p.C = n_img, H, W, a_H, a_W, Cc
    p.tile_rows = tile_rows
    p.a_sw, p.a_sh, p.a_sn = a_sw, a_sh, a_sn
    p.b = b.data_ptr(); p.b_terms = Tb; p.b_term_g = b_term_g; p.b_groups = b_groups
    p.b_batched = b_batched; p.n_out = n_out; p.b_sn = b_sn; p.b_sg = b_sg
    p.b_groups2 = b_groups2; p.b_sg2 = b_sg2 if b_groups2 > 1 else b_sg; p.b_batched_h = b_batched_h
    p.ntaps = len(taps)
    for i, (dy, dx, off) in enumerate(taps):
        p.tap_dy[i], p.tap_dx[i], p.tap_img_off[i] = dy, dx, off
    p.nterms = 3 if (T == 2 and Tb == 2) else 1
    p.d = d.data_ptr(); p.d_mode = d_mode
    p.d_terms = d.shape[0] if d_mode == OUT_PLANES else 0
    p.d_plane = d_plane
    p.d_sn, p.d_sh, p.d_sw, p.d_sc = d_strides
    p.bias = bias.data_ptr() if bias is not None else None
    p.bias_mode = bias_mode if bias is not None else BIAS_NONE
    p.act = act
    p.alpha = alpha
    p.residual = residual.data_ptr() if residual is not None else None
    p.gn_stats = gn_stats.data_ptr() if gn_stats is not None else None
    p.gn_cpg = gn_cpg if gn_stats is not None else 0
    p.k_split = k_split
    p.bias_sn = bias_sn
    p.a_mn, p.b_mn = a_mn, b_mn
    p.accumulate = 1 if accumulate else 0
    p.k_partials, p.d_slab = k_partials, d_slab
    if nb is not None:
        # norm-backward pass 1 in the epilogue: `residual` carries x (not added), see nb_context
        assert residual is None
        p.residual = nb["x"].data_ptr()
        p.nb_sums = nb["sums"].data_ptr(); p.nb_stats = nb["stats"].data_ptr()
        p.nb_gamma = nb["gamma"].data_ptr(); p.nb_beta = nb["beta"].data_ptr()
        p.nb_eps = nb["eps"]; p.nb_act = ACT_CODE[nb["act"]]; p.nb_groups = nb["groups"]
    if tap_w is not None:
        p.use_tap_w = 1
        for i, wi in enumerate(tap_w):
            p.tap_w[i] = wi
    _launch(lib.t2h_tapgemm, p, 2.0 * n_img * H * W * n_out * Cc * len(taps), (n_img, H, W, n_out, Cc * len(taps)))


def _launch(fn, p, algo, shape):
    """count one launch of ``fn(p)``; with profile_tapgemm on, bracket it with CUDA events and record it"""
    _count()
    if not _PROFILE["on"]:
        _lib.check(fn(C.byref(p), _stream()))
        return
    e0 = torch.cuda.Event(enable_timing=True)
    e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(fn(C.byref(p), _stream()))
    e1.record()
    _PROFILE["records"].append((algo, algo * p.nterms, e0, e1, shape))


def _alloc_out(shape, planes, terms, device):
    if planes:
        return torch.empty((terms,) + tuple(shape), dtype=torch.float16, device=device)
    return torch.empty(tuple(shape), dtype=torch.float32, device=device)


GN_GROUPS = 32


_ARENA = {"buf": None, "next": 0, "n": 0}


class stats_arena:
    """Context manager: all GroupNorm-statistics accumulators of one forward pass come out of ONE buffer zeroed by a
    single fill, instead of one ``torch.zeros`` launch per convolution (~80 per step).  Not re-entrant; one stream."""

    def __init__(self, n, device, slots=160):
        self.n, self.device, self.slots = n, device, slots

    def __enter__(self):
        buf = _ARENA["buf"]
        need = (self.slots, self.n, GN_GROUPS, 2)
        if buf is None or tuple(buf.shape) != need or buf.device != torch.device(self.device):
            buf = torch.zeros(need, dtype=torch.float64, device=self.device)
        else:
            buf.zero_()
        _ARENA.update(buf=buf, next=0, n=self.n, active=True)
        return self

    def __exit__(self, *exc):
        _ARENA["active"] = False


def new_gn_stats(n, device):
    """zeroed (sum, sumsq) accumulators [n, 32, 2] fp64 for a fused GroupNorm-statistics epilogue"""
    a = _ARENA
    if a.get("active") and a["n"] == n and a["next"] < a["buf"].shape[0] and a["buf"].device == torch.device(device):
        a["next"] += 1
        return a["buf"][a["next"] - 1]
    return torch.zeros((n, GN_GROUPS, 2), dtype=torch.float64, device=device)


def _stats_for(cout, n, device, want):
    """GroupNorm(32) statistics can ride in the epilogue when channels-per-group is a power of two >= 2"""
    cpg = cout // GN_GROUPS
    if not want or cout % GN_GROUPS != 0 or cpg < 2 or (cpg & (cpg - 1)) != 0:
        return None, 0
    return new_gn_stats(n, device), cpg


import os as _os_env


def conv3x3(a, w, bias, *, residual=None, planes_out=False, nchw_out=False, want_stats=False, taps=None,
            act=ACT_NONE):
    """3x3 stride-1 pad-1 conv (or, with taps=_TAPS_1 and a [T,1,Cout,C] weight, a 1x1 conv).
    a: planes [T,N,H,W,C]; w: packed planes [T,ntaps,Cout,C] (see pack_conv_weight); bias fp32 [Cout].
    Returns fp32 NHWC [N,H,W,Cout] (or NCHW with nchw_out) or planes [T,N,H,W,Cout]; with
    want_stats also the fused GroupNorm statistics of the fp32 output (or None if not applicable)."""
    taps = taps if taps is not None else _TAPS_3x3
    assert w.shape[1] == len(taps), (a.shape, w.shape)
    return tap_conv(a, w, bias, taps, n=a.shape[1], out_hw=a.shape[2:4], residual=residual, planes_out=planes_out,
                    nchw_out=nchw_out, want_stats=want_stats, act=act)


def pack_upsample_conv_weight(w, terms):
    """Weights of `nearest x2 upsample -> 3x3 conv` (Upsample, vqgan_arch.py:529-534) folded into four
    2x2 convs on the low-resolution input, one per output parity (a, b):
        out[2i+a, 2j+b] = sum_{r,s in 0..1} Wab[r,s] . in[i + a + r - 1, j + b + s - 1]
    with Wab[r,s] = sum of the 3x3 taps that read that input pixel (rows: a=0 -> {w0 | w1+w2},
    a=1 -> {w0+w1 | w2}; columns likewise).  36 tap-GEMMs at high resolution become 16 at low
    resolution (2.25x fewer FLOPs, 4x fewer activation bytes).  Returns planes [T, 16, Cout, Cin],
    tap index = ((a*2+b)*2 + r)*2 + s."""
    w = w.detach().float()
    Cout, Cin = w.shape[:2]
    rows = {0: (w[:, :, 0], w[:, :, 1] + w[:, :, 2]), 1: (w[:, :, 0] + w[:, :, 1], w[:, :, 2])}  # [Cout,Cin,3(kw)]
    taps = []
    for a in (0, 1):
        for b in (0, 1):
            for r in (0, 1):
                wr = rows[a][r]
                cols = (wr[:, :, 0], wr[:, :, 1] + wr[:, :, 2]) if b == 0 else (wr[:, :, 0] + wr[:, :, 1], wr[:, :, 2])
                for sidx in (0, 1):
                    taps.append(cols[sidx])
    wt = torch.stack(taps)  # [16, Cout, Cin]
    cp = (Cin + 7) // 8 * 8
    if cp != Cin:
        wt = torch.nn.functional.pad(wt, (0, cp - Cin))
    return split_planes(wt, terms)


def upsample_conv3x3(a, w16, bias, *, want_stats=False):
    """nearest x2 + 3x3 conv on low-resolution planes a [T,N,H,W,C] with pack_upsample_conv_weight()
    weights [T,16,Cout,C] -> fp32 NHWC [N,2H,2W,Cout] (+ fused GroupNorm statistics): four strided-output
    launches, one per output parity."""
    _need_cuda(a, w16)
    T, N, H, W, Cc = a.shape
    Cout = w16.shape[2]
    assert w16.shape[1] == 16 and w16.shape[3] == Cc
    H2, W2 = 2 * H, 2 * W
    out = torch.empty((N, H2, W2, Cout), dtype=torch.float32, device=a.device)
    stats, cpg = _stats_for(Cout, N, a.device, want_stats)
    for pa in (0, 1):
        for pb in (0, 1):
            par = pa * 2 + pb
            taps = tuple((pa + r - 1, pb + sidx - 1, 0) for r in (0, 1) for sidx in (0, 1))
            wv = w16[:, par * 4:(par + 1) * 4]  # [T,4,Cout,C] view: plane stride stays 16 taps
            dview = out[:, pa::2, pb::2, :]
            _tapgemm(a=a, a_term_imgs=N, a_imgs=T * N, a_bcast=0, n_img=N, H=H, W=W, a_H=H, a_W=W, Cc=Cc,
                     a_sw=Cc, a_sh=W * Cc, a_sn=H * W * Cc,
                     b=wv, b_term_g=16, b_groups=(w16.shape[0] - 1) * 16 + 4, b_batched=0, n_out=Cout, b_sn=Cc,
                     b_sg=Cout * Cc,
                     taps=taps, d=dview, d_mode=OUT_F32,
                     d_strides=(H2 * W2 * Cout, 2 * W2 * Cout, 2 * Cout, 1),
                     bias=bias, bias_mode=BIAS_COL, gn_stats=stats, gn_cpg=cpg)
    if want_stats:
        return out, stats
    return out


def conv1x1(a, w, bias, *, residual=None, planes_out=False, want_stats=False):
    """1x1 conv on planes [T,N,H,W,C] with a pack_linear_weight()-packed weight [T,1,Cout,C]; tiles stay
    inside one image so GroupNorm statistics can be fused."""
    return conv3x3(a, w, bias, residual=residual, planes_out=planes_out, want_stats=want_stats, taps=_TAPS_1)


def conv3x3_s2(a_ph, w, bias, *, want_stats=False):
    """Downsample conv: pad (0,1,0,1) then 3x3 stride 2 (vqgan_arch.py:547-551).
    a_ph: space-to-depth planes [T,4,N,Ho,Wo,C] from f32_to_planes(mode=S2D)."""
    from .conv_grad import fwd_taps  # conv_grad imports this module
    T, four, N, Ho, Wo, Cc = a_ph.shape
    assert four == 4
    return tap_conv(a_ph, w, bias, fwd_taps("down", N), n=N, out_hw=(Ho, Wo), want_stats=want_stats)


# Split-K GEMMs reduce their k-slices with fp32 atomics (TMA reduce-add), so their results depend on the
# arrival order at rounding level (~1e-7 relative).  Weight gradients use it by default (as cuDNN's wgrad
# does); inference stays bit-reproducible run to run unless the caller opts in.
SPLIT_K = {"wgrad": True, "inference": False, "small_batch": True}


def set_split_k(wgrad=None, inference=None, small_batch=None):
    """enable / disable the split-K paths; returns the previous settings.  ``wgrad`` / ``inference`` are the
    reduce-add (arrival-order) forms; ``small_batch`` is the deterministic stored-partials form the transformer
    uses when a projection has too few output tiles to fill the GPU."""
    old = dict(SPLIT_K)
    if small_batch is not None:
        SPLIT_K["small_batch"] = bool(small_batch)
    if wgrad is not None:
        SPLIT_K["wgrad"] = bool(wgrad)
    if inference is not None:
        SPLIT_K["inference"] = bool(inference)
    return old


def wgrad_k_split(M, Nout, K):
    """k-slices per output tile so that a GEMM with few [128 x 128] output tiles and a long contraction
    (weight gradients; proj / fc2 at small batch) fills the H100's 132 SMs; 0 when splitting does not pay"""
    tiles = ((M + 127) // 128) * ((Nout + 127) // 128)
    ks = min((K + 63) // 64, 132 // max(tiles, 1))
    return ks if ks >= 2 else 0


def linear(a, w, bias=None, *, residual=None, planes_out=False, act=ACT_NONE, alpha=1.0, out=None, k_split=0,
           w_kn=False):
    """a: planes [T,M,K] (any leading dims are flattened by the caller);
    w: planes [T,1,Nout,K] (pack_linear_weight).  -> fp32 [M,Nout] or planes [T,M,Nout].
    Serves 1x1 convs on NHWC activations and nn.Linear.  ``k_split`` >= 2 (small output, long contraction)
    ACCUMULATES into ``out``: out += alpha * a @ w^T (+ bias) -- a zeroed gradient buffer, or the residual stream."""
    assert k_split < 2 or (out is not None and residual is None and not planes_out)
    _need_cuda(a, w)
    T, M, K = a.shape
    if w_kn:
        # w: planes [T,1,K,Nout] -- the contraction index is the ROW of the stored matrix (e.g. the forward
        # weight [out,in] used for the data gradient dX = dY.W): consumed as an MN-major operand, no transpose
        Nout = w.shape[3]
        assert w.shape[2] == K and a.stride(2) == 1 and w.stride(3) == 1, (a.shape, w.shape)
    else:
        Nout = w.shape[2]
        assert w.shape[3] == K and a.stride(2) == 1, (a.shape, w.shape)
    if out is None:
        out = _alloc_out((M, Nout), planes_out, T, a.device)
    a_sw = a.stride(1)
    _tapgemm(a=a, a_term_imgs=1, a_imgs=T, a_bcast=0, n_img=1, H=1, W=M, a_H=1, a_W=M, Cc=K,
             a_sw=a_sw, a_sh=a.stride(0), a_sn=a.stride(0),
             b=w, b_term_g=1, b_groups=w.shape[0], b_batched=0, n_out=Nout, b_sn=w.stride(2),
             b_sg=w.stride(0),
             taps=_TAPS_1, d=out, d_mode=OUT_PLANES if planes_out else OUT_F32,
             d_strides=(0, 0, out.stride(-2), 1), d_plane=out.stride(0) if planes_out else 0,
             bias=bias, bias_mode=BIAS_COL, act=act, alpha=alpha, residual=residual, k_split=k_split,
             b_mn=1 if w_kn else 0)
    return out


def split_slices(K, k_partials):
    """number of k-slices t2h_tapgemm actually produces for a contraction of length K and a k_partials request"""
    kchunks = (K + 63) // 64
    ks = min(k_partials, kchunks)
    kper = (kchunks + ks - 1) // ks
    return (kchunks + kper - 1) // kper


def linear_partials(a, w, k_partials, alpha=1.0):
    """Deterministic split-K: the k-slices of a @ w^T are STORED to separate slabs -> fp32 [S, M, Nout]
    (S = split_slices(K, k_partials)); ``splitk_reduce_ln`` sums them in a fixed order."""
    _need_cuda(a, w)
    T, M, K = a.shape
    Nout = w.shape[2]
    assert w.shape[3] == K and a.stride(2) == 1
    S = split_slices(K, k_partials)
    out = torch.empty((S, M, Nout), dtype=torch.float32, device=a.device)
    _tapgemm(a=a, a_term_imgs=1, a_imgs=T, a_bcast=0, n_img=1, H=1, W=M, a_H=1, a_W=M, Cc=K,
             a_sw=a.stride(1), a_sh=a.stride(0), a_sn=a.stride(0),
             b=w, b_term_g=1, b_groups=w.shape[0], b_batched=0, n_out=Nout, b_sn=w.stride(2), b_sg=w.stride(0),
             taps=_TAPS_1, d=out, d_mode=OUT_F32, d_strides=(0, 0, Nout, 1), alpha=alpha,
             k_partials=k_partials, d_slab=M * Nout)
    return out


def splitk_reduce_ln(partials, bias, residual, gamma=None, beta=None, eps=1e-5, *, ln_out=None, row_map=None,
                     terms=None, want_ln=True):
    """x = residual + bias + sum_s partials[s] (fixed order) -> (x fp32 [M,C], LayerNorm(x) planes or None).
    ``ln_out`` / ``row_map``: scatter the normalised rows into an existing planes buffer [T, rows_out, C]."""
    _need_cuda(partials)
    S, M, Cc = partials.shape
    terms = terms or get_terms()
    x = torch.empty((M, Cc), dtype=torch.float32, device=partials.device)
    if want_ln and ln_out is None:
        ln_out = torch.empty((terms, M, Cc), dtype=torch.float16, device=partials.device)
    ln_rows = ln_out.shape[1] if ln_out is not None else 0
    _count(1)
    _lib.check(_lib.load().t2h_splitk_reduce_ln(_ptr(partials), S, M * Cc, _ptr(bias), _ptr(residual), _ptr(x),
                                                _ptr(gamma), _ptr(beta), eps, _ptr(ln_out) if want_ln else None,
                                                ln_out.shape[0] if ln_out is not None else terms, _ptr(row_map),
                                                ln_rows, M, Cc, _stream()))
    return x, (ln_out if want_ln else None)


def wgrad(dy, x, out, k_split=0, alpha=1.0, accumulate=False):
    """out[n_out, n_in] += alpha * dy^T @ x over the rows (tokens).  dy planes [T,M,n_out], x planes [T,M,n_in]
    exactly as the forward / backward passes hold them (row = token): both are consumed as MN-major operands,
    so no transposed copy exists.  With ``k_split`` >= 2 the token range is split over the SMs and reduce-added
    into ``out`` (which the caller zeroed); with 0 ``out`` is overwritten."""
    _need_cuda(dy, x, out)
    T, M, No = dy.shape
    Ni = x.shape[2]
    assert x.shape[:2] == dy.shape[:2] and dy.stride(2) == 1 and x.stride(2) == 1 and out.shape == (No, Ni)
    _tapgemm(a=dy, a_term_imgs=1, a_imgs=T, a_bcast=0, n_img=1, H=1, W=No, a_H=1, a_W=No, Cc=M,
             a_sw=dy.stride(1), a_sh=dy.stride(0), a_sn=dy.stride(0),
             b=x, b_term_g=1, b_groups=T, b_batched=0, n_out=Ni, b_sn=x.stride(1), b_sg=x.stride(0),
             taps=_TAPS_1, d=out, d_mode=OUT_F32, d_strides=(0, 0, out.stride(0), 1), alpha=alpha,
             k_split=k_split, a_mn=1, b_mn=1, accumulate=accumulate)
    return out


def bmm_nt(a, b, *, planes_out=False, alpha=1.0, bias_row=None, a_bcast=False, bias_col=None, act=ACT_NONE):
    """out[g] = a[g] @ b[g]^T.  a: planes [T,G,M,K] (or [T,1,M,K] with a_bcast);
    b: planes [T,G,N,K]; views with a unit last stride are accepted.
    -> fp32 [G,M,N] or planes [T,G,M,N].  bias_row fp32 [M] (shared) or bias_col fp32 [G,N] (per group)."""
    _need_cuda(a, b)
    T, Ga, M, K = a.shape
    Tb, G, N, Kb = b.shape
    assert K == Kb and a.stride(3) == 1 and b.stride(3) == 1
    assert (Ga == G) or (a_bcast and Ga == 1)
    out = _alloc_out((G, M, N), planes_out, T, a.device)
    a_sn = a.stride(1)
    a_term_imgs = 1 if T == 1 else a.stride(0) // a_sn
    assert T == 1 or a.stride(0) % a_sn == 0
    _tapgemm(a=a, a_term_imgs=a_term_imgs, a_imgs=(T - 1) * a_term_imgs + Ga, a_bcast=1 if a_bcast else 0,
             n_img=G, H=1, W=M, a_H=1, a_W=M, Cc=K, a_sw=a.stride(2), a_sh=a_sn, a_sn=a_sn,
             b=b, b_term_g=1, b_groups=Tb, b_sg=b.stride(0), b_groups2=G, b_sg2=b.stride(1), b_batched=1,
             n_out=N, b_sn=b.stride(2),
             taps=_TAPS_1, d=out, d_mode=OUT_PLANES if planes_out else OUT_F32,
             d_strides=(M * N, 0, N, 1), d_plane=G * M * N,
             bias=bias_row if bias_col is None else bias_col,
             bias_mode=BIAS_ROW if bias_col is None else BIAS_COL,
             bias_sn=0 if bias_col is None else N, alpha=alpha, act=act)
    return out


def mha_scores(q, B, Tn, nh, alpha=1.0, k=None):
    """Multi-head q @ k^T without head transposes (transformer_arch.py:41-58).
    q, k: planes [T, B*Tn, C] with the heads side by side -- possibly column-sliced views of a wider matrix
    (e.g. of the fused q|k|v projection); with ``k=None``, ``q`` is [T, B*Tn, 2C] holding q in columns [0,C)
    and k in [C,2C).  -> fp32 [B, nh, Tn, Tn].  (h, img) of the tap-GEMM act as (batch, head)."""
    if k is None:
        Cc = q.shape[2] // 2
        q, k = q[:, :, :Cc], q[:, :, Cc:]
    _need_cuda(q, k)
    T, M, Cc = q.shape
    hs = Cc // nh
    assert M == B * Tn and k.shape == q.shape and q.stride(2) == 1 and k.stride(2) == 1
    ldq, ldk = q.stride(1), k.stride(1)
    out = torch.empty((B, nh, Tn, Tn), dtype=torch.float32, device=q.device)
    plane = q.stride(0)
    assert plane % hs == 0 and (T == 1 or k.stride(0) == M * ldk)
    _tapgemm(a=q, a_term_imgs=plane // hs, a_imgs=(T - 1) * (plane // hs) + nh, a_bcast=0,
             n_img=nh, H=B, W=Tn, a_H=B, a_W=Tn, Cc=hs, a_sw=ldq, a_sh=Tn * ldq, a_sn=hs, tile_rows=1,
             b=k, b_term_g=B, b_groups=T * B, b_sg=Tn * ldk, b_batched_h=1,
             b_groups2=nh, b_sg2=hs, b_batched=1, n_out=Tn, b_sn=ldk,
             taps=_TAPS_1, d=out, d_mode=OUT_F32, d_strides=(Tn * Tn, nh * Tn * Tn, Tn, 1), alpha=alpha)
    return out


def mha_pv(p, vt, B, Tn, nh, out=None, planes_out=True, alpha=1.0, p_mn=False, v_tok=False):
    """Multi-head att @ v (transformer_arch.py:65-67).  p: planes [T,B,nh,Tn,Tn];
    vt: planes [T,B,C,Tn] (v transposed: channels x tokens), or with ``v_tok`` planes [T,B*Tn,C] token-major
    (possibly a column-sliced view of the fused q|k|v projection; consumed MN-major).  ``p_mn`` uses p^T
    (out[j] = sum_i p[i,j] v[i], the value / key gradients) without a transposed copy.
    -> planes [T, B*Tn, C] (or fp32 [B*Tn, C]) with the heads re-assembled side by side.  ``out`` may be a
    column-sliced view of a wider matrix."""
    _need_cuda(p, vt)
    T = p.shape[0]
    assert p.is_contiguous()
    if v_tok:
        Cc = vt.shape[2]
        ldv = vt.stride(1)
        assert vt.shape[1] == B * Tn and vt.stride(2) == 1 and (T == 1 or vt.stride(0) == B * Tn * ldv)
        b_kw = dict(b_sg=Tn * ldv, b_sg2=Cc // nh, b_sn=ldv, b_mn=1)
    else:
        Cc = vt.shape[2]
        assert vt.is_contiguous()
        b_kw = dict(b_sg=Cc * Tn, b_sg2=(Cc // nh) * Tn, b_sn=Tn, b_mn=0)
    hs = Cc // nh
    if out is None:
        out = _alloc_out((B * Tn, Cc), planes_out, T, p.device)
    ld = out.stride(-2)
    _tapgemm(a=p, a_term_imgs=B * nh, a_imgs=T * B * nh, a_bcast=0,
             n_img=nh, H=B, W=Tn, a_H=B, a_W=Tn, Cc=Tn, a_sw=Tn, a_sh=nh * Tn * Tn, a_sn=Tn * Tn,
             tile_rows=1,
             b=vt, b_term_g=B, b_groups=T * B, b_batched_h=1,
             b_groups2=nh, b_batched=1, n_out=hs,
             taps=_TAPS_1, d=out, d_mode=OUT_PLANES if planes_out else OUT_F32, d_strides=(hs, Tn * ld, ld, 1),
             d_plane=out.stride(0) if planes_out else 0, alpha=alpha, a_mn=1 if p_mn else 0, **b_kw)
    return out


# ----------------------------------------------------------------------------
# weight packing (one-time host-side preparation, cached by the modules)
# ----------------------------------------------------------------------------
def split_planes(x, terms):
    """fp32 tensor -> fp16 planes [terms, ...] (hi, lo)."""
    x = x.detach().float()
    hi = x.half()
    if terms == 1:
        return hi.unsqueeze(0).contiguous()
    lo = (x - hi.float()).half()
    return torch.stack((hi, lo)).contiguous()


def pack_conv_weight(w, terms, c_pad=None):
    """OIHW fp32 conv weight -> planes [T, kh*kw, Cout, Cin_pad] (tap-major, K-contiguous)."""
    Cout, Cin, kh, kw = w.shape
    wt = w.detach().float().permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin)
    cp = c_pad if c_pad is not None else (Cin + 7) // 8 * 8
    if cp != Cin:
        wt = torch.nn.functional.pad(wt, (0, cp - Cin))
    return split_planes(wt, terms)


def conv_weight_for_dgrad(w):
    """OIHW weight of a stride-1 'same' conv -> the OIHW weight whose FORWARD conv computes that conv's data
    gradient: dX = conv(dY, W') with W'[ci, co, kh, kw] = W[co, ci, K-1-kh, K-1-kw] (taps flipped, channels
    exchanged).  With it the data gradient of every 3x3 / 1x1 conv runs on the forward tap-GEMM kernels
    (DESIGN 4.5); tests/test_host_logic.py checks the identity against autograd."""
    return w.detach().flip(2, 3).transpose(0, 1).contiguous()


def pack_linear_weight(w, terms):
    """[out, in] fp32 (nn.Linear / 1x1 conv weight squeezed) -> planes [T,1,out,in]."""
    w2 = w.detach().float().reshape(w.shape[0], -1)
    return split_planes(w2.unsqueeze(0), terms)


# ----------------------------------------------------------------------------
# HBM-bound kernels
# ----------------------------------------------------------------------------
def nchw_to_planes(x, c_pad=None, terms=None):
    _need_cuda(x)
    x = _f32c(x)
    N, Cc, H, W = x.shape
    terms = terms or get_terms()
    cp = c_pad if c_pad is not None else (Cc + 7) // 8 * 8
    out = torch.empty((terms, N, H, W, cp), dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_nchw_to_planes(_ptr(x), _ptr(out), N, Cc, H, W, cp, terms, _stream()))
    return out


def nhwc_to_nchw(x):
    _need_cuda(x)
    N, H, W, Cc = x.shape
    out = torch.empty((N, Cc, H, W), dtype=torch.float32, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_nhwc_to_nchw(_ptr(x), _ptr(out), N, Cc, H, W, _stream()))
    return out


def nchw_to_nhwc(x):
    _need_cuda(x)
    x = _f32c(x)
    N, Cc, H, W = x.shape
    out = torch.empty((N, H, W, Cc), dtype=torch.float32, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_nchw_to_nhwc(_ptr(x), _ptr(out), N, Cc, H, W, _stream()))
    return out


def f32_to_planes(x, mode=CVT_PLAIN, terms=None):
    """fp32 NHWC [N,H,W,C] -> planes.  PLAIN: [T,N,H,W,C]; UP2X (nearest) / BILINEAR2X: [T,N,2H,2W,C];
    S2D: [T,4,N,H/2,W/2,C]; MAXPOOL2: [T,N,H/2,W/2,C]."""
    _need_cuda(x)
    N, H, W, Cc = x.shape
    terms = terms or get_terms()
    if mode in (CVT_UP2X, CVT_BILINEAR2X):
        shape = (terms, N, 2 * H, 2 * W, Cc)
    elif mode == CVT_MAXPOOL2:
        shape = (terms, N, H // 2, W // 2, Cc)
    elif mode == CVT_S2D:
        shape = (terms, 4, N, H // 2, W // 2, Cc)
    else:
        shape = (terms, N, H, W, Cc)
    out = torch.empty(shape, dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_f32_to_planes(_ptr(x), _ptr(out), N, H, W, Cc, mode, terms, _stream()))
    return out


def f32_to_planes_bcast(x, e, mode=CVT_PLAIN, terms=None):
    """fp32 NHWC x [N,H,W,C] (any C) and fp32 e [N,Ce] -> planes [T,N,h,w,c_pad] of
    cat([x, e broadcast over h,w], channels), zero-padded to c_pad = C+Ce rounded up to 8.
    PLAIN: (h,w) = (H,W); MAXPOOL2: (H/2,W/2), the pooled x (a constant channel pools to itself)."""
    _need_cuda(x, e)
    assert mode in (CVT_PLAIN, CVT_MAXPOOL2), mode
    x, e = _f32c(x), _f32c(e)
    N, H, W, Cc = x.shape
    Ce = e.shape[1]
    assert e.shape == (N, Ce), (x.shape, e.shape)
    terms = terms or get_terms()
    cp = (Cc + Ce + 7) // 8 * 8
    hw = (H // 2, W // 2) if mode == CVT_MAXPOOL2 else (H, W)
    out = torch.empty((terms, N) + hw + (cp,), dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_f32_to_planes_bcast(_ptr(x), _ptr(e), _ptr(out), N, H, W, Cc, Ce, cp, mode, terms,
                                                   _stream()))
    return out


def group_norm(x, gamma, beta, *, swish, groups=32, eps=1e-6, terms=None, stats=None):
    """GroupNorm(32, C, eps=1e-6) (+ swish) of fp32 NHWC x -> planes [T,N,H,W,C].
    ``stats``: (sum, sumsq) [N,groups,2] fp64 already accumulated by the producer's epilogue."""
    _need_cuda(x)
    N, H, W, Cc = x.shape
    terms = terms or get_terms()
    lib = _lib.load()
    _count(1)
    if stats is None:
        stats = torch.zeros((N, groups, 2), dtype=torch.float64, device=x.device)
        _count(1)
        _lib.check(lib.t2h_gn_stats(_ptr(x), _ptr(stats), N, H * W, Cc, groups, _stream()))
    out = torch.empty((terms, N, H, W, Cc), dtype=torch.float16, device=x.device)
    _lib.check(lib.t2h_gn_apply(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(out), N, H * W, Cc,
                                groups, eps, 1 if swish else 0, terms, _stream()))
    return out


def add_inplace(x, y):
    _need_cuda(x, y)
    assert x.shape == y.shape and x.is_contiguous() and y.is_contiguous()
    _count(1)
    _lib.check(_lib.load().t2h_add_inplace(_ptr(x), _ptr(y), x.numel(), _stream()))
    return x


def softmax_rows(s, scale=1.0, terms=None):
    """softmax(s * scale) over the last dim of fp32 s -> planes [T, *s.shape]."""
    _need_cuda(s)
    terms = terms or get_terms()
    cols = s.shape[-1]
    rows = s.numel() // cols
    out = torch.empty((terms,) + tuple(s.shape), dtype=torch.float16, device=s.device)
    _count(1)
    _lib.check(_lib.load().t2h_softmax_rows(_ptr(s), _ptr(out), rows, cols, scale, terms, _stream()))
    return out


# Multi-head attention as one kernel (csrc/attn_fused.cuh) where its shape constraints hold; T2H_FUSED_ATTN=0 (or
# set_fused_attn(False)) keeps the three-launch q k^T / softmax / p v path for A/B measurements.
FUSED_ATTN = {"on": _os_env.environ.get("T2H_FUSED_ATTN", "1") != "0"}


def set_fused_attn(on):
    old = FUSED_ATTN["on"]
    FUSED_ATTN["on"] = bool(on)
    return old


def can_fuse_attn(tokens, head_dim):
    return FUSED_ATTN["on"] and head_dim == 64 and tokens % 128 == 0 and 128 <= tokens <= 512


def attn_fused(qkv, B, Tn, nh, scale, out=None):
    """softmax(q k^T * scale) v per (sequence, head) in one launch (transformer_arch.py:41-67).
    qkv: planes [T, B*Tn, 3C], the fused q | k | v projection with the heads side by side (C = nh * 64).
    -> planes [T, B*Tn, C]."""
    _need_cuda(qkv)
    T, M, C3 = qkv.shape
    Cc = C3 // 3
    assert M == B * Tn and Cc == nh * 64 and qkv.stride(2) == 1 and qkv.dtype == torch.float16
    if out is None:
        out = torch.empty((T, M, Cc), dtype=torch.float16, device=qkv.device)
    assert out.shape == (T, M, Cc) and out.stride(2) == 1
    _count(1)
    _lib.check(_lib.load().t2h_attn_fwd(_ptr(qkv), T, qkv.stride(0), qkv.stride(1), M, 0, Cc, 2 * Cc, B, Tn, nh, 64,
                                        float(scale), _ptr(out), out.stride(0), out.stride(1), _stream()))
    return out


def layer_norm(x, gamma, beta, eps=1e-5, terms=None):
    """LayerNorm over the last dim of fp32 [rows, C] -> planes [T, rows, C]."""
    _need_cuda(x)
    terms = terms or get_terms()
    rows, Cc = x.shape
    out = torch.empty((terms, rows, Cc), dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_layernorm(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), rows, Cc, eps, terms,
                                         _stream()))
    return out


def layer_norm_scatter(x, gamma, beta, out, row_map, eps=1e-5):
    """LayerNorm of fp32 [rows, C]; row r lands in row row_map[r] of the planes buffer out [T, out_rows, C]
    (rows of ``out`` that no position maps to are left untouched)"""
    _need_cuda(x, out, row_map)
    rows, Cc = x.shape
    assert out.is_contiguous() and out.shape[2] == Cc and row_map.dtype == torch.int64 and row_map.numel() == rows
    _count(1)
    _lib.check(_lib.load().t2h_layernorm_scatter(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), rows, Cc, eps,
                                                 out.shape[0], _ptr(row_map), out.shape[1], _stream()))
    return out


def embed_sum(idx, segm, tex, tok_emb, pos_emb, segm_emb, tex_emb):
    _need_cuda(idx, tok_emb)
    B, T = idx.shape
    Cc = tok_emb.shape[1]
    x = torch.empty((B * T, Cc), dtype=torch.float32, device=idx.device)
    _count(1)
    _lib.check(_lib.load().t2h_embed_sum(_ptr(idx.contiguous()), _ptr(segm.contiguous()),
                                         _ptr(tex.contiguous()), _ptr(tok_emb), _ptr(pos_emb),
                                         _ptr(segm_emb), _ptr(tex_emb), _ptr(x), B, T, Cc, _stream()))
    return x


def onehot_to_planes(segm, n_classes, terms=None):
    """float class-id map [B,1,H,W] -> one-hot planes [T,B,H,W,c_pad]"""
    _need_cuda(segm)
    segm = _f32c(segm)
    B, _, H, W = segm.shape
    terms = terms or get_terms()
    cp = (n_classes + 7) // 8 * 8
    out = torch.empty((terms, B, H, W, cp), dtype=torch.float16, device=segm.device)
    _count(1)
    _lib.check(_lib.load().t2h_onehot_to_planes(_ptr(segm), _ptr(out), B, H, W, n_classes, cp, terms, _stream()))
    return out


# clothes groups of the DeepFashion parsing classes (data/segm_attr_dataset.py:63-65): 0 upper, 1 lower, 2 outer
CLS_GROUP = [-1] * 24
for _c in (1, 4):
    CLS_GROUP[_c] = 0
for _c in (3, 5, 21):
    CLS_GROUP[_c] = 1
CLS_GROUP[2] = 2


def texture_mask(segm, attrs):
    """parsing map [B,1,H,W] (float class ids) + fused attributes int [B,3] (upper, lower, outer; 17 = none) ->
    texture mask [B,1,H,W] float (0 = common codebook, attr+1 = texture codebook), segm_attr_dataset.py:138-151"""
    _need_cuda(segm, attrs)
    segm = _f32c(segm)
    B = segm.shape[0]
    attrs = attrs.to(torch.int32).contiguous()
    grp = torch.tensor(CLS_GROUP, dtype=torch.int32, device=segm.device)
    out = torch.empty_like(segm)
    _count(1)
    _lib.check(_lib.load().t2h_texture_mask(_ptr(segm), _ptr(attrs), _ptr(grp), len(CLS_GROUP), _ptr(out), B,
                                            segm.numel() // B, _stream()))
    return out


def u8_to_planes(img_u8, divisor=127.5, shift=-1.0, want_nchw=False, terms=None):
    """uint8 [B,H,W,C] -> planes [T,B,H,W,c_pad] of img / divisor + shift (and the fp32 NCHW tensor if asked)"""
    _need_cuda(img_u8)
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
    B, H, W, Cc = img_u8.shape
    terms = terms or get_terms()
    cp = (Cc + 7) // 8 * 8
    out = torch.empty((terms, B, H, W, cp), dtype=torch.float16, device=img_u8.device)
    nchw = torch.empty((B, Cc, H, W), dtype=torch.float32, device=img_u8.device) if want_nchw else None
    _count(1)
    _lib.check(_lib.load().t2h_u8_to_planes(_ptr(img_u8), _ptr(out), _ptr(nchw), B, H, W, Cc, cp, divisor, shift,
                                            terms, _stream()))
    return (out, nchw) if want_nchw else out


def mask_to_ids(mask, ht, wt):
    """float id map [B,1,Hs,Ws] -> int32 [B,ht,wt] (nearest)."""
    _need_cuda(mask)
    mask = _f32c(mask)
    B, _, Hs, Ws = mask.shape
    ids = torch.empty((B, ht, wt), dtype=torch.int32, device=mask.device)
    _count(1)
    _lib.check(_lib.load().t2h_mask_to_ids(_ptr(mask), _ptr(ids), B, Hs, Ws, ht, wt, _stream()))
    return ids


# ----------------------------------------------------------------------------
# quantizers
# ----------------------------------------------------------------------------
def vq_search(z_nhwc, codebook, book_id, *, ps=1, cont_stride=None, want_list=True, want_nchw=True,
              want_nhwc=True, want_err=True):
    """z_nhwc fp32 [B,Hz,Wz,Cz]; codebook fp32 [n_books,n_e,D]; book_id int32 [B,Hp,Wp] or None.
    Returns dict(idx, idx_cont, idx_list, zq_nhwc, zq_nchw, sqerr)."""
    _need_cuda(z_nhwc, codebook)
    lib = _lib.load()
    B, Hz, Wz, Cz = z_nhwc.shape
    n_books, n_e, D = codebook.shape
    assert D == Cz * ps * ps
    Hp, Wp = Hz // ps, Wz // ps
    rows = B * Hp * Wp
    dev = z_nhwc.device
    idx = torch.empty((B, Hp, Wp), dtype=torch.int64, device=dev)
    idx_cont = torch.empty((B, Hp, Wp), dtype=torch.int64, device=dev)
    idx_list = torch.empty((n_books, B, Hp, Wp), dtype=torch.int64, device=dev) if want_list else None
    zq_nhwc = torch.empty_like(z_nhwc) if want_nhwc else None
    zq_nchw = torch.empty((B, Cz, Hz, Wz), dtype=torch.float32, device=dev) if want_nchw else None
    sqerr = torch.zeros((1,), dtype=torch.float64, device=dev) if want_err else None
    wsb = lib.t2h_vq_workspace_bytes(rows, n_books, n_e)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
    _count(3)
    _lib.check(lib.t2h_vq_search(_ptr(z_nhwc), _ptr(codebook), _ptr(book_id), B, Hz, Wz, Cz, ps, n_books,
                                 n_e, n_e if cont_stride is None else cont_stride, _ptr(idx),
                                 _ptr(idx_cont), _ptr(idx_list), _ptr(zq_nhwc), _ptr(zq_nchw), _ptr(sqerr),
                                 _ptr(ws), wsb, _stream()))
    return dict(idx=idx, idx_cont=idx_cont, idx_list=idx_list, zq_nhwc=zq_nhwc, zq_nchw=zq_nchw,
                sqerr=sqerr)


def vq_gather(codebook, idx, book_id, *, B, Hz, Wz, Cz, ps=1, want_nchw=True, want_nhwc=False):
    _need_cuda(codebook, idx)
    n_books, n_e, D = codebook.shape
    dev = codebook.device
    zq_nhwc = torch.empty((B, Hz, Wz, Cz), dtype=torch.float32, device=dev) if want_nhwc else None
    zq_nchw = torch.empty((B, Cz, Hz, Wz), dtype=torch.float32, device=dev) if want_nchw else None
    _count(1)
    _lib.check(_lib.load().t2h_vq_gather(_ptr(codebook), _ptr(idx.contiguous()), _ptr(book_id), B, Hz, Wz,
                                         Cz, ps, n_books, n_e, _ptr(zq_nhwc), _ptr(zq_nchw), _stream()))
    return zq_nhwc, zq_nchw


# ----------------------------------------------------------------------------
# training (backward / optimiser) kernels
# ----------------------------------------------------------------------------
def f32_to_planes_rows(x, terms=None, scale=1.0):
    """fp32 [..., C] -> planes [T, ..., C] of scale*x (no layout change)"""
    _need_cuda(x)
    terms = terms or get_terms()
    assert x.is_contiguous() and x.dtype == torch.float32
    Cc = x.shape[-1]
    R = x.numel() // Cc
    out = torch.empty((terms,) + tuple(x.shape), dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_f32_to_planes_t(_ptr(x), None, _ptr(out), 1, R, Cc, terms, scale, _stream()))
    return out


def f32_to_planes_t(x, terms=None, want_plain=True, scale=1.0):
    """fp32 [G,R,C] (or [R,C]) -> (planes [T,G,R,C] or None, transposed planes [T,G,C,R]) of scale*x"""
    _need_cuda(x)
    terms = terms or get_terms()
    x3 = x if x.dim() == 3 else x.unsqueeze(0)
    assert x3.is_contiguous() and x3.dtype == torch.float32
    G, R, Cc = x3.shape
    out_t = torch.empty((terms, G, Cc, R), dtype=torch.float16, device=x.device)
    out_n = torch.empty((terms, G, R, Cc), dtype=torch.float16, device=x.device) if want_plain else None
    _count(1)
    _lib.check(_lib.load().t2h_f32_to_planes_t(_ptr(x3), _ptr(out_t), _ptr(out_n), G, R, Cc, terms, scale,
                                                 _stream()))
    if x.dim() == 2:
        return (out_n[:, 0] if want_plain else None), out_t[:, 0]
    return out_n, out_t


def planes_transpose(x, out=None):
    """planes [T,G,R,C] (unit last stride; may be a column-sliced view) -> [T,G,C,R]; ``out`` may be a
    column-sliced view [T,G,C,R] of a wider tensor (unit last stride)."""
    _need_cuda(x)
    T, G, R, Cc = x.shape
    assert x.stride(3) == 1
    if out is None:
        out = torch.empty((T, G, Cc, R), dtype=torch.float16, device=x.device)
    assert out.shape == (T, G, Cc, R) and out.stride(3) == 1
    _count(1)
    _lib.check(_lib.load().t2h_planes_transpose(_ptr(x), _ptr(out), G, R, Cc, x.stride(2), x.stride(1), x.stride(0),
                                                out.stride(2), out.stride(1), out.stride(0), T, _stream()))
    return out


def colsum_(out, x):
    """out[c] += sum_r x[r,c] (fp32)"""
    _need_cuda(x, out)
    rows, Cc = x.shape
    assert x.is_contiguous() and out.numel() == Cc
    _count(1)
    _lib.check(_lib.load().t2h_colsum(_ptr(x), _ptr(out), rows, Cc, _stream()))


def gelu_fwd(a, terms=None):
    _need_cuda(a)
    terms = terms or get_terms()
    out = torch.empty((terms,) + tuple(a.shape), dtype=torch.float16, device=a.device)
    _count(1)
    _lib.check(_lib.load().t2h_gelu_fwd(_ptr(a), _ptr(out), a.numel(), terms, _stream()))
    return out


def gelu_bwd(a, dg, want_planes=False, terms=None):
    """da = dg * gelu'(a) (fp32) [, and its fp16 planes for the following GEMMs, from the same pass]"""
    _need_cuda(a, dg)
    da = torch.empty_like(a)
    terms = terms or get_terms()
    planes = torch.empty((terms,) + tuple(a.shape), dtype=torch.float16, device=a.device) if want_planes else None
    _count(1)
    _lib.check(_lib.load().t2h_gelu_bwd(_ptr(a), _ptr(dg), _ptr(da), _ptr(planes), a.numel(), terms, _stream()))
    return (da, planes) if want_planes else da


def layernorm_bwd_(dx, dy, x, gamma, dgamma, dbeta, eps=1e-5, accumulate=True, want_planes=False, colsum_out=None,
                   terms=None):
    """dx (+)= LayerNorm backward of dy wrt x; dgamma/dbeta accumulated.  Optionally, from the same pass: the
    fp16 planes of the updated dx (returned) and its column sums accumulated into ``colsum_out`` [C]."""
    _need_cuda(dx, dy, x)
    rows, Cc = x.shape
    terms = terms or get_terms()
    planes = torch.empty((terms, rows, Cc), dtype=torch.float16, device=x.device) if want_planes else None
    _count(1)
    _lib.check(_lib.load().t2h_layernorm_bwd_fused(_ptr(dy), _ptr(x), _ptr(gamma), _ptr(dx), _ptr(dgamma),
                                                   _ptr(dbeta), rows, Cc, eps, 1 if accumulate else 0, _ptr(planes),
                                                   terms, _ptr(colsum_out), _stream()))
    return planes


def softmax_bwd(p, dp, scale):
    """p planes [T, ...rows, cols], dp fp32 [...rows, cols] -> ds fp32"""
    _need_cuda(p, dp)
    cols = dp.shape[-1]
    rows = dp.numel() // cols
    ds = torch.empty_like(dp)
    _count(1)
    _lib.check(_lib.load().t2h_softmax_bwd(_ptr(p), _ptr(dp), _ptr(ds), rows, cols, scale, p.shape[0], _stream()))
    return ds


def softmax_bwd_planes(p, dp, scale, out_scale=1.0):
    """as softmax_bwd, but out_scale*ds goes straight to fp16 planes [T, ...] (no fp32 round trip)"""
    _need_cuda(p, dp)
    cols = dp.shape[-1]
    rows = dp.numel() // cols
    out = torch.empty((p.shape[0],) + tuple(dp.shape), dtype=torch.float16, device=dp.device)
    _count(1)
    _lib.check(_lib.load().t2h_softmax_bwd_planes(_ptr(p), _ptr(dp), _ptr(out), rows, cols, scale, p.shape[0],
                                                  out_scale, _stream()))
    return out


def ce_heads(logits, target, head, w):
    """logits fp32 [M, nh, ncls]; target/head int64 [M]; w fp32 [M] -> (ce_rows [M] unweighted... see kernel,
    dlogits fp32 [M, nh*ncls] already multiplied by w)"""
    _need_cuda(logits)
    M, nh, ncls = logits.shape
    loss_rows = torch.empty((M,), dtype=torch.float32, device=logits.device)
    dlogits = torch.empty((M, nh * ncls), dtype=torch.float32, device=logits.device)
    _count(1)
    _lib.check(_lib.load().t2h_ce_heads(_ptr(logits), _ptr(target), _ptr(head), _ptr(w), _ptr(loss_rows),
                                        _ptr(dlogits), M, nh, ncls, _stream()))
    return loss_rows, dlogits


def embed_bwd_(dE, dx, idx=None, t_mod=0):
    _need_cuda(dE, dx)
    rows, Cc = dx.shape
    _count(1)
    _lib.check(_lib.load().t2h_embed_bwd(_ptr(dx), _ptr(idx), _ptr(dE), rows, Cc, t_mod, _stream()))


def adam_(p, g, m, v, lr, beta1, beta2, eps, step, grad_scale=1.0):
    _need_cuda(p, g, m, v)
    _count(1)
    _lib.check(_lib.load().t2h_adam(_ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), lr, beta1, beta2, eps, step,
                                    grad_scale, _stream()))


# ----------------------------------------------------------------------------
# index prediction (UNet + multi-head FCN) helpers
# ----------------------------------------------------------------------------
def argmax_heads(logits, head):
    """logits fp32 [G, M, ncls]; head int64 [M] -> int64 [M]: argmax (lowest index on ties) inside each row's
    own head, -1 where head is outside 0..G-1"""
    _need_cuda(logits, head)
    G, M, ncls = logits.shape
    assert logits.is_contiguous() and head.numel() == M and head.dtype == torch.int64
    out = torch.empty((M,), dtype=torch.int64, device=logits.device)
    _count(1)
    _lib.check(_lib.load().t2h_argmax_heads(_ptr(logits), _ptr(head.contiguous()), _ptr(out), M, G, ncls, _stream()))
    return out


def shape_attr_embed(attr, packed):
    """ShapeAttrEmbedding forward: attr int64 [B,n_attr] (already range-checked) -> fp32 [B,out_dim].
    packed: dict from ShapeAttrEmbedding's packed-parameter cache (cls_off, w1t, b1, w2, b2, wf1, bf1, wf2, bf2)."""
    p = packed
    _need_cuda(attr, p["w1t"])
    attr = attr.to(torch.int64).contiguous()
    B, A = attr.shape
    D, O = p["b1"].shape[1], p["bf1"].shape[0]
    assert p["cls_off"].numel() == A + 1 and p["b1"].shape[0] == A
    out = torch.empty((B, O), dtype=torch.float32, device=attr.device)
    _count(1)
    _lib.check(_lib.load().t2h_shape_attr_embed(
        _ptr(attr), _ptr(p["cls_off"]), _ptr(p["w1t"]), _ptr(p["b1"]), _ptr(p["w2"]), _ptr(p["b2"]), _ptr(p["wf1"]),
        _ptr(p["bf1"]), _ptr(p["wf2"]), _ptr(p["bf2"]), _ptr(out), B, A, D, O, _stream()))
    return out


def pack_u8(x, scale=1.0, shift=0.0):
    """fp32 NCHW image batch -> uint8 NHWC as torchvision's save_image quantises it (after an optional affine
    map and the clamp to [0,1])"""
    _need_cuda(x)
    x = _f32c(x)
    N, Cc, H, W = x.shape
    out = torch.empty((N, H, W, Cc), dtype=torch.uint8, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_pack_u8(_ptr(x), _ptr(out), N, Cc, H, W, scale, shift, _stream()))
    return out


# ----------------------------------------------------------------------------
# VQGAN training step: generic tap convolution (forward and data gradient), conv weight gradient, norm backward,
# losses (csrc/gemm_tc.cu t2h_conv_wgrad, csrc/gan.cu)
# ----------------------------------------------------------------------------
def tap_conv(a, w, bias, taps, *, n, out_hw, out=None, d_strides=None, planes_out=False, nchw_out=False, act=ACT_NONE,
             residual=None, want_stats=False, alpha=1.0, tap_w=None, nb=None):
    """out[img, h, w, :] = act(alpha * sum_i W[tap_w[i]] . a[img + off_i, h + dy_i, w + dx_i, :] + bias) over an
    (out_hw) output domain that may differ from a's spatial extent (reads outside a are zero).
    a: planes whose last three dims are (h, w, C) and whose dims between the plane dim and those flatten to the
    image index ([T,N,h,w,C] or the 4-phase [T,4,N,h,w,C]); w: planes [T, slots, Cout, C] (possibly a tap-sliced
    view); taps: ((dy, dx, img_off), ...).  Serves conv3x3 / conv1x1 / conv3x3_s2 above, the Discriminator's 4x4
    convs (vqgan_arch.py:1160-1197), all data gradients (forward kernel on the transposed weights with negated taps),
    the parity launches of the strided convs' data gradients."""
    _need_cuda(a, w)
    T = a.shape[0]
    aH, aW, Cc = a.shape[-3:]
    a_imgs = a.numel() // (aH * aW * Cc)
    H, W = out_hw
    Cout = w.shape[2]
    assert w.shape[3] == Cc and w.stride(3) == 1 and w.stride(2) == Cc, (a.shape, w.shape)
    b_term_g = (w.stride(0) // w.stride(1)) if w.shape[0] > 1 else max(w.shape[1], max(tap_w or (0,)) + 1)
    slots = w.shape[1] if tap_w is None else max(tap_w) + 1
    stats, cpg = _stats_for(Cout, n, a.device, want_stats and not planes_out and not nchw_out and out is None)
    if out is None:
        if nchw_out:
            out = torch.empty((n, Cout, H, W), dtype=torch.float32, device=a.device)
            d_strides = (Cout * H * W, W, 1, H * W)
        else:
            out = _alloc_out((n, H, W, Cout), planes_out, T, a.device)
            d_strides = (H * W * Cout, W * Cout, Cout, 1)
    _tapgemm(a=a, a_term_imgs=a_imgs // T, a_imgs=a_imgs, a_bcast=0, n_img=n, H=H, W=W, a_H=aH, a_W=aW, Cc=Cc,
             a_sw=Cc, a_sh=aW * Cc, a_sn=aH * aW * Cc,
             b=w, b_term_g=b_term_g, b_groups=(w.shape[0] - 1) * b_term_g + slots, b_batched=0, n_out=Cout, b_sn=Cc,
             b_sg=w.stride(1),
             taps=taps, d=out, d_mode=OUT_PLANES if planes_out else OUT_F32, d_strides=d_strides,
             d_plane=n * H * W * Cout, bias=bias, bias_mode=BIAS_COL, act=act, residual=residual, alpha=alpha,
             gn_stats=stats, gn_cpg=cpg, tap_w=tap_w, nb=nb)
    if want_stats:
        return out, stats
    return out


FUSE_NB = {"on": _os_env.environ.get("T2H_FUSE_NB", "1") != "0"}


def nb_context(x, stats, gamma, beta, *, act, groups, eps):
    """Context for fusing pass 1 of ``norm_bwd`` (the per-(image, channel) sums of du and du*xhat) into the epilogue of
    the data-gradient conv that produces dy = dL/d act(norm(x)*gamma+beta): pass it as ``nb=`` to a stride-1
    ``conv_grad.dgrad`` whose output has x's shape, then ``norm_bwd(..., sums=ctx["sums"])``.  Returns None when the
    conv would not run on the swapped-operand kernel (channels % 128, narrow images) or T2H_FUSE_NB=0 -- the caller
    then simply omits both arguments and norm_bwd runs its own reduce pass."""
    N, H, W, Cc = x.shape
    if not FUSE_NB["on"] or Cc % 128 or Cc % groups or H < 2 or not x.is_contiguous():
        return None
    sums = torch.zeros((N * Cc * 2,), dtype=torch.float64, device=x.device)
    return dict(x=x, stats=stats, gamma=_f32c(gamma), beta=_f32c(beta), act=act, groups=groups, eps=float(eps), sums=sums)


def conv_wgrad(dy, x, taps, dw, *, n, alpha=1.0, k_split=0):
    """dw[tap, co, ci] += alpha * sum_{img,h,w} dy[img,h,w,co] * x[img + off, h + dy_t, w + dx_t, ci].
    dy: planes [T,N,H,W,Co]; x: planes [T,(phases,)N,h,w,Ci] (the forward conv's input operand, as saved);
    dw: fp32 [ntaps, Co, Ci_ld] (rows 16-byte aligned), accumulated."""
    _need_cuda(dy, x, dw)
    lib = _lib.load()
    T = dy.shape[0]
    N, H, W, Co = dy.shape[1:]
    xH, xW, Ci = x.shape[-3:]
    x_imgs = x.numel() // (xH * xW * Ci)
    assert N == n and dy.is_contiguous() and x.is_contiguous() and x.shape[0] == T
    assert dw.dim() == 3 and dw.shape[0] == len(taps) and dw.shape[1] == Co and dw.shape[2] == Ci and dw.stride(2) == 1
    p = _lib.ConvWgradParams()
    p.dy = dy.data_ptr(); p.dy_terms = T; p.dy_term_imgs = N; p.dy_imgs = T * N
    p.n_img, p.H, p.W, p.cout = N, H, W, Co
    p.dy_sw, p.dy_sh, p.dy_sn = Co, W * Co, H * W * Co
    p.x = x.data_ptr(); p.x_terms = T; p.x_term_imgs = x_imgs // T; p.x_imgs = x_imgs
    p.x_H, p.x_W, p.cin = xH, xW, Ci
    p.x_sw, p.x_sh, p.x_sn = Ci, xW * Ci, xH * xW * Ci
    p.ntaps = len(taps)
    for i, (ty, tx, off) in enumerate(taps):
        p.tap_dy[i], p.tap_dx[i], p.tap_img_off[i] = ty, tx, off
    p.dw = dw.data_ptr(); p.dw_tap_stride = dw.stride(0); p.dw_ld = dw.stride(1)
    p.alpha = alpha
    p.nterms = 3 if T == 2 else 1
    p.k_split = k_split
    _launch(lib.t2h_conv_wgrad, p, 2.0 * N * H * W * Co * Ci * len(taps), ("wgrad", N, H, W, Co, Ci * len(taps)))
    return dw


ACT_CODE = {None: 0, "none": 0, "swish": 1, "lrelu": 2}


def norm_apply(x, stats, gamma, beta, *, act, groups, eps, n=None, terms=None):
    """act(norm(x)*gamma+beta) -> planes.  x fp32 [N,H,W,C]; with n=1 the whole batch is one normalisation domain
    (BatchNorm2d in training mode: groups = C)."""
    _need_cuda(x)
    N, H, W, Cc = x.shape
    terms = terms or get_terms()
    nn_, hw = (N, H * W) if n is None else (n, N * H * W // n)
    out = torch.empty((terms, N, H, W, Cc), dtype=torch.float16, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_gn_apply(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(out), nn_, hw, Cc, groups,
                                        eps, ACT_CODE[act], terms, _stream()))
    return out


def norm_stats(x, groups, n=None):
    """(sum, sumsq) [n, groups, 2] fp64 of fp32 [N,H,W,C] (n=1: over the whole batch)"""
    _need_cuda(x)
    N, H, W, Cc = x.shape
    nn_, hw = (N, H * W) if n is None else (n, N * H * W // n)
    stats = torch.zeros((nn_, groups, 2), dtype=torch.float64, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_gn_stats(_ptr(x), _ptr(stats), nn_, hw, Cc, groups, _stream()))
    return stats


def norm_bwd(x, stats, gamma, beta, dy, *, act, groups, eps, dgamma=None, dbeta=None, add=None, want_planes=False,
             n=None, terms=None, colsum_out=None, want_dx=True, sums=None):
    """backward of act(norm(x)*gamma+beta): -> dx fp32 (+ add) [, planes of dx]; dgamma/dbeta accumulated;
    ``colsum_out`` [C] += column sums of dx (the bias gradient of the conv that produced x); ``want_dx=False``
    (with ``want_planes``) skips the fp32 copy when only the conv gradients consume dx (4 of 14 B per element);
    ``sums``: pass 1's result from ``nb_context`` (the data-gradient conv accumulated it in its epilogue) -- the
    reduce launch and its 8 B per element are skipped"""
    _need_cuda(x, dy)
    N, H, W, Cc = x.shape
    terms = terms or get_terms()
    nn_, hw = (N, H * W) if n is None else (n, N * H * W // n)
    assert want_dx or want_planes
    dx = torch.empty_like(x) if want_dx else None
    planes = torch.empty((terms, N, H, W, Cc), dtype=torch.float16, device=x.device) if want_planes else None
    if sums is not None:
        assert sums.dtype == torch.float64 and sums.numel() == nn_ * Cc * 2
        ws = sums
    else:
        ws = torch.empty((nn_ * Cc * 2,), dtype=torch.float64, device=x.device)
    assert dy.is_contiguous() and x.is_contiguous() and (add is None or add.is_contiguous())
    _count(3 if sums is None else 2)
    _lib.check(_lib.load().t2h_norm_bwd(_ptr(x), _ptr(stats), _ptr(gamma), _ptr(beta), _ptr(dy), _ptr(add), _ptr(dx),
                                        _ptr(planes), terms, _ptr(dgamma), _ptr(dbeta), _ptr(ws), nn_, hw, Cc, groups,
                                        eps, ACT_CODE[act], _ptr(colsum_out), 0 if sums is None else 1, _stream()))
    return (dx, planes) if want_planes else dx


def bn_update_running(stats, running_mean, running_var, count, momentum):
    _count(1)
    _lib.check(_lib.load().t2h_bn_update_running(_ptr(stats), _ptr(running_mean), _ptr(running_var), count, momentum,
                                                 running_mean.numel(), _stream()))


def lrelu_bwd(y_planes, dy, want_planes=True, terms=None):
    """dpre = dy * LeakyReLU'(pre) from the sign of y = LeakyReLU(pre) (planes); -> (dpre fp32, planes or None)"""
    _need_cuda(y_planes, dy)
    terms = terms or y_planes.shape[0]
    dpre = torch.empty_like(dy)
    planes = torch.empty((terms,) + tuple(dy.shape), dtype=torch.float16, device=dy.device) if want_planes else None
    _count(1)
    _lib.check(_lib.load().t2h_lrelu_bwd(_ptr(y_planes), _ptr(dy), _ptr(dpre), _ptr(planes), terms, dy.numel(),
                                         _stream()))
    return dpre, planes


def planes_s2d(a):
    """planes [T,N,H,W,C] -> space-to-depth planes [T,4,N,H/2,W/2,C]"""
    _need_cuda(a)
    T, N, H, W, Cc = a.shape
    assert a.is_contiguous()
    out = torch.empty((T, 4, N, H // 2, W // 2, Cc), dtype=torch.float16, device=a.device)
    _count(1)
    _lib.check(_lib.load().t2h_planes_s2d(_ptr(a), _ptr(out), T, N, H, W, Cc, _stream()))
    return out


def sumpool2(x):
    """adjoint of nearest x2: fp32 [N,2H,2W,C] -> [N,H,W,C]"""
    _need_cuda(x)
    N, H2, W2, Cc = x.shape
    out = torch.empty((N, H2 // 2, W2 // 2, Cc), dtype=torch.float32, device=x.device)
    _count(1)
    _lib.check(_lib.load().t2h_sumpool2(_ptr(x), _ptr(out), N, H2 // 2, W2 // 2, Cc, _stream()))
    return out


def vq_bwd(z, codebook, idx, book_id, dzq, dcodebook, coef_z, coef_e):
    """dz = dzq + coef_z (z - e); dcodebook[book, idx] += coef_e (e - z).  z fp32 [B,H,W,D] (patch size 1)"""
    _need_cuda(z, codebook)
    n_books, n_e, D = codebook.shape
    assert z.shape[-1] == D and z.is_contiguous() and dcodebook.is_contiguous()
    dz = torch.empty_like(z)
    _count(1)
    _lib.check(_lib.load().t2h_vq_bwd(_ptr(z), _ptr(codebook), _ptr(idx.contiguous()), _ptr(book_id), _ptr(dzq),
                                      _ptr(dz), _ptr(dcodebook), z.numel() // D, D, n_books, n_e, coef_z, coef_e,
                                      _stream()))
    return dz


def l1_loss(x, xrec, sum_out, gscale=0.0, want_grad=True):
    """sum_out[0] += sum|x - xrec|; -> grad = gscale*sign(xrec - x) (or None)"""
    _need_cuda(x, xrec)
    assert x.is_contiguous() and xrec.is_contiguous() and x.shape == xrec.shape
    grad = torch.empty_like(xrec) if want_grad else None
    _count(1)
    _lib.check(_lib.load().t2h_l1_loss(_ptr(x), _ptr(xrec), _ptr(grad), _ptr(sum_out), x.numel(), gscale, _stream()))
    return grad


def bce_logits(logits, segm, sum_out, gscale=1.0, want_grad=True, colsum_out=None, terms=None):
    """BCE-with-logits of fp32 NHWC ``logits`` [N,H,W,C] against the one-hot of the class-id map ``segm`` (float
    [N,1,H,W], the ids onehot_to_planes reads; a non-integer or out-of-range id has an all-zero target row):
    sum_out[0] += the loss summed over all N*C*H*W elements; -> fp16 planes [T,N,H,W,c_pad] of
    gscale * (sigmoid(logits) - onehot) (or None); ``colsum_out`` [C] += the column sums of that gradient"""
    _need_cuda(logits, segm, sum_out)
    segm = _f32c(segm)
    N, H, W, Cc = logits.shape
    assert logits.is_contiguous() and logits.dtype == torch.float32 and segm.numel() == N * H * W
    assert sum_out.dtype == torch.float64 and (colsum_out is None or colsum_out.numel() == Cc)
    terms = terms or get_terms()
    cp = (Cc + 7) // 8 * 8
    planes = torch.empty((terms, N, H, W, cp), dtype=torch.float16, device=logits.device) if want_grad else None
    _count(1)
    _lib.check(_lib.load().t2h_bce_logits(_ptr(logits), _ptr(segm), N, H, W, Cc, cp, gscale, _ptr(sum_out),
                                          _ptr(planes), terms, _ptr(colsum_out), _stream()))
    return planes


def hinge_loss(logits, sum_out, sgn, gscale=0.0, want_grad=True):
    _need_cuda(logits)
    assert logits.is_contiguous()
    grad = torch.empty_like(logits) if want_grad else None
    _count(1)
    _lib.check(_lib.load().t2h_hinge_loss(_ptr(logits), _ptr(grad), _ptr(sum_out), logits.numel(), float(sgn), gscale,
                                          _stream()))
    return grad


def diffaug_fwd(x, r, t):
    """DiffAugment 'color,translation' of fp32 NCHW [B,3,H,W]; r fp32 [B,3], t int32 [B,2]"""
    _need_cuda(x, r, t)
    B, Cc, H, W = x.shape
    assert Cc == 3 and x.is_contiguous() and r.dtype == torch.float32 and t.dtype == torch.int32
    out = torch.empty_like(x)
    ws = torch.empty((B,), dtype=torch.float64, device=x.device)
    _count(2)
    _lib.check(_lib.load().t2h_diffaug_fwd(_ptr(x), _ptr(r), _ptr(t), _ptr(ws), _ptr(out), B, H, W, _stream()))
    return out


def diffaug_bwd(dout, r, t):
    _need_cuda(dout, r, t)
    B, Cc, H, W = dout.shape
    assert Cc == 3 and dout.is_contiguous()
    dx = torch.empty_like(dout)
    ws = torch.empty((B,), dtype=torch.float64, device=dout.device)
    _count(2)
    _lib.check(_lib.load().t2h_diffaug_bwd(_ptr(dout), _ptr(r), _ptr(t), _ptr(ws), _ptr(dx), B, H, W, _stream()))
    return dx


def adaptive_weight(rg, gg, out, inv_scale, wmax, enable):
    _need_cuda(rg, gg, out)
    assert rg.numel() == gg.numel() and rg.is_contiguous() and gg.is_contiguous()
    _count(1)
    _lib.check(_lib.load().t2h_adaptive_weight(_ptr(rg), _ptr(gg), rg.numel(), inv_scale, wmax, enable, _ptr(out),
                                               _stream()))
    return out


def axpy_dev(a, b, w):
    """a + w[0]*b with the scalar w on the device"""
    _need_cuda(a, b, w)
    assert a.shape == b.shape and a.is_contiguous() and b.is_contiguous()
    out = torch.empty_like(a)
    _count(1)
    _lib.check(_lib.load().t2h_axpy_dev(_ptr(a), _ptr(b), _ptr(w), _ptr(out), a.numel(), _stream()))
    return out


def sample_step(logits_own, u, tex, x_t, unmasked, *, t, temp, seed, step, n_heads, cont_stride=1024):
    """one reveal step of the diffusion sampler, in place on x_t [M] int64 / unmasked [M] uint8"""
    _need_cuda(logits_own, u, tex, x_t, unmasked)
    M, ncls = logits_own.shape
    assert logits_own.is_contiguous() and u.numel() == M and x_t.numel() == M and unmasked.dtype == torch.uint8
    _count(1)
    _lib.check(_lib.load().t2h_sample_step(_ptr(logits_own), _ptr(u), _ptr(tex), _ptr(x_t), _ptr(unmasked), M, ncls,
                                           n_heads, 1.0 / float(t), 1.0 / float(temp), int(seed), int(step), cont_stride,
                                           _stream()))
