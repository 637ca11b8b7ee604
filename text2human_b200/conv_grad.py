"""Forward / data-gradient / weight-gradient launch shapes of every convolution on the VQGAN training path
(reference: the nn.Conv2d layers of models/archs/vqgan_arch.py and what autograd derives for them).

A conv is described by its *kind* (kernel, stride, padding) and runs on three views of one weight tensor kept
tap-major in fp32 master storage ``[taps, Cout_p, Cin_p]`` (channel counts padded to 8, zero padding):

  * forward          ``t2h_tapgemm`` on planes ``wn [T, taps, Cout_p, Cin_p]`` of the master weights;
  * data gradient    the SAME forward kernel on the transposed planes ``wt [T, taps, Cin_p, Cout_p]`` with the taps
                     negated (stride 1), or -- stride 2 -- four launches, one per input parity, each using the
                     subset of taps that reaches that parity (``tap_w`` selects their weight slots in place) and
                     writing a strided quarter of dX;
  * weight gradient  ``t2h_conv_wgrad``: dW[tap] += dY^T . shift_tap(X) with both operands read MN-major.

Kinds:  "k3" 3x3 s1 p1 | "k1" 1x1 | "down" pad (0,1,0,1) + 3x3 s2 (Downsample, vqgan_arch.py:547-551) |
        "k4s2" 4x4 s2 p1 and "k4s1" 4x4 s1 p1 (Discriminator, :1160-1197).
Stride-2 kinds take their input as 4-phase space-to-depth planes ``[T, 4, N, H/2, W/2, C]``.
"""
import functools

import torch

from . import ops

KSIZE = {"k3": 3, "k1": 1, "down": 3, "k4s2": 4, "k4s1": 4}
STRIDE = {"k3": 1, "k1": 1, "down": 2, "k4s2": 2, "k4s1": 1}
PAD = {"k3": 1, "k1": 0, "down": 0, "k4s2": 1, "k4s1": 1}


def pad8(c):
    return (c + 7) // 8 * 8


def out_hw(kind, H, W):
    if kind in ("k3", "k1"):
        return H, W
    if kind == "k4s1":
        return H - 1, W - 1
    return H // 2, W // 2          # down, k4s2 (even H, W)


@functools.lru_cache(maxsize=None)
def fwd_taps(kind, n):
    """((dy, dx, img_off), ...) in weight-slot order kh*K + kw (cached: every strided conv launch asks for it)"""
    K, pad = KSIZE[kind], PAD[kind]
    taps = []
    for kh in range(K):
        for kw in range(K):
            if STRIDE[kind] == 1:
                taps.append((kh - pad, kw - pad, 0))
            else:                   # source row 2u + kh - pad = 2(u + dy) + phase
                ph, pw = (kh - pad) % 2, (kw - pad) % 2
                taps.append(((kh - pad - ph) // 2, (kw - pad - pw) // 2, (ph * 2 + pw) * n))
    return tuple(taps)


def dgrad_parity_taps(kind, a, b):
    """stride-2 data gradient of input parity (a, b): dX[2u+a, 2v+b] = sum W[kh,kw]^T dY[u + dy, v + dx] over the
    taps with kh = a + pad, kw = b + pad (mod 2).  -> (taps, weight slots)"""
    K, pad = KSIZE[kind], PAD[kind]
    taps, slots = [], []
    for kh in range(K):
        if (kh - a - pad) % 2:
            continue
        for kw in range(K):
            if (kw - b - pad) % 2:
                continue
            taps.append(((a + pad - kh) // 2, (b + pad - kw) // 2, 0))
            slots.append(kh * K + kw)
    return tuple(taps), tuple(slots)


def forward(kind, a, wn, bias, *, n, in_hw, **kw):
    """a: input planes (plain [T,N,H,W,C] or s2d [T,4,N,H/2,W/2,C]); wn [T,taps,Cout,Cin_p] -> see ops.tap_conv"""
    return ops.tap_conv(a, wn, bias, fwd_taps(kind, n), n=n, out_hw=out_hw(kind, *in_hw), **kw)


def dgrad(kind, dyp, wt, *, n, in_hw, cin=None, out=None, d_strides=None, nb=None):
    """dX fp32 [N,H,W,Cin_p] (or into ``out`` with element strides ``d_strides`` = (sn, sh, sw, sc) of the FULL
    input grid, e.g. an NCHW image gradient) from dY planes [T,N,Ho,Wo,Cout_p] and transposed planes
    wt [T,taps,Cin_p,Cout_p]; ``cin`` limits the computed input channels (image gradients: 3 of 8)."""
    H, W = in_hw
    if cin is not None and cin != wt.shape[2]:
        wt = wt[:, :, :cin]
    ci = wt.shape[2]
    if STRIDE[kind] == 1:
        taps = tuple((-ty, -tx, 0) for ty, tx, _ in fwd_taps(kind, n))
        if out is None:
            return ops.tap_conv(dyp, wt, None, taps, n=n, out_hw=(H, W), nb=nb)   # nb: ops.nb_context (norm-backward sums)
        assert nb is None
        return ops.tap_conv(dyp, wt, None, taps, n=n, out_hw=(H, W), out=out, d_strides=d_strides)
    assert nb is None, "norm-backward sums ride only on single-launch (stride-1) data gradients"
    if out is None:
        out = torch.empty((n, H, W, ci), dtype=torch.float32, device=dyp.device)
        d_strides = (H * W * ci, W * ci, ci, 1)
    sn, sh, sw, sc = d_strides
    for a in (0, 1):
        for b in (0, 1):
            taps, slots = dgrad_parity_taps(kind, a, b)
            view = out.reshape(-1)[a * sh + b * sw:]
            ops.tap_conv(dyp, wt, None, taps, n=n, out_hw=(H // 2, W // 2), out=view,
                         d_strides=(sn, 2 * sh, 2 * sw, sc), tap_w=slots)
    return out


def wgrad(kind, dyp, x_operand, gw, *, n, alpha=1.0):
    """gw fp32 [taps, Cout_p, Cin_p] += dY^T . shifted X (x_operand = the planes the forward conv consumed)"""
    return ops.conv_wgrad(dyp, x_operand, fwd_taps(kind, n), gw, n=n, alpha=alpha)


# ----------------------------------------------------------------------------
# master-weight layout helpers
# ----------------------------------------------------------------------------
def oihw_to_master(w):
    """[Cout, Cin, K, K] -> tap-major, channel-padded [K*K, Cout_p, Cin_p] fp32"""
    co, ci, kh, kw = w.shape
    m = torch.zeros((kh * kw, pad8(co), pad8(ci)), dtype=torch.float32, device=w.device)
    m[:, :co, :ci] = w.detach().float().permute(2, 3, 0, 1).reshape(kh * kw, co, ci)
    return m


def master_as_oihw(m, co, ci, k):
    """the OIHW view of a tap-major master tensor (no copy): what the nn.Parameter becomes"""
    return m.view(k, k, m.shape[1], m.shape[2]).permute(2, 3, 0, 1)[:co, :ci]


def weight_planes(m, terms=None):
    """-> (wn [T,taps,Cout_p,Cin_p], wt [T,taps,Cin_p,Cout_p]) of a master tensor, one conversion launch"""
    wn, wt = ops.f32_to_planes_t(m, terms=terms, want_plain=True)
    return wn, wt
