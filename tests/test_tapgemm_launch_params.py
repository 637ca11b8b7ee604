"""CPU: the t2h_tapgemm / t2h_conv_wgrad parameter blocks the convolution wrappers of ops.py build, field by field,
against a table.  The library is replaced by a recorder, so nothing reaches CUDA: the wrappers run on CPU tensors of
small shapes and every launch's struct is reduced to its non-default fields.  Pointers are recorded as (tensor, byte
offset) against the tensors the case passed in or got back.

``d_plane`` (the distance to the output's lo plane) is recorded only where the library reads it: when the output is a
pair of fp16 planes."""
import ctypes as C

import pytest
import torch

from text2human_b200 import _lib, conv_grad, ops

F16 = torch.float16


class _Recorder:
    def __init__(self):
        self.launches = []

    def _take(self, kind, ref):
        s = ref._obj
        self.launches.append((kind, {f: getattr(s, f) for f, _ in s._fields_}, type(s)))
        return 0

    def t2h_tapgemm(self, p, stream):
        return self._take("tapgemm", p)

    def t2h_conv_wgrad(self, p, stream):
        return self._take("wgrad", p)


def _canon(kind, fields, struct, tensors):
    spans = [(name, t.data_ptr(), t.numel() * t.element_size()) for name, t in tensors.items() if t is not None]
    out = {"kind": kind}
    for f, ctype in struct._fields_:
        v = fields[f]
        if ctype is C.c_void_p:
            if v:
                out[f] = next(((n, v - base) for n, base, size in spans if base <= v < base + size), "?")
            continue
        if isinstance(v, C.Array):
            v = list(v)
            while v and v[-1] == 0:
                v.pop()
            v = tuple(v)
        elif isinstance(v, float):
            v = round(v, 6)
        if kind == "tapgemm" and f == "d_plane" and not (fields["d_mode"] == ops.OUT_PLANES and fields["d_terms"] == 2):
            continue
        if v:
            out[f] = v
    return out


def _cases():
    """name -> callable returning (named tensors for pointer labels); each builds its inputs from shapes alone"""
    def planes(*shape):
        return torch.zeros(shape, dtype=F16)

    def conv(T, N, H, W, Ci, Co, taps=None, **kw):
        ntaps = 9 if taps is None else len(taps)
        a, w, b = planes(T, N, H, W, Ci), planes(T, ntaps, Co, Ci), torch.zeros(Co)
        res = torch.zeros(N, H, W, Co) if kw.pop("res", False) else None
        r = ops.conv3x3(a, w, b, residual=res, taps=taps, **kw)
        out, stats = r if kw.get("want_stats") else (r, None)
        return dict(a=a, w=w, bias=b, residual=res, out=out, stats=stats)

    def conv1(T, N, H, W, Ci, Co, **kw):
        a, w, b = planes(T, N, H, W, Ci), planes(T, 1, Co, Ci), torch.zeros(Co)
        r = ops.conv1x1(a, w, b, **kw)
        out, stats = r if kw.get("want_stats") else (r, None)
        return dict(a=a, w=w, bias=b, out=out, stats=stats)

    def down(T, N, Ho, Wo, Ci, Co, want_stats):
        a, w, b = planes(T, 4, N, Ho, Wo, Ci), planes(T, 9, Co, Ci), torch.zeros(Co)
        r = ops.conv3x3_s2(a, w, b, want_stats=want_stats)
        out, stats = r if want_stats else (r, None)
        return dict(a=a, w=w, bias=b, out=out, stats=stats)

    def up(T, N, H, W, Ci, Co, want_stats):
        a, w, b = planes(T, N, H, W, Ci), planes(T, 16, Co, Ci), torch.zeros(Co)
        r = ops.upsample_conv3x3(a, w, b, want_stats=want_stats)
        out, stats = r if want_stats else (r, None)
        return dict(a=a, w=w, bias=b, out=out, stats=stats)

    def k4s2(T, N, H, W, Ci, Co):
        a, w, b = planes(T, 4, N, H // 2, W // 2, Ci), planes(T, 16, Co, Ci), torch.zeros(Co)
        out = conv_grad.forward("k4s2", a, w, b, n=N, in_hw=(H, W), act=ops.ACT_LRELU)
        return dict(a=a, w=w, bias=b, out=out)

    def tap(T, N, H, W, Ci, Co, **kw):
        a, w, b = planes(T, N, H, W, Ci), planes(T, 9, Co, Ci), torch.zeros(Co)
        r = ops.tap_conv(a, w, b, conv_grad.fwd_taps("k3", N), n=N, out_hw=(H, W), **kw)
        out, stats = r if kw.get("want_stats") else (r, None)
        return dict(a=a, w=w, bias=b, out=out, stats=stats)

    def dgrad_s2(T, N, H, W, Ci, Co):
        dy, wt = planes(T, N, H // 2, W // 2, Co), planes(T, 9, Ci, Co)
        out = conv_grad.dgrad("down", dy, wt, n=N, in_hw=(H, W))
        return dict(dy=dy, wt=wt, out=out)

    def dgrad_nb(T, N, H, W, C):
        dy, wt, x = planes(T, N, H, W, C), planes(T, 9, C, C), torch.zeros(N, H, W, C)
        st, g, be = torch.zeros(N, 32, 2, dtype=torch.float64), torch.zeros(C), torch.zeros(C)
        nb = ops.nb_context(x, st, g, be, act="swish", groups=32, eps=1e-6)
        out = conv_grad.dgrad("k3", dy, wt, n=N, in_hw=(H, W), nb=nb)
        return dict(dy=dy, wt=wt, x=x, stats=st, gamma=nb["gamma"], beta=nb["beta"], sums=nb["sums"], out=out)

    def wgrad(T, N, H, W, Ci, Co):
        dy, x, gw = planes(T, N, H, W, Co), planes(T, N, H, W, Ci), torch.zeros(9, Co, Ci)
        conv_grad.wgrad("k3", dy, x, gw, n=N, alpha=0.5)
        return dict(dy=dy, x=x, gw=gw)

    return {
        "conv3x3_f32": lambda: conv(2, 2, 8, 8, 32, 64),
        "conv3x3_fast_planes_out": lambda: conv(1, 2, 8, 8, 32, 64, planes_out=True),
        "conv3x3_planes_out": lambda: conv(2, 2, 8, 8, 32, 64, planes_out=True),
        "conv3x3_nchw_out": lambda: conv(2, 1, 8, 8, 32, 8, nchw_out=True),
        "conv3x3_residual_stats": lambda: conv(2, 2, 8, 8, 32, 64, res=True, want_stats=True),
        "conv3x3_relu_1x1_taps": lambda: conv(1, 2, 8, 8, 32, 64, taps=ops._TAPS_1, planes_out=True, act=ops.ACT_RELU),
        "conv1x1_stats": lambda: conv1(2, 2, 8, 8, 32, 128, want_stats=True),
        "conv1x1_planes_out": lambda: conv1(2, 1, 4, 4, 64, 32, planes_out=True),
        "conv3x3_s2_stats": lambda: down(2, 2, 4, 4, 32, 64, True),
        "conv3x3_s2_fast": lambda: down(1, 1, 4, 4, 32, 128, False),
        "upsample_conv3x3_stats": lambda: up(2, 2, 4, 4, 32, 64, True),
        "upsample_conv3x3_fast": lambda: up(1, 1, 4, 4, 64, 128, False),
        "tap_conv_k4s2": lambda: k4s2(2, 2, 8, 8, 32, 64),
        "tap_conv_stats": lambda: tap(2, 2, 8, 8, 32, 64, want_stats=True, alpha=2.0),
        "tap_conv_planes_out": lambda: tap(2, 1, 8, 8, 32, 64, planes_out=True, act=ops.ACT_GELU),
        "tap_conv_nchw_out": lambda: tap(1, 1, 8, 8, 32, 8, nchw_out=True),
        "tap_conv_dgrad_s2": lambda: dgrad_s2(2, 2, 8, 8, 32, 64),
        "tap_conv_dgrad_nb": lambda: dgrad_nb(2, 1, 4, 4, 128),
        "conv_wgrad": lambda: wgrad(2, 2, 8, 8, 32, 64),
    }


def record(monkeypatch, case):
    rec = _Recorder()
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(ops, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setitem(ops.FUSE_NB, "on", True)
    tensors = _cases()[case]()
    return [_canon(kind, fields, struct, tensors) for kind, fields, struct in rec.launches]


@pytest.mark.parametrize("case", sorted(_cases()))
def test_launch_params(monkeypatch, case):
    assert record(monkeypatch, case) == EXPECTED[case]


# recorded from the wrappers as they built each launch by hand, before conv3x3 and conv3x3_s2 became calls of tap_conv
EXPECTED = {
    'conv3x3_f32': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 4096,
         'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
    ],
    'conv3x3_fast_planes_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 2, 'a_imgs': 2, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 1, 'b_term_g': 9,
         'b_groups': 9, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 1, 'd': ('out', 0), 'd_mode': 1,
         'd_terms': 1, 'd_sn': 4096, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha':
         1.0},
    ],
    'conv3x3_planes_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_mode': 1,
         'd_terms': 2, 'd_plane': 8192, 'd_sn': 4096, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0),
         'bias_mode': 1, 'alpha': 1.0},
    ],
    'conv3x3_nchw_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 1, 'a_imgs': 2, 'n_img': 1, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 8, 'b_sn': 32, 'b_sg': 256, 'b_sg2': 256, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 512,
         'd_sh': 8, 'd_sw': 1, 'd_sc': 64, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
    ],
    'conv3x3_residual_stats': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 4096,
         'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0, 'residual': ('residual',
         0), 'gn_stats': ('stats', 0), 'gn_cpg': 2},
    ],
    'conv3x3_relu_1x1_taps': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 2, 'a_imgs': 2, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 1, 'b_term_g': 1,
         'b_groups': 1, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 1, 'nterms': 1,
         'd': ('out', 0), 'd_mode': 1, 'd_terms': 1, 'd_sn': 4096, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias',
         0), 'bias_mode': 1, 'act': 2, 'alpha': 1.0},
    ],
    'conv1x1_stats': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 1,
         'b_groups': 2, 'b_groups2': 1, 'n_out': 128, 'b_sn': 32, 'b_sg': 4096, 'b_sg2': 4096, 'ntaps': 1, 'nterms': 3,
         'd': ('out', 0), 'd_sn': 8192, 'd_sh': 1024, 'd_sw': 128, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1,
         'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 4},
    ],
    'conv1x1_planes_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 1, 'a_imgs': 2, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 1,
         'b_groups': 2, 'b_groups2': 1, 'n_out': 32, 'b_sn': 64, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 1, 'nterms': 3,
         'd': ('out', 0), 'd_mode': 1, 'd_terms': 2, 'd_plane': 512, 'd_sn': 512, 'd_sh': 128, 'd_sw': 32, 'd_sc': 1,
         'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
    ],
    'conv3x3_s2_stats': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 8, 'a_imgs': 16, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (0,
         0, 0, 0, 0, 0, 1, 1, 1), 'tap_dx': (0, 0, 1, 0, 0, 1, 0, 0, 1), 'tap_img_off': (0, 2, 0, 4, 6, 4, 0, 2),
         'nterms': 3, 'd': ('out', 0), 'd_sn': 1024, 'd_sh': 256, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0),
         'bias_mode': 1, 'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 2},
    ],
    'conv3x3_s2_fast': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 4, 'a_imgs': 4, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 0), 'b_terms': 1, 'b_term_g': 9,
         'b_groups': 9, 'b_groups2': 1, 'n_out': 128, 'b_sn': 32, 'b_sg': 4096, 'b_sg2': 4096, 'ntaps': 9, 'tap_dy': (0,
         0, 0, 0, 0, 0, 1, 1, 1), 'tap_dx': (0, 0, 1, 0, 0, 1, 0, 0, 1), 'tap_img_off': (0, 1, 0, 2, 3, 2, 0, 1),
         'nterms': 1, 'd': ('out', 0), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 128, 'd_sc': 1, 'bias': ('bias', 0),
         'bias_mode': 1, 'alpha': 1.0},
    ],
    'upsample_conv3x3_stats': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 16,
         'b_groups': 20, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 4, 'tap_dy': (-1,
         -1), 'tap_dx': (-1, 0, -1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 4096, 'd_sh': 1024, 'd_sw': 128, 'd_sc': 1,
         'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 2},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 16384), 'b_terms': 2, 'b_term_g':
         16, 'b_groups': 20, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 4, 'tap_dy':
         (-1, -1), 'tap_dx': (0, 1, 0, 1), 'nterms': 3, 'd': ('out', 256), 'd_sn': 4096, 'd_sh': 1024, 'd_sw': 128,
         'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 2},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 32768), 'b_terms': 2, 'b_term_g':
         16, 'b_groups': 20, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 4, 'tap_dy':
         (0, 0, 1, 1), 'tap_dx': (-1, 0, -1), 'nterms': 3, 'd': ('out', 2048), 'd_sn': 4096, 'd_sh': 1024, 'd_sw': 128,
         'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 2},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 49152), 'b_terms': 2, 'b_term_g':
         16, 'b_groups': 20, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 4, 'tap_dy':
         (0, 0, 1, 1), 'tap_dx': (0, 1, 0, 1), 'nterms': 3, 'd': ('out', 2304), 'd_sn': 4096, 'd_sh': 1024, 'd_sw': 128,
         'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0, 'gn_stats': ('stats', 0), 'gn_cpg': 2},
    ],
    'upsample_conv3x3_fast': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 1, 'a_imgs': 1, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('w', 0), 'b_terms': 1, 'b_term_g': 16,
         'b_groups': 4, 'b_groups2': 1, 'n_out': 128, 'b_sn': 64, 'b_sg': 8192, 'b_sg2': 8192, 'ntaps': 4, 'tap_dy': (-1,
         -1), 'tap_dx': (-1, 0, -1), 'nterms': 1, 'd': ('out', 0), 'd_sn': 8192, 'd_sh': 2048, 'd_sw': 256, 'd_sc': 1,
         'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 1, 'a_imgs': 1, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('w', 65536), 'b_terms': 1, 'b_term_g':
         16, 'b_groups': 4, 'b_groups2': 1, 'n_out': 128, 'b_sn': 64, 'b_sg': 8192, 'b_sg2': 8192, 'ntaps': 4, 'tap_dy':
         (-1, -1), 'tap_dx': (0, 1, 0, 1), 'nterms': 1, 'd': ('out', 512), 'd_sn': 8192, 'd_sh': 2048, 'd_sw': 256,
         'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 1, 'a_imgs': 1, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('w', 131072), 'b_terms': 1,
         'b_term_g': 16, 'b_groups': 4, 'b_groups2': 1, 'n_out': 128, 'b_sn': 64, 'b_sg': 8192, 'b_sg2': 8192, 'ntaps':
         4, 'tap_dy': (0, 0, 1, 1), 'tap_dx': (-1, 0, -1), 'nterms': 1, 'd': ('out', 4096), 'd_sn': 8192, 'd_sh': 2048,
         'd_sw': 256, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 1, 'a_imgs': 1, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('w', 196608), 'b_terms': 1,
         'b_term_g': 16, 'b_groups': 4, 'b_groups2': 1, 'n_out': 128, 'b_sn': 64, 'b_sg': 8192, 'b_sg2': 8192, 'ntaps':
         4, 'tap_dy': (0, 0, 1, 1), 'tap_dx': (0, 1, 0, 1), 'nterms': 1, 'd': ('out', 4608), 'd_sn': 8192, 'd_sh': 2048,
         'd_sw': 256, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
    ],
    'tap_conv_k4s2': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 8, 'a_imgs': 16, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 32, 'a_sw': 32, 'a_sh': 128, 'a_sn': 512, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 16,
         'b_groups': 32, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 16, 'tap_dy':
         (-1, -1, -1, -1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1), 'tap_dx': (-1, 0, 0, 1, -1, 0, 0, 1, -1, 0, 0, 1, -1, 0,
         0, 1), 'tap_img_off': (6, 4, 6, 4, 2, 0, 2, 0, 6, 4, 6, 4, 2, 0, 2), 'nterms': 3, 'd': ('out', 0), 'd_sn': 1024,
         'd_sh': 256, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'act': 3, 'alpha': 1.0},
    ],
    'tap_conv_stats': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 4096,
         'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 2.0, 'gn_stats': ('stats', 0),
         'gn_cpg': 2},
    ],
    'tap_conv_planes_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 2, 'a_term_imgs': 1, 'a_imgs': 2, 'n_img': 1, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 64, 'b_sn': 32, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 9, 'tap_dy': (-1,
         -1, -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 3, 'd': ('out', 0), 'd_mode': 1,
         'd_terms': 2, 'd_plane': 4096, 'd_sn': 4096, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'bias': ('bias', 0),
         'bias_mode': 1, 'act': 1, 'alpha': 1.0},
    ],
    'tap_conv_nchw_out': [
        {'kind': 'tapgemm', 'a': ('a', 0), 'a_terms': 1, 'a_term_imgs': 1, 'a_imgs': 1, 'n_img': 1, 'H': 8, 'W': 8,
         'a_H': 8, 'a_W': 8, 'C': 32, 'a_sw': 32, 'a_sh': 256, 'a_sn': 2048, 'b': ('w', 0), 'b_terms': 1, 'b_term_g': 9,
         'b_groups': 9, 'b_groups2': 1, 'n_out': 8, 'b_sn': 32, 'b_sg': 256, 'b_sg2': 256, 'ntaps': 9, 'tap_dy': (-1, -1,
         -1, 0, 0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'nterms': 1, 'd': ('out', 0), 'd_sn': 512,
         'd_sh': 8, 'd_sw': 1, 'd_sc': 64, 'bias': ('bias', 0), 'bias_mode': 1, 'alpha': 1.0},
    ],
    'tap_conv_dgrad_s2': [
        {'kind': 'tapgemm', 'a': ('dy', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('wt', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 18, 'b_groups2': 1, 'n_out': 32, 'b_sn': 64, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 4, 'tap_dy': (0,
         0, -1, -1), 'tap_dx': (0, -1, 0, -1), 'nterms': 3, 'd': ('out', 0), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 64,
         'd_sc': 1, 'alpha': 1.0, 'use_tap_w': 1, 'tap_w': (0, 2, 6, 8)},
        {'kind': 'tapgemm', 'a': ('dy', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('wt', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 17, 'b_groups2': 1, 'n_out': 32, 'b_sn': 64, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 2, 'tap_dy': (0,
         -1), 'nterms': 3, 'd': ('out', 128), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'alpha': 1.0,
         'use_tap_w': 1, 'tap_w': (1, 7)},
        {'kind': 'tapgemm', 'a': ('dy', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('wt', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 15, 'b_groups2': 1, 'n_out': 32, 'b_sn': 64, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 2, 'tap_dx': (0,
         -1), 'nterms': 3, 'd': ('out', 1024), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'alpha': 1.0,
         'use_tap_w': 1, 'tap_w': (3, 5)},
        {'kind': 'tapgemm', 'a': ('dy', 0), 'a_terms': 2, 'a_term_imgs': 2, 'a_imgs': 4, 'n_img': 2, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 64, 'a_sw': 64, 'a_sh': 256, 'a_sn': 1024, 'b': ('wt', 0), 'b_terms': 2, 'b_term_g': 9,
         'b_groups': 14, 'b_groups2': 1, 'n_out': 32, 'b_sn': 64, 'b_sg': 2048, 'b_sg2': 2048, 'ntaps': 1, 'nterms': 3,
         'd': ('out', 1152), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 64, 'd_sc': 1, 'alpha': 1.0, 'use_tap_w': 1, 'tap_w':
         (4,)},
    ],
    'tap_conv_dgrad_nb': [
        {'kind': 'tapgemm', 'a': ('dy', 0), 'a_terms': 2, 'a_term_imgs': 1, 'a_imgs': 2, 'n_img': 1, 'H': 4, 'W': 4,
         'a_H': 4, 'a_W': 4, 'C': 128, 'a_sw': 128, 'a_sh': 512, 'a_sn': 2048, 'b': ('wt', 0), 'b_terms': 2, 'b_term_g':
         9, 'b_groups': 18, 'b_groups2': 1, 'n_out': 128, 'b_sn': 128, 'b_sg': 16384, 'b_sg2': 16384, 'ntaps': 9,
         'tap_dy': (1, 1, 1, 0, 0, 0, -1, -1, -1), 'tap_dx': (1, 0, -1, 1, 0, -1, 1, 0, -1), 'nterms': 3, 'd': ('out',
         0), 'd_sn': 2048, 'd_sh': 512, 'd_sw': 128, 'd_sc': 1, 'alpha': 1.0, 'residual': ('x', 0), 'nb_sums': ('sums',
         0), 'nb_stats': ('stats', 0), 'nb_gamma': ('gamma', 0), 'nb_beta': ('beta', 0), 'nb_eps': 1e-06, 'nb_act': 1,
         'nb_groups': 32},
    ],
    'conv_wgrad': [
        {'kind': 'wgrad', 'dy': ('dy', 0), 'dy_terms': 2, 'dy_term_imgs': 2, 'dy_imgs': 4, 'n_img': 2, 'H': 8, 'W': 8,
         'cout': 64, 'dy_sw': 64, 'dy_sh': 512, 'dy_sn': 4096, 'x': ('x', 0), 'x_terms': 2, 'x_term_imgs': 2, 'x_imgs':
         4, 'x_H': 8, 'x_W': 8, 'cin': 32, 'x_sw': 32, 'x_sh': 256, 'x_sn': 2048, 'ntaps': 9, 'tap_dy': (-1, -1, -1, 0,
         0, 0, 1, 1, 1), 'tap_dx': (-1, 0, 1, -1, 0, 1, -1, 0, 1), 'dw': ('gw', 0), 'dw_tap_stride': 2048, 'dw_ld': 32,
         'alpha': 0.5, 'nterms': 3},
    ],
}
