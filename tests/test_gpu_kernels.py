"""GPU parity of the individual libt2h kernels (through the C ABI) against fp64/fp32 PyTorch on the
same operands, and of the quantizer kernel against the C oracle (bit-exact)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_recipes as R

pytestmark = pytest.mark.gpu


def _rel(got, ref):
    return ((got.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-30)).item()


def _sum(p):
    return p.float().sum(0)


# ------------------------------------------------------------------ tapgemm
@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("M,K,N", [(128, 64, 16), (300, 512, 256), (2048, 512, 1536), (1000, 2048, 512),
                                   (4096, 32, 32), (64, 8, 24)])
def test_linear_matches_fp64(cuda, terms, M, K, N):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(M + K + N)
    x = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) / K ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    r = torch.randn(M, N, device=cuda, generator=g)
    a, wp = ops.split_planes(x, terms), ops.pack_linear_weight(w, terms)
    ref = _sum(a).double() @ _sum(wp)[0].double().t() + b.double()
    out = ops.linear(a, wp, b, residual=r)
    assert _rel(out, ref + r.double()) < 2e-5  # products of the split operands are exact; fp32 accumulate
    out = ops.linear(a, wp, b, act=ops.ACT_GELU, planes_out=True)
    tol = 1e-3 if terms == 1 else 2e-5  # single fp16 output plane rounds to 11 bits
    assert _rel(_sum(out), F.gelu(ref)) < tol
    if terms == 2:  # the 3-product split reproduces the fp32 GEMM of the ORIGINAL operands
        assert _rel(ops.linear(a, wp, b), x.double() @ w.double().t() + b.double()) < 2e-5


@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("N,H,W,Cin,Cout", [(2, 32, 16, 64, 128), (1, 16, 8, 512, 512), (1, 64, 32, 3, 128),
                                            (2, 64, 32, 128, 3), (2, 256, 128, 128, 128), (3, 24, 20, 24, 64),
                                            (1, 8, 4, 32, 32)])
def test_conv3x3_matches_fp64(cuda, terms, N, H, W, Cin, Cout):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(H * 7 + Cin + Cout)
    x = torch.randn(N, Cin, H, W, device=cuda, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device=cuda, generator=g) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=cuda, generator=g)
    a = ops.nchw_to_planes(x, terms=terms)
    wp = ops.pack_conv_weight(w, terms, c_pad=a.shape[-1])
    xe = _sum(a)[..., :Cin].permute(0, 3, 1, 2).double()
    we = _sum(wp)[..., :Cin].reshape(3, 3, Cout, Cin).permute(2, 3, 0, 1).double()
    ref = F.conv2d(xe, we, b.double(), padding=1)
    res = torch.randn(N, H, W, Cout, device=cuda, generator=g)
    out = ops.conv3x3(a, wp, b, residual=res)
    assert _rel(out.permute(0, 3, 1, 2), ref + res.permute(0, 3, 1, 2).double()) < 3e-5
    out = ops.conv3x3(a, wp, b, nchw_out=True)
    assert _rel(out, ref) < 3e-5
    if terms == 2:
        assert _rel(out, F.conv2d(x.double(), w.double(), b.double(), padding=1)) < 3e-5


@pytest.mark.parametrize("terms", [1, 2])
def test_conv3x3_stride2_and_upsample(cuda, terms):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randn(2, 64, 32, 128, device=cuda, generator=g)  # NHWC
    w = torch.randn(128, 128, 3, 3, device=cuda, generator=g) / (9 * 128) ** 0.5
    b = torch.randn(128, device=cuda, generator=g)
    wp = ops.pack_conv_weight(w, terms)
    we = _sum(wp).reshape(3, 3, 128, 128).permute(2, 3, 0, 1).double()
    xs = _sum(ops.split_planes(x, terms)).permute(0, 3, 1, 2).double()
    out = ops.conv3x3_s2(ops.f32_to_planes(x, ops.CVT_S2D, terms), wp, b)
    ref = F.conv2d(F.pad(xs, (0, 1, 0, 1)), we, b.double(), stride=2)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 3e-5
    out = ops.conv3x3(ops.f32_to_planes(x, ops.CVT_UP2X, terms), wp, b)
    ref = F.conv2d(F.interpolate(xs, scale_factor=2.0, mode="nearest"), we, b.double(), padding=1)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 3e-5


@pytest.mark.parametrize("terms", [1, 2])
def test_bmm_and_multihead_products(cuda, terms):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(9)
    a = torch.randn(3, 200, 96, device=cuda, generator=g)
    b = torch.randn(3, 130, 96, device=cuda, generator=g)
    ap, bp = ops.split_planes(a, terms), ops.split_planes(b, terms)
    ref = 0.5 * _sum(ap).double() @ _sum(bp).double().transpose(1, 2)
    assert _rel(ops.bmm_nt(ap, bp, alpha=0.5), ref) < 2e-5
    # multi-head: B=2, T=64, nh=4, hs=16
    B, Tn, nh, hs = 2, 64, 4, 16
    Cc = nh * hs
    qk = torch.randn(B * Tn, 2 * Cc, device=cuda, generator=g)
    qkp = ops.split_planes(qk, terms)
    qe = _sum(qkp).double()
    q = qe[:, :Cc].view(B, Tn, nh, hs).transpose(1, 2)
    k = qe[:, Cc:].view(B, Tn, nh, hs).transpose(1, 2)
    s = ops.mha_scores(qkp, B, Tn, nh)
    assert s.shape == (B, nh, Tn, Tn)
    assert _rel(s, q @ k.transpose(-2, -1)) < 2e-5
    p = ops.softmax_rows(s, scale=0.25, terms=terms)
    pe = _sum(p).double()
    assert _rel(pe, torch.softmax(s.double() * 0.25, -1)) < (1e-3 if terms == 1 else 1e-6)
    v = torch.randn(B, Tn, Cc, device=cuda, generator=g)
    vt = ops.split_planes(v.transpose(1, 2).contiguous(), terms)  # [T,B,C,Tn]
    y = ops.mha_pv(p, vt, B, Tn, nh)
    ve = _sum(vt).double().transpose(1, 2).reshape(B, Tn, nh, hs).transpose(1, 2)
    ref = (pe @ ve).transpose(1, 2).reshape(B * Tn, Cc)
    assert _rel(_sum(y), ref) < (1e-3 if terms == 1 else 2e-5)


# ------------------------------------------------------------- HBM kernels
@pytest.mark.parametrize("C,H,W", [(128, 64, 32), (64, 16, 8), (512, 32, 16), (32, 8, 4)])
def test_groupnorm_swish_matches_torch(cuda, C, H, W):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C + H)
    x = torch.randn(3, H, W, C, device=cuda, generator=g) * 2 + 0.5
    gamma = torch.randn(C, device=cuda, generator=g)
    beta = torch.randn(C, device=cuda, generator=g)
    xn = x.permute(0, 3, 1, 2).double()
    ref = F.group_norm(xn, 32, gamma.double(), beta.double(), eps=1e-6)
    out = _sum(ops.group_norm(x, gamma, beta, swish=False, terms=2)).permute(0, 3, 1, 2)
    assert _rel(out, ref) < 5e-6
    out = _sum(ops.group_norm(x, gamma, beta, swish=True, terms=2)).permute(0, 3, 1, 2)
    assert _rel(out, ref * torch.sigmoid(ref)) < 5e-6
    out1 = ops.group_norm(x, gamma, beta, swish=True, terms=1)[0].float().permute(0, 3, 1, 2)
    assert _rel(out1, ref * torch.sigmoid(ref)) < 1e-3


def test_layout_and_small_kernels(cuda):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(3)
    x = torch.randn(2, 37, 9, 5, device=cuda, generator=g)  # NCHW, awkward sizes
    assert torch.equal(ops.nchw_to_nhwc(x), x.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(ops.nhwc_to_nchw(ops.nchw_to_nhwc(x)), x)
    p = ops.nchw_to_planes(x, terms=2)
    assert p.shape == (2, 2, 9, 5, 40)
    assert _rel(_sum(p)[..., :37], x.permute(0, 2, 3, 1)) < 1e-6 and (_sum(p)[..., 37:] == 0).all()
    a = torch.randn(1001, device=cuda, generator=g).view(1, 1001)
    b = torch.randn(1001, device=cuda, generator=g).view(1, 1001)
    a2 = torch.zeros(4096, device=cuda)[:1001].copy_(a.view(-1))
    ref = a2 + b.view(-1)
    ops.add_inplace(a2, b.view(-1).contiguous())
    assert torch.equal(a2, ref)
    xl = torch.randn(100, 512, device=cuda, generator=g)
    gm, bt = torch.randn(512, device=cuda, generator=g), torch.randn(512, device=cuda, generator=g)
    assert _rel(_sum(ops.layer_norm(xl, gm, bt, terms=2)), F.layer_norm(xl.double(), (512,), gm.double(),
                                                                         bt.double())) < 5e-6
    m = R.blocky_mask(1, 2, 512, 256, 32, extra_ids=(20,)).to(cuda)
    ids = ops.mask_to_ids(m, 32, 16)
    assert torch.equal(ids.long(), F.interpolate(m, size=(32, 16), mode="nearest")[:, 0].long())


# ---------------------------------------------------------------- quantizers
@pytest.mark.parametrize("kind", ["default", "trained"])
@pytest.mark.parametrize("cfg", ["top", "bottom", "plain", "full_top"])
def test_quantizer_bit_exact_vs_oracle(cuda, kind, cfg):
    from oracle import vq_oracle
    from text2human_b200 import ops
    if cfg == "top":
        B, Hz, Wz, Cz, ps, nb, ne = 2, 32, 16, 256, 1, 18, 128
        mask = R.blocky_mask(13, B, 512, 256, 64, extra_ids=(20,))
    elif cfg == "full_top":  # the real vqvae_top.yml codebook geometry, ragged bins
        B, Hz, Wz, Cz, ps, nb, ne = 3, 32, 16, 256, 1, 18, 1024
        mask = R.iid_mask(14, B, 512, 256)
    elif cfg == "bottom":
        B, Hz, Wz, Cz, ps, nb, ne = 2, 32, 16, 32, 2, 18, 64
        mask = R.blocky_mask(23, B, 256, 128, 32)
    else:
        B, Hz, Wz, Cz, ps, nb, ne = 2, 32, 16, 32, 1, 1, 128
        mask = None
    cb = R.codebooks(11, nb, ne, Cz * ps * ps, kind)
    z = R.latent(12, (B, Hz, Wz, Cz), 1.0 if kind == "trained" else 0.02)  # NHWC
    ids_np = vq_oracle.nearest_ids(mask.numpy(), Hz // ps, Wz // ps) if mask is not None else None
    want = vq_oracle.search(z.numpy(), cb.numpy(), ids_np, ps=ps, cont_stride=1024)
    ids = ops.mask_to_ids(mask.to(cuda), Hz // ps, Wz // ps) if mask is not None else None
    if ids is not None:
        assert np.array_equal(ids.cpu().numpy(), ids_np)
    got = ops.vq_search(z.to(cuda), cb.to(cuda), ids, ps=ps, cont_stride=1024)
    assert np.array_equal(got["idx"].cpu().numpy(), want["idx"])
    assert np.array_equal(got["idx_cont"].cpu().numpy(), want["idx_cont"])
    assert np.array_equal(got["idx_list"].cpu().numpy(), want["idx_list"])
    assert np.array_equal(got["zq_nhwc"].cpu().numpy(), want["zq_nhwc"])  # bit-exact values too
    assert np.array_equal(got["zq_nchw"].cpu().numpy(), np.transpose(want["zq_nhwc"], (0, 3, 1, 2)))
    assert abs(got["sqerr"].item() - want["sqerr"]) <= 1e-9 * abs(want["sqerr"]) + 1e-12
    zq, _ = ops.vq_gather(cb.to(cuda), got["idx"], ids, B=B, Hz=Hz, Wz=Wz, Cz=Cz, ps=ps, want_nhwc=True,
                          want_nchw=False)
    assert np.array_equal(zq.cpu().numpy(), vq_oracle.gather(cb.numpy(), want["idx"], ids_np, B, Hz, Wz, Cz, ps))


def test_quantizer_edge_cases(cuda):
    """ties -> lowest index; every row unselected; a single row; duplicate codes"""
    from oracle import vq_oracle
    from text2human_b200 import ops
    cb = torch.zeros(2, 8, 16)
    cb[0, 3] = 1.0
    cb[0, 5] = 1.0  # duplicate of code 3: argmin must return 3
    cb[1] = torch.arange(8).view(8, 1).float().expand(8, 16)
    z = torch.ones(1, 2, 2, 16)
    ids = torch.tensor([[[0, 1], [7, -1]]], dtype=torch.int32)
    got = ops.vq_search(z.to(cuda), cb.to(cuda), ids.to(cuda), cont_stride=8)
    want = vq_oracle.search(z.numpy(), cb.numpy(), ids.numpy(), cont_stride=8)
    assert got["idx"].view(-1).tolist() == [3, 1, -1, -1] == want["idx"].reshape(-1).tolist()
    assert got["idx_cont"].view(-1).tolist() == [3, 9, -1, -1]
    assert torch.equal(got["zq_nhwc"][0, 1].cpu(), torch.zeros(2, 16))  # unselected rows -> 0
    assert np.array_equal(got["idx_list"].cpu().numpy(), want["idx_list"])


@pytest.mark.parametrize("C,Cout,H,W", [(64, 128, 32, 16), (128, 256, 16, 8), (64, 64, 40, 24), (256, 512, 8, 4)])
def test_fused_groupnorm_statistics_in_conv_epilogue(cuda, C, Cout, H, W):
    """the conv epilogue's (sum, sumsq) per (image, group) equal those of its own fp32 output"""
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(C + Cout + H)
    x = torch.randn(3, C, H, W, device=cuda, generator=g)
    w = torch.randn(Cout, C, 3, 3, device=cuda, generator=g) / (9 * C) ** 0.5
    b = torch.randn(Cout, device=cuda, generator=g)
    res = torch.randn(3, H, W, Cout, device=cuda, generator=g)
    a = ops.nchw_to_planes(x, terms=2)
    out, stats = ops.conv3x3(a, ops.pack_conv_weight(w, 2), b, residual=res, want_stats=True)
    assert stats is not None and stats.shape == (3, 32, 2)
    o = out.double().view(3, H * W, 32, Cout // 32)
    want = torch.stack((o.sum((1, 3)), (o * o).sum((1, 3))), -1)
    assert _rel(stats, want) < 1e-5
    # and GroupNorm fed with them matches GroupNorm that measures its own statistics
    gm, bt = torch.randn(Cout, device=cuda, generator=g), torch.randn(Cout, device=cuda, generator=g)
    a1 = ops.group_norm(out, gm, bt, swish=True, terms=2, stats=stats)
    a2 = ops.group_norm(out, gm, bt, swish=True, terms=2)
    assert _rel(_sum(a1), _sum(a2)) < 1e-5
    # 1x1 conv (spatial tiles) and stride-2 conv epilogues too
    o1, s1 = ops.conv1x1(a, ops.pack_linear_weight(w[:, :, 1, 1].contiguous(), 2), b, want_stats=True)
    o1d = o1.double().view(3, H * W, 32, Cout // 32)
    assert _rel(s1, torch.stack((o1d.sum((1, 3)), (o1d * o1d).sum((1, 3))), -1)) < 1e-5


GN_CONV_CASES = [  # N, H, W, Cin, Cout, terms, residual, nchw
    (2, 32, 16, 128, 128, 2, True, False), (1, 64, 32, 128, 256, 2, False, False), (2, 16, 8, 256, 256, 2, True, False),
    (2, 8, 4, 256, 128, 2, False, False), (2, 32, 16, 128, 3, 2, False, True), (2, 32, 16, 128, 128, 1, True, False),
    (3, 40, 24, 64, 128, 2, False, False), (1, 256, 128, 128, 128, 2, True, False),
]


@pytest.mark.parametrize("case", GN_CONV_CASES, ids=lambda c: "-".join(str(int(v)) for v in c))
def test_groupnorm_swish_then_conv3x3_matches_fp64(cuda, case):
    """swish(GroupNorm(x)) -> 3x3 conv (Normalize() + nonlinearity() + Conv2d of ResnetBlock / conv_out,
    vqgan_arch.py:599-609, :916-918, :1030-1032) as the gn_apply pass and the conv, against fp64 torch; the conv
    epilogue's GroupNorm sums against fp64 sums of its own output"""
    from text2human_b200 import ops
    N, H, W, Ci, Co, terms, residual, nchw = case
    g = torch.Generator().manual_seed(sum(int(v) for v in case))
    x = (torch.randn(N, H, W, Ci, generator=g) * 1.5 + 0.3).to(cuda)
    gamma = (1 + 0.1 * torch.randn(Ci, generator=g)).to(cuda)
    beta = (0.1 * torch.randn(Ci, generator=g)).to(cuda)
    w = torch.randn(Co, Ci, 3, 3, generator=g) / (9 * Ci) ** 0.5
    b = (0.1 * torch.randn(Co, generator=g)).to(cuda)
    res = torch.randn(N, H, W, Co, generator=g).to(cuda) if residual else None
    a = ops.group_norm(x, gamma, beta, swish=True, eps=1e-6, terms=terms, stats=ops.norm_stats(x, 32))
    out = ops.conv3x3(a, ops.pack_conv_weight(w.to(cuda), terms), b, residual=res, nchw_out=nchw,
                      want_stats=not nchw)
    if not nchw:
        out, stats = out
        if stats is not None:
            o = out.double().view(N, H * W, 32, Co // 32)
            assert _rel(stats, torch.stack((o.sum((1, 3)), (o * o).sum((1, 3))), -1)) < 1e-5
    xr = x.permute(0, 3, 1, 2).double()
    u = F.group_norm(xr, 32, gamma.double(), beta.double(), eps=1e-6)
    want = F.conv2d(u * torch.sigmoid(u), w.to(cuda).double(), b.double(), padding=1)
    if residual:
        want = want + res.permute(0, 3, 1, 2).double()
    got = out if nchw else out.permute(0, 3, 1, 2)
    assert _rel(got, want) < (3e-5 if terms == 2 else 4e-3)


@pytest.mark.parametrize("terms", [1, 2])
@pytest.mark.parametrize("N,H,W,Cin,Cout", [(1, 37, 19, 40, 128), (2, 21, 50, 128, 256), (1, 5, 3, 64, 128),
                                            (3, 33, 17, 72, 72), (1, 512, 256, 8, 128)])
def test_conv3x3_ragged_shapes_with_residual_and_stats(cuda, terms, N, H, W, Cin, Cout):
    """image extents that are not multiples of the 16x8 / 16x16 pixel tiles, channel counts that are not
    multiples of the 64-wide K chunk: TMA clipping on loads and stores, partial-tile GroupNorm sums"""
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(N * H + W + Cin)
    x = torch.randn(N, Cin, H, W, device=cuda, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device=cuda, generator=g) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=cuda, generator=g)
    res = torch.randn(N, H, W, Cout, device=cuda, generator=g)
    a = ops.nchw_to_planes(x, terms=terms)
    wp = ops.pack_conv_weight(w, terms, c_pad=a.shape[-1])
    out, stats = ops.conv3x3(a, wp, b, residual=res, want_stats=True)
    xe = _sum(a)[..., :Cin].permute(0, 3, 1, 2).double()
    we = _sum(wp)[..., :Cin].reshape(3, 3, Cout, Cin).permute(2, 3, 0, 1).double()
    ref = F.conv2d(xe, we, b.double(), padding=1) + res.permute(0, 3, 1, 2).double()
    assert _rel(out.permute(0, 3, 1, 2), ref) < 3e-5
    if Cout % 32 == 0 and (Cout // 32) & (Cout // 32 - 1) == 0 and Cout // 32 >= 2:
        o = out.double().view(N, H * W, 32, Cout // 32)
        assert _rel(stats, torch.stack((o.sum((1, 3)), (o * o).sum((1, 3))), -1)) < 1e-5
    else:
        assert stats is None


def test_upsample_fold_matches_interpolate_then_conv(cuda):
    from text2human_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(77)
    for (N, H, W, C) in [(2, 16, 8, 128), (1, 9, 5, 64), (1, 32, 16, 256)]:
        x = torch.randn(N, H, W, C, device=cuda, generator=g)
        w = torch.randn(C, C, 3, 3, device=cuda, generator=g) / (9 * C) ** 0.5
        b = torch.randn(C, device=cuda, generator=g)
        out, stats = ops.upsample_conv3x3(ops.f32_to_planes(x, ops.CVT_PLAIN, 2), ops.pack_upsample_conv_weight(w, 2), b,
                                          want_stats=True)
        ref = F.conv2d(F.interpolate(x.permute(0, 3, 1, 2).double(), scale_factor=2.0, mode="nearest"), w.double(),
                       b.double(), padding=1)
        assert out.shape == (N, 2 * H, 2 * W, C)
        assert _rel(out.permute(0, 3, 1, 2), ref) < 3e-5
        o = out.double().view(N, 4 * H * W, 32, C // 32)
        assert _rel(stats, torch.stack((o.sum((1, 3)), (o * o).sum((1, 3))), -1)) < 1e-5


def test_tapgemm_rejects_inconsistent_requests(cuda):
    from text2human_b200 import _lib, ops
    a = ops.split_planes(torch.randn(64, 64, device=cuda), 1)
    w = ops.pack_linear_weight(torch.randn(32, 64, device=cuda), 2)
    out = ops.linear(a, w)  # mixed plane counts fall back to one product and still work
    assert out.shape == (64, 32)
    bad = ops.split_planes(torch.randn(64, 60, device=cuda), 1)[:, :, :57]  # row stride 60 halves: not 16-byte aligned
    with pytest.raises(_lib.T2HError):
        ops.linear(bad, ops.pack_linear_weight(torch.randn(32, 57, device=cuda), 1))
