"""The swapped-operand tap-GEMM's channel ownership: a consumer warpgroup computes 64 output channels of every tile
of its work item (paired mode: one m64n256k16 wgmma per K step over both tiles' pixels), and a warpgroup whose 64
channels all lie at or beyond n_out sits the item out.

Every conv here runs once as a paired launch (at least two tiles per SM) and once per image as launches small enough
to run unpaired; both must write the same bits, into a destination with guard channels that must keep their sentinel.
References, bounds and launch helpers are those of test_gpu_tapgemm_paths.py, test_gpu_tapgemm_pairs.py and, for the
norm-backward sums, test_gpu_backward_paths.py.  A Cout that is neither a multiple of 128 nor at most 128 (192) runs
on the generic kernel and has no case here.
"""
import math

import pytest
import torch

import test_gpu_backward_paths as backward  # (as modules: their tests are called here, not collected again)
import test_gpu_tapgemm_paths as paths
from test_gpu_backward_paths import H100_SMS, NBS
from test_gpu_tapgemm_pairs import _sms, _tiles
from test_gpu_tapgemm_paths import SENTINEL, Case, _case_id, _label, _launch, _operands, _out_hw

GUARD = 4  # guard channels after the valid ones (a multiple of 4: the NHWC pixel stride stays 16-byte aligned)


def idle_warpgroup(n0, wg, n_out):
    """csrc/gemm_tc_swap.cuh, `idle`: warpgroup wg of the column block at n0 owns channels n0 + 64 wg .. + 63; when
    none of them exists it issues no MMA and runs no epilogue for the item (it still waits and releases)"""
    return n0 + 64 * wg >= n_out


# Cout 3, 64, 65, 128 through the strided NCHW epilogue and 128, 256, 384 through the TMA epilogue, one and two
# planes, plain and residual + GroupNorm sums; 131 rows at TH 8: 17 tile rows, the last pair's second tile is outside
OWNER_CASES = [
    Case(6, 131, 40, "k3", 64, 3, 2, "shared", 0.375, "none", False, 0, "nchw"),
    Case(6, 131, 40, "k3", 64, 64, 1, "shared", 1.0, "none", False, 0, "nchw"),
    Case(6, 131, 40, "k3", 64, 65, 2, "image", 1.0, "none", False, 0, "nchw"),
    Case(6, 131, 40, "k3", 64, 128, 1, "shared", 0.375, "none", False, 0, "nchw"),
    Case(6, 131, 40, "k3", 64, 128, 2, "shared", 1.0, "none", False, 0, "nhwc"),
    Case(6, 131, 40, "k3", 64, 128, 1, "shared", 1.0, "none", True, 4, "nhwc"),
    Case(3, 131, 40, "k3", 64, 256, 2, "image", 0.375, "relu", True, 16, "nhwc"),
    Case(3, 131, 40, "k3", 64, 256, 1, "none", 1.0, "none", False, 0, "nhwc"),
    Case(3, 131, 40, "k3", 64, 384, 2, "shared", 1.0, "lrelu", True, 1, "nhwc"),
]

# GroupNorm sums over both tiles of a pair: channels per group 1, 4, 16, 128 with the second tile of a column's last
# pair wholly (131 rows: 17 tile rows) and partly (140 rows: 17.5) below the image
GN_CASES = [Case(3, H, 40, "k3", 64, 256, t, "shared", 1.0, "none", res, cpg, "nhwc")
            for cpg, H, t, res in [(1, 131, 2, True), (1, 140, 1, False), (4, 140, 2, True), (4, 131, 1, False),
                                   (16, 131, 1, True), (16, 140, 2, False), (128, 140, 1, True),
                                   (128, 131, 2, False)]]
NB_CASES = [NBS(3, 131, 40, 256, 256, "swish"), NBS(3, 140, 40, 256, 64, "lrelu"), NBS(3, 131, 40, 256, 16, "none"),
            NBS(3, 140, 40, 256, 2, "swish")]


def _blocks(c):
    """(n0, wg) of every warpgroup of every column block of a case's launches"""
    return [(n0, wg) for n0 in range(0, math.ceil(c.cout / 128) * 128, 128) for wg in (0, 1)]


def test_owner_case_table():
    """the cases are swapped-kernel launches, paired as a whole and unpaired per image (on the 132 SMs of an H100 SXM);
    both kernels meet warpgroups with no channel, with some and with all 64, and both tables end a column on a pair
    whose second tile is outside the image"""
    for c in OWNER_CASES + GN_CASES:
        r = _label(c)
        assert r["kernel"] == "swap" and (r["TW"], r["TH"]) == (16, 8), (c, r)
        assert (r["epi"] == "direct") == (c.out == "nchw")
        assert _tiles(c) >= 2 * H100_SMS > _tiles(c._replace(N=1)), c
    for c in NB_CASES:
        tiles = math.ceil(c.H / 8) * math.ceil(c.W / 16) * c.C // 128
        assert c.N * tiles >= 2 * H100_SMS
    owned = lambda c, n0, wg: min(max(c.cout - n0 - 64 * wg, 0), 64)  # noqa: E731
    # (the one table runs on both kernels: as a whole on the paired one, image by image on the unpaired one)
    seen = {(idle_warpgroup(n0, wg, c.cout), owned(c, n0, wg)) for c in OWNER_CASES for n0, wg in _blocks(c)}
    assert {idle for idle, n in seen} == {True, False}
    assert all(idle == (n == 0) for idle, n in seen)
    assert {n for idle, n in seen} >= {0, 1, 3, 64}
    assert {c.cout for c in OWNER_CASES} >= {3, 64, 65, 128, 256, 384} and {c.terms for c in OWNER_CASES} == {1, 2}
    assert any(c.res and c.gn for c in OWNER_CASES) and any(not c.res and not c.gn for c in OWNER_CASES)
    rows = lambda H: math.ceil(H / 8)  # noqa: E731
    assert {c.gn for c in GN_CASES} == {1, 4, 16, 128} == {c.C // c.groups for c in NB_CASES}
    for cpg in (1, 4, 16, 128):
        hs = {c.H for c in GN_CASES if c.gn == cpg}
        assert any(rows(H) % 2 == 1 for H in hs) and any(rows(H) % 2 == 0 and H % 8 for H in hs), cpg
    assert any(rows(c.H) % 2 == 1 for c in NB_CASES) and any(rows(c.H) % 2 == 0 and c.H % 8 for c in NB_CASES)


def _run_guarded(c, a, wp, taps, bias, res_buf, dev):
    """one launch of the case into the first Cout channels of a sentinel-filled buffer of Cout + GUARD channels; the
    residual buffer has the destination's layout.  -> (valid view, guard view)"""
    Ho, Wo = _out_hw(c)
    N, Co, Ct = c.N, c.cout, c.cout + GUARD
    if c.out == "nchw":
        buf = torch.full((N, Ct, Ho, Wo), SENTINEL, device=dev)
        view, guard, strides = buf[:, :Co], buf[:, Co:], (Ct * Ho * Wo, Wo, 1, Ho * Wo)
        res = None
    else:
        buf = torch.full((N, Ho, Wo, Ct), SENTINEL, device=dev)
        view, guard, strides = buf[..., :Co], buf[..., Co:], (Ho * Wo * Ct, Wo * Ct, Ct, 1)
        res = res_buf[..., :Co] if c.res else None
    stats = torch.zeros(N * (Co // c.gn) * 2, dtype=torch.float64, device=dev) if c.gn else None
    r = _launch(a, wp, taps, n=N, out_hw=(Ho, Wo), d=view, d_strides=strides, bias=bias,
                bias_sn=Co if c.bias == "image" else 0, alpha=c.alpha, act=c.act, residual=res, stats=stats, cpg=c.gn)
    assert r["kernel"] == "swap" and (r["epi"] == "direct") == (c.out == "nchw"), r
    return view, guard


@pytest.mark.gpu
@pytest.mark.parametrize("c", OWNER_CASES, ids=_case_id)
def test_paired_launch_matches_fp64_and_unpaired_launches(cuda, c):
    """a paired launch against fp64 (and its GroupNorm sums), then into a destination with guard channels: they keep
    the sentinel, and the launch writes the bits that unpaired launches over one image each write"""
    dev = cuda
    one = c._replace(N=1)
    assert _tiles(c) >= 2 * _sms() > _tiles(one), f"{_tiles(c)} / {_tiles(one)} tiles on {_sms()} SMs"
    paths.test_tapgemm_path_matches_fp64(cuda, c)
    a, wp, _, _, taps = _operands(c, dev)
    g = torch.Generator().manual_seed(c.cout + 5)
    Ho, Wo = _out_hw(c)
    bias = None
    if c.bias != "none":
        bias = torch.randn((c.N, c.cout) if c.bias == "image" else (c.cout,), generator=g).to(dev)
    res = torch.randn(c.N, Ho, Wo, c.cout + GUARD, generator=g).to(dev) if c.res else None
    d, guard = _run_guarded(c, a, wp, taps, bias, res, dev)
    assert (guard == SENTINEL).all(), f"{int((guard != SENTINEL).sum())} writes beyond channel {c.cout}"
    assert (d != SENTINEL).all(), "valid elements left unwritten"
    for n in range(c.N):
        d1, guard1 = _run_guarded(one, a[:, n:n + 1].contiguous(), wp, taps,
                                  bias[n:n + 1] if c.bias == "image" else bias,
                                  res[n:n + 1].contiguous() if c.res else None, dev)
        assert (guard1 == SENTINEL).all(), f"image {n}, unpaired: writes beyond channel {c.cout}"
        assert torch.equal(d[n:n + 1], d1), f"image {n}: paired and unpaired launches differ"


@pytest.mark.gpu
@pytest.mark.parametrize("c", GN_CASES, ids=_case_id)
def test_group_norm_sums_over_both_tiles_match_fp64(cuda, c):
    """the output and the GroupNorm sums of a paired launch whose last pairs end partly or wholly below the image,
    through the mean and variance as test_gpu_tapgemm_paths.py checks them"""
    assert _tiles(c) >= 2 * _sms()
    paths.test_tapgemm_path_matches_fp64(cuda, c)


@pytest.mark.gpu
@pytest.mark.parametrize("c", NB_CASES, ids=lambda c: f"n{c.N}x{c.H}x{c.W}-C{c.C}-g{c.groups}-{c.act}")
def test_nb_sums_over_both_tiles_match_fp64(cuda, c):
    """norm-backward sums of a paired data-gradient conv at 1, 4, 16 and 128 channels per group"""
    assert c.N * math.ceil(c.H / 8) * math.ceil(c.W / 16) * c.C // 128 >= 2 * _sms()
    backward.test_nb_sums_in_the_data_gradient_conv_match_fp64(cuda, c)
