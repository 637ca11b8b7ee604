"""The swapped-operand tap-GEMM's paired mode (one CTA computes two vertically adjacent tiles that share every weight
tile and one activation slab), element by element against fp64.

t2h_tapgemm takes the paired kernel when a launch has at least two tiles per SM, so every case here is sized above
that and checks it.  References, bounds and launch helpers are those of test_gpu_tapgemm_paths.py and, for the
norm-backward sums, test_gpu_backward_paths.py.
"""
import math

import pytest
import torch

import test_gpu_backward_paths as backward  # (as modules: their tests are called here, not collected again)
import test_gpu_tapgemm_paths as paths
from test_gpu_backward_paths import NBS, _tile
from test_gpu_tapgemm_paths import Case, _case_id, _label, _operands, _out_hw, _run_case


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(c):
    """tiles of each launch of a case (the upsample fold's parity launches run over the low-resolution grid)"""
    r = _label(c)
    H, W = (c.H, c.W) if c.kind == "up" else _out_hw(c)
    return c.N * math.ceil(H / r["TH"]) * math.ceil(W / r["TW"]) * math.ceil(c.cout / 128)


# the second tile of the last pair of a column lies partly below the image (odd tile-row count, H % TH != 0) or wholly
# (H <= TH)
PAIR_CASES = [
    Case(3, 131, 40, "k3", 64, 256, 2, "shared", 1.0, "none", True, 4, "nhwc"),     # TW 16, 17 tile rows, res + gn
    Case(7, 200, 8, "k3", 64, 384, 1, "image", 0.375, "gelu", False, 0, "nhwc"),    # TW 8, 13 tile rows
    Case(45, 70, 7, "k3", 40, 128, 2, "none", 1.0, "relu", True, 16, "nhwc"),       # TW 4, 3 tile rows, ragged W
    Case(70, 5, 64, "k3", 64, 128, 2, "shared", 1.0, "lrelu", True, 8, "nhwc"),     # H < TH: second tile outside
    Case(35, 10, 64, "k3", 64, 128, 1, "shared", 1.0, "none", True, 32, "nhwc"),    # TH < H < 2 TH
    Case(2, 135, 128, "k3", 64, 3, 2, "shared", 0.375, "none", False, 0, "nchw"),   # strided NCHW, Cout 3
    Case(4, 67, 64, "up", 64, 256, 2, "shared", 1.0, "none", False, 4, "nhwc"),     # upsample-fold parity launches
    Case(4, 134, 128, "down", 64, 256, 2, "shared", 1.0, "none", True, 128, "nhwc"),  # stride 2 on 4 phases
]


def test_pair_case_table():
    """the pair cases are swapped-kernel launches at TW 16, 8 and 4 with Cout 128, 256, 384 and 3, one and two planes,
    an odd tile-row count and heights below TH and 2 TH"""
    labels = [(c, _label(c)) for c in PAIR_CASES]
    assert all(r["kernel"] == "swap" for c, r in labels)
    assert {r["TW"] for c, r in labels} >= {16, 8, 4}
    assert {c.cout for c in PAIR_CASES} >= {3, 128, 256, 384} and {c.terms for c in PAIR_CASES} == {1, 2}
    H = lambda c: c.H if c.kind == "up" else _out_hw(c)[0]  # noqa: E731
    assert any(math.ceil(H(c) / r["TH"]) % 2 == 1 and H(c) % r["TH"] for c, r in labels)
    assert any(H(c) < r["TH"] for c, r in labels) and any(r["TH"] < H(c) < 2 * r["TH"] for c, r in labels)
    assert any(c.res and c.gn for c in PAIR_CASES) and any(c.act == "gelu" for c in PAIR_CASES)
    assert {c.kind for c in PAIR_CASES} >= {"k3", "up", "down"} and any(r["epi"] == "direct" for c, r in labels)


@pytest.mark.gpu
@pytest.mark.parametrize("c", PAIR_CASES, ids=_case_id)
def test_paired_tapgemm_matches_fp64(cuda, c):
    """one paired launch (or four parity launches) against fp64, and again: bit-identical"""
    assert _tiles(c) >= 2 * _sms(), f"{_tiles(c)} tiles do not take the paired kernel on {_sms()} SMs"
    paths.test_tapgemm_path_matches_fp64(cuda, c)


@pytest.mark.gpu
def test_paired_output_equals_unpaired(cuda):
    """the MMA sequence per pixel is the unpaired one: a paired launch over three images and an unpaired launch over
    one of them write the same bits"""
    dev = cuda
    c = PAIR_CASES[0]
    one = c._replace(N=1)
    assert _tiles(c) >= 2 * _sms() > _tiles(one)
    a, wp, _, _, taps = _operands(c, dev)
    g = torch.Generator().manual_seed(11)
    Ho, Wo = _out_hw(c)
    bias = torch.randn(c.cout, generator=g).to(dev)
    res = torch.randn(c.N, Ho, Wo, c.cout, generator=g).to(dev)
    d, _, _ = _run_case(c, a, wp, taps, bias, res, dev)
    for n in range(c.N):
        d1, _, _ = _run_case(one, a[:, n:n + 1].contiguous(), wp, taps, bias, res[n:n + 1].contiguous(), dev)
        assert torch.equal(d[n:n + 1], d1), f"image {n}: paired and unpaired launches differ"


@pytest.mark.gpu
@pytest.mark.parametrize("c", [NBS(3, 133, 40, 256, 32, "swish"), NBS(33, 20, 64, 128, 8, "lrelu")],
                         ids=lambda c: f"n{c.N}x{c.H}x{c.W}-C{c.C}-g{c.groups}-{c.act}")
def test_paired_nb_sums_match_fp64(cuda, c):
    """norm-backward sums of a paired data-gradient conv: contiguous pair ranges per CTA that start and end inside an
    image and a 128-channel block"""
    TW, TH = _tile(c.W)
    tiles = c.N * math.ceil(c.H / TH) * math.ceil(c.W / TW) * c.C // 128
    pairs = c.N * math.ceil(math.ceil(c.H / TH) / 2) * math.ceil(c.W / TW) * c.C // 128
    per_block = pairs // (c.N * c.C // 128)
    assert tiles >= 2 * _sms()
    starts = [b * pairs // _sms() for b in range(_sms())]
    assert any(s % per_block for s in starts), "no CTA range starts inside an (image, channel block)"
    backward.test_nb_sums_in_the_data_gradient_conv_match_fp64(cuda, c)
