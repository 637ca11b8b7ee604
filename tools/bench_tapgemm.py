"""Time single tapgemm launches (CUDA events, L2-cold via rotating buffers) for a few conv shapes."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from text2human_b200 import ops  # noqa: E402

dev = "cuda"


def bench_conv(N, H, W, Cin, Cout, terms, residual, stats, iters=5):
    x = [torch.randn(N, H, W, Cin, device=dev) for _ in range(2)]
    a = [ops.f32_to_planes(t, ops.CVT_PLAIN, terms) for t in x]
    w = ops.pack_conv_weight(torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5, terms)
    b = torch.randn(Cout, device=dev)
    res = torch.randn(N, H, W, Cout, device=dev) if residual else None
    for i in range(2):
        ops.conv3x3(a[i % 2], w, b, residual=res, want_stats=stats)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        ops.conv3x3(a[i % 2], w, b, residual=res, want_stats=stats)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * N * H * W * Cout * Cin * 9
    return ms, fl / ms / 1e9


for (N, H, W, Ci, Co) in [(16, 512, 256, 128, 128), (16, 128, 64, 256, 256), (16, 64, 32, 256, 256),
                          (16, 32, 16, 512, 512)]:
    for terms in (1, 2):
        for residual, stats in ((False, False), (True, True)):
            ms, tf = bench_conv(N, H, W, Ci, Co, terms, residual, stats)
            print(f"conv {N}x{H}x{W} {Ci}->{Co} terms={terms} res={int(residual)} stats={int(stats)}: "
                  f"{ms * 1e3:8.1f} us  {tf:7.1f} TFLOP/s (algorithmic)", flush=True)
