"""CPU, two ranks over gloo: IndexPredTrainer's host-side DDP logic -- the parameters and optimiser state broadcast
from rank 0 at construction, and the bucketed gradient all-reduce fired by ``done(module)`` over the flat store with
the new layouts (the 18 conv_seg heads as one group, the 18 BatchNorms as one group, the stacked head convs), each
gradient element summed exactly once, every bucket all-reduced once."""
import os
import socket

import torch
import torch.multiprocessing as mp


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import golden_recipes as R
    from text2human_b200 import dist as D
    from text2human_b200.index_pred_arch import MultiHeadFCNHead, UNet
    from text2human_b200.index_pred_train import IndexPredTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    D.init("gloo")
    torch.manual_seed(100 + rank)                       # replicas are BUILT differently ...
    unet, fcn = UNet(**R.TINY_UNET), MultiHeadFCNHead(**R.TINY_FCN)
    w_before = fcn.convs_list[5][0].conv.weight.detach().clone()
    tr = IndexPredTrainer(unet, fcn, bucket_bytes=16 << 10)    # ... and synchronised from rank 0 by the trainer
    sp = tr.space
    psum = float(sp.flat_p.double().sum())
    same_as_built = torch.equal(fcn.convs_list[5][0].conv.weight.detach(), w_before)
    n = sp.flat_g.numel()
    sp.flat_g.copy_(torch.arange(n, dtype=torch.float32) % 97 + 1000.0 * rank)
    sp.arm(True)
    for mod, _, _ in sp.mod_span:                       # the order the backward pass finishes the modules in
        sp.done(mod)
    n_handles = len(sp.handles)
    sp.wait()
    want = 2 * (torch.arange(n, dtype=torch.float32) % 97) + 1000.0
    q.put((rank, psum, same_as_built, bool(torch.equal(sp.flat_g, want)), n_handles, len(sp.buckets),
           tuple(fcn.convs_list[5][0].conv.weight.shape)))
    torch.distributed.destroy_process_group()


def test_index_pred_flat_store_broadcast_and_gradient_buckets_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (_, psum0, same0, ok0, h0, b0, shape), (_, psum1, same1, ok1, h1, b1, _) = res
    assert psum0 == psum1, "replicas were not synchronised from rank 0"
    assert same0 and not same1, "rank 0 keeps its parameters, rank 1 takes rank 0's"
    assert shape == (8, 8, 3, 3)                        # a stacked head conv keeps the reference's OIHW shape
    assert ok0 and ok1                                  # every gradient element summed exactly once
    assert h0 == b0 == h1 == b1 >= 4
