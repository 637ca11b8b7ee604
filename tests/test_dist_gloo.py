"""world_size-2 gloo test (CPU) of the replica sharding used for N>1 runs: every image is processed by
exactly one rank, the gathered result equals the single-process result, and the timing reduction takes
the slowest rank."""
import os
import socket

import torch
import torch.multiprocessing as mp

from text2human_b200 import dist as D


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    r, lr, w = D.init("gloo")
    assert (r, w) == (rank, world)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(7, 3, 4, 4, generator=g)        # 7 images over 2 ranks: 4 + 3
    m = torch.arange(7).float().view(7, 1, 1, 1)
    xs, ms = D.shard_batch((x, m), rank, world)
    y = xs * 2 + ms                                  # stand-in for the per-image (collective-free) path
    full = D.gather_concat(y)
    D.barrier()
    t = D.max_over_ranks(1.0 + rank)
    n = D.sum_over_ranks(xs.shape[0])
    if rank == 0:   # plain python values: a tensor in the queue is a shared-memory handle that dies with this process
        q.put((full.numpy().tolist(), t, n, xs.shape[0]))
    torch.distributed.destroy_process_group()


def test_replica_sharding_two_ranks_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    full, t, n, n0 = q.get(timeout=120)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    g = torch.Generator().manual_seed(0)
    x = torch.randn(7, 3, 4, 4, generator=g)
    want = x * 2 + torch.arange(7).float().view(7, 1, 1, 1)
    assert torch.equal(torch.tensor(full), want)
    assert t == 2.0 and n == 7 and n0 == 4


def test_shard_range_covers_everything_once():
    for n in (0, 1, 5, 16, 17):
        for world in (1, 2, 3, 8):
            seen = []
            for r in range(world):
                a, b = D.shard_range(n, r, world)
                assert 0 <= a <= b <= n
                seen += list(range(a, b))
            assert seen == list(range(n))


def _train_worker(rank, world, port, q):
    """the trainer's bucketed gradient all-reduce (host logic) on CPU tensors over gloo"""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import golden_recipes as R
    from text2human_b200.transformer_arch import TransformerMultiHead
    from text2human_b200.transformer_train import SamplerTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    D.init("gloo")
    cfg = dict(R.TINY_TRANSFORMER, bert_n_layers=5)
    tr = SamplerTrainer(TransformerMultiHead(**cfg), bucket_layers=2)
    sp, m = tr.space, tr.m
    n = sp.flat_g.numel()
    sp.flat_g.copy_(torch.arange(n, dtype=torch.float32) % 97 + 1000.0 * rank)
    # the modules the backward pass reports finished: head, blocks last to first, embeddings
    sp.arm(True)
    sp.done(m.ln_f)
    for li in range(4, -1, -1):
        sp.done(m.blocks[li].ln1)
    sp.done(m.texture_emb)
    n_handles = len(sp.handles)
    sp.wait()
    if rank == 0:
        q.put((sp.flat_g.numpy().tolist(), n_handles))
    torch.distributed.destroy_process_group()


def test_sampler_flat_store_buckets_cover_flat_buffer_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    g, n_handles = q.get(timeout=120)
    g = torch.tensor(g, dtype=torch.float32)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    n = g.numel()
    want = 2 * (torch.arange(n, dtype=torch.float32) % 97) + 1000.0   # every element summed exactly once
    assert torch.equal(g, want)
    assert n_handles == 1 + 3 + 1                                     # head, 3 block buckets, embeddings


def _vqgan_worker(rank, world, port, q):
    """VQGANTrainer's host-side DDP logic on CPU tensors over gloo: parameter broadcast at construction and the
    bucketed all-reduce fired by the backward pass's `done(module)` notifications"""
    import contextlib
    import io
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import golden_recipes as R
    from text2human_b200.pipeline import VQImageSegmTextureModel
    from text2human_b200.vqgan_arch import Discriminator
    from text2human_b200.vqgan_train import VQGANTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    D.init("gloo")
    cfg = R.TINY_VQGAN_TRAIN
    e = cfg["enc"]
    opt = dict(embed_dim=cfg["embed_dim"], n_embed=cfg["n_embed"], double_z=False, z_channels=e["z_channels"],
               resolution=e["resolution"], in_channels=3, out_ch=3, ch=e["ch"], ch_mult=e["ch_mult"],
               num_res_blocks=e["num_res_blocks"], attn_resolutions=e["attn_resolutions"], dropout=0.0)
    torch.manual_seed(100 + rank)                       # replicas are BUILT differently ...
    with contextlib.redirect_stdout(io.StringIO()):
        m = VQImageSegmTextureModel(opt)
    disc = Discriminator(3, cfg["ndf"], n_layers=cfg["disc_layers"])
    w_before = m.decoder.conv_out.weight.detach().clone()
    tr = VQGANTrainer(m, disc, bucket_bytes=256 << 10)  # ... and synchronised from rank 0 by the trainer
    psum = float(tr.gen.flat_p.double().sum()) + float(tr.dsc.flat_p.double().sum())
    same_as_built = torch.equal(m.decoder.conv_out.weight.detach(), w_before)
    out = {}
    for name, sp in (("gen", tr.gen), ("dsc", tr.dsc)):
        n = sp.flat_g.numel()
        sp.flat_g.copy_(torch.arange(n, dtype=torch.float32) % 97 + 1000.0 * rank)
        sp.arm(True)
        for mod, _, _ in sp.mod_span:                   # the order the backward pass finishes the modules in
            sp.done(mod)
        n_handles = len(sp.handles)
        sp.wait()
        want = 2 * (torch.arange(n, dtype=torch.float32) % 97) + 1000.0     # every element summed exactly once
        out[name] = (bool(torch.equal(sp.flat_g, want)), n_handles, len(sp.buckets))
    q.put((rank, psum, same_as_built, out if rank == 0 else None, tuple(m.decoder.conv_out.weight.shape)))
    torch.distributed.destroy_process_group()


def test_vqgan_flat_stores_broadcast_and_gradient_buckets_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_vqgan_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    (r0, psum0, same0, out, shape), (r1, psum1, same1, _, _) = res
    assert psum0 == psum1, "replicas were not synchronised from rank 0"
    assert same0 and not same1, "rank 0 keeps its parameters, rank 1 takes rank 0's"
    assert shape == (3, 32, 3, 3)                       # the nn.Parameter kept the reference's OIHW shape
    for name in ("gen", "dsc"):
        ok, n_handles, n_buckets = out[name]
        assert ok, name                                 # every gradient element summed exactly once
        assert n_handles == n_buckets >= (3 if name == "gen" else 1)
