"""2-GPU (NCCL) gradient equivalence of the VQGAN training step (SURVEY §4 iv / §8e): the gradients two ranks
all-reduce, each on its own image, equal the gradients one process accumulates over the same two images as
micro-batches (a micro-batch IS one DDP rank: own BatchNorm statistics, own adaptive weight, own DiffAugment draws),
and after Adam both ranks hold the same parameters as the single process.  Skipped with fewer than 2 GPUs
(run: gpurun --gpus 2 -- python -m pytest tests/test_gpu_ddp.py -m gpu)."""
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

import golden_recipes as R

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _draws(seed, skip):
    from test_gpu_vqgan_train import recorded_draws
    fn = recorded_draws(seed)
    for _ in range(skip):          # advance past the draws the lower ranks / earlier micro-batches consume
        fn(1, 64, 32, "cpu")
    return fn


def _worker(rank, world, port, q):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    from test_gpu_vqgan_train import build
    from text2human_b200 import ops
    from text2human_b200.vqgan_train import VQGANTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    ops.set_precision("fp32")
    m, disc, cfg = build(dev)
    tr = VQGANTrainer(m, disc, bucket_bytes=256 << 10)      # several buckets even for the reduced nets
    x, mask = R.image(7, world, 3, 64, 32), R.blocky_mask(8, world, 64, 32, 8)
    tr.aug_draw_fn = _draws(5, 2 * rank)                     # 2 DiffAugment calls (fake, real) per image
    tr.training_step(dict(image=x[rank:rank + 1], texture_mask=mask[rank:rank + 1]), 3)
    n_reduces = len(tr.gen.handles) + len(tr.dsc.handles)
    tr.wait_reduced()
    torch.cuda.synchronize()
    g_gen, g_dsc = tr.gen.flat_g.clone(), tr.dsc.flat_g.clone()
    tr.adam_step()
    torch.cuda.synchronize()
    out = dict(rank=rank, n_reduces=n_reduces, n_buckets=len(tr.gen.buckets) + len(tr.dsc.buckets),
               psum=float(tr.gen.flat_p.double().sum()))
    if rank == 0:
        # the single-process reference on the same device: both images as two micro-batches
        m1, disc1, _ = build(dev)
        t1 = VQGANTrainer(m1, disc1, micro_batch=1)
        t1.aug_draw_fn = _draws(5, 0)
        t1.force_no_reduce = True
        t1.training_step(dict(image=x, texture_mask=mask), 3)
        torch.cuda.synchronize()
        out["gen_rel"] = float((g_gen - t1.gen.flat_g).abs().max() / t1.gen.flat_g.abs().max())
        out["dsc_rel"] = float((g_dsc - t1.dsc.flat_g).abs().max() / t1.dsc.flat_g.abs().max())
        world_save = dist.get_world_size
        t1.n_micro = 2
        # Adam on the single process: gradients are sums over 2 micro-batches -> divide by 2 (world = 1 there)
        from text2human_b200 import ops as _o
        t1.gen.adam(t1.lr, t1.betas, t1.eps, 1.0 / (2 * t1.loss_scale))
        big = t1.gen.flat_g.abs() > 1e-3 * t1.gen.flat_g.abs().max()     # Adam amplifies rounding noise of ~zero grads
        out["p_dev"] = float((tr.gen.flat_p - t1.gen.flat_p)[big].abs().max())
    import json
    with open(os.path.join(q, f"rank{rank}.json"), "w") as f:     # q: a directory; plain files instead of an mp.Queue
        json.dump(out, f)
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
    os._exit(0)        # skip interpreter teardown (CUDA / NCCL atexit handlers of a spawned worker can stall it)


def test_two_rank_gradients_equal_single_process_micro_batches(cuda, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import json
    import time
    port = _free_port()
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    files = [os.path.join(str(tmp_path), f"rank{r}.json") for r in range(2)]
    t0 = time.time()
    while not all(os.path.exists(f) for f in files) and time.time() - t0 < 600 and all(p.is_alive() or p.exitcode == 0 for p in procs):
        time.sleep(0.5)
    time.sleep(1.0)
    assert all(os.path.exists(f) for f in files), [p.exitcode for p in procs]
    r0, r1 = (json.load(open(f)) for f in files)
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.kill()
    print(f"[ddp] buckets {r0['n_buckets']} all-reduces launched during backward {r0['n_reduces']}; gradient rel diff "
          f"generator {r0['gen_rel']:.2e} discriminator {r0['dsc_rel']:.2e}; parameter deviation after Adam {r0['p_dev']:.2e}")
    assert r0["n_reduces"] == r0["n_buckets"] >= 4
    assert r0["gen_rel"] < 1e-4 and r0["dsc_rel"] < 1e-4
    assert r0["psum"] == r1["psum"]                          # both ranks took the identical Adam step
    assert r0["p_dev"] < 1e-6
