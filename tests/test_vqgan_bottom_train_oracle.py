"""CPU checks of the hierarchical VQGAN's bottom-level training step: the restatement
(oracle/vqgan_bottom_train_ref.training_step) against the fixture made from the real reference
`HierarchyVQSpatialTextureAwareModel.training_step` + `loss.backward()` + `d_loss.backward()`
(oracle/make_golden_vqgan_bottom_train.py), the fixture's distance from the step's discontinuities, the new
quantizer-backward entry point of the C ABI, and which tensors the trainer broadcasts and all-reduces (two gloo
ranks)."""
import os
import socket

import numpy as np
import torch
import torch.multiprocessing as mp

import golden_recipes as R
import vqgan_bottom_train_recipes as BR
from oracle import vqgan_bottom_train_ref as BT

GOLD = os.path.join(os.path.dirname(__file__), "golden", "vqgan_bottom_train.npz")


def _run(dtype, noise=None, probe=None):
    sd, top, bot, sdd = BR.restatement_state(dtype)
    if noise is not None:           # relative weight noise on every generator / discriminator tensor
        g = torch.Generator().manual_seed(noise[1])
        with torch.no_grad():
            for t in list(sd.values()) + bot + [v for v in sdd.values() if v.is_floating_point()]:
                t.mul_(1 + noise[0] * torch.randn(t.shape, generator=g, dtype=dtype))
    d = BR.batch()
    torch.manual_seed(BR.AUG_SEED)
    r = BT.training_step(sd, top, bot, sdd, d["image"].to(dtype), d["texture_mask"], BR.STEP,
                         disc_start_step=BR.DISC_START_STEP, disc_layers=BR.DISC_LAYERS, probe=probe)
    r["loss"].backward(retain_graph=True)
    gen = {k: v.detach().clone() for k, v in BR.gen_grads(sd, bot).items()}
    for p in sdd.values():
        p.grad = None                       # disc_optimizer.zero_grad() before d_loss.backward()
    r["d_loss"].backward()
    dsc = {k: v.grad.detach().clone() for k, v in sdd.items() if v.requires_grad}
    return r, gen, dsc


def test_restatement_matches_reference_fixture():
    gold = np.load(GOLD)
    r, gen, dsc = _run(torch.float32)
    for k in ("loss", "d_loss", "nll_loss", "g_loss", "d_weight", "codebook_loss"):
        assert abs(float(r[k]) - float(gold[k])) <= 1e-5 * max(1.0, abs(float(gold[k]))), k
    assert np.array_equal(r["bot_idx"].numpy(), gold["bot_idx"])
    for prefix, grads in (("g", gen), ("d", dsc)):
        keys = [k for k in gold.files if k.startswith(prefix + "norm/")]
        assert sorted(k[6:] for k in keys) == sorted(grads), prefix        # the same optimised tensors
        for key in keys:
            name = key[6:]
            g, want = grads[name], float(gold[key])
            assert abs(float(g.norm()) - want) <= 1e-5 * max(want, 1e-6) + 1e-8, name
            head = torch.from_numpy(gold[prefix + "head/" + name])
            assert float((g.reshape(-1)[:8] - head).abs().max()) <= 1e-5 * max(want, 1e-6) + 1e-8, name
    assert len(gen) > 150 and len(dsc) >= 10


def test_fixture_is_not_at_a_kink():
    """fp64 gradients under 3e-7 relative weight noise move by less than 1e-4 per tensor: no argmin, LeakyReLU or
    hinge decision flips within the rounding of an fp32 implementation"""
    _, g0, d0 = _run(torch.float64)
    _, g1, d1 = _run(torch.float64, noise=(3e-7, 7))
    worst = 0.0
    for a, b in ((g0, g1), (d0, d1)):
        # gradients that are zero in exact arithmetic (a conv bias in front of a GroupNorm) are rounding noise
        floor = 1e-6 * max(float(v.norm()) for v in a.values())
        for k in a:
            n = float(a[k].norm())
            if n > floor:
                worst = max(worst, float((a[k] - b[k]).norm()) / n)
    assert worst < 1e-4, worst


def test_recorded_margins_hold():
    probe = {}
    _run(torch.float64, probe=probe)
    argmin = float(min(probe["argmin"]))
    kink = min(min(p) for p in probe["kink"])
    assert argmin >= BR.ARGMIN_MARGIN, argmin
    assert kink >= BR.KINK_MARGIN, kink


def test_abi_lists_the_patch_quantizer_backward():
    from text2human_b200 import _lib
    from test_abi import declared_symbols
    assert "t2h_vq_bwd_patch" in declared_symbols() and "t2h_vq_bwd_patch" in _lib.SIGNATURES
    lib = _lib.load()
    rc = lib.t2h_vq_bwd_patch(None, None, None, None, None, None, None, None, None, 1, 4, 4, 8, 2, 18, 16, 1.0, 1.0,
                              None)
    assert rc == -1 and b"null pointer" in lib.t2h_last_error()


# ---------------------------------------------------------------- two gloo ranks
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    """HierarchyVQGANTrainer's host-side DDP logic on CPU tensors: what it broadcasts at construction and what its
    backward pass's bucketed all-reduce covers"""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import vqgan_bottom_train_recipes as BR
    from text2human_b200 import dist as D
    from text2human_b200.vqgan_bottom_train import HierarchyVQGANTrainer
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    D.init("gloo")
    out = {}
    for fix in (False, True):
        m, disc = BR.modules()
        with torch.no_grad():                           # replicas start different ...
            for p in list(m.parameters()) + list(disc.parameters()):
                p.add_(0.01 * rank)
        built = {n: p.detach().clone() for n, p in m.named_parameters()}
        tr = HierarchyVQGANTrainer(m, disc, fix_decoder=fix, bucket_bytes=64 << 10)   # ... and are synchronised
        in_gen = {id(p) for p, _, _ in tr.gen.slots}
        in_fixed = {id(p) for p, _, _ in tr.fixed.slots}
        names = {}
        for n, p in m.named_parameters():
            names[n] = (id(p) in in_gen, id(p) in in_fixed, torch.equal(p.detach(), built[n]))
        sums = []
        for sp in (tr.gen, tr.dsc, tr.fixed):
            n = sp.flat_g.numel()
            sp.flat_g.copy_(torch.arange(n, dtype=torch.float32) % 97 + 1000.0 * rank)
            if sp is not tr.fixed:
                sp.arm(True)
            for mod, _, _ in sp.mod_span:
                sp.done(mod)
            sums.append(len(sp.handles))
            sp.wait()
            want = (2 * (torch.arange(n, dtype=torch.float32) % 97) + 1000.0) if sp is not tr.fixed else \
                torch.arange(n, dtype=torch.float32) % 97 + 1000.0 * rank
            sums.append(bool(torch.equal(sp.flat_g, want)))
        out[fix] = (names, sums, float(tr.gen.flat_p.double().sum()))
    q.put((rank, out))
    torch.distributed.destroy_process_group()


def test_only_trainable_tensors_are_broadcast_and_bucketed_gloo():
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for fix in (False, True):
        names0, sums0, psum0 = res[0][fix]
        names1, sums1, psum1 = res[1][fix]
        assert psum0 == psum1                                   # the stepped tensors come from rank 0
        n_gen = 0
        for n, (g, f, kept0) in names0.items():
            dec = n.startswith("decoder.")
            stepped = BR.stepped(n) and not (fix and dec)
            assert g == stepped, n                              # the generator store holds the stepped tensors only
            fixed = dec and (n.startswith(("decoder.conv_out.", "decoder.norm_out.")) or (fix and BR.stepped(n)))
            assert f == fixed, n                                # computed, never stepped
            assert kept0 and names1[n][2] == (not g), n         # rank 1 takes rank 0's stepped tensors, keeps the rest
            n_gen += g
        assert n_gen > 100
        assert sums0[1] and sums0[3] and sums0[5]               # gen / disc summed over ranks once, fixed untouched
        assert sums0[0] >= 2 and sums0[2] >= 1 and sums0[4] == 0
