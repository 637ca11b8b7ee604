"""Flat parameter store of the native trainers (``transformer_train``, ``vqgan_train``, ``segm_train``).

Parameters, gradients and Adam moments of an ordered list of modules live in four flat fp32 buffers and the
``nn.Parameter``s (and their ``.grad``) become views of them, so state_dict keys and shapes are unchanged and Adam is
one launch.  The modules are laid out in the order the backward pass finishes their gradients, and the gradient
buffer is cut into contiguous buckets of whole modules: the backward pass reports each finished module with
``done(mod)``, and the all-reduce (sum over the default process group) of a bucket starts as soon as its last module
is done, overlapping the rest of the backward pass.
"""
import torch
import torch.distributed as dist
import torch.nn as nn

from . import conv_grad as G
from . import ops
from .dist import world_size


class ConvP:
    """one conv layer's views into the flat buffers"""
    __slots__ = ("mod", "k", "co", "ci", "co_p", "ci_p", "w", "gw", "b", "gb", "wn", "wt")


class ConvStack:
    """Convolutions of equal shape that always run as ONE convolution with their outputs stacked along the output
    channels (the index-prediction heads' 3x3 ConvModules).  ParamSpace keeps their weights as one tap-major block
    ``[K*K, n*Cout, Cin]``, so the stacked forward operand and weight gradient need no per-step copy; each member's
    ``weight`` / ``.grad`` is a view of its ``Cout``-row slice.  ``done(stack)`` reports the whole block."""

    def __init__(self, convs):
        self.convs = tuple(convs)
        co, ci, kh, kw = self.convs[0].weight.shape
        assert kh == kw and co % 8 == 0 and ci % 8 == 0, "stacked convs need channel counts that are multiples of 8"
        assert all(tuple(c.weight.shape) == (co, ci, kh, kw) and c.bias is None for c in self.convs)


class ParamSpace:
    """Flat fp32 parameter / gradient / Adam-moment buffers for ``order``, modules in backward-completion order.

    A Conv2d's weight is kept TAP-MAJOR ``[K*K, Cout_p, Cin_p]`` (the layout the kernels' packed operands and the
    weight-gradient kernel's output share) and the conv gets a ``ConvP`` in ``convs``.  A tuple of Conv2d or Linear
    modules is one group laid out weights first, then biases, so that a fused projection (q | k | v, the sampler's
    18 heads) reads them as one matrix (``joint``); a conv alone is a group of one; a tuple of BatchNorm2d is one
    group too (gammas back to back, then betas).  A ``ConvStack`` is one conv of ``n*Cout`` output channels.  Any other module contributes its
    own parameters (``parameters(recurse=False)``).  Every slot starts 32-byte aligned.

    A gradient bucket closes after the module (a group: its last member) that brings it to ``bucket_bytes`` or more,
    after every module in ``close_after``, and at the end of ``order``."""

    def __init__(self, order, device, bucket_bytes=48 << 20, close_after=()):
        self.device = device
        self.convs = {}
        self.slots = []          # (param, offset, ConvP for a conv weight / ("bias", ConvP) / None)
        self.mod_span = []       # (module, start, end)
        total = 0

        def take(p, n, tag=None):
            nonlocal total
            self.slots.append((p, total, tag))
            total += (n + 7) // 8 * 8

        for mod in order:
            start = total
            group = mod if isinstance(mod, tuple) else (mod,)
            if isinstance(mod, ConvStack):
                co, ci, k, _ = mod.convs[0].weight.shape
                cp = ConvP()
                cp.mod, cp.k, cp.co, cp.ci = mod, k, co * len(mod.convs), ci
                cp.co_p, cp.ci_p = cp.co, cp.ci
                take(mod.convs[0].weight, k * k * cp.co * cp.ci, ("stack", cp))
                self.convs[mod] = cp
            elif isinstance(mod, (tuple, nn.Conv2d)):
                for m_ in group:
                    if isinstance(m_, nn.Conv2d):
                        co, ci, kh, kw = m_.weight.shape
                        assert kh == kw
                        cp = ConvP()
                        cp.mod, cp.k, cp.co, cp.ci, cp.co_p, cp.ci_p = m_, kh, co, ci, G.pad8(co), G.pad8(ci)
                        take(m_.weight, kh * kw * cp.co_p * cp.ci_p, cp)
                        self.convs[m_] = cp
                    else:
                        take(m_.weight, m_.weight.numel())
                for m_ in group:
                    if m_.bias is not None:
                        take(m_.bias, m_.bias.numel(), ("bias", self.convs[m_]) if m_ in self.convs else None)
            else:
                for p in mod.parameters(recurse=False):
                    take(p, p.numel())
            for m_ in group[:-1]:
                self.mod_span.append((m_, start, start))   # empty spans: a group closes with its last member
            self.mod_span.append((group[-1], start, total))
        self.total = total
        self.flat_p = torch.zeros(total, dtype=torch.float32, device=device)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=device)
        self.flat_m = torch.zeros(total, dtype=torch.float32, device=device)
        self.flat_v = torch.zeros(total, dtype=torch.float32, device=device)
        self.gview = {}
        with torch.no_grad():
            for p, off, tag in self.slots:
                if isinstance(tag, tuple) and tag[0] == "stack":
                    cp = tag[1]
                    n = cp.k * cp.k * cp.co * cp.ci
                    cp.w = self.flat_p[off:off + n].view(cp.k * cp.k, cp.co, cp.ci)
                    cp.gw = self.flat_g[off:off + n].view(cp.k * cp.k, cp.co, cp.ci)
                    cp.b = cp.gb = None
                    per = cp.co // len(cp.mod.convs)
                    for j, c in enumerate(cp.mod.convs):
                        rows = slice(j * per, (j + 1) * per)
                        cp.w[:, rows].copy_(G.oihw_to_master(c.weight.detach().to(device)))
                        c.weight.data = G.master_as_oihw(cp.w[:, rows], per, cp.ci, cp.k)
                        c.weight.grad = G.master_as_oihw(cp.gw[:, rows], per, cp.ci, cp.k)
                        self.gview[id(c.weight)] = c.weight.grad
                    continue
                if isinstance(tag, ConvP):
                    cp = tag
                    n = cp.k * cp.k * cp.co_p * cp.ci_p
                    m = self.flat_p[off:off + n].view(cp.k * cp.k, cp.co_p, cp.ci_p)
                    m.copy_(G.oihw_to_master(p.detach().to(device)))
                    cp.w = m
                    cp.gw = self.flat_g[off:off + n].view(cp.k * cp.k, cp.co_p, cp.ci_p)
                    p.data = G.master_as_oihw(m, cp.co, cp.ci, cp.k)
                    p.grad = G.master_as_oihw(cp.gw, cp.co, cp.ci, cp.k)
                    cp.b = cp.gb = None
                elif tag is not None:
                    cp = tag[1]
                    self.flat_p[off:off + cp.co].copy_(p.detach().reshape(-1))
                    cp.b = self.flat_p[off:off + cp.co_p]
                    cp.gb = self.flat_g[off:off + cp.co_p]
                    p.data = self.flat_p[off:off + cp.co]
                    p.grad = self.flat_g[off:off + cp.co]
                else:
                    n = p.numel()
                    self.flat_p[off:off + n].copy_(p.detach().reshape(-1))
                    p.data = self.flat_p[off:off + n].view_as(p)
                    p.grad = self.flat_g[off:off + n].view_as(p)
                self.gview[id(p)] = p.grad
        # gradient buckets: contiguous runs of whole modules, in backward-completion order
        close_after = set(close_after)
        self.buckets, self.bucket_last = [], {}
        b0 = 0
        for i, (mod, s, e) in enumerate(self.mod_span):
            if (e - b0) * 4 >= bucket_bytes or mod in close_after or i == len(self.mod_span) - 1:
                self.bucket_last[mod] = len(self.buckets)
                self.buckets.append((b0, e))
                b0 = e
        self._armed = [False] * len(self.buckets)
        self.handles = []        # all-reduces in flight
        self.step_count = 0

    def g(self, p):
        return self.gview[id(p)]

    def joint(self, params, cols=None):
        """-> (parameter view, gradient view) of ``params``, which must lie back to back without padding (a group's
        weights or biases), as one [rows, cols] matrix each, or 1-D without ``cols``"""
        off = self.g(params[0]).storage_offset()
        n = 0
        for p in params:
            assert self.g(p).storage_offset() == off + n, "the parameters are not adjacent in the flat buffer"
            n += p.numel()
        shape = (-1,) if cols is None else (-1, cols)
        return self.flat_p[off:off + n].view(shape), self.flat_g[off:off + n].view(shape)

    def prepare(self, terms):
        """fp16 planes of every conv weight for this step: forward operand wn and transposed (data-gradient) wt"""
        for cp in self.convs.values():
            cp.wn, cp.wt = G.weight_planes(cp.w, terms)

    def release(self):
        for cp in self.convs.values():
            cp.wn = cp.wt = None

    # ---- bucketed gradient all-reduce
    def arm(self, on):
        """``done`` starts the all-reduces of this backward pass only when armed (and there is more than one rank),
        each bucket's at most once per arming"""
        self._armed = [bool(on) and world_size() > 1] * len(self.buckets)

    def done(self, mod):
        """all gradients of ``mod`` are final: if it closes an armed bucket, start that bucket's all-reduce (sum,
        asynchronous) while the backward pass continues"""
        b = self.bucket_last.get(mod)
        if b is not None and self._armed[b]:
            a, e = self.buckets[b]
            self.handles.append(dist.all_reduce(self.flat_g[a:e], op=dist.ReduceOp.SUM, async_op=True))
            self._armed[b] = False

    def wait(self):
        assert not any(self._armed), "an armed gradient bucket was never closed by done()"
        for h in self.handles:
            h.wait()
        self.handles = []

    # ---- optimiser
    def adam(self, lr, betas, eps, grad_scale):
        """torch.optim.Adam(lr, betas, eps, weight_decay=0) on the flat buffers, gradients multiplied by
        ``grad_scale`` first"""
        p, off, _ = self.slots[0]
        assert p.data_ptr() == self.flat_p.data_ptr() + 4 * off, \
            "the parameters no longer alias the flat buffer (model.to() / .half() after the trainer was built?)"
        self.step_count += 1
        ops.adam_(self.flat_p, self.flat_g, self.flat_m, self.flat_v, lr, betas[0], betas[1], eps, self.step_count,
                  grad_scale=grad_scale)

    def sync_from_rank0(self):
        """replicas start (and resume) from identical parameters and optimiser state, as torch DDP guarantees"""
        if world_size() > 1:
            for t in (self.flat_p, self.flat_m, self.flat_v):
                dist.broadcast(t, 0)

    def state(self):
        return dict(flat_m=self.flat_m.clone(), flat_v=self.flat_v.clone(), step=self.step_count)

    def load_state(self, st):
        self.flat_m.copy_(st["flat_m"])
        self.flat_v.copy_(st["flat_v"])
        self.step_count = int(st["step"])


def drop_packed_caches(*roots):
    """Forget the packed-weight caches and captured sampler graphs (they bake in packed-weight pointers) of every
    module under ``roots``.  The caches are keyed on torch's version counters, which the flat-buffer Adam kernel and
    the broadcast from rank 0 do not bump: call this after either, and after loading a checkpoint."""
    for root in roots:
        for mod in root.modules():
            mod.__dict__.pop("_t2h_cache", None)
            mod.__dict__.pop("_t2h_graphs", None)


def save_checkpoint(path, nets, optimizer):
    """{name: state_dict} of the modules in ``nets`` plus ``optimizer`` (the optimiser state) -> ``path``"""
    # clones: a state_dict entry is a view of the flat buffer, and torch.save would write the whole buffer with it
    ck = {k: {kk: v.detach().clone().contiguous() for kk, v in mod.state_dict().items()} for k, mod in nets.items()}
    torch.save(dict(ck, optimizer=optimizer), path)


def load_checkpoint(path, nets, device):
    """loads every module of ``nets`` strictly from its entry in the checkpoint; -> the optimiser state or None"""
    ck = torch.load(path, map_location=device)
    for k, mod in nets.items():
        mod.load_state_dict(ck[k], strict=True)
    return ck.get("optimizer")
