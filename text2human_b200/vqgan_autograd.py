"""Drop-in training boundary: the arch-module mirrors as torch.autograd nodes.

The reference trains through ``loss.backward()`` on modules built by its wrapper (models/vqgan_model.py:329-344,
:444-488: ``training_step`` / ``optimize_parameters`` with two ``torch.optim.Adam`` over ``module.parameters()`` and two
``torch.autograd.grad`` calls on ``decoder.conv_out.weight``, vqgan_loss.py:5-12).  For those files to run UNMODIFIED
on the mirrors, each mirror's ``forward`` -- when autograd is recording and something requires grad -- is ONE custom
autograd node whose ``backward`` is the hand-written backward of ``vqgan_train`` (wgmma data / weight gradients,
norm / attention / quantizer backward kernels), returning gradients for the input and for every parameter in the
parameter's own (OIHW) layout.  torch's autograd engine and optimiser are only the plumbing between those nodes.

``Decoder`` is two nodes (trunk | norm_out + conv_out) so that ``autograd.grad(loss, decoder.conv_out.weight)`` only
runs the tail's backward, as in the reference.  The native, faster path for the same step is
``vqgan_train.VQGANTrainer`` (flat buffers, one fused backward, bucketed all-reduce).
"""
import torch
import torch.nn as nn

from . import conv_grad as G
from . import ops
from . import vqgan_train as VT
from .flat_params import ConvP, ConvStack
from .vqgan_bottom_train import RES_LEVEL


# ----------------------------------------------------------------------------
# parameter provider for modules whose parameters are ordinary (OIHW) nn.Parameters
# ----------------------------------------------------------------------------
class _Convs:
    def __init__(self, space):
        self.space = space
        self.d = {}

    def __getitem__(self, mod):
        cp = self.d.get(mod)
        if cp is None:
            cp = self.space._make(mod)
            self.d[mod] = cp
        return cp


class StandaloneSpace:
    """Builds ``ConvP`` views (tap-major master copy, packed planes, gradient buffers) on demand from a module's own
    parameters; gradient buffers are fresh zeros per backward.  A ``ConvStack`` is one conv of ``n*Cout`` outputs
    gathered from its members' weights, and ``joint`` gathers a group of parameters (the BatchNorms of a stacked
    ConvModule) into one vector; each member's gradient is handed out in its own shape."""

    def __init__(self, want_grads):
        self.want_grads = want_grads
        self.convs = _Convs(self)
        self.gbuf = {}
        self.members = {}        # member conv of a ConvStack -> (ConvP of the stack, its row slice)
        self.jview = {}          # id(param) of a joint group -> its slice of the group's gradient

    def _make_stack(self, st):
        co, ci, k, _ = st.convs[0].weight.shape
        cp = ConvP()
        n = co * len(st.convs)
        cp.mod, cp.k, cp.co, cp.ci, cp.co_p, cp.ci_p = st, k, n, ci, n, ci
        cp.w = G.oihw_to_master(torch.cat([c.weight.detach() for c in st.convs]))
        cp.wn, cp.wt = G.weight_planes(cp.w)
        cp.gw = torch.zeros_like(cp.w) if self.want_grads else None
        cp.b = cp.gb = None
        for j, c in enumerate(st.convs):
            self.members[c] = (cp, slice(j * co, (j + 1) * co))
        return cp

    def joint(self, params, cols=None):
        """-> (the parameters gathered into one fp32 vector (or [rows, cols] matrix), a zeroed gradient of that shape)"""
        shape = (-1,) if cols is None else (-1, cols)
        p = torch.cat([q.detach().float().reshape(-1) for q in params])
        g = torch.zeros_like(p)
        self.gbuf[("joint", id(params[0]))] = g
        off = 0
        for q in params:
            self.jview[id(q)] = g[off:off + q.numel()].view_as(q)
            off += q.numel()
        return p.view(shape), g.view(shape)

    def _make(self, mod):
        if isinstance(mod, ConvStack):
            return self._make_stack(mod)
        w = mod.weight
        co, ci, k, _ = w.shape
        cp = ConvP()
        cp.mod, cp.k, cp.co, cp.ci, cp.co_p, cp.ci_p = mod, k, co, ci, G.pad8(co), G.pad8(ci)
        cp.w = G.oihw_to_master(w.detach())
        cp.wn, cp.wt = G.weight_planes(cp.w)
        cp.gw = torch.zeros_like(cp.w) if self.want_grads else None
        if mod.bias is not None:
            cp.b = torch.zeros(cp.co_p, dtype=torch.float32, device=w.device)
            cp.b[:co] = mod.bias.detach()
            cp.gb = torch.zeros_like(cp.b) if self.want_grads else None
        else:
            cp.b = cp.gb = None
        return cp

    def g(self, p):
        buf = self.gbuf.get(id(p))
        if buf is None:
            buf = torch.zeros_like(p, dtype=torch.float32)
            self.gbuf[id(p)] = buf
        return buf

    def grad_of(self, p, owner):
        """gradient of parameter ``p`` of module ``owner`` in the parameter's own layout"""
        if isinstance(owner, nn.Conv2d):
            cp = self.convs.d.get(owner)
            if cp is None and owner in self.members:
                cp, rows = self.members[owner]
                return G.master_as_oihw(cp.gw[:, rows], rows.stop - rows.start, cp.ci, cp.k)
            if cp is None:
                return None
            if p is owner.weight:
                return G.master_as_oihw(cp.gw, cp.co, cp.ci, cp.k)
            return cp.gb[:cp.co]
        if id(p) in self.jview:
            return self.jview[id(p)]
        return self.gbuf.get(id(p))

    def done(self, mod):
        """no gradient buckets: the gradients are handed to autograd"""


class _Host:
    """the ``tr`` interface the layers expect (space lookup) over one StandaloneSpace"""

    def __init__(self, want_grads):
        self.space = StandaloneSpace(want_grads)

    def space_of(self, mod):
        return self.space

    def space_of_param(self, p):
        return self.space


def _params_with_owner(module):
    out = []
    for m in module.modules():
        for p in m.parameters(recurse=False):
            out.append((p, m))
    return out


def _recording(module, *tensors):
    """the training path is taken when the module is in training mode (the reference's optimize_parameters calls
    .train() on every net, vqgan_model.py:330-334) and autograd is recording something that needs a gradient"""
    return module.training and torch.is_grad_enabled() and (
        any(t is not None and t.requires_grad for t in tensors) or any(p.requires_grad for p in module.parameters()))


# ----------------------------------------------------------------------------
# gradient scaling at node boundaries
# ----------------------------------------------------------------------------
def _pow2_scale(dy, target=64.0):
    """torch hands the nodes raw gradients (d nll / d xrec = sign / numel ~ 1e-8): the backward kernels take fp16
    hi/lo planes (absolute resolution 2^-24), so every node rescales its incoming gradient to ~``target`` by a power
    of two and divides what it returns (one device->host read per node; the native trainer uses static scales)."""
    amax = float(dy.abs().max())
    # (the Encoder and Decoder-trunk nodes use target 1, the magnitude the native trainers' loss scales give: over
    # their ~20 layers the gradient grows, and the attention backward near the far end writes 2^8-scaled score
    # gradients to fp16 planes, which overflowed for the parsing tokenizer's gradients at target 64)
    if not (amax > 0.0) or amax != amax or amax == float("inf"):
        return 1.0
    import math
    return 2.0 ** math.floor(math.log2(target / amax))


def _unscale(grads, s):
    gs = [g for g in grads if g is not None]
    if s != 1.0 and gs:
        torch._foreach_mul_(gs, 1.0 / s)
    return grads


def _all_layers(objs):
    out = []
    for o in objs:
        if isinstance(o, VT.Seq):
            out += o.layers
        elif isinstance(o, VT.DiscNet):
            out += [o] + o.mid
        elif o is not None:
            out.append(o)
    return out


class _Replayable:
    """A node's backward may run more than once (``retain_graph=True``: calculate_adaptive_weight calls
    autograd.grad twice before loss.backward(), vqgan_loss.py:6-8): the layers pop their saved tensors, so they are
    snapshotted before and restored after each call, and the gradient buffers are handed out as copies and cleared."""

    def __init__(self, host, layers):
        self.host, self.layers = host, _all_layers(layers)

    def __enter__(self):
        self.snap = [(ly, [list(r) if isinstance(r, list) else r for r in ly.saved]) for ly in self.layers]
        return self

    def __exit__(self, *exc):
        for ly, saved in self.snap:
            ly.saved = saved

    def take(self, grads):
        return take_grads(self.host, grads)


def take_grads(host, grads):
    """copies of ``grads`` (views of ``host``'s gradient buffers) for autograd, which may keep them as ``.grad``; the
    buffers are zeroed for the next backward of the same graph"""
    out = [g.clone() if g is not None else None for g in grads]
    sp = host.space
    for cp in sp.convs.d.values():
        if cp.gw is not None:
            cp.gw.zero_()
        if cp.gb is not None:
            cp.gb.zero_()
    for buf in sp.gbuf.values():
        buf.zero_()
    return out


# ----------------------------------------------------------------------------
# Discriminator
# ----------------------------------------------------------------------------
class _DiscFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, disc, x, *params):
        host = _Host(want_grads=True)
        net = VT.DiscNet(host, disc)
        with torch.no_grad():
            logits = net.fwd(x.detach().float().contiguous())
        ctx.host, ctx.net, ctx.disc = host, net, disc
        ctx.x_shape = x.shape
        N, h, w, _ = logits.shape
        return logits.view(N, 1, h, w)

    @staticmethod
    def backward(ctx, dlogits):
        disc, host, net = ctx.disc, ctx.host, ctx.net
        N, _, h, w = dlogits.shape
        dx = torch.empty(ctx.x_shape, dtype=torch.float32, device=dlogits.device) if ctx.needs_input_grad[1] else None
        s = _pow2_scale(dlogits)
        with torch.no_grad(), _Replayable(host, [net]) as rp:
            net.bwd((dlogits * s).contiguous().float().view(N, h, w, 1), want_params=True, want_input=dx is not None,
                    dx_out=dx)
            grads = rp.take([host.space.grad_of(p, m) for p, m in _params_with_owner(disc)])
        out = _unscale([dx] + grads, s)
        return (None,) + tuple(out)


def discriminator_forward(disc, x):
    if _recording(disc, x):
        return _DiscFn.apply(disc, x, *[p for p, _ in _params_with_owner(disc)])
    host = _Host(want_grads=False)
    with torch.no_grad():
        logits = VT.DiscNet(host, disc).fwd(x.detach().float().contiguous())
    N, h, w, _ = logits.shape
    return logits.view(N, 1, h, w)


# ----------------------------------------------------------------------------
# Encoder
# ----------------------------------------------------------------------------
class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, x, *params):
        host = _Host(want_grads=True)
        inl, body, out = VT.encoder_layers(host, enc)
        with torch.no_grad():
            z = out.fwd(body.fwd(inl.fwd(x.detach().float().contiguous())))
        ctx.host, ctx.layers, ctx.enc = host, (inl, body, out), enc
        return ops.nhwc_to_nchw(z)

    @staticmethod
    def backward(ctx, dz):
        inl, body, out = ctx.layers
        s = _pow2_scale(dz, target=1.0)
        with torch.no_grad(), _Replayable(ctx.host, [inl, body, out]) as rp:
            g = ops.nchw_to_nhwc((dz * s).contiguous())
            inl.bwd(body.bwd(out.bwd(g)))
            grads = rp.take([ctx.host.space.grad_of(p, m) for p, m in _params_with_owner(ctx.enc)])
        return (None, None) + tuple(_unscale(grads, s))


def encoder_forward(enc, x):
    assert not x.requires_grad, "the image input of the Encoder mirror is not differentiable"
    return _EncoderFn.apply(enc, x, *[p for p, _ in _params_with_owner(enc)])


# ----------------------------------------------------------------------------
# Decoder: trunk node | tail node (norm_out -> swish -> conv_out)
# ----------------------------------------------------------------------------
def _trunk_params(dec):
    tail = {id(p) for p in list(dec.norm_out.parameters()) + list(dec.conv_out.parameters())}
    return [(p, m) for p, m in _params_with_owner(dec) if id(p) not in tail]


class _DecTrunkFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dec, z, *params):
        host = _Host(want_grads=True)
        inl, body, _ = VT.decoder_layers(host, dec)
        with torch.no_grad():
            zin = ops.nchw_to_nhwc(z.detach().float().contiguous())
            h = body.fwd(inl.fwd(VT.Act(zin)))
        ctx.host, ctx.layers, ctx.dec = host, (inl, body), dec
        dec.__dict__["_t2h_tail_stats"] = (h.x.data_ptr(), h.stats)
        return h.x

    @staticmethod
    def backward(ctx, dh):
        inl, body = ctx.layers
        s = _pow2_scale(dh, target=1.0)
        with torch.no_grad(), _Replayable(ctx.host, [inl, body]) as rp:
            g = inl.bwd(body.bwd(VT.Grad((dh * s).contiguous())))
            dz = ops.nhwc_to_nchw(g.g)
            grads = rp.take([ctx.host.space.grad_of(p, m) for p, m in _trunk_params(ctx.dec)])
        out = _unscale([dz] + grads, s)
        return (None,) + tuple(out)


class _DecTailFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dec, h, gamma, beta, w, b):
        host = _Host(want_grads=True)
        tail = VT.NormConvOutL(host, dec.norm_out, dec.conv_out, nchw=True)
        st = dec.__dict__.pop("_t2h_tail_stats", (None, None))
        with torch.no_grad():
            y = tail.fwd(VT.Act(h.detach(), st[1] if st[0] == h.data_ptr() else None))
        ctx.host, ctx.tail, ctx.dec = host, tail, dec
        return y

    @staticmethod
    def backward(ctx, dy):
        dec = ctx.dec
        s = _pow2_scale(dy)
        sp = ctx.host.space
        with torch.no_grad(), _Replayable(ctx.host, [ctx.tail]) as rp:
            g = ctx.tail.bwd((dy * s).contiguous())
            grads = rp.take([g.g, sp.grad_of(dec.norm_out.weight, dec.norm_out),
                             sp.grad_of(dec.norm_out.bias, dec.norm_out),
                             sp.grad_of(dec.conv_out.weight, dec.conv_out),
                             sp.grad_of(dec.conv_out.bias, dec.conv_out)])
        return (None,) + tuple(_unscale(grads, s))


def _upper_modules(dec):
    """the trunk above the residual point: conv_in, mid and the levels from the top down to RES_LEVEL"""
    return [dec.conv_in, dec.mid] + [dec.up[i] for i in range(RES_LEVEL, dec.num_resolutions)]


class _DecTrunkResFn(torch.autograd.Function):
    """the trunk with the hierarchy residual: upper part (conv_in, mid, levels down to RES_LEVEL) -> + bot_h -> lower
    part (levels RES_LEVEL-1 .. 0).  The gradient leaving the lower part is d bot_h; the upper part's backward runs
    only when one of its parameters or z needs a gradient (the reference fills .grad of conv_in, mid and up.4 although
    its Adam never steps them; quant_top comes from no_grad)."""

    @staticmethod
    def forward(ctx, dec, z, bot_h, *params):
        host = _Host(want_grads=True)
        upper_ids = {id(p) for m in _upper_modules(dec) for p in m.parameters()}
        need = ctx.needs_input_grad
        ctx.run_upper = need[1] or any(n for (p, _), n in zip(_trunk_params(dec), need[3:]) if id(p) in upper_ids)
        inl = VT.ConvL(host, dec.conv_in, "k3", need_dx=need[1])
        upper = VT.Seq(VT.mid_layers(host, dec.mid) + VT.decoder_up_layers(host, dec, dec.num_resolutions - 1,
                                                                            bottom_level=RES_LEVEL))
        lower = VT.Seq(VT.decoder_up_layers(host, dec, RES_LEVEL - 1))
        with torch.no_grad():
            h = upper.fwd(inl.fwd(VT.Act(ops.nchw_to_nhwc(z.detach().float().contiguous()))))
            # the statistics of the sum are not known: the first level-3 block computes them
            h = lower.fwd(VT.Act(ops.add_inplace(h.x, ops.nchw_to_nhwc(bot_h.detach().float().contiguous()))))
        ctx.host, ctx.layers, ctx.dec = host, (inl, upper, lower), dec
        dec.__dict__["_t2h_tail_stats"] = (h.x.data_ptr(), h.stats)
        return h.x

    @staticmethod
    def backward(ctx, dh):
        inl, upper, lower = ctx.layers
        s = _pow2_scale(dh, target=1.0)
        dz = None
        with torch.no_grad(), _Replayable(ctx.host, [inl, upper, lower]) as rp:
            g = lower.bwd(VT.Grad((dh * s).contiguous()))
            dbot = ops.nhwc_to_nchw(g.g)
            if ctx.run_upper:
                g = inl.bwd(upper.bwd(g))
                if g is not None:
                    dz = ops.nhwc_to_nchw(g.g)
            grads = rp.take([ctx.host.space.grad_of(p, m) if n else None
                             for (p, m), n in zip(_trunk_params(ctx.dec), ctx.needs_input_grad[3:])])
        out = _unscale([dz, dbot] + grads, s)
        return (None,) + tuple(out)


def decoder_forward(dec, z, bot_h=None):
    assert not dec.give_pre_end
    if bot_h is None:
        h = _DecTrunkFn.apply(dec, z, *[p for p, _ in _trunk_params(dec)])
    else:
        if dec.num_resolutions <= RES_LEVEL:
            raise ValueError(f"a decoder of {dec.num_resolutions} levels has no level {RES_LEVEL} to add bot_h after")
        h = _DecTrunkResFn.apply(dec, z, bot_h, *[p for p, _ in _trunk_params(dec)])
    return _DecTailFn.apply(dec, h, dec.norm_out.weight, dec.norm_out.bias, dec.conv_out.weight, dec.conv_out.bias)


# ----------------------------------------------------------------------------
# DecoderRes (conv_in -> mid: the bottom level's bot_h, reference vqgan_arch.py:1136-1151)
# ----------------------------------------------------------------------------
class _DecResFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dres, z, *params):
        host = _Host(want_grads=True)
        inl = VT.ConvL(host, dres.conv_in, "k3", need_dx=ctx.needs_input_grad[1])
        body = VT.Seq(VT.mid_layers(host, dres.mid))
        with torch.no_grad():
            h = body.fwd(inl.fwd(VT.Act(ops.nchw_to_nhwc(z.detach().float().contiguous()))))
        ctx.host, ctx.layers, ctx.dres = host, (inl, body), dres
        return ops.nhwc_to_nchw(h.x)

    @staticmethod
    def backward(ctx, dh):
        inl, body = ctx.layers
        s = _pow2_scale(dh, target=1.0)
        with torch.no_grad(), _Replayable(ctx.host, [inl, body]) as rp:
            g = inl.bwd(body.bwd(VT.Grad(ops.nchw_to_nhwc((dh * s).contiguous()))))
            dz = ops.nhwc_to_nchw(g.g) if g is not None else None
            grads = rp.take([ctx.host.space.grad_of(p, m) for p, m in _params_with_owner(ctx.dres)])
        return (None,) + tuple(_unscale([dz] + grads, s))


def decoder_res_forward(dres, z):
    return _DecResFn.apply(dres, z, *[p for p, _ in _params_with_owner(dres)])


# ----------------------------------------------------------------------------
# the texture quantizers (straight-through + legacy-beta codebook loss): VectorQuantizerTexture on single positions
# (vqgan_arch.py:270-281) and VectorQuantizerSpatialTextureAware on ps x ps patches (:449-458)
# ----------------------------------------------------------------------------
def _books_selected(ids, n_books):
    """which codebooks some position selects: one device->host read of ``n_books`` flags"""
    flat = ids.reshape(-1).long()
    flat = flat[(flat >= 0) & (flat < n_books)]
    return (torch.bincount(flat, minlength=n_books)[:n_books] > 0).tolist()


class _VQTexFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, ps, z, segm_map, *weights):
        with torch.no_grad():
            zh = ops.nchw_to_nhwc(z.detach().float().contiguous())
            cb = torch.stack([w.detach().float() for w in weights]).contiguous()
            B, H, W, _ = zh.shape
            ids = ops.mask_to_ids(segm_map, H // ps, W // ps)
            # the reference hard-codes 1024 as the top quantizer's continual-index stride (:262), n_e for the patches
            r = ops.vq_search(zh, cb, ids, ps=ps, cont_stride=1024 if ps == 1 else q.n_e)
            loss = ((1.0 + q.beta) * r["sqerr"][0] / zh.numel()).to(torch.float32)
        ctx.q, ctx.ps, ctx.saved_vq = q, ps, (zh, cb, r["idx"], ids)
        idx_list = r["idx_list"]
        ctx.mark_non_differentiable(r["idx_cont"], idx_list)
        if ps != 1 and not ctx.needs_input_grad[2]:
            # z_q = z + (z_q - z).detach() (:458) carries a gradient only when z does
            ctx.mark_non_differentiable(r["zq_nchw"])
        return r["zq_nchw"], loss, r["idx_cont"], idx_list

    @staticmethod
    def backward(ctx, dzq, dloss, *_):
        zh, cb, idx, ids = ctx.saved_vq
        nel = zh.numel()
        dl = float(dloss) if dloss is not None else 0.0
        # legacy: loss = mean((zq.detach()-z)^2) + beta*mean((zq-z.detach())^2); otherwise beta weighs the z term
        w_z, w_e = (1.0, ctx.q.beta) if ctx.q.legacy else (ctx.q.beta, 1.0)
        cz, ce = 2.0 * w_z * dl / nel, 2.0 * w_e * dl / nel
        with torch.no_grad():
            s = _pow2_scale(dzq) if dzq is not None else 1.0
            dzq_h = ops.nchw_to_nhwc((dzq * s).contiguous()) if dzq is not None else None
            dcb = torch.zeros_like(cb)
            if ctx.ps == 1:
                dz = ops.vq_bwd(zh, cb, idx, ids, dzq_h, dcb, cz * s, ce * s)
            else:
                dz = ops.vq_bwd_patch(zh, cb, idx, ids, dzq_h, dcb, cz * s, ce * s, ps=ctx.ps)
            dzn = ops.nhwc_to_nchw(dz)
        grads = _unscale([dzn, dcb], s)
        books = list(grads[1].unbind(0))
        if ctx.ps != 1:
            # the reference only looks up embedding_list[k] when some patch selects book k (:416): the others keep
            # .grad None, so that torch.optim.Adam skips them instead of moving them by their first moment
            books = [g if used else None for g, used in zip(books, _books_selected(ids, len(books)))]
        return (None, None, grads[0], None) + tuple(books)


def quantizer_texture_forward(q, z, segm_map):
    zq, loss, cont, lst = _VQTexFn.apply(q, 1, z, segm_map, *[e.weight for e in q.embedding_list])
    return zq, loss, (None, cont, list(lst.unbind(0)))


def quantizer_spatial_forward(q, z, segm_map):
    """-> (z_q, loss, (None, idx_cont flat, 18 index maps)) as VectorQuantizerSpatialTextureAware.forward"""
    zq, loss, cont, lst = _VQTexFn.apply(q, q.spatial_size, z, segm_map, *[e.weight for e in q.embedding_list])
    return zq, loss, (None, cont.reshape(-1), list(lst.unbind(0)))


# ----------------------------------------------------------------------------
# VectorQuantizer (one codebook; straight-through + beta codebook loss, vqgan_arch.py:79-122)
# ----------------------------------------------------------------------------
class _VQFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, z, weight):
        with torch.no_grad():
            zh = ops.nchw_to_nhwc(z.detach().float().contiguous())
            cb = weight.detach().float().unsqueeze(0).contiguous()
            r = ops.vq_search(zh, cb, None, want_list=False, want_nhwc=False)
            loss = ((1.0 + q.beta) * r["sqerr"][0] / zh.numel()).to(torch.float32)
        ctx.q, ctx.saved_vq = q, (zh, cb, r["idx"])
        ctx.mark_non_differentiable(r["idx"])
        return r["zq_nchw"], loss, r["idx"]

    @staticmethod
    def backward(ctx, dzq, dloss, _):
        zh, cb, idx = ctx.saved_vq
        nel = zh.numel()
        dl = float(dloss) if dloss is not None else 0.0
        # legacy: loss = mean((zq.detach()-z)^2) + beta*mean((zq-z.detach())^2); otherwise beta weighs the z term
        w_z, w_e = (1.0, ctx.q.beta) if ctx.q.legacy else (ctx.q.beta, 1.0)
        with torch.no_grad():
            s = _pow2_scale(dzq) if dzq is not None else 1.0
            dzq_h = ops.nchw_to_nhwc((dzq * s).contiguous()) if dzq is not None else None
            dcb = torch.zeros_like(cb)
            dz = ops.vq_bwd(zh, cb, idx, None, dzq_h, dcb, 2.0 * w_z * dl * s / nel, 2.0 * w_e * dl * s / nel)
            dzn = ops.nhwc_to_nchw(dz)
        grads = _unscale([dzn, dcb], s)
        return None, grads[0], grads[1][0]


def quantizer_forward(q, z):
    """-> (z_q, loss, (None, None, idx)) as VectorQuantizer.forward; idx flat unless ``sane_index_shape``"""
    zq, loss, idx = _VQFn.apply(q, z, q.embedding.weight)
    return zq, loss, (None, None, idx if q.sane_index_shape else idx.reshape(-1))


def recording(module, *tensors):
    return _recording(module, *tensors)
