"""Drop-in training boundary of the parsing generator: ShapeAttrEmbedding, ShapeUNet and FCNHead as torch.autograd
nodes, so that the reference's ``ParsingGenModel.optimize_parameters`` (models/parsing_gen_model.py:80-95: three nets
in training mode, CrossEntropyLoss, ``loss.backward()``, ``torch.optim.Adam``) runs unmodified on the mirrors.

Each mirror's ``forward`` in training mode is one node (when autograd records something that needs a gradient) whose
forward and backward are the native trainer's (``parsing_gen_train``): ``train_layers.UNetL`` / ``ConvModuleL`` with
batch-statistics BatchNorm, running statistics updated as nn.BatchNorm2d does, Dropout2d in the norm apply, and
``shape_attr_embed_bwd``.  The nodes hand NCHW fp32 tensors to each other, as the reference's modules do; the head's
incoming logit gradient becomes conv_seg's operand planes and bias gradient in one pass
(``ops.nchw_grad_to_planes``).  In training mode without recording (``torch.no_grad``) the same forward runs and
nothing is saved.  The native, faster path for the same step is ``parsing_gen_train.ParsingGenTrainer``.  The UNet
node also serves index_pred_arch's UNet (no embedding; the input gradient when the input requires one).
"""
import torch

from . import conv_grad as G
from . import ops
from .flat_params import drop_packed_caches
from .parsing_gen_train import dropout2d_mask, embedder_linears
from .train_layers import UNetL, conv_module
from .vqgan_autograd import _Host, _params_with_owner, _pow2_scale, _recording, _unscale, take_grads


# ----------------------------------------------------------------------------
# the layers' saved stacks through ctx.save_for_backward
# ----------------------------------------------------------------------------
class _Slot:
    __slots__ = ("i",)

    def __init__(self, i):
        self.i = i


def _stash(ctx, layers, *extra):
    """move every tensor on the layers' saved stacks (and ``extra``) into ``ctx.save_for_backward``, so that they are
    released with the graph and kept for a ``retain_graph`` replay; the stacks' structure stays on ctx"""
    tensors = []

    def enc(v):
        if isinstance(v, torch.Tensor):
            tensors.append(v)
            return _Slot(len(tensors) - 1)
        if isinstance(v, (list, tuple)):
            return type(v)(enc(u) for u in v)
        return v

    ctx.skel = [enc(ly.saved) for ly in layers]
    for ly in layers:
        ly.saved = []
    ctx.n_stashed = len(tensors)
    ctx.save_for_backward(*tensors, *extra)


def _restore(ctx, layers):
    """refill the layers' stacks (fresh lists: each backward of the graph pops its own) -> the ``extra`` tensors"""
    ts = ctx.saved_tensors

    def dec(v):
        if isinstance(v, _Slot):
            return ts[v.i]
        if isinstance(v, (list, tuple)):
            return type(v)(dec(u) for u in v)
        return v

    for ly, sk in zip(layers, ctx.skel):
        ly.saved = dec(sk)
    return ts[ctx.n_stashed:]


# ----------------------------------------------------------------------------
# ShapeAttrEmbedding
# ----------------------------------------------------------------------------
_PACKED = ("cls_off", "w1t", "b1", "w2", "b2", "wf1", "bf1", "wf2", "bf2")


def _embedder_grad_layout(emb):
    """per parameter (in ``embedder_linears`` order, weight then bias) its 8-aligned offset in one flat buffer"""
    offs, total = {}, 0
    for m in embedder_linears(emb):
        for p in (m.weight, m.bias):
            offs[id(p)] = total
            total += (p.numel() + 7) // 8 * 8
    return offs, total


class _EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, attr, *params):
        packed = emb._packed()
        out = ops.shape_attr_embed(attr, packed)
        ctx.save_for_backward(attr, *[packed[k] for k in _PACKED])
        ctx.emb = emb
        return out

    @staticmethod
    def backward(ctx, d):
        # fp32 throughout (no operand planes): the incoming gradient is used as it is, without rescaling
        emb = ctx.emb
        attr, *pk = ctx.saved_tensors
        offs, total = _embedder_grad_layout(emb)
        flat = torch.zeros(total, dtype=torch.float32, device=d.device)
        order = [p for m in embedder_linears(emb) for p in (m.weight, m.bias)]
        goff = torch.tensor([offs[id(p)] for p in order], dtype=torch.int64).to(d.device)
        with torch.no_grad():
            ops.shape_attr_embed_bwd(attr, dict(zip(_PACKED, pk)), d.float().contiguous(), flat, goff)
        grads = [flat[offs[id(p)]:offs[id(p)] + p.numel()].view_as(p) if n else None
                 for p, n in zip(emb.parameters(), ctx.needs_input_grad[2:])]
        return (None, None) + tuple(grads)


def shape_attr_embedding_forward(emb, attr):
    """ShapeAttrEmbedding.forward in training mode: attr int [B, n_attr] -> fp32 [B, out_dim]"""
    emb.check_attributes(attr)
    attr = attr.to(emb.fusion[0].weight.device).to(torch.int64).contiguous()
    if _recording(emb):
        return _EmbedFn.apply(emb, attr, *emb.parameters())
    with torch.no_grad():
        return ops.shape_attr_embed(attr, emb._packed())


# ----------------------------------------------------------------------------
# UNet / ShapeUNet
# ----------------------------------------------------------------------------
def _unet_layers(ul):
    out = [ul]
    for st in ul.stages:
        out += st.convs
    for d in ul.dec:
        out += [d, d.up] + d.block.convs
    return out


def _unet_run(unet, host, x, e, need_dx):
    """the training-mode forward: -> (UNetL, the five decoder outputs fp32 NHWC, coarsest first)"""
    # the running statistics are updated by a kernel that torch's version counters do not see
    drop_packed_caches(unet)
    ul = UNetL(host, unet, need_dx=need_dx)
    B, C, H, W = x.shape
    xh = x.detach().float().reshape(B, H, W, 1) if C == 1 else ops.nchw_to_nhwc(x.detach())
    return ul, ul.fwd(xh, None if e is None else e.detach().float().contiguous(), all_outs=True)


class _UNetFn(torch.autograd.Function):
    """The UNet of index_pred_arch (``e`` None) or ShapeUNet (``e`` the attribute embedding) in training mode: returns
    the five decoder outputs and takes a gradient on any of them.  The gradient of ``x`` is computed and returned when
    ``x`` requires one; ShapeUNet's embedding always needs stage 0's data gradient."""

    @staticmethod
    def forward(ctx, unet, x, e, *params):
        ctx.set_materialize_grads(False)       # a decoder output the loss does not use arrives as None
        host = _Host(want_grads=True)
        ul, outs = _unet_run(unet, host, x, e, need_dx=e is not None or ctx.needs_input_grad[1])
        ctx.unet, ctx.host, ctx.ul, ctx.last_shape = unet, host, ul, outs[-1].shape
        ctx.x_shape, ctx.e_shape = x.shape, None if e is None else e.shape
        _stash(ctx, _unet_layers(ul))
        return tuple(ops.nhwc_to_nchw(o) for o in outs)

    @staticmethod
    def backward(ctx, *douts):
        unet, host, ul = ctx.unet, ctx.host, ctx.ul
        n_in = 3 + len(list(unet.parameters()))
        gs = [g for g in douts if g is not None]
        if not gs:
            return (None,) * n_in
        _restore(ctx, _unet_layers(ul))
        s = _pow2_scale(torch.stack([g.detach().abs().amax() for g in gs]), target=1.0)
        dx = None
        with torch.no_grad():
            nhwc = [ops.nchw_to_nhwc((g * s).contiguous()) if g is not None else None for g in douts]
            last = nhwc[-1]
            if last is None:
                last = torch.zeros(ctx.last_shape, dtype=torch.float32, device=gs[0].device)
            de = None if ctx.e_shape is None else torch.zeros(ctx.e_shape, dtype=torch.float32, device=gs[0].device)
            da = ul.bwd(last, de, d_coarser=nhwc[:-1])
            if ctx.needs_input_grad[1]:
                C = ctx.x_shape[1]
                dx = ops.nhwc_to_nchw(da if da.shape[-1] == C else da[..., :C].contiguous())
            grads = take_grads(host, [host.space.grad_of(p, m) for p, m in _params_with_owner(unet)])
        dx, de, *out = _unscale([dx, de] + grads, s)
        return (None, dx, de if ctx.needs_input_grad[2] else None) + tuple(out)


def unet_node_forward(unet, x, e=None):
    """a UNet (``e`` None) or ShapeUNet in training mode: -> the five decoder outputs NCHW, coarsest first; one
    autograd node when autograd records, else the same forward (batch statistics, running statistics updated)"""
    if _recording(unet, x, e):
        return list(_UNetFn.apply(unet, x, e, *unet.parameters()))
    with torch.no_grad():
        _, outs = _unet_run(unet, _Host(want_grads=False), x, e, need_dx=False)
        return [ops.nhwc_to_nchw(o) for o in outs]


def shape_unet_forward(unet, x, e):
    """ShapeUNet.forward in training mode: x NCHW (the pose), e fp32 [B, attr_embedding] -> the five decoder outputs
    NCHW, coarsest first (unet_arch.py:657-674)"""
    if x.requires_grad and torch.is_grad_enabled():
        raise NotImplementedError("ShapeUNet: no gradient with respect to the pose input (the reference never asks "
                                  "for one)")
    return unet_node_forward(unet, x, e)


# ----------------------------------------------------------------------------
# FCNHead
# ----------------------------------------------------------------------------
def _head_run(head, host, x):
    """3x3 ConvModule (batch statistics, Dropout2d drawn as nn.Dropout2d draws it) -> 1x1 conv_seg: -> (the
    ConvModuleL, conv_seg's operand planes, NCHW fp32 logits)"""
    drop_packed_caches(head)
    B, _, H, W = x.shape
    drop = None
    if head.dropout is not None:
        p = head.dropout.p
        drop = dropout2d_mask(B, head.channels, p, x.device).div_(1.0 - p)
    hc = conv_module(host, head.convs[0])
    y = hc.fwd(ops.nchw_to_planes(x.detach()), out="planes", drop=drop)
    cps = host.space.convs[head.conv_seg]
    C = head.num_classes
    wn = cps.wn[:, :, :C] if cps.co != cps.co_p else cps.wn
    logits = G.forward("k1", y, wn, cps.b[:C], n=B, in_hw=(H, W), nchw_out=True)
    return hc, y, logits


class _FCNHeadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, head, x, *params):
        host = _Host(want_grads=True)
        hc, y, logits = _head_run(head, host, x)
        ctx.head, ctx.host, ctx.hc, ctx.x_shape = head, host, hc, x.shape
        _stash(ctx, [hc], y)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        head, host, hc = ctx.head, ctx.host, ctx.hc
        (y,) = _restore(ctx, [hc])
        B, Cin, H, W = ctx.x_shape
        # the magnitude ce_logits gives the native trainer's conv_seg gradient: |d| <= 1
        s = _pow2_scale(dlogits, target=1.0)
        cps = host.space.convs[head.conv_seg]
        with torch.no_grad():
            dlp, _ = ops.nchw_grad_to_planes(dlogits, cps.co_p, s, sums=cps.gb)
            G.wgrad("k1", dlp, y, cps.gw, n=B)
            d = hc.bwd(G.dgrad("k1", dlp, cps.wt, n=B, in_hw=(H, W)))
            dx = ops.nhwc_to_nchw(d if d.shape[-1] == Cin else d[..., :Cin].contiguous())
            grads = take_grads(host, [host.space.grad_of(p, m) for p, m in _params_with_owner(head)])
        return (None,) + tuple(_unscale([dx] + grads, s))


def fcn_head_forward(head, inputs):
    """FCNHead.forward in training mode: NCHW logits [B, num_classes, H, W] of inputs[in_index]"""
    x = inputs[head.in_index]
    if _recording(head, x):
        return _FCNHeadFn.apply(head, x, *head.parameters())
    with torch.no_grad():
        return _head_run(head, _Host(want_grads=False), x)[2]
