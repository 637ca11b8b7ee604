"""Drop-in training boundary of the index-prediction nets: UNet and MultiHeadFCNHead as torch.autograd nodes, so that
the reference's ``VQGANTextureAwareSpatialHierarchyInferenceModel.optimize_parameters``
(models/hierarchy_inference_model.py:227-245: both nets in training mode, the sum over the 18 heads of
CrossEntropyLoss(ignore_index=-1), ``loss.backward()``, ``torch.optim.Adam`` or ``SGD``) runs unmodified on the mirrors.

* ``UNet`` is the UNet node of ``parsing_gen_autograd`` without an embedding: ``train_layers.UNetL`` with
  batch-statistics BatchNorm, the five decoder outputs, and the input gradient whenever the input requires one (the
  wrapper's ``feature_t`` comes out of its own ``top_post_quant_conv``, whose ``.grad`` the reference fills).
* ``MultiHeadFCNHead``: the 18 3x3 ConvModules run as ONE ``train_layers.ConvModuleL`` of 18*channels outputs with one
  BatchNorm over them, as ``index_pred_train.IndexPredTrainer`` runs them; the 18 Dropout2d draws are made one head
  after the other, as the reference's single ``nn.Dropout2d`` called once per head makes them; conv_seg is one batched
  GEMM over the heads.  Its backward turns the 18 logit gradients torch hands over into conv_seg's operand planes and
  the 18 bias gradients in one read (``ops.head_grads_to_planes_sums``), then runs one batched weight-gradient GEMM,
  one batched data-gradient GEMM and the stacked ConvModule's backward.

Parameters are gathered from the modules at every forward (a few hundred KB) and every gradient is returned in its
parameter's own shape; the running statistics are written into each BatchNorm's own buffers.  In training mode without
recording (``torch.no_grad``) the same forward runs and nothing is saved.  The native, faster path for the same step
(and the one for several GPUs) is ``index_pred_train.IndexPredTrainer``.
"""
import torch

from . import ops
from .flat_params import ConvStack, drop_packed_caches
from .parsing_gen_autograd import _restore, _stash, unet_node_forward
from .parsing_gen_train import dropout2d_mask
from .train_layers import ConvModuleL
from .vqgan_autograd import _Host, _params_with_owner, _pow2_scale, _recording, _unscale, take_grads


def _check_feature(unet, x):
    f = 2 ** (unet.num_stages - 1)
    if x.dim() != 4 or x.shape[2] % f or x.shape[3] % f:
        raise ValueError(f"UNet: the feature must be [B, C, h, w] with h, w multiples of {f} (the UNet pools "
                         f"{unet.num_stages - 1} times), got {tuple(x.shape)}")


def unet_forward(unet, x):
    """index_pred_arch.UNet.forward in training mode: x NCHW -> the five decoder outputs NCHW, coarsest first"""
    _check_feature(unet, x)
    return unet_node_forward(unet, x)


# ----------------------------------------------------------------------------
# MultiHeadFCNHead
# ----------------------------------------------------------------------------
def _drop_factor(head, B, device):
    """the 18 Dropout2d draws of one forward, in head order, packed head-major and divided by 1-p: [B, 18*channels]"""
    if head.dropout is None:
        return None
    p = head.dropout.p
    masks = [dropout2d_mask(B, head.channels, p, device) for _ in range(head.num_head)]
    return torch.stack(masks, 1).div_(1.0 - p).reshape(B, -1)


def _heads_run(head, host, x):
    """stacked 3x3 ConvModule (batch statistics, Dropout2d) -> the 18 conv_seg: -> (the ConvModuleL, its output
    planes [T,B,h,w,18*ch], conv_seg's weight planes [T,18,ncls,ch], logits fp32 [18, B*h*w, ncls])"""
    drop_packed_caches(head)
    B, _, H, W = x.shape
    drop = _drop_factor(head, B, x.device)
    bns = [seq[0].bn for seq in head.convs_list]
    hc = ConvModuleL(host, ConvStack(seq[0].conv for seq in head.convs_list), bns, "k3", "relu", bind_stats=False)
    y = hc.fwd(ops.nchw_to_planes(x.detach()), out="planes", drop=drop)
    G_, ch, ncls = head.num_head, head.channels, head.num_classes
    segs = head.conv_seg_head_list
    w1 = ops.split_planes(torch.stack([c.weight.detach().float().view(ncls, ch) for c in segs]), ops.get_terms())
    b1 = torch.stack([c.bias.detach().float() for c in segs]).contiguous()
    T = y.shape[0]
    logits = ops.bmm_nt(y.view(T, B * H * W, G_, ch).permute(0, 2, 1, 3), w1, bias_col=b1)
    return hc, y, w1, logits


def _views(head, logits, B, H, W):
    return tuple(logits[k].view(B, H, W, head.num_classes).permute(0, 3, 1, 2) for k in range(head.num_head))


class _HeadsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, head, x, *params):
        ctx.set_materialize_grads(False)       # a head the loss does not use arrives as None, read as zeros
        host = _Host(want_grads=True)
        hc, y, w1, logits = _heads_run(head, host, x)
        ctx.head, ctx.host, ctx.hc, ctx.x_shape = head, host, hc, x.shape
        _stash(ctx, [hc], y, w1)
        B, _, H, W = x.shape
        return _views(head, logits, B, H, W)

    @staticmethod
    def backward(ctx, *dlogits):
        head, host, hc = ctx.head, ctx.host, ctx.hc
        n_params = len(list(head.parameters()))
        if all(g is None for g in dlogits):
            return (None, None) + (None,) * n_params
        y, w1 = _restore(ctx, [hc])
        B, Cin, H, W = ctx.x_shape
        G_, ch, ncls = head.num_head, head.channels, head.num_classes
        M = B * H * W
        T = y.shape[0]
        with torch.no_grad():
            # [B, h*w, ncls] views of the NCHW gradients, whatever their strides: no copy
            table, shape = ops.head_grads_table([g.flatten(2).transpose(1, 2) if g is not None else None
                                                 for g in dlogits])
            # the magnitude routed_head_ce gives the native trainer's conv_seg gradient: |d| <= 1
            s = _pow2_scale(ops.head_grads_absmax(table, shape), target=1.0)   # the one device->host read
            dlp, gb = ops.head_grads_to_planes_sums(table, shape, s)
            dl = dlp.view(T, M, G_, ncls).permute(0, 2, 1, 3)
            gw = torch.empty((G_, ncls, ch), dtype=torch.float32, device=y.device)
            ops.wgrad_batched(dl, y.view(T, M, G_, ch).permute(0, 2, 1, 3), gw)
            dy = torch.empty((B, H, W, G_ * ch), dtype=torch.float32, device=y.device)
            ops.bmm_nt(dl, w1, b_kn=True, out=dy.view(M, G_, ch).permute(1, 0, 2))
            d = hc.bwd(dy)
            del dy, dlp
            dx = ops.nhwc_to_nchw(d if d.shape[-1] == Cin else d[..., :Cin].contiguous()) \
                if ctx.needs_input_grad[1] else None
            seg = {}
            for k, c in enumerate(head.conv_seg_head_list):
                seg[id(c.weight)], seg[id(c.bias)] = gw[k].view_as(c.weight), gb[k]
            grads = take_grads(host, [seg[id(p)] if id(p) in seg else host.space.grad_of(p, m)
                                      for p, m in _params_with_owner(head)])
        out = _unscale([dx] + grads, s)
        return (None,) + tuple(g if n else None for g, n in zip(out, ctx.needs_input_grad[1:]))


def heads_forward(head, inputs):
    """MultiHeadFCNHead.forward in training mode: -> the 18 NCHW logit maps [B, num_classes, h, w] of
    inputs[in_index], in head order"""
    x = inputs[head.in_index]
    if x.dim() != 4 or x.shape[1] != head.in_channels:
        raise ValueError(f"MultiHeadFCNHead: the input must be [B, {head.in_channels}, h, w], got {tuple(x.shape)}")
    if _recording(head, x):
        return list(_HeadsFn.apply(head, x, *head.parameters()))
    with torch.no_grad():
        B, _, H, W = x.shape
        return list(_views(head, _heads_run(head, _Host(want_grads=False), x)[3], B, H, W))
