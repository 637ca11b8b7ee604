"""Training step of the index-prediction transformer on the H100 kernels, with data-parallel
gradient all-reduce over NCCL.

Mirrors ``TransformerTextureAwareModel._train_loss`` / ``q_sample`` / ``optimize_parameters``
(models/transformer_model.py:212-303: absorbing-diffusion masking, 18 masked cross-entropies,
re-weighted ELBO, ``loss.backward()``, ``torch.optim.Adam.step()``) for the ``TransformerMultiHead``
mirror.  Forward and backward contractions (dgrad, wgrad, attention gradients) all run on
``t2h_tapgemm``; a gradient GEMM that contracts over the rows of a stored matrix (dY^T X, P^T dY, dY W) reads it
as an MN-major tensor-core operand (``a_mn`` / ``b_mn``), so no transposed copy of any activation, gradient or
weight is made.  Parameters, gradients and Adam moments live in a ``flat_params.ParamSpace`` (the
``nn.Parameter``s are views of its flat fp32 buffers), so the optimiser is one kernel launch and the gradient
all-reduce works on contiguous buckets (the heads with ``ln_f``, each run of ``bucket_layers`` blocks, the
embeddings) that are launched as soon as the backward pass has finished the layers they cover (overlap with the
remaining backward).
"""
import math

import torch

from . import ops
from .dist import world_size
from .flat_params import ParamSpace, drop_packed_caches


def targets_from_gt_list(gt_list):
    """the reference's 18 per-texture ground-truth lists (-1 outside the texture; transformer_model.py:
    get_quantized_img) -> (own-codebook target [B,T], with -1 where no list covers the position)"""
    own = torch.full_like(gt_list[0], -1)
    for gt in gt_list:
        own = torch.where(gt >= 0, gt, own)
    return own


# ---------------------------------------------------------------------- forward with saved activations
def weight_planes(m, wqkv, w_heads):
    """fp16 planes [T,1,out,in] of every GEMM weight for this step (one conversion launch each); ``wqkv`` holds each
    block's q | k | v weights as one [3C, C] matrix, ``w_heads`` the 18 heads as one [18*ncls, C] matrix.  The
    forward uses the planes K-major (y = x W^T); the data-gradient GEMMs read the SAME planes MN-major (dX = dY W)."""
    def planes(w):
        return ops.f32_to_planes_rows(w.detach()).unsqueeze(1)

    wp = []
    for blk, w in zip(m.blocks, wqkv):
        wp.append(dict(qkv=planes(w), proj=planes(blk.attn.proj.weight), fc1=planes(blk.mlp[0].weight),
                       fc2=planes(blk.mlp[2].weight)))
    return wp, planes(w_heads)


SAVED_KEYS = ("x_in", "h1", "qkv", "p", "y", "x_mid", "h2", "pre", "g")   # per block, what the backward reads


def forward_saved(m, idx, segm, tex, wp, w_heads, bqkv):
    """the TransformerMultiHead forward keeping what the backward needs; ``bqkv`` holds each block's q | k | v bias
    as one [3C] vector.  -> (logits [B*T, num_head, ncls], per-block saved activations, last stream x, ln_f planes)"""
    B, T = idx.shape
    C = m.n_embd
    nh = m.blocks[0].attn.n_head
    x = ops.embed_sum(idx, segm, tex, m.tok_emb.weight.detach(), m.pos_emb.detach()[0],
                      m.segm_emb.weight.detach(), m.texture_emb.weight.detach())
    saved = []
    for blk, w, b_qkv in zip(m.blocks, wp, bqkv):
        a = blk.attn
        s = {"x_in": x}
        h1 = ops.layer_norm(x, blk.ln1.weight.detach(), blk.ln1.bias.detach(), blk.ln1.eps)
        qkv = ops.linear(h1, w["qkv"], b_qkv, planes_out=True)                     # [Tt, M, 3C]: q | k | v
        sc = ops.mha_scores(qkv[:, :, :C], B, T, nh, k=qkv[:, :, C:2 * C])
        p = ops.softmax_rows(sc, scale=1.0 / math.sqrt(C // nh))
        y = ops.mha_pv(p, qkv[:, :, 2 * C:], B, T, nh, v_tok=True)
        x_mid = ops.linear(y, w["proj"], a.proj.bias.detach(), residual=x)
        h2 = ops.layer_norm(x_mid, blk.ln2.weight.detach(), blk.ln2.bias.detach(), blk.ln2.eps)
        pre = ops.linear(h2, w["fc1"], blk.mlp[0].bias.detach())
        g = ops.gelu_fwd(pre)
        x = ops.linear(g, w["fc2"], blk.mlp[2].bias.detach(), residual=x_mid)
        s.update(h1=h1, qkv=qkv, p=p, y=y, x_mid=x_mid, h2=h2, pre=pre, g=g)
        saved.append(s)
    hf = ops.layer_norm(x, m.ln_f.weight.detach(), m.ln_f.bias.detach(), m.ln_f.eps)
    logits = ops.linear(hf, w_heads)
    return logits.view(B * T, m.num_head, m.head_class_num), saved, x, hf


# ---------------------------------------------------------------------- backward from the heads' output gradient
def _wgrad(dy, x, out):
    """out[n_out, n_in] = dy^T x over all tokens; dy [T,M,n_out], x [T,M,n_in] token-major planes, read
    MN-major.  The output has few tiles and the contraction is long, so k-slices are spread over the SMs
    and reduce-added into the (zeroed) gradient buffer."""
    ks = ops.wgrad_k_split(dy.shape[2], x.shape[2], dy.shape[1]) if ops.SPLIT_K["wgrad"] else 0
    ops.wgrad(dy, x, out, k_split=ks)


def backward_from_planes(m, dl, saved, x_last, hf, wp, w_heads, x_t, segm, tex, grads):
    """The whole backward pass below the logits, shared by ``SamplerTrainer`` and the drop-in autograd node.
    dl: fp16 planes [Tt, B*T, 18*ncls] of the (scaled) logit gradient; saved, x_last, hf, wp, w_heads: what
    ``forward_saved`` / ``weight_planes`` returned (``saved`` entries are dropped as the blocks finish); x_t, segm,
    tex [B,T]: the token inputs.  ``grads`` provides the zeroed gradient buffers: ``g(p)`` for one parameter,
    ``joint(params, cols)[1]`` for q | k | v and the 18 heads as one matrix each, and ``done(mod)`` as each
    module's gradients become final (``flat_params.ParamSpace``, or ``NodeGrads`` for the node)."""
    B, T = x_t.shape
    C = m.n_embd
    M = B * T
    nh = m.blocks[0].attn.n_head
    scale = 1.0 / math.sqrt(C // nh)
    DS = 256.0  # extra scale of the (much smaller) score gradients, undone by the consuming GEMMs' alpha
    g = grads.g

    # ---- heads + final LayerNorm
    _wgrad(dl, hf, grads.joint([h.weight for h in m.head_list], C)[1])  # dW_heads [NK, C] = dlogits^T hf
    d_hf = ops.linear(dl, w_heads, w_kn=True)                        # [M, C] = dlogits W_heads
    del dl
    dx = torch.zeros((M, C), dtype=torch.float32, device=x_last.device)  # running gradient of the stream
    # every LayerNorm backward also emits what the next stage needs from the dx it just wrote: its fp16
    # planes and its column sums (the bias gradient of the linear layer that produced that activation)
    dxo = ops.layernorm_bwd_(dx, d_hf, x_last, m.ln_f.weight.detach(), g(m.ln_f.weight), g(m.ln_f.bias),
                             m.ln_f.eps, accumulate=False, want_planes=True,
                             colsum_out=g(m.blocks[-1].mlp[2].bias))
    grads.done(m.ln_f)

    # ---- blocks, last to first; dx is updated in place
    for li in range(len(m.blocks) - 1, -1, -1):
        blk, s, w = m.blocks[li], saved[li], wp[li]
        a = blk.attn
        fc1, fc2 = blk.mlp[0], blk.mlp[2]
        q, k, v = s["qkv"][:, :, :C], s["qkv"][:, :, C:2 * C], s["qkv"][:, :, 2 * C:]
        # MLP: x_out = x_mid + fc2(gelu(fc1(ln2(x_mid))))
        _wgrad(dxo, s["g"], g(fc2.weight))                                       # dW2 [C,F] = dxo^T g
        d_g = ops.linear(dxo, w["fc2"], w_kn=True)                                # [M,F]  = dxo W2
        d_a, da = ops.gelu_bwd(s["pre"], d_g, want_planes=True)                   # fp32 (bias grad) + planes
        ops.colsum_(g(fc1.bias), d_a)
        _wgrad(da, s["h2"], g(fc1.weight))                                       # dW1 [F,C]
        d_h2 = ops.linear(da, w["fc1"], w_kn=True)                                # [M,C]
        dxm = ops.layernorm_bwd_(dx, d_h2, s["x_mid"], blk.ln2.weight.detach(), g(blk.ln2.weight),
                                 g(blk.ln2.bias), blk.ln2.eps, accumulate=True, want_planes=True,
                                 colsum_out=g(a.proj.bias))                       # dx = d x_mid
        # attention output projection: x_mid = x_in + proj(y)
        _wgrad(dxm, s["y"], g(a.proj.weight))                                    # dWp [C,C]
        d_y = ops.linear(dxm, w["proj"], w_kn=True, planes_out=True)              # planes [Tt,M,C]
        # attention core; the three gradients land side by side in d_qkv [M, 3C]
        d_qkv = torch.empty((M, 3 * C), dtype=torch.float32, device=dx.device)
        ops.mha_pv(s["p"], d_y, B, T, nh, planes_out=False, out=d_qkv[:, 2 * C:], p_mn=True, v_tok=True)  # dV
        dp = ops.mha_scores(d_y, B, T, nh, k=v)                                   # dP = dY V^T
        dsp = ops.softmax_bwd_planes(s["p"], dp, scale, out_scale=DS)             # planes [Tt,B,nh,T,T] of DS*dS
        ops.mha_pv(dsp, k, B, T, nh, planes_out=False, out=d_qkv[:, :C], alpha=1.0 / DS, v_tok=True)     # dQ
        ops.mha_pv(dsp, q, B, T, nh, planes_out=False, out=d_qkv[:, C:2 * C], alpha=1.0 / DS, p_mn=True,
                   v_tok=True)                                                    # dK = dS^T Q
        # fused q|k|v projection
        dqkv = ops.f32_to_planes_rows(d_qkv)
        gwqkv = grads.joint([a.query.weight, a.key.weight, a.value.weight], C)[1]
        gbqkv = grads.joint([a.query.bias, a.key.bias, a.value.bias])[1]
        ops.colsum_(gbqkv, d_qkv)
        _wgrad(dqkv, s["h1"], gwqkv)
        d_h1 = ops.linear(dqkv, w["qkv"], w_kn=True)                              # [M,C]
        dxo = ops.layernorm_bwd_(dx, d_h1, s["x_in"], blk.ln1.weight.detach(), g(blk.ln1.weight),
                                 g(blk.ln1.bias), blk.ln1.eps, accumulate=True, want_planes=li > 0,
                                 colsum_out=g(m.blocks[li - 1].mlp[2].bias) if li > 0 else None)
        # dx = d x_in = the gradient of the previous layer's output
        saved[li] = None
        grads.done(blk.ln1)

    # ---- embeddings
    ops.embed_bwd_(g(m.tok_emb.weight), dx, x_t.reshape(-1).contiguous())
    ops.embed_bwd_(g(m.pos_emb).view(-1, C), dx, None, T)
    ops.embed_bwd_(g(m.segm_emb.weight), dx, segm.reshape(-1).contiguous())
    ops.embed_bwd_(g(m.texture_emb.weight), dx, tex.reshape(-1).contiguous())
    grads.done(m.texture_emb)


class SamplerTrainer:
    """Owns a TransformerMultiHead, its flat parameter / gradient / Adam buffers and the training step."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, num_timesteps=1000, mask_id=None,
                 loss_type="reweighted_elbo", bucket_layers=6):
        self.m = model
        self.lr, self.betas, self.eps = lr, betas, eps
        self.num_timesteps = num_timesteps
        self.mask_id = model.codebook_size if mask_id is None else mask_id
        self.loss_type = loss_type
        self.loss_scale = 1.0
        self.bucket_layers = bucket_layers
        self.device = next(model.parameters()).device
        m = model
        C = m.n_embd
        assert C % 8 == 0, "flat parameter slots are 32-byte aligned; n_embd must be a multiple of 8"
        # backward-completion order; q | k | v and the 18 heads are groups, each read as one matrix
        order = [tuple(m.head_list), m.ln_f]
        for blk in reversed(list(m.blocks)):
            a = blk.attn
            order += [blk.mlp[2], blk.mlp[0], blk.ln2, a.proj, (a.query, a.key, a.value), blk.ln1]
        order += [m, m.tok_emb, m.segm_emb, m.texture_emb]     # m: its own pos_emb and start_tok
        close = [m.ln_f] + [blk.ln1 for li, blk in enumerate(m.blocks) if li % bucket_layers == 0]
        self.space = sp = ParamSpace(order, self.device, bucket_bytes=math.inf, close_after=close)
        self.flat_p = sp.flat_p
        self.heads = sp.joint([h.weight for h in m.head_list], C)                       # (W, dW) [18*1024, C]
        self.qkv = [sp.joint([b.attn.query.weight, b.attn.key.weight, b.attn.value.weight], C) +
                    sp.joint([b.attn.query.bias, b.attn.key.bias, b.attn.value.bias]) for b in m.blocks]  # W dW b db
        self.sync_from_rank0()

    @property
    def step_count(self):
        return self.space.step_count

    def sync_from_rank0(self):
        """Replicas must start (and resume) from identical parameters and optimiser state -- torch DDP broadcasts
        them at construction; call this again after loading a checkpoint on one rank.  The random draws
        (``q_sample`` masks, diffusion times) should differ per rank: pass each rank its own ``generator``."""
        self.space.sync_from_rank0()
        drop_packed_caches(self.m)

    def g(self, p):
        return self.space.g(p)

    def _weight_planes(self):
        return weight_planes(self.m, [qkv[0] for qkv in self.qkv], self.heads[0])

    # ------------------------------------------------------------------ diffusion bookkeeping (torch RNG)
    def q_sample(self, x_0, t, generator=None):
        """mask each token with probability t/T (transformer_model.py:212-230)"""
        r = torch.rand(x_0.shape, device=x_0.device, generator=generator)
        mask = r < (t.float().unsqueeze(-1) / self.num_timesteps)
        x_t = torch.where(mask, torch.full_like(x_0, self.mask_id), x_0)
        return x_t, mask

    # ------------------------------------------------------------------ loss + backward
    def loss_and_grads(self, x_0, target_own, segm, tex, t, generator=None, reduce=True, mask=None):
        """x_0 [B,T] continual tokens; target_own [B,T] each position's index inside its own texture
        codebook; segm, tex [B,T]; t [B] diffusion times.  Fills the flat gradient buffer (all-reduced over
        the data-parallel group when ``reduce``) and returns (loss, vb_loss) like the reference.  The
        gradients (``p.grad`` views) are left multiplied by ``self.loss_scale``; ``adam_step`` divides."""
        m = self.m
        B, T = x_0.shape
        sp = self.space
        sp.flat_g.zero_()
        sp.arm(reduce)
        # Static loss scale (a power of two, undone inside the Adam kernel): the gradient operands of the
        # backward GEMMs are fp16 hi/lo planes, whose absolute resolution is 2^-24; scaling the loss so that
        # |dlogits| <= 256 keeps every gradient tensor well inside fp16's normal range.  The bound on the
        # per-row loss weight is known on the host, so no device->host sync is needed to choose it.
        w_bound = (1.0 if self.loss_type == "reweighted_elbo" else float(self.num_timesteps)) / (math.log(2) * T * B)
        S = self.loss_scale = 2.0 ** math.floor(math.log2(256.0 / w_bound))

        if mask is None:
            x_t, mask = self.q_sample(x_0, t, generator)
        else:
            x_t = torch.where(mask, torch.full_like(x_0, self.mask_id), x_0)
        wp, w_heads = self._weight_planes()
        logits, saved, x_last, hf = forward_saved(m, x_t, segm, tex, wp, w_heads, [qkv[2] for qkv in self.qkv])

        # ---- re-weighted ELBO over the masked positions' own heads (transformer_model.py:250-270)
        tgt = torch.where(mask, target_own, torch.full_like(target_own, -1)).reshape(-1).contiguous()
        tf = t.float()
        if self.loss_type == "reweighted_elbo":
            wb = (1.0 - tf / self.num_timesteps) / (math.log(2) * T)
        elif self.loss_type == "elbo":
            wb = self.num_timesteps / tf / (math.log(2) * T)
        else:
            raise NotImplementedError(self.loss_type)
        w_rows = (wb * (S / B)).repeat_interleave(T).contiguous()
        ce_rows, dlogits = ops.ce_heads(logits, tgt, tex.reshape(-1).contiguous(), w_rows)
        ce_b = ce_rows.view(B, T).sum(1)
        loss = (wb * ce_b).mean()
        vb_loss = (ce_b * self.num_timesteps / tf / (math.log(2) * T)).mean()

        # ---- heads, final LayerNorm, blocks, embeddings
        dl = ops.f32_to_planes_rows(dlogits)                              # [Tt, M, NK]
        del logits, dlogits
        backward_from_planes(m, dl, saved, x_last, hf, wp, w_heads, x_t, segm, tex, sp)
        sp.wait()
        return loss, vb_loss

    # ------------------------------------------------------------------ optimiser
    def adam_step(self):
        """torch.optim.Adam(lr, weight_decay=0) on the flat buffers; gradients averaged over ranks"""
        self.space.adam(self.lr, self.betas, self.eps, 1.0 / (world_size() * self.loss_scale))
        drop_packed_caches(self.m)

    def optimize_parameters(self, x_0, target_own, segm, tex, generator=None):
        """one reference training step: sample t ~ U{1..T}, loss, backward, all-reduce, Adam"""
        B = x_0.shape[0]
        t = torch.randint(1, self.num_timesteps + 1, (B,), device=x_0.device, generator=generator)
        loss, vb = self.loss_and_grads(x_0, target_own, segm, tex, t, generator)
        self.adam_step()
        return loss, vb


# ---------------------------------------------------------------------- the drop-in autograd node
class NodeGrads:
    """Gradient provider of the autograd node: ONE fresh zeroed fp32 buffer per backward pass, every slot 32-byte
    aligned, q | k | v (weights, then biases) and the 18 heads each laid out back to back so that they are one matrix,
    as in ``SamplerTrainer``'s ``ParamSpace``.  The parameters themselves are not touched: a ParamSpace built over the
    module would re-point them into its own flat buffers, under an optimiser (or a SamplerTrainer) already holding
    them.  ``start_tok`` gets no slot: nothing reads it."""

    def __init__(self, m, device):
        groups = [tuple(h.weight for h in m.head_list)]
        for blk in m.blocks:
            a = blk.attn
            groups += [(a.query.weight, a.key.weight, a.value.weight), (a.query.bias, a.key.bias, a.value.bias)]
        seen = {id(p) for grp in groups for p in grp} | {id(m.start_tok)}
        groups += [(p,) for p in m.parameters() if id(p) not in seen]
        slots, total = [], 0
        for grp in groups:
            for p in grp:
                slots.append((p, total))
                total += (p.numel() + 7) // 8 * 8
        self.flat = torch.zeros(total, dtype=torch.float32, device=device)
        self.view = {id(p): self.flat[off:off + p.numel()].view_as(p) for p, off in slots}

    def g(self, p):
        return self.view.get(id(p))

    def joint(self, params, cols=None):
        first = self.view[id(params[0])]
        off, n = first.storage_offset(), 0
        for p in params:
            assert self.view[id(p)].storage_offset() == off + n, "the parameters are not adjacent in the buffer"
            n += p.numel()
        return None, self.flat[off:off + n].view((-1,) if cols is None else (-1, cols))

    def done(self, mod):
        """no gradient buckets: the gradients are handed to autograd"""


WP_KEYS = ("qkv", "proj", "fc1", "fc2")
DL_BOUND = 256.0   # largest |scaled logit gradient|: what the static loss scale of SamplerTrainer guarantees


def head_grad_scale(amax):
    """power of two s with s * amax <= DL_BOUND (1 when the gradient is zero or not finite)"""
    if not (0.0 < amax < math.inf):
        return 1.0
    return 2.0 ** min(100, max(-100, math.floor(math.log2(DL_BOUND / amax))))


class _SamplerNode(torch.autograd.Function):
    """TransformerMultiHead.forward as one autograd node: the forward of ``forward_saved`` returning the reference's
    18 [B, T, ncls] logit views, and a backward that turns the 18 logit gradients torch hands over into the planes
    operand (``ops.head_grads_to_planes``, scaled by a power of two chosen from their maximum) and runs
    ``backward_from_planes`` -- the native trainer's backward -- into a fresh ``NodeGrads``."""

    @staticmethod
    def forward(ctx, m, idx, segm, tex, *params):
        ctx.set_materialize_grads(False)      # a head the loss does not use arrives as None, read as zeros
        blocks = list(m.blocks)
        wqkv = [torch.cat([b.attn.query.weight, b.attn.key.weight, b.attn.value.weight]) for b in blocks]
        bqkv = [torch.cat([b.attn.query.bias, b.attn.key.bias, b.attn.value.bias]) for b in blocks]
        wp, w_heads = weight_planes(m, wqkv, torch.cat([h.weight for h in m.head_list]))
        del wqkv
        logits, saved, x_last, hf = forward_saved(m, idx, segm, tex, wp, w_heads, bqkv)
        # saved through autograd, so that they are released with the graph (and kept for a retain_graph replay)
        ctx.save_for_backward(idx, segm, tex, x_last, hf, w_heads, *[s[k] for s in saved for k in SAVED_KEYS],
                              *[w[k] for w in wp for k in WP_KEYS])
        ctx.m, ctx.params = m, params
        B, T = idx.shape
        lg = logits.view(B, T, m.num_head, m.head_class_num)
        return tuple(lg[:, :, i, :] for i in range(m.num_head))

    @staticmethod
    def backward(ctx, *dheads):
        m, params = ctx.m, ctx.params
        if all(d is None for d in dheads):
            return (None,) * (4 + len(params))
        idx, segm, tex, x_last, hf, w_heads, *rest = ctx.saved_tensors
        L, ns = len(m.blocks), len(SAVED_KEYS)
        saved = [dict(zip(SAVED_KEYS, rest[i * ns:(i + 1) * ns])) for i in range(L)]
        rest = rest[L * ns:]
        wp = [dict(zip(WP_KEYS, rest[i * len(WP_KEYS):(i + 1) * len(WP_KEYS)])) for i in range(L)]
        table, shape = ops.head_grads_table(dheads)
        s = head_grad_scale(float(ops.head_grads_absmax(table, shape)[0]))   # the one device->host read
        grads = NodeGrads(m, x_last.device)
        backward_from_planes(m, ops.head_grads_to_planes(table, shape, s), saved, x_last, hf, wp, w_heads, idx, segm,
                             tex, grads)
        if s != 1.0:
            grads.flat.mul_(1.0 / s)
        out = [grads.g(p) if ctx.needs_input_grad[4 + i] else None for i, p in enumerate(params)]
        return (None, None, None, None) + tuple(out)


def sampler_node(m, idx, segm, tex):
    """TransformerMultiHead.forward while training: the 18 logit tensors [B, T, ncls] of one autograd node"""
    pdrop = [m.drop.p] + [d.p for b in m.blocks for d in (b.attn.attn_drop, b.attn.resid_drop, b.mlp[3])]
    if any(p > 0 for p in pdrop):
        raise NotImplementedError("training the sampler with dropout > 0: no dropout kernel (every Text2Human "
                                  "config uses embd_pdrop = resid_pdrop = attn_pdrop = 0)")
    if m.causal:
        raise NotImplementedError("sampler='autoregressive' is never used by Text2Human")
    return list(_SamplerNode.apply(m, idx.contiguous(), segm.contiguous(), tex.contiguous(), *m.parameters()))
