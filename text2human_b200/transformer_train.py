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
        """fp16 planes [T,1,out,in] of every GEMM weight for this step (one conversion launch each).  The forward
        uses them K-major (y = x W^T); the data-gradient GEMMs read the SAME planes MN-major (dX = dY W)."""
        def planes(w):
            return ops.f32_to_planes_rows(w.detach()).unsqueeze(1)

        wp = []
        for blk, qkv in zip(self.m.blocks, self.qkv):
            wp.append(dict(qkv=planes(qkv[0]), proj=planes(blk.attn.proj.weight), fc1=planes(blk.mlp[0].weight),
                           fc2=planes(blk.mlp[2].weight)))
        return wp, planes(self.heads[0])

    # ------------------------------------------------------------------ diffusion bookkeeping (torch RNG)
    def q_sample(self, x_0, t, generator=None):
        """mask each token with probability t/T (transformer_model.py:212-230)"""
        r = torch.rand(x_0.shape, device=x_0.device, generator=generator)
        mask = r < (t.float().unsqueeze(-1) / self.num_timesteps)
        x_t = torch.where(mask, torch.full_like(x_0, self.mask_id), x_0)
        return x_t, mask

    # ------------------------------------------------------------------ forward with saved activations
    def _forward(self, idx, segm, tex, wp, w_heads):
        m = self.m
        B, T = idx.shape
        C = m.n_embd
        nh = m.blocks[0].attn.n_head
        x = ops.embed_sum(idx, segm, tex, m.tok_emb.weight.detach(), m.pos_emb.detach()[0],
                          m.segm_emb.weight.detach(), m.texture_emb.weight.detach())
        saved = []
        for blk, w, (_, _, bqkv, _) in zip(m.blocks, wp, self.qkv):
            a = blk.attn
            s = {"x_in": x}
            h1 = ops.layer_norm(x, blk.ln1.weight.detach(), blk.ln1.bias.detach(), blk.ln1.eps)
            qkv = ops.linear(h1, w["qkv"], bqkv, planes_out=True)                      # [Tt, M, 3C]: q | k | v
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

    # ------------------------------------------------------------------ loss + backward
    def loss_and_grads(self, x_0, target_own, segm, tex, t, generator=None, reduce=True, mask=None):
        """x_0 [B,T] continual tokens; target_own [B,T] each position's index inside its own texture
        codebook; segm, tex [B,T]; t [B] diffusion times.  Fills the flat gradient buffer (all-reduced over
        the data-parallel group when ``reduce``) and returns (loss, vb_loss) like the reference.  The
        gradients (``p.grad`` views) are left multiplied by ``self.loss_scale``; ``adam_step`` divides."""
        m = self.m
        B, T = x_0.shape
        C = m.n_embd
        M = B * T
        nh = m.blocks[0].attn.n_head
        scale = 1.0 / math.sqrt(C // nh)
        sp = self.space
        sp.flat_g.zero_()
        sp.arm(reduce)
        # Static loss scale (a power of two, undone inside the Adam kernel): the gradient operands of the
        # backward GEMMs are fp16 hi/lo planes, whose absolute resolution is 2^-24; scaling the loss so that
        # |dlogits| <= 256 keeps every gradient tensor well inside fp16's normal range.  The bound on the
        # per-row loss weight is known on the host, so no device->host sync is needed to choose it.
        w_bound = (1.0 if self.loss_type == "reweighted_elbo" else float(self.num_timesteps)) / (math.log(2) * T * B)
        S = self.loss_scale = 2.0 ** math.floor(math.log2(256.0 / w_bound))
        DS = 256.0  # extra scale of the (much smaller) score gradients, undone by the consuming GEMMs' alpha

        if mask is None:
            x_t, mask = self.q_sample(x_0, t, generator)
        else:
            x_t = torch.where(mask, torch.full_like(x_0, self.mask_id), x_0)
        wp, w_heads = self._weight_planes()
        logits, saved, x_last, hf = self._forward(x_t, segm, tex, wp, w_heads)

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

        # ---- heads + final LayerNorm
        NK = m.num_head * m.head_class_num
        dl = ops.f32_to_planes_rows(dlogits)                              # [Tt, M, NK]
        self._wgrad(dl, hf, self.heads[1])                               # dW_heads [NK, C] = dlogits^T hf
        d_hf = ops.linear(dl, w_heads, w_kn=True)                        # [M, C] = dlogits W_heads
        del dlogits, dl
        dx = torch.zeros((M, C), dtype=torch.float32, device=x_0.device)  # running gradient of the stream
        # every LayerNorm backward also emits what the next stage needs from the dx it just wrote: its fp16
        # planes and its column sums (the bias gradient of the linear layer that produced that activation)
        dxo = ops.layernorm_bwd_(dx, d_hf, x_last, m.ln_f.weight.detach(), self.g(m.ln_f.weight), self.g(m.ln_f.bias),
                                 m.ln_f.eps, accumulate=False, want_planes=True,
                                 colsum_out=self.g(m.blocks[-1].mlp[2].bias))
        sp.done(m.ln_f)

        # ---- blocks, last to first; dx is updated in place
        for li in range(len(m.blocks) - 1, -1, -1):
            blk, s, w = m.blocks[li], saved[li], wp[li]
            a = blk.attn
            fc1, fc2 = blk.mlp[0], blk.mlp[2]
            q, k, v = s["qkv"][:, :, :C], s["qkv"][:, :, C:2 * C], s["qkv"][:, :, 2 * C:]
            # MLP: x_out = x_mid + fc2(gelu(fc1(ln2(x_mid))))
            self._wgrad(dxo, s["g"], self.g(fc2.weight))                              # dW2 [C,F] = dxo^T g
            d_g = ops.linear(dxo, w["fc2"], w_kn=True)                                # [M,F]  = dxo W2
            d_a, da = ops.gelu_bwd(s["pre"], d_g, want_planes=True)                   # fp32 (bias grad) + planes
            ops.colsum_(self.g(fc1.bias), d_a)
            self._wgrad(da, s["h2"], self.g(fc1.weight))                              # dW1 [F,C]
            d_h2 = ops.linear(da, w["fc1"], w_kn=True)                                # [M,C]
            dxm = ops.layernorm_bwd_(dx, d_h2, s["x_mid"], blk.ln2.weight.detach(), self.g(blk.ln2.weight),
                                     self.g(blk.ln2.bias), blk.ln2.eps, accumulate=True, want_planes=True,
                                     colsum_out=self.g(a.proj.bias))                  # dx = d x_mid
            # attention output projection: x_mid = x_in + proj(y)
            self._wgrad(dxm, s["y"], self.g(a.proj.weight))                           # dWp [C,C]
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
            _, gwqkv, _, gbqkv = self.qkv[li]
            ops.colsum_(gbqkv, d_qkv)
            self._wgrad(dqkv, s["h1"], gwqkv)
            d_h1 = ops.linear(dqkv, w["qkv"], w_kn=True)                              # [M,C]
            dxo = ops.layernorm_bwd_(dx, d_h1, s["x_in"], blk.ln1.weight.detach(), self.g(blk.ln1.weight),
                                     self.g(blk.ln1.bias), blk.ln1.eps, accumulate=True, want_planes=li > 0,
                                     colsum_out=self.g(m.blocks[li - 1].mlp[2].bias) if li > 0 else None)
            # dx = d x_in = the gradient of the previous layer's output
            saved[li] = None
            sp.done(blk.ln1)

        # ---- embeddings
        ops.embed_bwd_(self.g(m.tok_emb.weight), dx, x_t.reshape(-1).contiguous())
        ops.embed_bwd_(self.g(m.pos_emb).view(-1, C), dx, None, T)
        ops.embed_bwd_(self.g(m.segm_emb.weight), dx, segm.reshape(-1).contiguous())
        ops.embed_bwd_(self.g(m.texture_emb.weight), dx, tex.reshape(-1).contiguous())
        sp.done(m.texture_emb)
        sp.wait()
        return loss, vb_loss

    @staticmethod
    def _wgrad(dy, x, out):
        """out[n_out, n_in] = dy^T x over all tokens; dy [T,M,n_out], x [T,M,n_in] token-major planes, read
        MN-major.  The output has few tiles and the contraction is long, so k-slices are spread over the SMs
        and reduce-added into the (zeroed) gradient buffer."""
        ks = ops.wgrad_k_split(dy.shape[2], x.shape[2], dy.shape[1]) if ops.SPLIT_K["wgrad"] else 0
        ops.wgrad(dy, x, out, k_split=ks)

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
