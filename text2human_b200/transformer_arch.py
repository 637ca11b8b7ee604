"""H100-native mirror of the reference's ``models/archs/transformer_arch.py``.

Same class names, constructor/forward signatures and ``state_dict`` keys as the
reference (SURVEY.md §8b).  torch ``nn.Linear`` / ``nn.LayerNorm`` /
``nn.Embedding`` objects are parameter containers only; the arithmetic runs in
libt2h: embedding-sum, LayerNorm, wgmma GEMMs (fused q|k|v projection, per-head
q k^T and att v without head or v transposes, MLP with fused
GELU, one N=18*1024 GEMM for the 18 heads), row softmax.  While training (the
reference's ``TransformerTextureAwareModel.optimize_parameters``) ``TransformerMultiHead.forward`` is one
autograd node whose backward is ``transformer_train``'s hand-written one.

The sampler is always non-causal on the Text2Human path (sampler='absorbing',
transformer_arch.py:200,30), so no mask and no KV cache exist.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .vqgan_arch import _cached, _f32, _lin_w


def _linear_residual(a, lin, x_res):
    """x_res + lin(a).  With ``ops.set_split_k(inference=True)`` and few output tiles (small batch) the
    contraction is split over the SMs and the k-slices are reduce-added into the residual stream in place
    (faster, but the fp32 summation order then varies run to run); otherwise a fresh tensor is written."""
    M, K = a.shape[1], a.shape[2]
    ks = ops.wgrad_k_split(M, lin.out_features, K) if ops.SPLIT_K["inference"] else 0
    if ks >= 2:
        return ops.linear(a, _lin_w(lin), _f32(lin.bias), out=x_res, k_split=ks)
    return ops.linear(a, _lin_w(lin), _f32(lin.bias), residual=x_res)


class CausalSelfAttention(nn.Module):
    """multi-head self-attention (reference :9-71; runs non-causal)."""

    def __init__(self, bert_n_emb, bert_n_head, attn_pdrop, resid_pdrop, latent_shape, sampler):
        super().__init__()
        assert bert_n_emb % bert_n_head == 0
        self.key = nn.Linear(bert_n_emb, bert_n_emb)
        self.query = nn.Linear(bert_n_emb, bert_n_emb)
        self.value = nn.Linear(bert_n_emb, bert_n_emb)
        self.attn_drop = nn.Dropout(attn_pdrop)
        self.resid_drop = nn.Dropout(resid_pdrop)
        self.proj = nn.Linear(bert_n_emb, bert_n_emb)
        self.n_head = bert_n_head
        self.causal = True if sampler == 'autoregressive' else False
        if self.causal:
            block_size = np.prod(latent_shape)
            mask = torch.tril(torch.ones(block_size, block_size))
            self.register_buffer("mask", mask.view(1, 1, block_size, block_size))

    def _qkv_packed(self):
        """q | k | v projections as ONE [3C, C] weight (and bias): one GEMM instead of three"""
        t = ops.get_terms()
        ws = (self.query.weight, self.key.weight, self.value.weight)
        bs = (self.query.bias, self.key.bias, self.value.bias)
        w = _cached(self, ("wqkv", t), ws, lambda: ops.pack_linear_weight(torch.cat(ws, 0), t))
        b = _cached(self, ("bqkv",), bs, lambda: torch.cat(bs, 0).float().contiguous())
        return w, b

    def attend(self, hn, x_res, B, T):
        """hn: LayerNorm'ed planes [Tt, B*T, C]; x_res: fp32 [B*T, C] residual stream.
        Returns x_res + proj(attention(hn)) as fp32 [B*T, C]; at small batch, with
        ``ops.set_split_k(inference=True)``, the projection is accumulated INTO ``x_res``."""
        if self.causal:
            raise NotImplementedError("sampler='autoregressive' is never used by Text2Human")
        Tt, M, Cc = hn.shape
        nh = self.n_head
        wqkv, bqkv = self._qkv_packed()
        qkv = ops.linear(hn, wqkv, bqkv, planes_out=True)  # [Tt, M, 3C]  (q | k | v), heads side by side
        if ops.can_fuse_attn(T, Cc // nh):
            return _linear_residual(ops.attn_fused(qkv, B, T, nh, 1.0 / math.sqrt(Cc // nh)), self.proj, x_res)
        s = ops.mha_scores(qkv[:, :, :Cc], B, T, nh, k=qkv[:, :, Cc:2 * Cc])  # fp32 [B, nh, T, T]
        p = ops.softmax_rows(s, scale=1.0 / math.sqrt(Cc // nh))  # planes [Tt, B, nh, T, T]
        # v stays token-major inside qkv: the tensor core reads it as an MN-major operand (no v^T copy)
        y = ops.mha_pv(p, qkv[:, :, 2 * Cc:], B, T, nh, v_tok=True)  # planes [Tt, M, C]
        return _linear_residual(y, self.proj, x_res)

    @torch.no_grad()
    def forward(self, x, layer_past=None):
        assert layer_past is None, "layer_past is only used by the (unused) autoregressive sampler"
        B, T, Cc = x.shape
        x2 = x.reshape(B * T, Cc).float().contiguous()
        hn = ops.split_planes(x2, ops.get_terms())
        zero = torch.zeros_like(x2)
        y = self.attend(hn, zero, B, T).view(B, T, Cc)
        # `present` (stacked k, v) is built by the reference and discarded by Block (:51, :97-99)
        return y, None


class Block(nn.Module):
    """pre-LN attention + pre-LN MLP (reference :74-99)."""

    def __init__(self, bert_n_emb, resid_pdrop, bert_n_head, attn_pdrop, latent_shape, sampler):
        super().__init__()
        self.ln1 = nn.LayerNorm(bert_n_emb)
        self.ln2 = nn.LayerNorm(bert_n_emb)
        self.attn = CausalSelfAttention(bert_n_emb, bert_n_head, attn_pdrop, resid_pdrop, latent_shape,
                                        sampler)
        self.mlp = nn.Sequential(
            nn.Linear(bert_n_emb, 4 * bert_n_emb),
            nn.GELU(),
            nn.Linear(4 * bert_n_emb, bert_n_emb),
            nn.Dropout(resid_pdrop),
        )

    def forward_rows_split(self, x, h, B, T, ks, next_ln, ln_out=None, row_map=None):
        """Small-batch form of the block (few [128 x 256] output tiles): the two N=C projections (proj, fc2) are
        split over the contraction so that >= 128 SMs work on them; the k-slices are stored separately and one
        kernel sums them in a FIXED order (bit-reproducible), adds bias + residual and applies the NEXT LayerNorm.
        x: fp32 residual stream [M, C]; h: LayerNorm1(x) planes.  -> (x_out fp32, planes of next_ln(x_out))"""
        a = self.attn
        Tt, M, Cc = h.shape
        wqkv, bqkv = a._qkv_packed()
        qkv = ops.linear(h, wqkv, bqkv, planes_out=True)
        if ops.can_fuse_attn(T, Cc // a.n_head):
            y = ops.attn_fused(qkv, B, T, a.n_head, 1.0 / math.sqrt(Cc // a.n_head))
        else:
            s = ops.mha_scores(qkv[:, :, :Cc], B, T, a.n_head, k=qkv[:, :, Cc:2 * Cc])
            p = ops.softmax_rows(s, scale=1.0 / math.sqrt(Cc // a.n_head))
            y = ops.mha_pv(p, qkv[:, :, 2 * Cc:], B, T, a.n_head, v_tok=True)
        part = ops.linear_partials(y, _lin_w(a.proj), ks)
        x, h2 = ops.splitk_reduce_ln(part, _f32(a.proj.bias), x, _f32(self.ln2.weight), _f32(self.ln2.bias), self.ln2.eps)
        m = ops.linear(h2, _lin_w(self.mlp[0]), _f32(self.mlp[0].bias), planes_out=True, act=ops.ACT_GELU)
        part = ops.linear_partials(m, _lin_w(self.mlp[2]), ks)
        return ops.splitk_reduce_ln(part, _f32(self.mlp[2].bias), x, _f32(next_ln.weight), _f32(next_ln.bias),
                                    next_ln.eps, ln_out=ln_out, row_map=row_map)

    def forward_rows(self, x, B, T):
        """x: fp32 [B*T, C] residual stream -> fp32 [B*T, C]"""
        h = ops.layer_norm(x, _f32(self.ln1.weight), _f32(self.ln1.bias), self.ln1.eps)
        x = self.attn.attend(h, x, B, T)
        h = ops.layer_norm(x, _f32(self.ln2.weight), _f32(self.ln2.bias), self.ln2.eps)
        m = ops.linear(h, _lin_w(self.mlp[0]), _f32(self.mlp[0].bias), planes_out=True, act=ops.ACT_GELU)
        return _linear_residual(m, self.mlp[2], x)

    @torch.no_grad()
    def forward(self, x, layer_past=None, return_present=False):
        assert layer_past is None
        B, T, Cc = x.shape
        y = self.forward_rows(x.reshape(B * T, Cc).float().clone(), B, T).view(B, T, Cc)  # updated in place
        if return_present:
            return y, None
        return y


class TransformerMultiHead(nn.Module):
    """the index-prediction transformer with 18 per-texture heads (reference :184-273)."""

    def __init__(self, codebook_size, segm_codebook_size, texture_codebook_size, bert_n_emb, bert_n_layers,
                 bert_n_head, block_size, latent_shape, embd_pdrop, resid_pdrop, attn_pdrop, num_head,
                 sampler='absorbing'):
        super().__init__()
        self.vocab_size = codebook_size + 1
        self.n_embd = bert_n_emb
        self.block_size = block_size
        self.n_layers = bert_n_layers
        self.codebook_size = codebook_size
        self.segm_codebook_size = segm_codebook_size
        self.texture_codebook_size = texture_codebook_size
        self.causal = sampler == 'autoregressive'
        if self.causal:
            self.vocab_size = codebook_size

        self.tok_emb = nn.Embedding(self.vocab_size, self.n_embd)
        self.pos_emb = nn.Parameter(torch.zeros(1, self.block_size, self.n_embd))
        self.segm_emb = nn.Embedding(self.segm_codebook_size, self.n_embd)
        self.texture_emb = nn.Embedding(self.texture_codebook_size, self.n_embd)
        self.start_tok = nn.Parameter(torch.zeros(1, 1, self.n_embd))
        self.drop = nn.Dropout(embd_pdrop)

        self.blocks = nn.Sequential(*[
            Block(bert_n_emb, resid_pdrop, bert_n_head, attn_pdrop, latent_shape, sampler)
            for _ in range(self.n_layers)
        ])
        self.num_head = num_head
        self.head_class_num = codebook_size // self.num_head
        self.ln_f = nn.LayerNorm(self.n_embd)
        self.head_list = nn.ModuleList(
            [nn.Linear(self.n_embd, self.head_class_num, bias=False) for _ in range(self.num_head)])

    def get_block_size(self):
        return self.block_size

    def _init_weights(self, module):
        # defined but never applied by the reference either (:240, no self.apply)
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def _heads_packed(self):
        t = ops.get_terms()
        ws = tuple(h.weight for h in self.head_list)
        return _cached(self, ("heads", t), ws,
                       lambda: ops.pack_linear_weight(torch.cat([w.detach() for w in ws], 0), t))

    @torch.no_grad()
    def forward_logits(self, idx, segm_tokens, texture_tokens):
        """-> fp32 [B, T, num_head, head_class_num]: all heads from one GEMM"""
        if self.causal:
            raise NotImplementedError("sampler='autoregressive' is never used by Text2Human")
        B, T = idx.shape
        assert T <= self.block_size, "Cannot forward, model block size is exhausted."
        x = ops.embed_sum(idx, segm_tokens, texture_tokens, _f32(self.tok_emb.weight),
                          _f32(self.pos_emb)[0], _f32(self.segm_emb.weight), _f32(self.texture_emb.weight))
        h = self._trunk(x, B, T)
        logits = ops.linear(h, self._heads_packed())  # [B*T, num_head*head_class_num]
        return logits.view(B, T, self.num_head, self.head_class_num)

    def _trunk(self, x, B, T, ln_out=None, row_map=None):
        """24 blocks + final LayerNorm of the fp32 stream x [B*T, C] -> planes of ln_f(x) (scattered by ``row_map``
        into ``ln_out`` for the grouped-head GEMM).  At small batch the deterministic split-K form of the blocks
        is used (each block's closing kernel already applies the next LayerNorm)."""
        M, Cc = x.shape
        ks = ops.wgrad_k_split(M, Cc, Cc) if ops.SPLIT_K["small_batch"] else 0
        if ks >= 2 and len(self.blocks) > 0:
            b0 = self.blocks[0]
            h = ops.layer_norm(x, _f32(b0.ln1.weight), _f32(b0.ln1.bias), b0.ln1.eps)
            for i, block in enumerate(self.blocks):
                last = i == len(self.blocks) - 1
                nxt = self.ln_f if last else self.blocks[i + 1].ln1
                x, h = block.forward_rows_split(x, h, B, T, ks, nxt, ln_out=ln_out if last else None,
                                                row_map=row_map if last else None)
            return h
        for block in self.blocks:
            x = block.forward_rows(x, B, T)
        if ln_out is not None:
            return ops.layer_norm_scatter(x, _f32(self.ln_f.weight), _f32(self.ln_f.bias), ln_out, row_map,
                                          self.ln_f.eps)
        return ops.layer_norm(x, _f32(self.ln_f.weight), _f32(self.ln_f.bias), self.ln_f.eps)

    @staticmethod
    def group_by_texture(texture_tokens, num_head):
        """texture ids [B,T] -> (dest int64 [B*T], rows_per_head): position m's row in a [num_head, rows_per_head]
        grouping by its texture id (ids outside 0..num_head-1 are clamped), each group padded to a multiple of
        128 rows.  Constant over a sampling run (the texture mask does not change), so it is computed once;
        ``rows_per_head`` costs one device->host read."""
        flat = texture_tokens.reshape(-1).clamp(0, num_head - 1)
        counts = torch.bincount(flat, minlength=num_head)
        need = max(128, int(counts.max().item()))
        rows = 128
        while rows < need:      # powers of two: a handful of distinct sizes (and captured graphs) for any mask
            rows *= 2
        order = torch.argsort(flat, stable=True)
        start = torch.cumsum(counts, 0) - counts
        rank = torch.arange(flat.numel(), device=flat.device) - start[flat[order]]
        dest = torch.empty_like(flat)
        dest[order] = flat[order] * rows + rank
        return dest, rows

    @torch.no_grad()
    def forward_own_logits(self, idx, segm_tokens, texture_tokens, dest, hf_grouped):
        """-> fp32 [B*T, head_class_num]: each position's logits in its OWN texture head only (all the sampler
        ever reads, sample_model.py:300-306).  The final LayerNorm scatters the positions into ``hf_grouped``
        (planes [T, num_head*rows_per_head, C], zero-initialised by the caller) by ``dest`` from
        ``group_by_texture``; one batched GEMM then multiplies each group by its own head: 1/18th .. 1x of the
        all-heads GEMM's work depending on how evenly the textures are spread.  Bit-identical to
        ``forward_logits`` gathered at the own head."""
        if self.causal:
            raise NotImplementedError("sampler='autoregressive' is never used by Text2Human")
        B, T = idx.shape
        x = ops.embed_sum(idx, segm_tokens, texture_tokens, _f32(self.tok_emb.weight),
                          _f32(self.pos_emb)[0], _f32(self.segm_emb.weight), _f32(self.texture_emb.weight))
        self._trunk(x, B, T, ln_out=hf_grouped, row_map=dest)
        Tt, rows_all, Cc = hf_grouped.shape
        rows = rows_all // self.num_head
        w = self._heads_packed().view(Tt, self.num_head, self.head_class_num, Cc)
        out = ops.bmm_nt(hf_grouped.view(Tt, self.num_head, rows, Cc), w)       # [num_head, rows, ncls]
        return out.view(rows_all, self.head_class_num).index_select(0, dest)

    def forward(self, idx, segm_tokens, texture_tokens, t=None):
        """``t`` is ignored, as in the reference.  In training mode, with autograd recording and a parameter that
        requires grad (the reference's optimize_parameters), the call is ONE autograd node whose backward is the
        native trainer's (``transformer_train.sampler_node``); otherwise the inference path below."""
        from .vqgan_autograd import recording
        if recording(self):
            from .transformer_train import sampler_node
            return sampler_node(self, idx, segm_tokens, texture_tokens)
        logits = self.forward_logits(idx, segm_tokens, texture_tokens)
        # reference returns a list of num_head tensors [B, T, head_class_num] (:271-273)
        return [logits[:, :, i, :] for i in range(self.num_head)]
