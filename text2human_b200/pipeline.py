"""Wrapper-level sequences of the Text2Human hot path on the H100 kernels.

Mirrors the inference methods of the reference's model wrappers (same method
names and ``opt`` keys), chaining the arch modules through their NHWC entry
points so no layout round trip happens between encoder, quantizer and decoder:

  VQImageSegmTextureModel.encode/decode/forward_step   models/vqgan_model.py:532-551
  HierarchyVQSpatialTextureAwareModel.top_encode/bot_encode/decode/forward_step
                                                       models/hierarchy_vqgan_model.py:215-239
  BaseSampleModel.sample_fn                            models/sample_model.py:256-328
  SampleFromParsingModel / SampleFromPoseModel         models/sample_model.py:215-254, :343-436

Training-only members of the reference wrappers (losses, optimisers, LPIPS,
discriminator, logging) are outside this round's scope.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .index_pred_arch import MultiHeadFCNHead, UNet, bot_index_prediction
from .parsing_gen_arch import FCNHead, ShapeAttrEmbedding, ShapeUNet, generate_parsing_map
from .transformer_arch import TransformerMultiHead
from .vqgan_arch import (Decoder, DecoderRes, Encoder, VectorQuantizer, VectorQuantizerSpatialTextureAware,
                         VectorQuantizerTexture, conv1x1_nhwc)


class VQImageSegmTextureModel(nn.Module):
    """top-level VQGAN: Encoder -> 1x1 -> VectorQuantizerTexture -> 1x1 -> Decoder
    (constructor keys as configs/vqvae_top.yml; reference vqgan_model.py:389-422)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.encoder = Encoder(ch=opt['ch'], num_res_blocks=opt['num_res_blocks'],
                               attn_resolutions=opt['attn_resolutions'], ch_mult=opt['ch_mult'],
                               in_channels=opt['in_channels'], resolution=opt['resolution'],
                               z_channels=opt['z_channels'], double_z=opt['double_z'],
                               dropout=opt['dropout'])
        self.decoder = Decoder(in_channels=opt['in_channels'], resolution=opt['resolution'],
                               z_channels=opt['z_channels'], ch=opt['ch'], out_ch=opt['out_ch'],
                               num_res_blocks=opt['num_res_blocks'],
                               attn_resolutions=opt['attn_resolutions'], ch_mult=opt['ch_mult'],
                               dropout=opt['dropout'], resamp_with_conv=True, give_pre_end=False)
        self.quantize = VectorQuantizerTexture(opt['n_embed'], opt['embed_dim'], beta=0.25)
        self.quant_conv = torch.nn.Conv2d(opt["z_channels"], opt['embed_dim'], 1)
        self.post_quant_conv = torch.nn.Conv2d(opt['embed_dim'], opt["z_channels"], 1)

    @torch.no_grad()
    def encode_nhwc(self, x, mask):
        h = self.encoder.forward_nhwc(x)
        h = conv1x1_nhwc(h, self.quant_conv)
        return self.quantize.forward_nhwc(h, mask), h

    @torch.no_grad()
    def encode(self, x, mask):
        r, _ = self.encode_nhwc(x, mask)
        quant = ops.nhwc_to_nchw(r["zq_nhwc"])
        return quant, r["loss"], (None, r["idx_cont"], list(r["idx_list"].unbind(0)))

    @torch.no_grad()
    def decode(self, quant):
        return self.decoder.forward_nhwc(conv1x1_nhwc(ops.nchw_to_nhwc(quant), self.post_quant_conv))

    @torch.no_grad()
    def forward_step(self, input, mask, return_info=False, streams=1):
        """``streams`` > 1: the batch is cut into that many slices (images are independent on this path) that run
        concurrently on their own CUDA streams, so one slice's HBM-bound kernels (GroupNorm apply, plane
        conversions) and small late-level launches overlap the other slice's tensor-bound convolutions."""
        if streams > 1 and input.shape[0] >= streams and not return_info:
            return self._forward_step_streams(input, mask, streams)
        with ops.stats_arena(input.shape[0], input.device):   # one fill for all fused GroupNorm statistics of the step
            r, z = self.encode_nhwc(input, mask)
            dec = self.decoder.forward_nhwc(conv1x1_nhwc(r["zq_nhwc"], self.post_quant_conv))
        if return_info:
            return dec, r["loss"], dict(idx_cont=r["idx_cont"], idx_list=r["idx_list"], z_nhwc=z,
                                        zq_nhwc=r["zq_nhwc"])
        return dec, r["loss"]

    def _forward_step_streams(self, input, mask, streams):
        B = input.shape[0]
        main = torch.cuda.current_stream()
        sig = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self.__dict__.get("_t2h_streams_sig") != sig:
            # the packed-weight caches are (re)built on first use: do that once on the current stream, so the
            # concurrent slices below only read them
            self.forward_step(input[:1], mask[:1])
            self.__dict__["_t2h_streams_sig"] = sig
        pool = self.__dict__.setdefault("_t2h_streams", [])
        while len(pool) < streams:
            pool.append(torch.cuda.Stream())
        cuts = [(B * i) // streams for i in range(streams + 1)]
        decs, sq = [], []
        for i in range(streams):
            st = pool[i]
            st.wait_stream(main)
            with torch.cuda.stream(st):
                xs, ms = input[cuts[i]:cuts[i + 1]], mask[cuts[i]:cuts[i + 1]]
                r, _ = self.encode_nhwc(xs, ms)
                d = self.decoder.forward_nhwc(conv1x1_nhwc(r["zq_nhwc"], self.post_quant_conv))
                decs.append(d)
                sq.append((r["sqerr"], r["zq_nhwc"].numel()))
        for i in range(streams):
            main.wait_stream(pool[i])
            decs[i].record_stream(main)
            sq[i][0].record_stream(main)
        dec = torch.cat(decs, 0)
        from .vqgan_arch import _loss_from_sqerr
        tot = sq[0][0].clone()
        for s_, _ in sq[1:]:
            tot += s_
        return dec, _loss_from_sqerr(tot, sum(n for _, n in sq), self.quantize.beta)


class HierarchyVQSpatialTextureAwareModel(nn.Module):
    """two-level VQGAN (constructor keys as configs/vqvae_bottom.yml;
    reference hierarchy_vqgan_model.py:24-85)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.top_encoder = Encoder(ch=opt['top_ch'], num_res_blocks=opt['top_num_res_blocks'],
                                   attn_resolutions=opt['top_attn_resolutions'], ch_mult=opt['top_ch_mult'],
                                   in_channels=opt['top_in_channels'], resolution=opt['top_resolution'],
                                   z_channels=opt['top_z_channels'], double_z=opt['top_double_z'],
                                   dropout=opt['top_dropout'])
        self.decoder = Decoder(in_channels=opt['top_in_channels'], resolution=opt['top_resolution'],
                               z_channels=opt['top_z_channels'], ch=opt['top_ch'], out_ch=opt['top_out_ch'],
                               num_res_blocks=opt['top_num_res_blocks'],
                               attn_resolutions=opt['top_attn_resolutions'], ch_mult=opt['top_ch_mult'],
                               dropout=opt['top_dropout'], resamp_with_conv=True, give_pre_end=False)
        self.top_quantize = VectorQuantizerTexture(1024, opt['embed_dim'], beta=0.25)
        self.top_quant_conv = torch.nn.Conv2d(opt["top_z_channels"], opt['embed_dim'], 1)
        self.top_post_quant_conv = torch.nn.Conv2d(opt['embed_dim'], opt["top_z_channels"], 1)

        self.bot_encoder = Encoder(ch=opt['bot_ch'], num_res_blocks=opt['bot_num_res_blocks'],
                                   attn_resolutions=opt['bot_attn_resolutions'], ch_mult=opt['bot_ch_mult'],
                                   in_channels=opt['bot_in_channels'], resolution=opt['bot_resolution'],
                                   z_channels=opt['bot_z_channels'], double_z=opt['bot_double_z'],
                                   dropout=opt['bot_dropout'])
        self.bot_decoder_res = DecoderRes(in_channels=opt['bot_in_channels'],
                                          resolution=opt['bot_resolution'],
                                          z_channels=opt['bot_z_channels'], ch=opt['bot_ch'],
                                          num_res_blocks=opt['bot_num_res_blocks'],
                                          ch_mult=opt['bot_ch_mult'], dropout=opt['bot_dropout'],
                                          give_pre_end=False)
        self.bot_quantize = VectorQuantizerSpatialTextureAware(
            opt['bot_n_embed'], opt['embed_dim'], beta=0.25, spatial_size=opt['codebook_spatial_size'])
        self.bot_quant_conv = torch.nn.Conv2d(opt["bot_z_channels"], opt['embed_dim'], 1)
        self.bot_post_quant_conv = torch.nn.Conv2d(opt['embed_dim'], opt["bot_z_channels"], 1)

    @torch.no_grad()
    def top_encode_nhwc(self, x, mask):
        h = conv1x1_nhwc(self.top_encoder.forward_nhwc(x), self.top_quant_conv)
        r = self.top_quantize.forward_nhwc(h, mask)
        return conv1x1_nhwc(r["zq_nhwc"], self.top_post_quant_conv), r

    @torch.no_grad()
    def bot_encode_nhwc(self, x, mask):
        h = conv1x1_nhwc(self.bot_encoder.forward_nhwc(x), self.bot_quant_conv)
        r = self.bot_quantize.forward_nhwc(h, mask)
        quant = conv1x1_nhwc(r["zq_nhwc"], self.bot_post_quant_conv)
        return self.bot_decoder_res.forward_nhwc(quant), r

    @torch.no_grad()
    def top_encode(self, x, mask):
        return ops.nhwc_to_nchw(self.top_encode_nhwc(x, mask)[0])

    @torch.no_grad()
    def bot_encode(self, x, mask):
        res, r = self.bot_encode_nhwc(x, mask)
        return ops.nhwc_to_nchw(res), r["loss"], (None, r["idx_cont"].reshape(-1), list(r["idx_list"].unbind(0)))

    @torch.no_grad()
    def decode(self, quant_top, bot_dec_res):
        return self.decoder(quant_top, bot_h=bot_dec_res)

    @torch.no_grad()
    def forward_step(self, input, mask, return_info=False):
        quant_top, rt = self.top_encode_nhwc(input, mask)
        bot_dec_res, rb = self.bot_encode_nhwc(input, mask)
        dec = self.decoder.forward_nhwc(quant_top, bot_h=bot_dec_res)
        if return_info:
            return dec, rb["loss"], dict(top_idx=rt["idx_cont"], bot_idx=rb["idx_cont"])
        return dec, rb["loss"]

    @torch.no_grad()
    def decode_from_indices(self, top_list, bot_list, mask):
        """tokens -> image (the decode half of sample_and_refine, sample_model.py:225-243, batched)"""
        B = mask.shape[0]
        zt = self.top_quantize.get_codebook_entry(top_list, mask, (B, 32, 16, self.opt["top_z_channels"]),
                                                  nhwc=True)
        quant_top = conv1x1_nhwc(zt, self.top_post_quant_conv)
        zb = self.bot_quantize.get_codebook_entry(bot_list, mask, (B, 32, 16, self.opt["bot_z_channels"]),
                                                  nhwc=True)
        res = self.bot_decoder_res.forward_nhwc(conv1x1_nhwc(zb, self.bot_post_quant_conv))
        return self.decoder.forward_nhwc(quant_top, bot_h=res)


class SegmTokenizer(nn.Module):
    """parsing map -> 32x16 segmentation tokens: one-hot -> segm Encoder -> 1x1 -> VectorQuantizer
    (BaseSampleModel.get_quantized_segm, sample_model.py:330-340; constructor keys as the segm_* entries of
    configs/sample_from_parsing.yml)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.segm_encoder = Encoder(ch=opt['segm_ch'], num_res_blocks=opt['segm_num_res_blocks'],
                                    attn_resolutions=opt['segm_attn_resolutions'], ch_mult=opt['segm_ch_mult'],
                                    in_channels=opt['segm_in_channels'], resolution=opt['segm_resolution'],
                                    z_channels=opt['segm_z_channels'], double_z=opt['segm_double_z'],
                                    dropout=opt['segm_dropout'])
        self.segm_quantizer = VectorQuantizer(opt['segm_n_embed'], opt['segm_embed_dim'], beta=0.25,
                                              sane_index_shape=True)
        self.segm_quant_conv = torch.nn.Conv2d(opt["segm_z_channels"], opt['segm_embed_dim'], 1)

    @torch.no_grad()
    def get_quantized_segm(self, segm):
        """segm: [B,1,H,W] class ids -> int64 tokens [B,h,w]"""
        a = ops.onehot_to_planes(segm, self.opt['segm_num_segm_classes'])
        z = conv1x1_nhwc(self.segm_encoder.forward_planes(a), self.segm_quant_conv)
        return self.segm_quantizer.forward_nhwc(z)["idx"]


class GraphedStep:
    """Capture a fixed-shape, allocation-stable sequence of libt2h launches into a CUDA graph and replay
    it (CUDA streams + graphs instead of a tracing compiler).  ``fn(*static_inputs) -> tensor | tuple``.
    Inputs are copied into static buffers before each replay; outputs are static buffers (clone them
    if they must outlive the next replay)."""

    def __init__(self, fn, example_inputs, warmup=2):
        self.static_in = [t.clone() for t in example_inputs]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):  # first calls configure kernels (cudaFuncSetAttribute) and caches
                fn(*self.static_in)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        before = ops.COUNTERS["launches"]
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = fn(*self.static_in)
        self.launches = ops.COUNTERS["launches"] - before  # libt2h kernels per replay

    def __call__(self, *inputs):
        for dst, src in zip(self.static_in, inputs):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        ops.COUNTERS["launches"] += self.launches
        return self.static_out


class Sampler(nn.Module):
    """The absorbing-diffusion sampling loop of BaseSampleModel (sample_model.py:256-328) around
    TransformerMultiHead, without the reference's per-codebook host synchronisations.

    RNG: torch's generator supplies ONE ``torch.rand`` of all reveal uniforms [steps, B, T] before the loop (the
    reference draws one [B, T] per step from the same kind of stream) and one integer seed; inside the loop the
    categorical draws come from ``t2h_sample_step`` (Gumbel-max over each position's OWN texture head with
    Philox4x32-10 keyed by (seed, step, position, class)) -- the reference draws every head for every position with
    18 ``Categorical.sample()`` calls and keeps one.  The law of every token is the same
    (softmax(logits/temp) of the own head); the loop body has no ATen launches."""

    MAX_GRAPHS = 4

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.sampler_fn = TransformerMultiHead(
            codebook_size=opt['codebook_size'], segm_codebook_size=opt['segm_codebook_size'],
            texture_codebook_size=opt['texture_codebook_size'], bert_n_emb=opt['bert_n_emb'],
            bert_n_layers=opt['bert_n_layers'], bert_n_head=opt['bert_n_head'], block_size=opt['block_size'],
            latent_shape=opt['latent_shape'], embd_pdrop=opt['embd_pdrop'], resid_pdrop=opt['resid_pdrop'],
            attn_pdrop=opt['attn_pdrop'], num_head=opt['num_head'])
        self.shape = tuple(opt['latent_shape'])
        self.mask_id = opt['codebook_size']
        self.sample_steps = opt['sample_steps']

    @property
    def _graphs(self):
        """captured graphs live ON the transformer module (next to its packed-weight cache) so that whoever
        invalidates the packed weights (``flat_params.drop_packed_caches``) drops them too"""
        return self.sampler_fn.__dict__.setdefault("_t2h_graphs", {})

    def _weights_signature(self):
        """a captured graph bakes in pointers to the packed fp16 weight planes: it is only valid for the exact
        parameter storage / version it was captured with"""
        return tuple((p.data_ptr(), p._version) for p in self.sampler_fn.parameters())

    def _own_logits_fn(self, B, T, device, use_graph, rows_per_head):
        """the transformer forward for fixed (B, T, rows_per_head), returning each position's own-head logits:
        ~220 small launches per step are CPU-launch-bound, so they are captured once into a CUDA graph and
        replayed every diffusion step.  -> (fn, hf, static inputs or None)"""
        m = self.sampler_fn
        Tt = ops.get_terms()
        key = (B, T, str(device), Tt, ops.SPLIT_K["inference"], rows_per_head, use_graph, self._weights_signature())
        graphs = self._graphs
        hit = graphs.get(key)
        if hit is None:
            while len(graphs) >= self.MAX_GRAPHS:   # bounded: each entry pins a private pool of all activations
                graphs.pop(next(iter(graphs)))
            # rows no position maps to stay zero for the lifetime of the buffer
            hf = torch.zeros((Tt, m.num_head * rows_per_head, m.n_embd), dtype=torch.float16, device=device)

            def fn(x_t, segm, tex, dest):
                return m.forward_own_logits(x_t, segm, tex, dest, hf)
            static = None
            if use_graph:
                ex = (torch.full((B, T), self.mask_id, dtype=torch.long, device=device),
                      torch.zeros((B, T), dtype=torch.long, device=device),
                      torch.zeros((B, T), dtype=torch.long, device=device),
                      torch.arange(B * T, dtype=torch.long, device=device))
                fn = GraphedStep(fn, ex)
                static = fn.static_in
            hit = (fn, hf, static)
            graphs[key] = hit
        else:
            graphs[key] = graphs.pop(key)           # most recently used last
        return hit

    @torch.no_grad()
    def sample_fn(self, segm_tokens, texture_mask, temp=1.0, sample_steps=None, generator=None, use_graph=True,
                  reveal_u=None, seed=None, trace=None):
        """segm_tokens int64 [B, T]; texture_mask float [B,1,H,W] of ids 0..17.
        Returns (list of 18 int64 [B,T] per-codebook index maps with -1 elsewhere, final x_t).
        ``reveal_u`` [steps, B, T] / ``seed``: the random inputs, drawn from ``generator`` when not given.
        ``trace``: a list that receives (x_t before the step, positions revealed in the step) per step."""
        m = self.sampler_fn
        B = segm_tokens.shape[0]
        T = int(np.prod(self.shape))
        dev = segm_tokens.device
        steps = sample_steps or self.sample_steps
        tex = ops.mask_to_ids(texture_mask, self.shape[0], self.shape[1]).view(B, T).long()
        nh = m.num_head
        tex_c = tex.clamp(0, nh - 1)
        valid_tex = (tex >= 0) & (tex < nh)
        if reveal_u is None:
            reveal_u = torch.rand((steps, B, T), device=dev, generator=generator)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,), device=dev, generator=generator).item())
        # positions grouped by texture once per run: every step's head GEMM then only computes each position's
        # own head (the reference computes all 18 heads for every position and keeps one)
        dest, rows_per_head = m.group_by_texture(tex_c, nh)
        logits_fn, hf, static = self._own_logits_fn(B, T, dev, use_graph, rows_per_head)
        hf.zero_()  # padding rows of a previous run's grouping must not leak in
        if static is not None:   # run the loop directly on the graph's input buffers: no per-step copies
            x_t, segm_s, tex_s, dest_s = static
            x_t.fill_(self.mask_id)
            segm_s.copy_(segm_tokens)
            tex_s.copy_(tex_c)
            dest_s.copy_(dest)
        else:
            x_t = torch.full((B, T), self.mask_id, dtype=torch.long, device=dev)
            segm_s, tex_s, dest_s = segm_tokens, tex_c, dest
        unmasked = torch.zeros((B * T,), dtype=torch.uint8, device=dev)
        tex_flat = tex.reshape(-1).contiguous()
        reveal_u = reveal_u.contiguous()
        for i, t in enumerate(range(steps, 0, -1)):
            own = logits_fn(x_t, segm_s, tex_s, dest_s)   # [B*T, ncls]: each position's own texture head
            if trace is not None:
                before, x_before = unmasked.clone(), x_t.clone()
            ops.sample_step(own, reveal_u[i].view(-1), tex_flat, x_t.view(-1), unmasked, t=t, temp=temp, seed=seed,
                            step=i, n_heads=nh)
            if trace is not None:
                trace.append((x_before, (unmasked != before).view(B, T)))
        x_t = x_t.clone()
        um = unmasked.view(B, T).bool()
        final = torch.where(um & valid_tex, x_t - 1024 * tex_c, torch.full_like(x_t, -1))
        out = [torch.where(tex == k, final, torch.full_like(final, -1)) for k in range(nh)]
        return out, x_t


class SampleFromParsingModel(nn.Module):
    """parsing map + texture mask -> image: the whole of ``BaseSampleModel.sample_and_refine``
    (sample_model.py:215-254) with the reference's component names and ``opt`` keys
    (configs/sample_from_parsing.yml): segm tokenizer -> diffusion sampler -> top codebook gather ->
    index-prediction UNet/FCN -> bottom codebook gather -> DecoderRes -> Decoder.  The reference decodes one
    sample at a time; here the whole batch goes through every stage at once."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.decoder = Decoder(in_channels=opt['top_in_channels'], resolution=opt['top_resolution'],
                               z_channels=opt['top_z_channels'], ch=opt['top_ch'], out_ch=opt['top_out_ch'],
                               num_res_blocks=opt['top_num_res_blocks'],
                               attn_resolutions=opt['top_attn_resolutions'], ch_mult=opt['top_ch_mult'],
                               dropout=opt['top_dropout'], resamp_with_conv=True, give_pre_end=False)
        self.top_quantize = VectorQuantizerTexture(1024, opt['embed_dim'], beta=0.25)
        self.top_post_quant_conv = torch.nn.Conv2d(opt['embed_dim'], opt["top_z_channels"], 1)
        self.bot_decoder_res = DecoderRes(in_channels=opt['bot_in_channels'], resolution=opt['bot_resolution'],
                                          z_channels=opt['bot_z_channels'], ch=opt['bot_ch'],
                                          num_res_blocks=opt['bot_num_res_blocks'], ch_mult=opt['bot_ch_mult'],
                                          dropout=opt['bot_dropout'], give_pre_end=False)
        self.bot_quantize = VectorQuantizerSpatialTextureAware(
            opt['bot_n_embed'], opt['embed_dim'], beta=0.25, spatial_size=opt['bot_codebook_spatial_size'])
        self.bot_post_quant_conv = torch.nn.Conv2d(opt['embed_dim'], opt["bot_z_channels"], 1)
        self.index_pred_guidance_encoder = UNet(in_channels=opt['index_pred_encoder_in_channels'])
        self.index_pred_decoder = MultiHeadFCNHead(
            in_channels=opt['index_pred_fc_in_channels'], in_index=opt['index_pred_fc_in_index'],
            channels=opt['index_pred_fc_channels'], num_convs=opt['index_pred_fc_num_convs'],
            concat_input=opt['index_pred_fc_concat_input'], dropout_ratio=opt['index_pred_fc_dropout_ratio'],
            num_classes=opt['index_pred_fc_num_classes'], align_corners=opt['index_pred_fc_align_corners'],
            num_head=18)
        self.segm = SegmTokenizer(opt)
        self.sampler = Sampler(opt)
        self.shape = tuple(opt['latent_shape'])

    @property
    def sampler_fn(self):
        return self.sampler.sampler_fn

    @torch.no_grad()
    def bot_index_prediction(self, feature_top, texture_mask):
        """feature_top fp32 NCHW [B,256,32,16] -> 18 int64 maps [B,32,16] (-1 outside each texture)"""
        return bot_index_prediction(self.index_pred_guidance_encoder, self.index_pred_decoder, feature_top,
                                    texture_mask, self.shape)

    @torch.no_grad()
    def decode_top_tokens(self, top_list, texture_mask):
        """sampled top tokens -> image in [0,1] (sample_model.py:225-246, batched)"""
        B = texture_mask.shape[0]
        h, w = self.shape
        zt = self.top_quantize.get_codebook_entry(top_list, texture_mask, (B, h, w, self.opt["top_z_channels"]),
                                                  nhwc=True)
        quant_top = conv1x1_nhwc(zt, self.top_post_quant_conv)
        own, _ = bot_index_prediction(self.index_pred_guidance_encoder, self.index_pred_decoder, quant_top,
                                      texture_mask, self.shape, as_list=False, nhwc_in=True)
        zb = self.bot_quantize.get_codebook_entry(own, texture_mask, (B, h, w, self.opt["bot_z_channels"]),
                                                  nhwc=True)
        res = self.bot_decoder_res.forward_nhwc(conv1x1_nhwc(zb, self.bot_post_quant_conv))
        dec = self.decoder.forward_nhwc(quant_top, bot_h=res)
        return dec.add_(1.0).mul_(0.5).clamp_(0, 1)

    @torch.no_grad()
    def sample_and_refine(self, segm, texture_mask, temp=1.0, sample_steps=None, generator=None, save_dir=None,
                          img_name=None):
        """segm [B,1,H,W] parsing ids, texture_mask [B,1,H,W] texture ids -> images [B,3,512,256] in [0,1].
        With ``save_dir`` and ``img_name`` (a list of B file names) the images are also written as the
        reference does (sample_model.py:249-253: one file per sample, save_image quantisation)."""
        B = segm.shape[0]
        segm_tokens = self.segm.get_quantized_segm(segm).view(B, -1)
        top_list, _ = self.sampler.sample_fn(segm_tokens, texture_mask, temp=temp, sample_steps=sample_steps,
                                             generator=generator)
        h, w = self.shape
        dec = self.decode_top_tokens([t.view(B, h, w) for t in top_list], texture_mask)
        if save_dir is not None and img_name is not None:
            save_images(dec, save_dir, img_name)
        return dec


class SampleFromPoseModel(SampleFromParsingModel):
    """pose + shape attributes + texture attributes -> image: ``SampleFromPoseModel.inference``
    (sample_model.py:363-436) with the reference's component names and ``opt`` keys (configs/sample_from_pose.yml):
    parsing generator (ShapeAttrEmbedding -> ShapeUNet -> FCNHead -> argmax) -> texture mask -> everything
    ``SampleFromParsingModel.sample_and_refine`` runs.  The whole batch goes through every stage at once."""

    def __init__(self, opt):
        super().__init__(opt)
        self.shape_attr_embedder = ShapeAttrEmbedding(dim=opt['shape_embedder_dim'],
                                                      out_dim=opt['shape_embedder_out_dim'],
                                                      cls_num_list=opt['shape_attr_class_num'])
        self.shape_parsing_encoder = ShapeUNet(in_channels=opt['shape_encoder_in_channels'],
                                               attr_embedding=opt['shape_embedder_out_dim'])
        self.shape_parsing_decoder = FCNHead(
            in_channels=opt['shape_fc_in_channels'], in_index=opt['shape_fc_in_index'],
            channels=opt['shape_fc_channels'], num_convs=opt['shape_fc_num_convs'],
            concat_input=opt['shape_fc_concat_input'], dropout_ratio=opt['shape_fc_dropout_ratio'],
            num_classes=opt['shape_fc_num_classes'], align_corners=opt['shape_fc_align_corners'])

    def load_shape_generation_models(self, path=None):
        """parsing_gen.pth: {'embedder', 'encoder', 'decoder'} state dicts, loaded strictly (sample_model.py:397-410)"""
        ck = torch.load(path or self.opt['pretrained_parsing_gen'], map_location="cpu")
        for name, key in (("shape_attr_embedder", "embedder"), ("shape_parsing_encoder", "encoder"),
                          ("shape_parsing_decoder", "decoder")):
            getattr(self, name).load_state_dict(ck[key], strict=True)
            getattr(self, name).eval()

    @torch.no_grad()
    def generate_parsing_map(self, pose, shape_attr):
        """pose fp32 [B,1,H,W], shape attributes int [B,15] -> float parsing map [B,1,H,W]"""
        return generate_parsing_map(self.shape_attr_embedder, self.shape_parsing_encoder, self.shape_parsing_decoder,
                                    pose, shape_attr)

    @torch.no_grad()
    def generate(self, pose, shape_attr, upper, lower, outer, temp=1.0, sample_steps=None, generator=None,
                 save_dir=None, img_name=None):
        """pose [B,1,H,W], shape attributes [B,15], fused texture attributes upper / lower / outer [B] (17 = none)
        -> images [B,3,H,W] in [0,1] (and the files, with ``save_dir`` / ``img_name``)"""
        dev = self.shape_attr_embedder.fusion[0].weight.device
        segm = self.generate_parsing_map(pose.to(dev), shape_attr.to(dev))
        attrs = torch.stack([torch.as_tensor(a, device=dev).view(-1) for a in (upper, lower, outer)], 1)
        texture_mask = ops.texture_mask(segm, attrs)
        return self.sample_and_refine(segm, texture_mask, temp=temp, sample_steps=sample_steps, generator=generator,
                                      save_dir=save_dir, img_name=img_name)

    @torch.no_grad()
    def inference(self, data_loader, save_dir, generator=None):
        """DeepFashionAttrPoseDataset batches ('densepose', 'shape_attr', '*_fused_attr', 'img_name') -> one image
        file per 'img_name' under save_dir (sample_model.py:425-436)"""
        for data in data_loader:
            self.generate(data['densepose'], data['shape_attr'], data['upper_fused_attr'], data['lower_fused_attr'],
                          data['outer_fused_attr'], sample_steps=self.opt.get('sample_steps'), generator=generator,
                          save_dir=save_dir, img_name=list(data['img_name']))


def save_images(images, save_dir, names):
    """images fp32 NCHW in [0,1] -> one image file per sample (what torchvision's save_image writes for a
    single image: uint8(x*255+0.5)); the packing runs on the GPU, the encoder (PIL) on the host"""
    import os
    from PIL import Image
    u8 = ops.pack_u8(images).cpu().numpy()                      # [B,H,W,C]
    os.makedirs(save_dir, exist_ok=True)
    for arr, name in zip(u8, names):
        Image.fromarray(arr if arr.shape[-1] != 1 else arr[..., 0]).save(os.path.join(save_dir, name))


class TransformerTextureAwareModel(nn.Module):
    """The sampler's training wrapper (reference models/transformer_model.py:18-303) with its component names
    and ``opt`` keys (configs/sampler.yml): frozen image tokenizer (top Encoder + VectorQuantizerTexture), frozen
    segm tokenizer, and the trainable ``_denoise_fn`` driven by ``SamplerTrainer``."""

    def __init__(self, opt):
        super().__init__()
        from .transformer_train import SamplerTrainer
        self.opt = opt
        self.img_encoder = Encoder(ch=opt['img_ch'], num_res_blocks=opt['img_num_res_blocks'],
                                   attn_resolutions=opt['img_attn_resolutions'], ch_mult=opt['img_ch_mult'],
                                   in_channels=opt['img_in_channels'], resolution=opt['img_resolution'],
                                   z_channels=opt['img_z_channels'], double_z=opt['img_double_z'],
                                   dropout=opt['img_dropout'])
        self.img_quantizer = VectorQuantizerTexture(opt['img_n_embed'], opt['img_embed_dim'], beta=0.25)
        self.img_quant_conv = torch.nn.Conv2d(opt["img_z_channels"], opt['img_embed_dim'], 1)
        self.segm = SegmTokenizer(opt)
        self._denoise_fn = TransformerMultiHead(
            codebook_size=opt['codebook_size'], segm_codebook_size=opt['segm_codebook_size'],
            texture_codebook_size=opt['texture_codebook_size'], bert_n_emb=opt['bert_n_emb'],
            bert_n_layers=opt['bert_n_layers'], bert_n_head=opt['bert_n_head'], block_size=opt['block_size'],
            latent_shape=opt['latent_shape'], embd_pdrop=opt['embd_pdrop'], resid_pdrop=opt['resid_pdrop'],
            attn_pdrop=opt['attn_pdrop'], num_head=opt['num_head'])
        self.shape = tuple(opt['latent_shape'])
        self.num_timesteps = 1000
        self._trainer_cls = SamplerTrainer
        self.trainer = None
        self.log_dict = {}

    @torch.no_grad()
    def get_quantized_img(self, image, texture_mask):
        """-> (continual tokens [B,T], own-codebook targets [B,T], texture ids [B,T]); the reference returns the
        targets as 18 lists with -1 fills (:154-170), of which each position uses exactly one"""
        B = image.shape[0]
        z = conv1x1_nhwc(self.img_encoder.forward_nhwc(image), self.img_quant_conv)   # NCHW in, NHWC out
        r = self.img_quantizer.forward_nhwc(z, texture_mask)
        return r["idx_cont"].view(B, -1), r["idx"].view(B, -1), r["ids"].view(B, -1).long()

    @torch.no_grad()
    def feed_data(self, data):
        """data: {'image' [B,3,H,W], 'segm' [B,1,H,W], 'texture_mask' [B,1,H,W]} (reference :273-288)"""
        dev = next(self._denoise_fn.parameters()).device
        image, segm, tm = data['image'].to(dev), data['segm'].to(dev), data['texture_mask'].to(dev)
        self.input_indices, self.gt_own, _ = self.get_quantized_img(image, tm)
        B = image.shape[0]
        self.texture_tokens = ops.mask_to_ids(tm, self.shape[0], self.shape[1]).view(B, -1).long()
        self.segm_tokens = self.segm.get_quantized_segm(segm).view(B, -1)

    def optimize_parameters(self, generator=None):
        if self.trainer is None:
            self.trainer = self._trainer_cls(self._denoise_fn, lr=self.opt.get('lr', 1e-4),
                                             num_timesteps=self.num_timesteps,
                                             loss_type=self.opt.get('loss_type', 'reweighted_elbo'))
        loss, vb = self.trainer.optimize_parameters(self.input_indices, self.gt_own, self.segm_tokens,
                                                    self.texture_tokens.clamp(0, 17), generator)
        self.log_dict['loss'], self.log_dict['vb_loss'] = loss, vb
        return loss, vb
