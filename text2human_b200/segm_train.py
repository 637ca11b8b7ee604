"""Training step of the parsing tokenizer (``VQSegmentationModel``, models/vqgan_model.py:86-96, :169-192; trained by
train_parsing_token.py with configs/parsing_token.yml) on the H100 kernels.

The net is the top VQGAN's Encoder / Decoder at ``ch=64`` with a 24-channel one-hot input, 24 logit outputs and one
``VectorQuantizer`` codebook; the loss is ``BCELossWithQuant`` (models/losses/segmentation_loss.py:12-25):
BCE-with-logits against the one-hot input plus the codebook loss; the optimiser is one Adam with betas (0.5, 0.9).
There is no discriminator.  ``SegmTokenizerTrainer.optimize_parameters`` is the native equivalent of the
reference's ``training_step`` + ``loss.backward()`` + ``optimizer.step()``:

  * input: the integer parsing map goes to one-hot fp16 planes in one launch (``onehot_to_planes``), the operand of
    ``conv_in`` -- the reference's F.one_hot (int64) / permute / .float() never exist;
  * forward / backward: the layers of ``vqgan_train`` (wgmma convs, data and weight gradients, GroupNorm and
    attention backward) and ``vq_search`` / ``vq_bwd`` for the quantizer;
  * loss: ``bce_logits`` reads the decoder's NHWC logits and the ids once and writes the output gradient as the
    fp16 planes conv_out's gradients read, plus conv_out's bias gradient (DESIGN §4.4);
  * parameters, gradients and Adam moments in one flat buffer; gradient buckets are all-reduced over the default
    process group while the backward pass runs, as in ``VQGANTrainer``.

The drop-in path for the same step (the reference's own ``optimize_parameters`` on the arch mirrors) goes through
the autograd nodes of ``vqgan_autograd``.
"""
import contextlib
import io
import math

import torch
import torch.distributed as dist
import torch.nn as nn

from . import conv_grad as G
from . import ops
from . import vqgan_train as VT
from .vqgan_arch import Decoder, Encoder, VectorQuantizer


class SegmTokenizerModel(nn.Module):
    """encoder / decoder / quantize / quant_conv / post_quant_conv built as VQModel.__init__ does
    (vqgan_model.py:19-50; ``opt`` holds the keys of configs/parsing_token.yml).  Its submodules' state_dicts are the
    reference checkpoint's entries."""

    def __init__(self, opt):
        super().__init__()
        with contextlib.redirect_stdout(io.StringIO()):
            self.encoder = Encoder(ch=opt['ch'], num_res_blocks=opt['num_res_blocks'],
                                   attn_resolutions=opt['attn_resolutions'], ch_mult=opt['ch_mult'],
                                   in_channels=opt['in_channels'], resolution=opt['resolution'],
                                   z_channels=opt['z_channels'], double_z=opt['double_z'], dropout=opt['dropout'])
            self.decoder = Decoder(in_channels=opt['in_channels'], resolution=opt['resolution'],
                                   z_channels=opt['z_channels'], ch=opt['ch'], out_ch=opt['out_ch'],
                                   num_res_blocks=opt['num_res_blocks'], attn_resolutions=opt['attn_resolutions'],
                                   ch_mult=opt['ch_mult'], dropout=opt['dropout'], resamp_with_conv=True,
                                   give_pre_end=False)
        self.quantize = VectorQuantizer(opt['n_embed'], opt['embed_dim'], beta=0.25)
        self.quant_conv = nn.Conv2d(opt['z_channels'], opt['embed_dim'], 1)
        self.post_quant_conv = nn.Conv2d(opt['embed_dim'], opt['z_channels'], 1)


class ConvInPlanesL(VT.ConvInImageL):
    """network-entry conv on fp16 planes that already exist (the one-hot parsing map): no data gradient"""

    def fwd(self, a):
        _, N, H, W, _ = a.shape
        cp = self.cp(self.conv)
        assert a.shape[-1] == cp.ci_p, (a.shape, cp.ci_p)
        y, st = G.forward("k3", a, cp.wn, cp.b, n=N, in_hw=(H, W), want_stats=True)
        self.saved.append((a, N))
        return VT.Act(y, st)


NETS = ("encoder", "decoder", "quantize", "quant_conv", "post_quant_conv")


class SegmTokenizerTrainer:
    """Owns a model with ``encoder``, ``decoder``, ``quantize`` (VectorQuantizer), ``quant_conv``,
    ``post_quant_conv`` (e.g. ``SegmTokenizerModel``); ``optimize_parameters(data)`` is one reference training step
    on ``data['segm']``, the parsing map of MaskDataset (class ids [B,H,W] or [B,1,H,W]).  ``lr`` may be changed
    between steps (the reference's step decay runs on the host)."""

    def __init__(self, model, lr=4.5e-5, betas=(0.5, 0.9), eps=1e-8, bucket_bytes=48 << 20):
        self.model = model
        self.lr, self.betas, self.eps = lr, betas, eps
        q = model.quantize
        self.beta, self.legacy = q.beta, q.legacy
        self.n_classes = model.decoder.conv_out.out_channels
        assert model.encoder.conv_in.in_channels == self.n_classes and not model.decoder.give_pre_end
        self.device = next(model.parameters()).device
        enc, dec = model.encoder, model.decoder
        self.enc_in = ConvInPlanesL(self, enc.conv_in)
        _, self.enc_body, self.enc_out = VT.encoder_layers(self, enc)
        self.dec_in, self.dec_body, _ = VT.decoder_layers(self, dec)
        self.dec_out = VT.NormConvOutL(self, dec.norm_out, dec.conv_out, nchw=False)     # logits NHWC
        self.qconv, self.pqconv = VT.Lin1x1L(self, model.quant_conv), VT.Lin1x1L(self, model.post_quant_conv)
        self.space = VT.ParamSpace(VT.backward_order(model), self.device, bucket_bytes)
        w = q.embedding.weight
        n_e, D = w.shape
        off = self.space.g(w).storage_offset()
        self.codebook = self.space.flat_p[off:off + n_e * D].view(1, n_e, D)
        self.g_codebook = self.space.flat_g[off:off + n_e * D].view(1, n_e, D)
        self._handles = []
        self._reduce = False
        self._out = None
        self.space.sync_from_rank0()

    # ---- plumbing used by the layers
    def space_of(self, mod):
        return self.space

    def space_of_param(self, p):
        return self.space

    def done(self, mod):
        """all gradients of ``mod`` are final: if it closes a bucket, start that bucket's all-reduce (asynchronously)
        while the backward pass continues"""
        if not self._reduce:
            return
        b = self.space.bucket_last.get(mod)
        if b is not None:
            a, e = self.space.buckets[b]
            self._handles.append(dist.all_reduce(self.space.flat_g[a:e], op=dist.ReduceOp.SUM, async_op=True))

    def wait_reduced(self):
        for h in self._handles:
            h.wait()
        self._handles = []

    @staticmethod
    def _world():
        return dist.get_world_size() if dist.is_initialized() else 1

    # ---- one step
    def training_step(self, data):
        """forward, loss and backward on this rank's batch; gradients are left in the flat buffer, multiplied by
        ``loss_scale`` and summed over ranks"""
        segm = data['segm'] if isinstance(data, dict) else data
        segm = segm.to(self.device).float()
        if segm.dim() == 3:
            segm = segm.unsqueeze(1)
        segm = segm.contiguous()
        B, _, H, W = segm.shape
        C = self.n_classes
        nel = B * C * H * W
        # static loss scale (a power of two, undone inside Adam): d bce / d logit ~ 1/nel is below fp16 resolution
        S = self.loss_scale = 2.0 ** math.floor(math.log2(nel))
        sp, dev = self.space, self.device
        sp.flat_g.zero_()
        self._handles = []
        sp.prepare(ops.get_terms())
        h = self.enc_out.fwd(self.enc_body.fwd(self.enc_in.fwd(ops.onehot_to_planes(segm, C))))
        z = self.qconv.fwd(h)
        del h
        r = ops.vq_search(z, self.codebook, None, want_list=False, want_nchw=False)
        q, stq = self.pqconv.fwd(r["zq_nhwc"], want_stats=True)
        logits = self.dec_out.fwd(self.dec_body.fwd(self.dec_in.fwd(VT.Act(q, stq))))
        del q
        bce = torch.zeros(1, dtype=torch.float64, device=dev)
        cs = torch.zeros(C, dtype=torch.float32, device=dev)
        dlp = ops.bce_logits(logits, segm, bce, gscale=S / nel, colsum_out=cs)
        del logits
        self._reduce = self._world() > 1
        g = self.dec_in.bwd(self.dec_body.bwd(self.dec_out.bwd(VT.Grad(None, dlp, cs))))
        g = self.pqconv.bwd(g)
        # codebook loss (legacy beta placement, vqgan_arch.py:98-103): coef_z on (z - e), coef_e on (e - z)
        w_z, w_e = (1.0, self.beta) if self.legacy else (self.beta, 1.0)
        zn = z.numel()
        dz = ops.vq_bwd(z, self.codebook, r["idx"], None, g.g, self.g_codebook, 2.0 * w_z * S / zn,
                        2.0 * w_e * S / zn)
        self.done(self.model.quantize.embedding)
        g = self.qconv.bwd(VT.Grad(dz))
        self.enc_in.bwd(self.enc_body.bwd(self.enc_out.bwd(g.g)))
        if self._reduce:
            assert len(self._handles) == len(sp.buckets), (len(self._handles), len(sp.buckets))
        self._reduce = False
        sp.release()
        self._out = dict(bce=bce, sqerr=r["sqerr"], nel=nel, z_numel=zn, idx=r["idx"])
        return self._out

    def losses(self):
        """the reference's log_dict scalars (split 'train', segmentation_loss.py:21-25); one device->host read"""
        o = self._out
        bce = float(o["bce"][0]) / o["nel"]
        quant = (1.0 + self.beta) * float(o["sqerr"][0]) / o["z_numel"]
        return dict(total_loss=bce + quant, bce_loss=bce, quant_loss=quant)

    def adam_step(self):
        self.wait_reduced()
        self.space.adam(self.lr, self.betas, self.eps, 1.0 / (self._world() * self.loss_scale))
        for mod in self.model.modules():       # packed-weight caches of the mirrors' inference path
            mod.__dict__.pop("_t2h_cache", None)

    def optimize_parameters(self, data):
        self.training_step(data)
        self.adam_step()

    # ---- checkpoint / resume: the reference layout (what load_pretrained_segm_token reads, sample_model.py:154-166)
    # plus the optimiser state
    def save(self, path):
        m = self.model
        net = {k: {kk: vv.detach().clone().contiguous() for kk, vv in getattr(m, k).state_dict().items()}
               for k in NETS}
        torch.save(dict(net, optimizer=self.space.state()), path)

    def load(self, path):
        ck = torch.load(path, map_location=self.device)
        for k in NETS:
            getattr(self.model, k).load_state_dict(ck[k], strict=True)
        if "optimizer" in ck:
            self.space.load_state(ck["optimizer"])
        for mod in self.model.modules():
            mod.__dict__.pop("_t2h_cache", None)
        self.space.sync_from_rank0()
