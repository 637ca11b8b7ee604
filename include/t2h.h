/*
 * t2h.h — C ABI of libt2h.so, the H100 (sm_90a) kernel library under the
 * Text2Human hot path (hierarchical VQGAN encode/quantize/decode + the
 * index-prediction transformer).
 *
 * The reference (yumingj/Text2Human) is pure Python/PyTorch and has no FFI of
 * its own (SURVEY.md §8b): its boundary is the nn.Module API of
 * models/archs/vqgan_arch.py and models/archs/transformer_arch.py.  This header
 * is the seam *beneath* the Python classes in text2human_b200/ that mirror
 * those modules; every entry point names the reference call(s) it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, a negative T2H_E* code otherwise;
 *     t2h_last_error() returns a thread-local human-readable message.
 *   - functions never allocate device memory, never synchronise and never
 *     throw; all device pointers are caller-owned; `stream` is a cudaStream_t.
 *   - "f16 planes" = an fp16 tensor stored as `terms` stacked planes
 *     [terms][...]: plane 0 holds hi = fp16(x), plane 1 (terms==2) holds
 *     lo = fp16(x - hi).  terms==1 is the TF32-like fast mode, terms==2 gives
 *     fp32-equivalent tensor-core products via the 3-product split
 *     (hi*hi + hi*lo + lo*hi) inside t2h_tapgemm.
 *   - activations are NHWC inside the library; NCHW only at module boundaries.
 */
#ifndef T2H_H_
#define T2H_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define T2H_VERSION 202

#define T2H_OK 0
#define T2H_EINVAL (-1)   /* bad argument / unsupported shape            */
#define T2H_ECUDA (-2)    /* CUDA runtime / driver error                  */
#define T2H_EARCH (-3)    /* device is not sm_90                          */

typedef void* t2h_stream_t; /* cudaStream_t */

int t2h_version(void);
const char* t2h_last_error(void);
/* compute capability and SM count of the current device */
int t2h_device_info(int* cc_major, int* cc_minor, int* num_sms);

/* ------------------------------------------------------------------------
 * t2h_tapgemm — wgmma/TMA implicit-GEMM.
 *
 *   D[n,h,w,:] = epilogue( sum_{tap} sum_{c} A[n, h+dy(tap), w+dx(tap), c] *
 *                                             B[tap, :, c] )
 *
 * One kernel serves every dense contraction on the path:
 *   3x3 conv s1 p1      torch.nn.Conv2d in ResnetBlock/conv_in/conv_out/Upsample
 *                       (vqgan_arch.py:573,579,526,840,885,954,997)
 *   3x3 conv s2 (0,1,0,1) pad   Downsample (vqgan_arch.py:544-551) — A is the
 *                       4-phase space-to-depth view, taps carry a phase offset
 *   1x1 conv / Linear   nin_shortcut :590, AttnBlock q/k/v/proj :627-634,
 *                       quant_conv/post_quant_conv (vqgan_model.py:418-422),
 *                       nn.Linear in transformer_arch.py:21-28,85-87,233
 *   batched bmm         AttnBlock torch.bmm :648,:655; q@k^T, att@v
 *                       (transformer_arch.py:58,65)
 *
 * A is an fp16-plane tensor addressed as (c, w, h, img) with element strides
 * (1, a_sw, a_sh, a_sn); out-of-range (h,w,c) reads are zero (TMA OOB fill),
 * which implements the conv zero padding.  B is an fp16-plane tensor addressed
 * as (k, n, g, g2) with strides (1, b_sn, b_sg, b_sg2); g = tap index (conv),
 * plane index and, for two-level batches, the h index; g2 = image index (bmm).
 * With tile_rows the (h, img) dims of A and D act as two batch dims of a plain
 * row-major GEMM (multi-head attention: h = batch, img = head).
 * Accumulation is fp32 in registers.
 * ---------------------------------------------------------------------- */
#define T2H_MAX_TAPS 16   /* 3x3 convs use 9; the Discriminator's 4x4 convs (vqgan_arch.py:1160-1197) 16 */

#define T2H_OUT_F32 0        /* fp32 output                                  */
#define T2H_OUT_PLANES 1     /* fp16 planes output (d_terms planes)          */

#define T2H_BIAS_NONE 0
#define T2H_BIAS_COL 1       /* bias[n_out]   (conv / Linear bias)            */
#define T2H_BIAS_ROW 2       /* bias[h*W + w] (transposed products, V^T)      */

#define T2H_ACT_NONE 0
#define T2H_ACT_GELU 1       /* exact erf GELU, nn.GELU() transformer_arch.py:86 */
#define T2H_ACT_RELU 2       /* ConvModule's ReLU in the index-prediction UNet / FCN head (unet_arch.py:160) */
#define T2H_ACT_LRELU 3      /* nn.LeakyReLU(0.2) of the Discriminator (vqgan_arch.py:1163,1180,1195) */

typedef struct t2h_tapgemm_params {
  /* ---- A operand (activations) ---- */
  const void* a;         /* fp16 planes                                      */
  int32_t a_terms;       /* 1 or 2 planes present                            */
  int32_t a_term_imgs;   /* img-index distance between plane 0 and plane 1   */
  int32_t a_imgs;        /* total img slots addressable in the map (all planes, phases) */
  int32_t a_bcast;       /* 1: A has a single image shared by all n (batch-broadcast) */
  int32_t n_img, H, W;   /* output domain: n_img images of HxW rows           */
  int32_t tile_rows;     /* 1: tiles are 128 consecutive w of one (h,img) (GEMM rows);
                            0: auto (rows when H==1, else 2-D spatial boxes)   */
  int32_t a_H, a_W;      /* extents of A's (h,w) dims (OOB beyond => 0)      */
  int32_t C;             /* contraction length per tap (valid channels)      */
  int64_t a_sw, a_sh, a_sn; /* element strides of A                          */
  /* ---- B operand (weights / second matrix) ---- */
  const void* b;         /* fp16 planes, (k, n, g)                           */
  int32_t b_terms;       /* 1 or 2                                           */
  int32_t b_term_g;      /* g-index distance between plane 0 and plane 1     */
  int32_t b_groups;      /* total g slots addressable (taps/planes/h-batches) */
  int32_t b_groups2;     /* extent of the second group dim g2 (>= 1)          */
  int32_t b_batched;     /* 1: g2 = image index n (bmm over images)           */
  int32_t b_batched_h;   /* 1: g += h (row-tile mode: h is a second batch dim) */
  int32_t n_out;         /* valid output columns (rows of B)                 */
  int64_t b_sn, b_sg, b_sg2; /* element strides of B                         */
  /* ---- taps ---- */
  int32_t ntaps;
  int32_t tap_dy[T2H_MAX_TAPS];
  int32_t tap_dx[T2H_MAX_TAPS];
  int32_t tap_img_off[T2H_MAX_TAPS]; /* added to A's img index (stride-2 phases) */
  /* ---- products ---- */
  int32_t nterms;        /* 1: hi*hi   3: hi*hi + hi*lo + lo*hi               */
  /* ---- epilogue ---- */
  void* d;               /* output                                           */
  int32_t d_mode;        /* T2H_OUT_*                                        */
  int32_t d_terms;       /* planes written when d_mode == PLANES             */
  int64_t d_plane;       /* element distance between output planes           */
  int64_t d_sn, d_sh, d_sw, d_sc; /* element strides of D (d_sc==1 => NHWC)   */
  const float* bias;     /* fp32, may be NULL                                */
  int32_t bias_mode;     /* T2H_BIAS_*                                       */
  int32_t act;           /* T2H_ACT_*                                        */
  float alpha;           /* acc *= alpha before bias                         */
  const float* residual; /* fp32, same addressing as D (f32 mode), or NULL   */
  double* gn_stats;      /* optional [n_img][32][2] (sum, sumsq) accumulators
                            of the fp32 output, for the following GroupNorm   */
  int32_t gn_cpg;        /* channels per group when gn_stats != NULL         */
  int32_t a_mn;          /* 1: A is stored contraction-major -- element (row w, k) at a + k*a_sw + w (rows
                            contiguous, a_sw = distance between consecutive k): A^T products without a
                            transposed copy (weight gradients dY^T.X, P^T.dY).  Row GEMMs with one tap only */
  int32_t b_mn;          /* 1: B is stored contraction-major -- element (n, k) at b + k*b_sn + n (output
                            columns contiguous): X.W with W as stored [k][n] (dgrad with the forward's
                            weight planes, att.V with V token-major)                                      */
  int64_t bias_sn;       /* BIAS_COL with n_img > 1: element distance between the bias vectors of consecutive
                            images (per-head biases of a batched GEMM); 0 = one shared vector          */
  int32_t k_split;       /* >= 2: D += alpha*A.B (+ column bias, once): the contraction of every output tile
                            is split over up to k_split CTAs whose partial sums are reduce-added (TMA .add)
                            into the existing contents of D -- a zeroed gradient buffer (weight gradients:
                            few output tiles, contraction over all tokens) or the residual stream itself
                            (x += proj(y) at small batch).  Needs a 16-byte-aligned fp32 D and no row bias /
                            act / residual / gn_stats.  0/1: off (D is overwritten)                     */
  int32_t use_tap_w;     /* 1: tap i reads weight slot tap_w[i] of B instead of slot i (the data gradient of a
                            strided conv uses a subset of the taps per output parity, in place)          */
  int32_t tap_w[T2H_MAX_TAPS];
  int32_t accumulate;    /* 1: D += result (TMA reduce-add) even without split-K -- gradient accumulation over
                            micro-batches; same requirements as k_split                                  */
  int32_t k_partials;    /* >= 2: deterministic split-K: the contraction of every output tile is split over up to
                            k_partials CTAs, slice s (s < ceil(kchunks / ceil(kchunks / k_partials)), kchunks =
                            ceil(C / 64)) STORES alpha*A.B to d + s*d_slab; t2h_splitk_reduce_ln sums the slabs in
                            a fixed order.  Single-image row GEMMs, no bias / act / residual                 */
  int64_t d_slab;        /* element distance between the k_partials slabs                                  */
  /* Norm-backward sums in the epilogue (swapped-operand kernel: spatial convs with n_out % 128 == 0 and a plain fp32
   * NHWC destination): for a data-gradient conv whose output D is the gradient w.r.t. act(norm(x)*gamma+beta), with
   * nb_sums != NULL `residual` holds x (fp32, D's geometry; it is NOT added) and the epilogue accumulates
   * nb_sums[(img*n_out + c)*2 + {0,1}] += sum over the pixels of {du, du*xhat}, du = D * act'(xhat*gamma+beta),
   * xhat from nb_stats (as t2h_gn_stats / the conv epilogue produced them) -- pass 1 of t2h_norm_bwd rides along.
   * nb_act: 0 none, 1 swish, 2 LeakyReLU(0.2); nb_groups: GroupNorm groups (n_out % nb_groups == 0). */
  double* nb_sums;
  const double* nb_stats;
  const float* nb_gamma;
  const float* nb_beta;
  float nb_eps;
  int32_t nb_act;
  int32_t nb_groups;
} t2h_tapgemm_params;

int t2h_tapgemm(const t2h_tapgemm_params* p, t2h_stream_t stream);
/* profiling aid: with T2H_DEBUG bit 16 set, CTA 0 of every tap-GEMM / fused-attention launch appends a record of 8
 * words to a device ring: globaltimer ns at {entry, dependency wait passed, first operands landed, last MMA issued,
 * accumulator complete, CTA done}, {work items, contraction chunks per item | kind << 32}.  out[0] = records so far,
 * out[1..] = the ring (synchronises the device). */
int t2h_debug_read(long long* out, int n);

/* ------------------------------------------------------------------------
 * Layout / precision conversion (HBM-bound)
 * ---------------------------------------------------------------------- */
/* fp32 NCHW [N,C,H,W] -> fp16 planes NHWC [terms][N][H][W][c_pad], zero
 * channel padding.  Entry of Encoder/Decoder.forward (vqgan_arch.py:899,1008). */
int t2h_nchw_to_planes(const float* x, void* out, int n, int c, int h, int w,
                       int c_pad, int terms, t2h_stream_t stream);
/* fp32 NHWC [N,H,W,C] -> fp32 NCHW.  Exit of the modules. */
int t2h_nhwc_to_nchw(const float* x, float* out, int n, int c, int h, int w,
                     t2h_stream_t stream);
/* Image write-out (sample_model.py:244-253 + torchvision.utils.save_image): fp32 NCHW x -> uint8 NHWC
 * out = uint8(clamp(clamp(x*scale + shift, 0, 1) * 255 + 0.5, 0, 255)); c <= 4 */
int t2h_pack_u8(const float* x, uint8_t* out, int n, int c, int h, int w, float scale, float shift,
                t2h_stream_t stream);
/* fp32 NCHW -> fp32 NHWC */
int t2h_nchw_to_nhwc(const float* x, float* out, int n, int c, int h, int w,
                     t2h_stream_t stream);

#define T2H_CVT_PLAIN 0
#define T2H_CVT_UP2X 1   /* nearest x2: F.interpolate in Upsample (vqgan_arch.py:530) */
#define T2H_CVT_S2D 2    /* 4-phase space-to-depth for Downsample (vqgan_arch.py:547-551):
                            out[(p*2+q)][n][oh][ow][c] = x[n][2*oh+p][2*ow+q][c]  */
#define T2H_CVT_MAXPOOL2 3   /* nn.MaxPool2d(2) between the index-prediction UNet's encoder stages (unet_arch.py:441) */
#define T2H_CVT_BILINEAR2X 4 /* nn.Upsample(x2, bilinear, align_corners=False) of InterpConv (unet_arch.py:303-304) */
/* fp32 NHWC [N,H,W,C] -> fp16 planes.  Output spatial size is (2H,2W) for UP2X / BILINEAR2X,
 * (H/2,W/2) x 4 phases for S2D, (H/2,W/2) for MAXPOOL2.  Plane layout: [terms][phases][N][h][w][C]. */
int t2h_f32_to_planes(const float* x, void* out, int n, int h, int w, int c,
                      int mode, int terms, t2h_stream_t stream);

/* ------------------------------------------------------------------------
 * GroupNorm(32, C, eps) (+ swish)  — Normalize()/nonlinearity(),
 * vqgan_arch.py:510-517, used at :599-600,:606-607,:638,:916-917,:1030-1031
 * ---------------------------------------------------------------------- */
/* stats[n][g] = (sum, sumsq) in fp64 over fp32 NHWC x.  stats must be zeroed
 * by the caller (or produced by t2h_tapgemm's gn_stats epilogue instead). */
int t2h_gn_stats(const float* x, double* stats, int n, int hw, int c, int groups,
                 t2h_stream_t stream);
/* y = act(gn(x)*gamma+beta) -> fp16 planes NHWC; swish: 0 none, 1 swish (nonlinearity(), :513-517), 2 LeakyReLU(0.2).
 * With n = 1, hw = N*H*W and groups = c the same two kernels are BatchNorm2d in training mode (batch statistics,
 * eps 1e-5) of the Discriminator (vqgan_arch.py:1178,1193). */
int t2h_gn_apply(const float* x, const double* stats, const float* gamma,
                 const float* beta, void* out, int n, int hw, int c, int groups,
                 float eps, int swish, int terms, t2h_stream_t stream);

/* x += y (fp32): `h += bot_h`, vqgan_arch.py:1024 */
int t2h_add_inplace(float* x, const float* y, int64_t numel, t2h_stream_t stream);

/* softmax over the last dim of fp32 [rows, cols] * scale -> fp16 planes
 * (F.softmax, vqgan_arch.py:649-650, transformer_arch.py:58-63) */
int t2h_softmax_rows(const float* s, void* out, int64_t rows, int cols, float scale,
                     int terms, t2h_stream_t stream);

/* Multi-head attention of the index-prediction transformer as one kernel: out = softmax(q k^T * scale) v per
 * (sequence, head) -- CausalSelfAttention.forward with causal=False, transformer_arch.py:41-67 (the k/q/v
 * .view().transpose(1, 2) head splits, `att = q @ k^T * (1/sqrt(hs))`, F.softmax, `att @ v`, the transpose back).
 * qkv: fp16 planes [terms][rows][ld] (hi [, lo]; `plane` elements apart) holding q, k, v of head h in columns
 * q_col / k_col / v_col + 64 h (e.g. the fused q|k|v projection); rows >= batch * tokens, sequence s = rows
 * s*tokens ..; out: fp16 planes [terms][rows][ld_out], heads side by side.  head_dim must be 64 and tokens a
 * multiple of 128 in 128..512 (one 128-query block per CTA) -- other shapes take
 * t2h_tapgemm (q k^T), t2h_softmax_rows, t2h_tapgemm (p v). */
int t2h_attn_fwd(const void* qkv, int terms, int64_t plane, int64_t ld, int64_t rows, int q_col, int k_col,
                 int v_col, int batch, int tokens, int heads, int head_dim, float scale, void* out,
                 int64_t out_plane, int64_t ld_out, t2h_stream_t stream);

/* ------------------------------------------------------------------------
 * Codebook quantizers (fp32 CUDA-core math, bit-reproducible; see
 * oracle/vq_oracle.c for the exact operation order)
 *   VectorQuantizer.forward                  vqgan_arch.py:79-122
 *   VectorQuantizerTexture.forward           vqgan_arch.py:212-287
 *   VectorQuantizerSpatialTextureAware.fwd   vqgan_arch.py:375-461
 *
 * z:        fp32 NHWC [B, Hz, Wz, Cz]
 * codebook: fp32 [n_books][n_e][D],  D = Cz * ps * ps  (ps = patch size 1|2);
 *           row element order is (c, kh, kw) as F.unfold produces (:324)
 * book_id:  int32 [B * Hz/ps * Wz/ps] codebook chosen per row (value outside
 *           [0,n_books) => row untouched: z_q row = 0, indices = -1), or NULL
 *           for the single-codebook quantizer
 * idx:      int64 [rows] argmin (lowest index wins ties), -1 when unselected
 * idx_cont: int64 [rows] idx + n_e_cont_stride*book (reference uses 1024*k for
 *           the top quantizer :262 and n_e*k for the bottom :436), may be NULL
 * idx_list: int64 [n_books][rows] per-codebook maps filled with -1 elsewhere
 *           (:238-242,:257-259), may be NULL
 * zq_nhwc:  fp32 NHWC quantized values (straight-through value z + (z_q - z),
 *           :281), may be NULL
 * zq_nchw:  fp32 NCHW of the same, may be NULL
 * sqerr:    double[1] += sum (z_q - z)^2 (for the codebook loss :273-278), may be NULL
 * ---------------------------------------------------------------------- */
int t2h_vq_search(const float* z, const float* codebook, const int32_t* book_id,
                  int b, int hz, int wz, int cz, int ps, int n_books, int n_e,
                  int64_t cont_stride, int64_t* idx, int64_t* idx_cont,
                  int64_t* idx_list, float* zq_nhwc, float* zq_nchw, double* sqerr,
                  void* workspace, int64_t workspace_bytes, t2h_stream_t stream);
/* bytes of workspace t2h_vq_search needs for `rows` rows */
int64_t t2h_vq_workspace_bytes(int64_t rows, int n_books, int n_e);

/* get_codebook_entry (vqgan_arch.py:124-139, :289-309, :463-486): gather rows
 * by index -> fp32 NHWC [B, Hz, Wz, Cz] (patch-folded when ps == 2).
 * idx: int64 [rows] per-row index inside its codebook (already resolved from
 * indices_list by the caller), book_id as above. */
int t2h_vq_gather(const float* codebook, const int64_t* idx, const int32_t* book_id,
                  int b, int hz, int wz, int cz, int ps, int n_books, int n_e,
                  float* zq_nhwc, float* zq_nchw, t2h_stream_t stream);

/* segmentation ids [B,1,H,W] (float) -> one-hot fp16 planes NHWC [terms][B][H][W][c_pad]: the input of the
 * segm tokeniser's Encoder; replaces F.one_hot(...).permute(0,3,1,2).float() (sample_model.py:331-335) */
int t2h_onehot_to_planes(const float* ids, void* out, int b, int h, int w, int n_classes, int c_pad, int terms,
                         t2h_stream_t stream);

/* Dataset-side preparation (data/segm_attr_dataset.py:120-164) on the device.
 * texture mask (:138-151): mask = attrs[b][g] + 1 where the parsing class segm value belongs to clothes group
 * g = cls_group[cls] (0 upper, 1 lower, 2 outer, -1 other) and attrs[b][g] != 17, else 0.  segm/mask float [b][per_img] */
int t2h_texture_mask(const float* segm, const int32_t* attrs, const int32_t* cls_group, int n_cls, float* mask, int b,
                     int64_t per_img, t2h_stream_t stream);
/* uint8 HWC images [b][h][w][c] -> fp16 planes NHWC [terms][b][h][w][c_pad] of x / divisor + shift (image / 127.5 - 1,
 * :154) -- the operand of Encoder.conv_in -- and optionally (nchw != NULL) the fp32 NCHW tensor the reference's
 * DataLoader yields */
int t2h_u8_to_planes(const uint8_t* x, void* out, float* nchw, int b, int h, int w, int c, int c_pad, float divisor,
                     float shift, int terms, t2h_stream_t stream);

/* nearest-neighbour resize of a float id map [B,1,Hs,Ws] to int32 [B,Ht,Wt]
 * (F.interpolate(mode='nearest'), vqgan_arch.py:222,:385-389) */
int t2h_mask_to_ids(const float* mask, int32_t* ids, int b, int hs, int ws, int ht,
                    int wt, t2h_stream_t stream);

/* ------------------------------------------------------------------------
 * Transformer pieces (transformer_arch.py)
 * ---------------------------------------------------------------------- */
/* bot_index_prediction's per-position argmax (sample_model.py:199-207): logits [n_heads][rows][ncls] fp32,
 * head[rows] = the texture id selecting the head; out[rows] = lowest index of the maximum in the row's own
 * head, -1 where head is outside 0..n_heads-1 */
int t2h_argmax_heads(const float* logits, const int64_t* head, int64_t* out, int64_t rows, int n_heads, int ncls,
                     t2h_stream_t stream);

/* x[b,t,:] = tok_emb[idx] + pos_emb[t] + segm_emb[segm] + tex_emb[tex]  (:251-266) fp32 */
int t2h_embed_sum(const int64_t* idx, const int64_t* segm, const int64_t* tex,
                  const float* tok_emb, const float* pos_emb, const float* segm_emb,
                  const float* tex_emb, float* x, int b, int t, int c,
                  t2h_stream_t stream);
/* LayerNorm over the last dim (eps 1e-5) of fp32 [rows, c] -> fp16 planes (:80-81,:231) */
int t2h_layernorm(const float* x, const float* gamma, const float* beta, void* out,
                  int64_t rows, int c, float eps, int terms, t2h_stream_t stream);
/* the same, row r written to row row_map[r] of a planes buffer of out_rows rows (the sampler's final LayerNorm
 * groups the positions by texture so that each position only meets its own head, transformer_arch.py:268-273) */
int t2h_layernorm_scatter(const float* x, const float* gamma, const float* beta, void* out, int64_t rows, int c,
                          float eps, int terms, const int64_t* row_map, int64_t out_rows, t2h_stream_t stream);

/* x_out[m,:] = residual[m,:] + bias + sum_{s<n_slabs} partials[s][m,:] (slabs summed in index order: bit-reproducible),
 * then optionally LayerNorm(x_out[m,:]) -> fp16 planes, row m written to row row_map[m] (or m) of a planes buffer of
 * ln_rows rows.  Completes a k_partials GEMM and fuses the residual add (x = x + proj(y), x = x + mlp(.),
 * transformer_arch.py:97-99) with the next LayerNorm (:80-81, :231).  residual may alias x_out. */
int t2h_splitk_reduce_ln(const float* partials, int n_slabs, int64_t slab, const float* bias, const float* residual,
                         float* x_out, const float* gamma, const float* beta, float eps, void* ln_out, int terms,
                         const int64_t* row_map, int64_t ln_rows, int64_t rows, int c, t2h_stream_t stream);

/* ------------------------------------------------------------------------
 * Training step of the index-prediction transformer
 * (TransformerTextureAwareModel._train_loss / optimize_parameters, models/transformer_model.py:232-303;
 *  loss.backward() + torch.optim.Adam.step()).  Dense gradients (dgrad / wgrad / attention) run on
 * t2h_tapgemm; these are the HBM-bound pieces around it.
 * ---------------------------------------------------------------------- */
/* fp32 [g][r][c] -> fp16 planes of scale*x, transposed out_t[terms][g][c][r] and / or untransposed out_n (either
 * may be NULL, not both): wgrad contracts over rows, so both operands are needed row-contiguous.  `scale` (a power of two,
 * undone by the consuming GEMM's alpha) keeps small gradients out of fp16's subnormal range */
int t2h_f32_to_planes_t(const float* x, void* out_t, void* out_n, int g, int r, int c, int terms, float scale,
                        t2h_stream_t stream);
/* fp16 planes [terms][g][r][c] (row stride ld, group stride g_stride, plane stride in_plane, elements)
 * -> [terms][g][c][r] with output row stride out_ld, group stride out_g_stride, plane stride out_plane */
int t2h_planes_transpose(const void* x, void* out, int g, int r, int c, int64_t ld, int64_t g_stride,
                         int64_t in_plane, int64_t out_ld, int64_t out_g_stride, int64_t out_plane, int terms,
                         t2h_stream_t stream);
/* out[c] += sum_r x[r][c]   (bias gradients) */
int t2h_colsum(const float* x, float* out, int64_t rows, int c, t2h_stream_t stream);
/* exact-erf GELU forward to fp16 planes, and backward da = dg * gelu'(a) (nn.GELU, transformer_arch.py:86) */
int t2h_gelu_fwd(const float* a, void* out, int64_t n, int terms, t2h_stream_t stream);
int t2h_gelu_bwd(const float* a, const float* dg, float* da, void* da_planes /* optional fp16 planes of da */,
                 int64_t n, int terms, t2h_stream_t stream);
/* LayerNorm backward; dx is overwritten or (accumulate=1) added to; dgamma/dbeta are accumulated */
int t2h_layernorm_bwd(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                      float* dbeta, int64_t rows, int c, float eps, int accumulate, t2h_stream_t stream);
/* the same with two optional fused outputs of the updated dx: its fp16 planes [terms][rows][c] (the operand of the
 * next backward GEMMs) and its column sums, accumulated into dx_colsum[c] (the bias gradient of the linear layer
 * this dx is the output gradient of) */
int t2h_layernorm_bwd_fused(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                            float* dbeta, int64_t rows, int c, float eps, int accumulate, void* dx_planes, int terms,
                            float* dx_colsum, t2h_stream_t stream);
/* ds = scale * p * (dp - sum_j dp_j p_j) over the last dim; p as fp16 planes */
int t2h_softmax_bwd(const void* p, const float* dp, float* ds, int64_t rows, int cols, float scale, int terms,
                    t2h_stream_t stream);
/* the same, written straight to fp16 planes of out_scale*ds (the operand of the dQ / dK GEMMs) */
int t2h_softmax_bwd_planes(const void* p, const float* dp, void* ds_planes, int64_t rows, int cols, float scale,
                           int terms, float out_scale, t2h_stream_t stream);
/* masked multi-head cross-entropy: row m belongs to head[m], target[m] (-1 = ignored), weight w[m]:
 * loss_rows[m] = CE (unweighted), dlogits [rows][nh][ncls] = w*(softmax - onehot) in the own head, 0 elsewhere
 * (F.cross_entropy(ignore_index=-1) over 18 heads, transformer_model.py:250-256) */
int t2h_ce_heads(const float* logits, const int64_t* target, const int64_t* head, const float* w,
                 float* loss_rows, float* dlogits, int64_t rows, int nh, int ncls, t2h_stream_t stream);
/* de[idx[m]] += dx[m] (idx NULL: row index m % t_mod, the positional table) */
int t2h_embed_bwd(const float* dx, const int64_t* idx, float* de, int64_t rows, int c, int t_mod,
                  t2h_stream_t stream);
/* torch.optim.Adam step (weight_decay 0); g is multiplied by grad_scale first (1/world after a sum all-reduce) */
int t2h_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
             float eps, int step, float grad_scale, t2h_stream_t stream);

/* ------------------------------------------------------------------------
 * Training step of the VQGAN (VQImageSegmTextureModel.training_step / optimize_parameters,
 * models/vqgan_model.py:444-488, :329-344; models/losses/vqgan_loss.py; loss.backward()).
 * Conv data gradients are t2h_tapgemm launches on the transposed weight planes with negated taps; these are
 * the remaining pieces.
 * ---------------------------------------------------------------------- */
/* Conv weight gradient (what autograd computes for nn.Conv2d.weight, vqgan_arch.py:526,548,573-590,840-1197):
 *   dw[tap][co][ci] += alpha * sum_{n,h,w} dy[n,h,w,co] * x[n + tap_img_off, h + tap_dy, w + tap_dx, ci]
 * dy, x: NHWC fp16 planes (channel stride 1; plane p of dy / x starts dy_term_imgs / x_term_imgs images after
 * plane 0); reads of x outside (x_H, x_W) are zero (= the conv's padding); tap_img_off addresses the phases of a
 * space-to-depth input (stride-2 convs).  dw is accumulated (TMA reduce-add) -- zero it first. */
typedef struct t2h_conv_wgrad_params {
  const void* dy;
  int32_t dy_terms, dy_term_imgs, dy_imgs;
  int32_t n_img, H, W, cout;          /* extents of dy's (img, h, w, c) dims                          */
  int64_t dy_sw, dy_sh, dy_sn;        /* element strides of dy                                        */
  const void* x;
  int32_t x_terms, x_term_imgs, x_imgs;
  int32_t x_H, x_W, cin;
  int64_t x_sw, x_sh, x_sn;
  int32_t ntaps;
  int32_t tap_dy[T2H_MAX_TAPS], tap_dx[T2H_MAX_TAPS], tap_img_off[T2H_MAX_TAPS];
  float* dw;                          /* fp32 [ntaps][cout][dw_ld >= cin]                             */
  int64_t dw_tap_stride, dw_ld;
  float alpha;
  int32_t nterms;                     /* 1 or 3 tensor-core products, as t2h_tapgemm                  */
  int32_t k_split;                    /* 0: choose so that the GPU is filled                          */
} t2h_conv_wgrad_params;
int t2h_conv_wgrad(const t2h_conv_wgrad_params* p, t2h_stream_t stream);

/* Backward of y = act(norm(x)*gamma + beta) for GroupNorm(groups) per image (Normalize(), vqgan_arch.py:510) or,
 * with n = 1 / hw = N*H*W / groups = c, training-mode BatchNorm2d.  stats as t2h_gn_stats / the conv epilogue
 * produced them.  dx = add (optional) + dL/dx as fp32 and / or fp16 planes (either may be NULL, not both: a
 * gradient only the following conv gradients consume needs no fp32 copy); dgamma/dbeta accumulated (may be NULL).
 * ws: 2*n*c doubles of scratch.  act: 0 none, 1 swish, 2 LeakyReLU(0.2).  dx_colsum (optional, [c], accumulated):
 * column sums of the dx written = the bias gradient of the conv whose output x is.  sums_ready != 0: ws already
 * holds pass 1's per-(image, channel) sums {sum du, sum du*xhat} -- the data-gradient conv that produced dy
 * accumulated them in its epilogue (t2h_tapgemm_params.nb_sums) -- and only the apply pass runs. */
int t2h_norm_bwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* dy,
                 const float* add, float* dx, void* dx_planes, int terms, float* dgamma, float* dbeta, double* ws,
                 int n, int hw, int c, int groups, float eps, int act, float* dx_colsum, int sums_ready,
                 t2h_stream_t stream);
/* BatchNorm2d running statistics: r = (1-momentum) r + momentum * batch (unbiased variance); stats [c][2] */
int t2h_bn_update_running(const double* stats, float* running_mean, float* running_var, int64_t count,
                          float momentum, int c, t2h_stream_t stream);
/* dpre = dy * (y > 0 ? 1 : 0.2), y = LeakyReLU(pre) given by (the hi plane of) its fp16 planes; optional planes */
int t2h_lrelu_bwd(const void* y_planes, const float* dy, float* dpre, void* dpre_planes, int terms, int64_t n,
                  t2h_stream_t stream);
/* fp16 planes [terms][n][h][w][c] -> 4-phase space-to-depth planes [terms][4][n][h/2][w/2][c] (T2H_CVT_S2D's layout),
 * the operand of the stride-2 convs when the producer already wrote planes (Discriminator, vqgan_arch.py:1160-1180) */
int t2h_planes_s2d(const void* x, void* out, int terms, int n, int h, int w, int c, t2h_stream_t stream);
/* adjoint of F.interpolate(scale_factor=2, mode='nearest') (Upsample, :530): x [n,2h,2w,c] -> out [n,h,w,c] */
int t2h_sumpool2(const float* x, float* out, int n, int h, int w, int c, t2h_stream_t stream);
/* Quantizer backward (straight-through + legacy-beta loss, vqgan_arch.py:270-281): dz = dzq + coef_z (z - e),
 * dcodebook[book][idx] += coef_e (e - z); rows whose book_id selects no codebook have e = 0 */
int t2h_vq_bwd(const float* z, const float* codebook, const int64_t* idx, const int32_t* book_id, const float* dzq,
               float* dz, float* dcodebook, int64_t rows, int d, int n_books, int n_e, float coef_z, float coef_e,
               t2h_stream_t stream);
/* sum[0] += sum |x - xrec|; grad (may be NULL) = gscale * sign(xrec - x)   (torch.abs, vqgan_model.py:449) */
int t2h_l1_loss(const float* x, const float* xrec, float* grad, double* sum, int64_t n, float gscale,
                t2h_stream_t stream);
/* sgn = +1 / -1: sum += relu(1 - sgn*l), grad = -sgn*gscale where positive (hinge_d_loss, vqgan_loss.py:21-26);
 * sgn = 0: sum += l, grad = gscale (g_loss = -mean(logits_fake), vqgan_model.py:461) */
int t2h_hinge_loss(const float* logits, float* grad, double* sum, int64_t n, float sgn, float gscale,
                   t2h_stream_t stream);
/* DiffAugment(x, 'color,translation') (vqgan_loss.py:29-80) on fp32 NCHW [b,3,h,w]; r [b][3] the brightness /
 * saturation / contrast uniforms, t [b][2] the integer translations (drawn by the caller in the reference's
 * order); ssum / dsum: b doubles of scratch */
int t2h_diffaug_fwd(const float* x, const float* r, const int32_t* t, double* ssum, float* out, int b, int h, int w,
                    t2h_stream_t stream);
int t2h_diffaug_bwd(const float* dout, const float* r, const int32_t* t, double* dsum, float* dx, int b, int h,
                    int w, t2h_stream_t stream);
/* out[0] = clamp(|rg| / (|gg| + 1e-4), 0, wmax) * enable, gradients scaled by 1/inv_scale
 * (calculate_adaptive_weight, vqgan_loss.py:5-12) */
int t2h_adaptive_weight(const float* rg, const float* gg, int64_t n, float inv_scale, float wmax, float enable,
                        float* out, t2h_stream_t stream);
/* out = a + w[0]*b with w on the device */
int t2h_axpy_dev(const float* a, const float* b, const float* w, float* out, int64_t n, t2h_stream_t stream);

/* One reveal step of BaseSampleModel.sample_fn (sample_model.py:283-317): rows with u < inv_t that are still masked
 * draw a token from softmax(logits[row] * inv_temp) (their own texture head's logits [rows][ncls]; Gumbel-max with
 * Philox4x32-10 keyed by (seed, step, row, class)) and write x_t[row] = token + cont_stride * tex[row]. */
int t2h_sample_step(const float* logits, const float* u, const int64_t* tex, int64_t* x_t, uint8_t* unmasked,
                    int64_t rows, int ncls, int n_heads, float inv_t, float inv_temp, uint64_t seed, uint32_t step,
                    int64_t cont_stride, t2h_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* T2H_H_ */
