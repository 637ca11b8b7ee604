// HBM-bound kernels of the VQGAN GAN training step (reference models/vqgan_model.py:444-488 `training_step`,
// :329-344 `optimize_parameters`; losses models/losses/vqgan_loss.py; `loss.backward()`): GroupNorm / BatchNorm
// (+ swish / LeakyReLU) backward, the adjoint of the nearest x2 upsample, the quantizer's straight-through +
// legacy-beta gradients, L1 / hinge / DiffAugment forward+backward, the adaptive discriminator weight, and the
// sampler's per-step categorical draw.  The dense gradients (conv dgrad / wgrad) run on t2h_tapgemm /
// t2h_conv_wgrad (gemm_tc.cu).  Reference call sites are listed next to each entry point in include/t2h.h.
#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

struct alignas(16) H8 {
  __half v[8];
};

// (tests/test_gpu_image_kernels.py::grid_route restates this rule)
static inline int grid_cap(long long work, int block, int per_sm = 16) {
  long long g = ceil_div64(work, block);
  long long cap = (long long)num_sms() * per_sm;
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

// per-channel constants of one image's normalisation, in shared memory: mean, rstd, gamma, beta
__device__ __forceinline__ void norm_consts(const double* __restrict__ stats, const float* __restrict__ gamma,
                                            const float* __restrict__ beta, int n, int C, int groups, int HW,
                                            float eps, float* mean, float* rstd, float* ga, float* be) {
  const int cpg = C / groups;
  const double cnt = (double)HW * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double s = stats[((long long)n * groups + g) * 2 + 0];
    const double q = stats[((long long)n * groups + g) * 2 + 1];
    const double m = s / cnt;
    double var = q / cnt - m * m;
    if (var < 0) var = 0;
    mean[c] = (float)m;
    rstd[c] = (float)(1.0 / sqrt(var + (double)eps));
    ga[c] = gamma[c];
    be[c] = beta[c];
  }
}

// ----------------------------------------------------------------------------
// GroupNorm / BatchNorm backward, pass 1: S[n][c] = (sum du, sum du*xhat) over the pixels, du = dy * act'(u)
// grid (chunks, N); a thread owns 4 consecutive channels and walks pixels (the gn_stats_kernel layout)
// ----------------------------------------------------------------------------
__global__ void norm_bwd_reduce_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       const float* __restrict__ dy, double* __restrict__ S, int HW, int C,
                                       int groups, float eps, int act, int pix_per_block) {
  extern __shared__ float sm[];  // mean, rstd, gamma, beta [C]; s1, s2 [C]
  float *mean = sm, *rstd = sm + C, *ga = sm + 2 * C, *be = sm + 3 * C, *a1 = sm + 4 * C, *a2 = sm + 5 * C;
  const int n = blockIdx.y;
  norm_consts(stats, gamma, beta, n, C, groups, HW, eps, mean, rstd, ga, be);
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) a1[c] = 0.f;
  __syncthreads();
  const int c4 = C >> 2;
  const int slots = blockDim.x / c4;
  const int cs = threadIdx.x % c4;
  const int pl = threadIdx.x / c4;
  const int p_begin = blockIdx.x * pix_per_block;
  const int p_end = min(HW, p_begin + pix_per_block);
  if (pl < slots) {
    float s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
    const long long base = (long long)n * HW * C + cs * 4;
    for (int p = p_begin + pl; p < p_end; p += slots) {
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + base + (long long)p * C));
      const float4 dv = __ldg(reinterpret_cast<const float4*>(dy + base + (long long)p * C));
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
      const float ds[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = cs * 4 + e;
        const float xh = (xs[e] - mean[c]) * rstd[c];
        const float du = ds[e] * act_grad(xh * ga[c] + be[c], act);
        s1[e] += du;
        s2[e] += du * xh;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      atomicAdd(&a1[cs * 4 + e], s1[e]);
      atomicAdd(&a2[cs * 4 + e], s2[e]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(&S[((long long)n * C + c) * 2 + 0], (double)a1[c]);
    atomicAdd(&S[((long long)n * C + c) * 2 + 1], (double)a2[c]);
  }
}

// pass 2: dx = rstd * (du*gamma - mean_g(du*gamma) - xhat * mean_g(du*gamma*xhat)) [+ add]; optional fp16 planes
__global__ void norm_bwd_apply_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ dy, const double* __restrict__ S,
                                      const float* __restrict__ add, float* __restrict__ dx,
                                      __half* __restrict__ planes, int terms, long long plane, int HW, int C,
                                      int groups, float eps, int act, int pix_per_block,
                                      float* __restrict__ dx_colsum) {
  extern __shared__ float sm[];  // mean, rstd, gamma, beta, m1, m2, colsum [C]
  float *mean = sm, *rstd = sm + C, *ga = sm + 2 * C, *be = sm + 3 * C, *m1 = sm + 4 * C, *m2 = sm + 5 * C;
  float* csum = sm + 6 * C;
  if (dx_colsum)
    for (int c = threadIdx.x; c < C; c += blockDim.x) csum[c] = 0.f;
  const int n = blockIdx.y;
  norm_consts(stats, gamma, beta, n, C, groups, HW, eps, mean, rstd, ga, be);
  const int cpg = C / groups;
  const double cnt = (double)HW * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g0 = (c / cpg) * cpg;
    double a = 0, b = 0;
    for (int k = 0; k < cpg; ++k) {
      const double gk = (double)gamma[g0 + k];
      a += gk * S[((long long)n * C + g0 + k) * 2 + 0];
      b += gk * S[((long long)n * C + g0 + k) * 2 + 1];
    }
    m1[c] = (float)(a / cnt);
    m2[c] = (float)(b / cnt);
  }
  __syncthreads();
  const int c4 = C >> 2;
  const long long p_begin = (long long)blockIdx.x * pix_per_block;
  const long long work = (long long)min((long long)pix_per_block, HW - p_begin) * c4;
  const long long base = ((long long)n * HW + p_begin) * C;
  // column sums of the dx written (= the bias gradient of the conv that produced x): when blockDim is a multiple of
  // C/4 a thread always meets the same 4 channels and keeps them in registers, otherwise it adds each element to
  // the block's shared column sums (tests/test_gpu_backward_paths.py::norm_bwd_route restates this choice)
  const bool fixed_cols = (blockDim.x % c4) == 0;
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long i = threadIdx.x; i < work; i += blockDim.x) {
    const int c0 = (int)(i % c4) * 4;
    const long long o = base + i * 4;
    const float4 xv = __ldg(reinterpret_cast<const float4*>(x + o));
    const float4 dv = __ldg(reinterpret_cast<const float4*>(dy + o));
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
    if (add) av = __ldg(reinterpret_cast<const float4*>(add + o));
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
    const float ds[4] = {dv.x, dv.y, dv.z, dv.w};
    const float as[4] = {av.x, av.y, av.z, av.w};
    float r[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + e;
      const float xh = (xs[e] - mean[c]) * rstd[c];
      const float du = ds[e] * act_grad(xh * ga[c] + be[c], act);
      r[e] = rstd[c] * (du * ga[c] - m1[c] - xh * m2[c]) + as[e];
    }
    if (dx) *reinterpret_cast<float4*>(dx + o) = make_float4(r[0], r[1], r[2], r[3]);  // null: only the planes are consumed
    if (dx_colsum) {
      if (fixed_cols) {
#pragma unroll
        for (int e = 0; e < 4; ++e) cs[e] += r[e];
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) atomicAdd(&csum[c0 + e], r[e]);
      }
    }
    if (planes) {
      __align__(8) __half hi[4];
      __align__(8) __half lo[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) split_f16(r[e], hi[e], lo[e]);
      *reinterpret_cast<uint2*>(planes + o) = *reinterpret_cast<uint2*>(hi);
      if (terms == 2) *reinterpret_cast<uint2*>(planes + plane + o) = *reinterpret_cast<uint2*>(lo);
    }
  }
  if (dx_colsum) {
    if (fixed_cols && threadIdx.x < work) {
      const int c0 = (int)(threadIdx.x % c4) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) atomicAdd(&csum[c0 + e], cs[e]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&dx_colsum[c], csum[c]);
  }
}

// dgamma[c] += sum_n S[n][c][1], dbeta[c] += sum_n S[n][c][0]
__global__ void norm_bwd_params_kernel(const double* __restrict__ S, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, int N, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0, b = 0;
  for (int n = 0; n < N; ++n) {
    a += S[((long long)n * C + c) * 2 + 0];
    b += S[((long long)n * C + c) * 2 + 1];
  }
  if (dbeta) dbeta[c] += (float)a;
  if (dgamma) dgamma[c] += (float)b;
}

// BatchNorm running statistics (momentum update with the unbiased batch variance), stats = (sum, sumsq) per channel
__global__ void bn_running_kernel(const double* __restrict__ stats, float* __restrict__ rmean,
                                  float* __restrict__ rvar, long long count, float momentum, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double m = stats[2 * c] / (double)count;
  double var = stats[2 * c + 1] / (double)count - m * m;
  if (var < 0) var = 0;
  const double unb = count > 1 ? var * (double)count / (double)(count - 1) : var;
  rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)m;
  rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unb;
}

// dpre = dy * (y > 0 ? 1 : slope) where y = LeakyReLU(pre) (sign preserved) given as the hi plane of its fp16 planes.
// The slope is read from hi: 0 < y <= 2^-25 rounds to an fp16 0 and gets 0.2 where autograd uses 1 (planes cannot
// tell those y from 0; tests/test_gpu_image_kernels.py::test_lrelu_bwd_bit_exact pins this rule)
__global__ void lrelu_bwd_kernel(const __half* __restrict__ y, const float* __restrict__ dy,
                                 float* __restrict__ dpre, __half* __restrict__ planes, int terms, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float g = dy[i] * (__half2float(y[i]) > 0.f ? 1.0f : 0.2f);
    dpre[i] = g;
    if (planes) {
      __half hi, lo;
      split_f16(g, hi, lo);
      planes[i] = hi;
      if (terms == 2) planes[n + i] = lo;
    }
  }
}

// fp16 planes [T][N][H][W][C] -> 4-phase space-to-depth planes [T][4][N][H/2][W/2][C] (the operand layout of the
// stride-2 convs), 16-byte copies
__global__ void planes_s2d_kernel(const __half* __restrict__ x, __half* __restrict__ out, int T, int N, int H, int W,
                                  int C) {
  const int c8 = C >> 3, Ho = H / 2, Wo = W / 2;
  const long long total = (long long)T * 4 * N * Ho * Wo * c8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c8);
    long long r = i / c8;
    const int ow = (int)(r % Wo); r /= Wo;
    const int oh = (int)(r % Ho); r /= Ho;
    const int n = (int)(r % N); r /= N;
    const int ph = (int)(r % 4);
    const int t = (int)(r / 4);
    const long long src = ((((long long)t * N + n) * H + 2 * oh + (ph >> 1)) * W + 2 * ow + (ph & 1)) * C + cc * 8;
    reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(x + src));
  }
}

// adjoint of the nearest x2 upsample: out[n,h,w,c] = sum of the 2x2 block of x [N,2H,2W,C]
__global__ void sumpool2_kernel(const float* __restrict__ x, float* __restrict__ out, int N, int H, int W, int C) {
  const int c4 = C >> 2;
  const long long total = (long long)N * H * W * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c4);
    long long r = i / c4;
    const int w = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int n = (int)(r / H);
    const float* b = x + (((long long)n * 2 * H + 2 * h) * 2 * W + 2 * w) * C + cc * 4;
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(b));
    const float4 a1 = __ldg(reinterpret_cast<const float4*>(b + C));
    const float4 a2 = __ldg(reinterpret_cast<const float4*>(b + (long long)2 * W * C));
    const float4 a3 = __ldg(reinterpret_cast<const float4*>(b + (long long)2 * W * C + C));
    reinterpret_cast<float4*>(out)[i] = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y),
                                                    (a0.z + a1.z) + (a2.z + a3.z), (a0.w + a1.w) + (a2.w + a3.w));
  }
}

// Quantizer backward (VectorQuantizerTexture.forward :270-281): zq_st = z + (e - z).detach(),
// loss = mean((e.detach()-z)^2) + beta*mean((e - z.detach())^2):
//   dz = dzq + coef_z * (z - e),  dE[book][idx] += coef_e * (e - z)     (e = 0 for rows no codebook selects)
__global__ void vq_bwd_kernel(const float* __restrict__ z, const float* __restrict__ cb,
                              const long long* __restrict__ idx, const int* __restrict__ book,
                              const float* __restrict__ dzq, float* __restrict__ dz, float* __restrict__ dcb,
                              long long rows, int D, int n_books, int n_e, float coef_z, float coef_e) {
  const long long row = blockIdx.x;
  const int bk = book ? book[row] : 0;
  const long long id = idx[row];
  const bool sel = bk >= 0 && bk < n_books && id >= 0 && id < n_e;
  const float* e = sel ? cb + ((long long)bk * n_e + id) * D : nullptr;
  float* de = sel ? dcb + ((long long)bk * n_e + id) * D : nullptr;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float zv = z[row * D + d];
    const float ev = sel ? e[d] : 0.f;
    dz[row * D + d] = (dzq ? dzq[row * D + d] : 0.f) + coef_z * (zv - ev);
    if (sel) atomicAdd(&de[d], coef_e * (ev - zv));
  }
}

// block-wide sum into a double accumulator
__device__ __forceinline__ void block_add(double v, double* out) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    v = lane < (blockDim.x >> 5) ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) atomicAdd(out, v);
  }
  __syncthreads();
}

// L1: sum += |x - xrec|; grad = gscale * sign(xrec - x)     (torch.abs backward: sign, 0 at 0)
__global__ void l1_kernel(const float* __restrict__ x, const float* __restrict__ xrec, float* __restrict__ grad,
                          double* __restrict__ sum, long long n, float gscale) {
  double acc = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float d = xrec[i] - x[i];
    acc += fabsf(d);
    if (grad) grad[i] = d > 0.f ? gscale : (d < 0.f ? -gscale : 0.f);
  }
  block_add(acc, sum);
}

// BCE-with-logits against the one-hot of a class-id map (BCELossWithQuant, segmentation_loss.py:12-25, with the target
// of VQSegmentationModel.feed_data, vqgan_model.py:117-124).  Per element x, t = [c == id(pixel)]:
//   loss += max(x,0) - x t + log1p(exp(-|x|)),   g = gscale (sigmoid(x) - t)
// g goes straight to fp16 hi/lo planes [terms][pix][c_pad] (pad channels 0) and its column sums to colsum[c].
// A thread owns 8 channels of one pixel (two float4 loads, one 16-byte store per plane); blockDim is a multiple of
// c_pad/8, so a thread meets the same 8 channels at every pixel and keeps their column sums in registers.
// sigmoid(x) - 1 is formed as -sigmoid(-x), so saturated logits keep their tiny gradients.
__global__ void bce_logits_kernel(const float* __restrict__ x, const float* __restrict__ ids, long long npix, int C,
                                  int c_pad, float gscale, double* __restrict__ loss, __half* __restrict__ planes,
                                  int terms, float* __restrict__ colsum) {
  extern __shared__ double cs_sm[];  // [c_pad]: the block's column sums
  const int c8 = c_pad >> 3;
  const int lanes = blockDim.x / c8;
  const int c0 = (threadIdx.x % c8) * 8;
  const int lane = threadIdx.x / c8;
  const long long plane = npix * c_pad;
  for (int c = threadIdx.x; c < c_pad; c += blockDim.x) cs_sm[c] = 0.0;
  __syncthreads();
  float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  double acc = 0.0;
  if (lane < lanes) {
    for (long long p = (long long)blockIdx.x * lanes + lane; p < npix; p += (long long)gridDim.x * lanes) {
      const float v = __ldg(ids + p);
      const int cls = (v == floorf(v) && v >= 0.f && v < (float)C) ? (int)v : -1;
      float xs[8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + 4 * h < C) q = __ldg(reinterpret_cast<const float4*>(x + p * C + c0 + 4 * h));
        xs[4 * h + 0] = q.x;
        xs[4 * h + 1] = q.y;
        xs[4 * h + 2] = q.z;
        xs[4 * h + 3] = q.w;
      }
      H8 hi, lo;
      float part = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int c = c0 + e;
        float g = 0.f;
        if (c < C) {
          const float xv = xs[e];
          const float en = expf(-fabsf(xv));
          const float r = 1.f / (1.f + en);
          const float sp = xv >= 0.f ? r : en * r;   // sigmoid(x)
          const float sn = xv >= 0.f ? en * r : r;   // sigmoid(-x) = 1 - sigmoid(x)
          const bool t = c == cls;
          part += fmaxf(xv, 0.f) - (t ? xv : 0.f) + log1pf(en);
          g = gscale * (t ? -sn : sp);
          cs[e] += g;
        }
        split_f16(g, hi.v[e], lo.v[e]);
      }
      acc += (double)part;
      if (planes) {
        *reinterpret_cast<H8*>(planes + p * c_pad + c0) = hi;
        if (terms == 2) *reinterpret_cast<H8*>(planes + plane + p * c_pad + c0) = lo;
      }
    }
  }
  if (colsum) {
    if (lane < lanes) {
#pragma unroll
      for (int e = 0; e < 8; ++e) atomicAdd(&cs_sm[c0 + e], (double)cs[e]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&colsum[c], (float)cs_sm[c]);
  }
  block_add(acc, loss);
}

// hinge term: sum += relu(1 - sgn*l); grad = -sgn*gscale where 1 - sgn*l > 0   (hinge_d_loss, vqgan_loss.py:21-26)
// sgn = 0: plain sum of l (g_loss = -mean(logits_fake)) with constant gradient gscale
__global__ void hinge_kernel(const float* __restrict__ l, float* __restrict__ grad, double* __restrict__ sum,
                             long long n, float sgn, float gscale) {
  double acc = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    if (sgn == 0.f) {
      acc += l[i];
      if (grad) grad[i] = gscale;
    } else {
      const float m = 1.0f - sgn * l[i];
      acc += m > 0.f ? m : 0.f;
      if (grad) grad[i] = m > 0.f ? -sgn * gscale : 0.f;
    }
  }
  block_add(acc, sum);
}

// per-sample sums of an NCHW batch (DiffAugment's contrast mean; its backward's sum of dz)
__global__ void sample_sum_kernel(const float* __restrict__ x, double* __restrict__ out, long long per) {
  const int b = blockIdx.y;
  double acc = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < per;
       i += (long long)gridDim.x * blockDim.x)
    acc += x[(long long)b * per + i];
  block_add(acc, out + b);
}

// DiffAugment(x, 'color,translation') (vqgan_loss.py:29-80), 3-channel NCHW.  r = per-sample (brightness r1,
// saturation r2, contrast r3) uniforms; t = per-sample integer (tx, ty).  With m_c the channel mean of a pixel and
// M the sample mean:  y = s*(x+b) + (1-s)*(m_c+b),  z = c*(y - (M+b)) + (M+b),  out[h,w] = z[h+tx, w+ty] (0 outside)
__global__ void diffaug_fwd_kernel(const float* __restrict__ x, const float* __restrict__ r,
                                   const int* __restrict__ t, const double* __restrict__ ssum,
                                   float* __restrict__ out, int H, int W) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  const float bb = r[b * 3 + 0] - 0.5f, s = r[b * 3 + 1] * 2.0f, c = r[b * 3 + 2] + 0.5f;
  const int tx = t[b * 2 + 0], ty = t[b * 2 + 1];
  const float M = (float)(ssum[b] / (double)(3 * HW)) + bb;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < HW;
       i += (long long)gridDim.x * blockDim.x) {
    const int h = (int)(i / W), w = (int)(i % W);
    const int sh = h + tx, sw = w + ty;
    float o[3] = {0.f, 0.f, 0.f};
    if (sh >= 0 && sh < H && sw >= 0 && sw < W) {
      const long long p = (long long)sh * W + sw;
      float v[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) v[k] = x[((long long)b * 3 + k) * HW + p] + bb;
      const float mc = (v[0] + v[1] + v[2]) * (1.0f / 3.0f);
#pragma unroll
      for (int k = 0; k < 3; ++k) o[k] = ((v[k] - mc) * s + mc - M) * c + M;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) out[((long long)b * 3 + k) * HW + i] = o[k];
  }
}

// backward, pass 1: per-sample sum of dz (dout over the in-range window)
__global__ void diffaug_bwd_sum_kernel(const float* __restrict__ dout, const int* __restrict__ t,
                                       double* __restrict__ dsum, int H, int W) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  const int tx = t[b * 2 + 0], ty = t[b * 2 + 1];
  double acc = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < HW;
       i += (long long)gridDim.x * blockDim.x) {
    const int h = (int)(i / W), w = (int)(i % W);
    const int sh = h + tx, sw = w + ty;  // out[h,w] reads z[sh,sw]
    if (sh >= 0 && sh < H && sw >= 0 && sw < W)
      for (int k = 0; k < 3; ++k) acc += dout[((long long)b * 3 + k) * HW + i];
  }
  block_add(acc, dsum + b);
}

// pass 2: dz[p] = dout[p - t];  dy = c*dz + (1-c)/(3HW)*sum(dz);  dx_k = s*dy_k + (1-s)/3*sum_k dy
__global__ void diffaug_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ r,
                                   const int* __restrict__ t, const double* __restrict__ dsum,
                                   float* __restrict__ dx, int H, int W) {
  const int b = blockIdx.y;
  const long long HW = (long long)H * W;
  const float s = r[b * 3 + 1] * 2.0f, c = r[b * 3 + 2] + 0.5f;
  const int tx = t[b * 2 + 0], ty = t[b * 2 + 1];
  const float mterm = (1.0f - c) * (float)(dsum[b] / (double)(3 * HW));
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < HW;
       i += (long long)gridDim.x * blockDim.x) {
    const int h = (int)(i / W), w = (int)(i % W);
    const int oh = h - tx, ow = w - ty;  // the output pixel that read z[h,w]
    float dy[3];
    const bool in = oh >= 0 && oh < H && ow >= 0 && ow < W;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      dy[k] = c * (in ? dout[((long long)b * 3 + k) * HW + (long long)oh * W + ow] : 0.f) + mterm;
    const float ms = (dy[0] + dy[1] + dy[2]) * (1.0f / 3.0f);
#pragma unroll
    for (int k = 0; k < 3; ++k) dx[((long long)b * 3 + k) * HW + i] = s * dy[k] + (1.0f - s) * ms;
  }
}

// d_weight = clamp(|rg| / (|gg| + 1e-4), 0, wmax) * enable  (calculate_adaptive_weight, vqgan_loss.py:5-12);
// both gradients carry the loss scale 1/inv_scale.  One block.
__global__ void adaptive_weight_kernel(const float* __restrict__ rg, const float* __restrict__ gg, long long n,
                                       float inv_scale, float wmax, float enable, float* __restrict__ out) {
  __shared__ double acc[2];
  if (threadIdx.x < 2) acc[threadIdx.x] = 0;
  __syncthreads();
  double a = 0, b = 0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const double r = (double)rg[i] * inv_scale, g = (double)gg[i] * inv_scale;
    a += r * r;
    b += g * g;
  }
  block_add(a, &acc[0]);
  block_add(b, &acc[1]);
  if (threadIdx.x == 0) {
    float w = (float)(sqrt(acc[0]) / (sqrt(acc[1]) + 1e-4));
    w = fminf(fmaxf(w, 0.f), wmax);
    out[0] = w * enable;
  }
}

// out = a + w[0] * b  (w on the device: no host sync between the adaptive weight and the generator backward)
__global__ void axpy_dev_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                const float* __restrict__ w, float* __restrict__ out, long long n) {
  const float ww = w[0];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    out[i] = a[i] + ww * b[i];
}

// ----------------------------------------------------------------------------
// One reveal step of the absorbing-diffusion sampler (BaseSampleModel.sample_fn, sample_model.py:283-317):
// position m is revealed when u[m] < 1/t and it is still masked; its token is a categorical draw from
// softmax(logits[m] / temp) over its own texture head, done as Gumbel-max with Philox4x32-10 uniforms keyed by
// (seed, step, position, class).  One warp per position; rows that are not revealed cost one load.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                               uint32_t k1, uint32_t (&o)[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
    c0 = n0; c1 = l1; c2 = n2; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  o[0] = c0; o[1] = c1; o[2] = c2; o[3] = c3;
}

__global__ void sample_step_kernel(const float* __restrict__ logits, const float* __restrict__ u,
                                   const long long* __restrict__ tex, long long* __restrict__ x_t,
                                   unsigned char* __restrict__ unmasked, long long M, int ncls, int n_heads,
                                   float inv_t, float inv_temp, unsigned long long seed, unsigned int step,
                                   long long cont_stride) {
  const long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  const int lane = threadIdx.x & 31;
  if (!(u[m] < inv_t) || unmasked[m]) return;  // warp-uniform
  const long long tx = tex[m];
  const bool valid = tx >= 0 && tx < n_heads;
  float best = -INFINITY;
  int bi = 0;
  const float* row = logits + m * ncls;
  for (int c0 = lane * 4; c0 < ncls; c0 += 128) {
    uint32_t rnd[4];
    philox4x32_10((uint32_t)c0, (uint32_t)m, (uint32_t)(m >> 32), step, (uint32_t)seed, (uint32_t)(seed >> 32), rnd);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + e;
      if (c < ncls) {
        const float uu = ((float)(rnd[e] >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
        const float v = row[c] * inv_temp - __logf(-__logf(uu));
        if (v > best) { best = v; bi = c; }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) {
    unmasked[m] = 1;
    if (valid) x_t[m] = (long long)bi + cont_stride * tx;
  }
}

// t2h_norm_bwd's kernels keep per-channel constants in dynamic shared memory: 6 C floats (reduce) and 7 C floats
// (apply), 56 KB at the largest C.  Above the default 48 KB a kernel must be opted in, once per device (the
// attribute lives in the device's copy of the function); model shapes stay below it and never call this.
constexpr int kNormBwdMaxC = 2048;
static int smem_opt_in(const void* kernel, size_t bytes, int max_bytes, bool (&configured)[64]) {
  if (bytes <= 48 * 1024) return T2H_OK;
  int dev = 0;
  T2H_CUDA(cudaGetDevice(&dev));
  if (!configured[dev & 63]) {
    T2H_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_bytes));
    configured[dev & 63] = true;
  }
  return T2H_OK;
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int t2h_norm_bwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* dy,
                 const float* add, float* dx, void* dx_planes, int terms, float* dgamma, float* dbeta, double* ws,
                 int n, int hw, int c, int groups, float eps, int act, float* dx_colsum, int sums_ready,
                 t2h_stream_t stream) {
  T2H_CHECK_ARG(x && stats && gamma && beta && dy && (dx || dx_planes) && ws && n > 0 && hw > 0, "norm_bwd: bad args");
  T2H_CHECK_ARG(c % groups == 0 && c % 4 == 0 && c <= kNormBwdMaxC, "norm_bwd: C=%d groups=%d unsupported", c,
                groups);
  T2H_CHECK_ARG(act >= 0 && act <= 2 && (terms == 1 || terms == 2 || !dx_planes), "norm_bwd: act=%d terms=%d", act,
                terms);
  cudaStream_t st = as_stream(stream);
  // (tests/test_gpu_backward_paths.py::norm_bwd_route restates the block, lane and pixels-per-block choices below)
  if (!sums_ready) {  // pass 1 (skipped when the conv that produced dy accumulated the sums in its epilogue)
    T2H_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * 2 * (size_t)n * c, st));
    const int c4 = c / 4;
    int block = 256;
    if (c4 > block) block = ((c4 + 31) / 32) * 32;
    T2H_CHECK_ARG(block <= 1024, "norm_bwd: C=%d too large", c);
    block = (block / c4) * c4;  // C > 1024: block = C/4, one pixel lane
    const int lanes = block / c4;
    int blocks_x = ceil_div(num_sms() * 4, n);
    int ppb = ceil_div(hw, blocks_x);
    if (ppb < lanes * 8) ppb = lanes * 8;
    blocks_x = ceil_div(hw, ppb);
    static bool reduce_configured[64] = {};
    const size_t smem = 6 * (size_t)c * sizeof(float);
    int rc = smem_opt_in((const void*)norm_bwd_reduce_kernel, smem, 6 * kNormBwdMaxC * (int)sizeof(float),
                         reduce_configured);
    if (rc) return rc;
    norm_bwd_reduce_kernel<<<dim3(blocks_x, n), block, smem, st>>>(x, stats, gamma, beta, dy, ws, hw, c, groups, eps,
                                                                   act, ppb);
    T2H_LAUNCH_OK();
  }
  int bx2 = ceil_div(num_sms() * 8, n);
  int ppb2 = ceil_div(hw, bx2);
  if (ppb2 < 16) ppb2 = 16;
  bx2 = ceil_div(hw, ppb2);
  static bool apply_configured[64] = {};
  const size_t smem2 = 7 * (size_t)c * sizeof(float);
  int rc = smem_opt_in((const void*)norm_bwd_apply_kernel, smem2, 7 * kNormBwdMaxC * (int)sizeof(float),
                       apply_configured);
  if (rc) return rc;
  norm_bwd_apply_kernel<<<dim3(bx2, n), 256, smem2, st>>>(
      x, stats, gamma, beta, dy, ws, add, dx, reinterpret_cast<__half*>(dx_planes), terms, (long long)n * hw * c, hw,
      c, groups, eps, act, ppb2, dx_colsum);
  T2H_LAUNCH_OK();
  if (dgamma || dbeta) {  // either may be given alone
    norm_bwd_params_kernel<<<ceil_div(c, 128), 128, 0, st>>>(ws, dgamma, dbeta, n, c);
    T2H_LAUNCH_OK();
  }
  return T2H_OK;
}

int t2h_bn_update_running(const double* stats, float* running_mean, float* running_var, int64_t count,
                          float momentum, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(stats && running_mean && running_var && count > 0 && c > 0, "bn_update_running: bad args");
  bn_running_kernel<<<ceil_div(c, 128), 128, 0, as_stream(stream)>>>(stats, running_mean, running_var, count,
                                                                     momentum, c);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_lrelu_bwd(const void* y_planes, const float* dy, float* dpre, void* dpre_planes, int terms, int64_t n,
                  t2h_stream_t stream) {
  T2H_CHECK_ARG(y_planes && dy && dpre && n > 0, "lrelu_bwd: bad args");
  lrelu_bwd_kernel<<<grid_cap(n, 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const __half*>(y_planes), dy, dpre, reinterpret_cast<__half*>(dpre_planes), terms, n);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_planes_s2d(const void* x, void* out, int terms, int n, int h, int w, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && h > 0 && w > 0 && c > 0, "planes_s2d: bad args");
  T2H_CHECK_ARG(h % 2 == 0 && w % 2 == 0 && c % 8 == 0 && (terms == 1 || terms == 2), "planes_s2d: shape");
  planes_s2d_kernel<<<grid_cap((long long)terms * n * h * w * (c / 8), 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(out), terms, n, h, w, c);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_sumpool2(const float* x, float* out, int n, int h, int w, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && h > 0 && w > 0 && c > 0 && c % 4 == 0, "sumpool2: bad args");
  sumpool2_kernel<<<grid_cap((long long)n * h * w * (c / 4), 256), 256, 0, as_stream(stream)>>>(x, out, n, h, w, c);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_vq_bwd(const float* z, const float* codebook, const int64_t* idx, const int32_t* book_id, const float* dzq,
               float* dz, float* dcodebook, int64_t rows, int d, int n_books, int n_e, float coef_z, float coef_e,
               t2h_stream_t stream) {
  T2H_CHECK_ARG(z && codebook && idx && dz && dcodebook && rows > 0 && d > 0, "vq_bwd: bad args");
  vq_bwd_kernel<<<(unsigned)rows, 128, 0, as_stream(stream)>>>(z, codebook, reinterpret_cast<const long long*>(idx),
                                                              book_id, dzq, dz, dcodebook, rows, d, n_books, n_e,
                                                              coef_z, coef_e);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_l1_loss(const float* x, const float* xrec, float* grad, double* sum, int64_t n, float gscale,
                t2h_stream_t stream) {
  T2H_CHECK_ARG(x && xrec && sum && n > 0, "l1_loss: bad args");
  // (tests/test_gpu_image_kernels.py::loss_route restates this grid, as for hinge_kernel)
  l1_kernel<<<grid_cap(n, 256, 4), 256, 0, as_stream(stream)>>>(x, xrec, grad, sum, n, gscale);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_bce_logits(const float* logits, const float* ids, int n, int h, int w, int c, int c_pad, float gscale,
                   double* loss_sum, void* grad_planes, int terms, float* colsum, t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && ids && loss_sum && n > 0 && h > 0 && w > 0 && c > 0, "bce_logits: bad args");
  T2H_CHECK_ARG(c % 4 == 0 && c_pad >= c && c_pad % 8 == 0 && c_pad <= 256, "bce_logits: c=%d c_pad=%d", c, c_pad);
  T2H_CHECK_ARG(!grad_planes || terms == 1 || terms == 2, "bce_logits: terms=%d", terms);
  const long long npix = (long long)n * h * w;
  const int c8 = c_pad / 8;
  // whole warps (block_add) and a whole number of pixels per block (fixed channels per thread)
  const int block = 32 * c8 * (c8 < 8 ? 8 / c8 : 1);  // (tests/test_gpu_image_kernels.py::bce_route restates this choice)
  bce_logits_kernel<<<grid_cap(npix, block / c8, 4), block, c_pad * sizeof(double), as_stream(stream)>>>(
      logits, ids, npix, c, c_pad, gscale, loss_sum, reinterpret_cast<__half*>(grad_planes), terms, colsum);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_hinge_loss(const float* logits, float* grad, double* sum, int64_t n, float sgn, float gscale,
                   t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && sum && n > 0, "hinge_loss: bad args");
  hinge_kernel<<<grid_cap(n, 256, 4), 256, 0, as_stream(stream)>>>(logits, grad, sum, n, sgn, gscale);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_diffaug_fwd(const float* x, const float* r, const int32_t* t, double* ssum, float* out, int b, int h, int w,
                    t2h_stream_t stream) {
  T2H_CHECK_ARG(x && r && t && ssum && out && b > 0 && h > 0 && w > 0, "diffaug_fwd: bad args");
  cudaStream_t st = as_stream(stream);
  T2H_CUDA(cudaMemsetAsync(ssum, 0, sizeof(double) * b, st));
  const long long per = 3LL * h * w;  // (tests/test_gpu_image_kernels.py::diffaug_route restates both capped grids)
  const int gx = grid_cap(per, 256, 2) < 64 ? grid_cap(per, 256, 2) : 64;
  sample_sum_kernel<<<dim3(gx, b), 256, 0, st>>>(x, ssum, per);
  T2H_LAUNCH_OK();
  const int gy = grid_cap((long long)h * w, 256, 2) < 128 ? grid_cap((long long)h * w, 256, 2) : 128;
  diffaug_fwd_kernel<<<dim3(gy, b), 256, 0, st>>>(x, r, t, ssum, out, h, w);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_diffaug_bwd(const float* dout, const float* r, const int32_t* t, double* dsum, float* dx, int b, int h, int w,
                    t2h_stream_t stream) {
  T2H_CHECK_ARG(dout && r && t && dsum && dx && b > 0 && h > 0 && w > 0, "diffaug_bwd: bad args");
  cudaStream_t st = as_stream(stream);
  T2H_CUDA(cudaMemsetAsync(dsum, 0, sizeof(double) * b, st));
  const int gy = grid_cap((long long)h * w, 256, 2) < 128 ? grid_cap((long long)h * w, 256, 2) : 128;
  diffaug_bwd_sum_kernel<<<dim3(gy, b), 256, 0, st>>>(dout, t, dsum, h, w);
  T2H_LAUNCH_OK();
  diffaug_bwd_kernel<<<dim3(gy, b), 256, 0, st>>>(dout, r, t, dsum, dx, h, w);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_adaptive_weight(const float* rg, const float* gg, int64_t n, float inv_scale, float wmax, float enable,
                        float* out, t2h_stream_t stream) {
  T2H_CHECK_ARG(rg && gg && out && n > 0, "adaptive_weight: bad args");
  // (tests/test_gpu_image_kernels.py::adaptive_weight_route restates this single block)
  adaptive_weight_kernel<<<1, 1024, 0, as_stream(stream)>>>(rg, gg, n, inv_scale, wmax, enable, out);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_axpy_dev(const float* a, const float* b, const float* w, float* out, int64_t n, t2h_stream_t stream) {
  T2H_CHECK_ARG(a && b && w && out && n > 0, "axpy_dev: bad args");
  axpy_dev_kernel<<<grid_cap(n, 256), 256, 0, as_stream(stream)>>>(a, b, w, out, n);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_sample_step(const float* logits, const float* u, const int64_t* tex, int64_t* x_t, uint8_t* unmasked,
                    int64_t rows, int ncls, int n_heads, float inv_t, float inv_temp, uint64_t seed, uint32_t step,
                    int64_t cont_stride, t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && u && tex && x_t && unmasked && rows > 0 && ncls > 0, "sample_step: bad args");
  const int warps = 8;
  sample_step_kernel<<<(unsigned)ceil_div64(rows, warps), warps * 32, 0, as_stream(stream)>>>(
      logits, u, reinterpret_cast<const long long*>(tex), reinterpret_cast<long long*>(x_t), unmasked, rows, ncls,
      n_heads, inv_t, inv_temp, (unsigned long long)seed, step, cont_stride);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

}  // extern "C"
