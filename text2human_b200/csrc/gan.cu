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

// act'(u) of the activation after a norm at element x (xhat its normalised value).  ReLU (act 3) forms u as the
// apply kernels do (x * scale + shift, scale = gamma * rstd), so the gradient passes exactly where their output
// is positive (torch's threshold_backward on the output)
__device__ __forceinline__ float norm_act_grad(float x, float xh, float mean, float rstd, float ga, float be, int act) {
  if (act == 3) {
    const float sc = ga * rstd;
    const float sh = be - mean * sc;
    return x * sc + sh > 0.f ? 1.0f : 0.0f;
  }
  return act_grad(xh * ga + be, act);
}

// ----------------------------------------------------------------------------
// GroupNorm / BatchNorm backward, pass 1: S[n][c] = (sum du, sum du*xhat) over the pixels, du = dy * act'(u)
// (dy first multiplied by dys[image][c] when given: the Dropout2d factor between the activation and its consumer,
// image = pixel / img_hw over the whole batch)
// grid (chunks, N); a thread owns 4 consecutive channels and walks pixels (the gn_stats_kernel layout)
// ----------------------------------------------------------------------------
__global__ void norm_bwd_reduce_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                       const float* __restrict__ dy, double* __restrict__ S, int HW, int C,
                                       int groups, float eps, int act, int pix_per_block,
                                       const float* __restrict__ dys, int img_hw) {
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
      float ds[4] = {dv.x, dv.y, dv.z, dv.w};
      if (dys) {
        const float* f = dys + (((long long)n * HW + p) / img_hw) * C + cs * 4;
#pragma unroll
        for (int e = 0; e < 4; ++e) ds[e] *= f[e];
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = cs * 4 + e;
        const float xh = (xs[e] - mean[c]) * rstd[c];
        const float du = ds[e] * norm_act_grad(xs[e], xh, mean[c], rstd[c], ga[c], be[c], act);
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
                                      float* __restrict__ dx_colsum, const float* __restrict__ dys, int img_hw) {
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
    float ds[4] = {dv.x, dv.y, dv.z, dv.w};
    const float as[4] = {av.x, av.y, av.z, av.w};
    if (dys) {
      const float* f = dys + (((long long)n * HW + p_begin + i / c4) / img_hw) * C + c0;
#pragma unroll
      for (int e = 0; e < 4; ++e) ds[e] *= f[e];
    }
    float r[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + e;
      const float xh = (xs[e] - mean[c]) * rstd[c];
      const float du = ds[e] * norm_act_grad(xs[e], xh, mean[c], rstd[c], ga[c], be[c], act);
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
// chunks per image of the broadcast-channel gradient sums of t2h_maxpool2_bcast_bwd (its ws: n * kBcastChunks * c_e)
constexpr int kBcastChunks = 32;
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

static int norm_bwd_impl(const float* x, const double* stats, const float* gamma, const float* beta, const float* dy,
                         const float* add, float* dx, void* dx_planes, int terms, float* dgamma, float* dbeta, double* ws,
                         int n, int hw, int c, int groups, float eps, int act, float* dx_colsum, int sums_ready,
                         const float* dy_scale, int img_hw, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && stats && gamma && beta && dy && (dx || dx_planes) && ws && n > 0 && hw > 0, "norm_bwd: bad args");
  T2H_CHECK_ARG(c % groups == 0 && c % 4 == 0 && c <= kNormBwdMaxC, "norm_bwd: C=%d groups=%d unsupported", c,
                groups);
  T2H_CHECK_ARG(act >= 0 && act <= 3 && (terms == 1 || terms == 2 || !dx_planes), "norm_bwd: act=%d terms=%d", act,
                terms);
  T2H_CHECK_ARG(!dy_scale || (img_hw > 0 && ((long long)n * hw) % img_hw == 0), "norm_bwd: img_hw=%d", img_hw);
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
                                                                   act, ppb, dy_scale, img_hw);
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
      c, groups, eps, act, ppb2, dx_colsum, dy_scale, img_hw);
  T2H_LAUNCH_OK();
  if (dgamma || dbeta) {  // either may be given alone
    norm_bwd_params_kernel<<<ceil_div(c, 128), 128, 0, st>>>(ws, dgamma, dbeta, n, c);
    T2H_LAUNCH_OK();
  }
  return T2H_OK;
}

// ----------------------------------------------------------------------------
// Training of the parsing generator (ParsingGenModel.optimize_parameters, parsing_gen_model.py:80-95): the
// backward of the pieces only the ShapeUNet / FCNHead path has.
// ----------------------------------------------------------------------------
// BatchNorm / GroupNorm apply with an fp32 output and / or fp16 planes, and an optional per-(image, channel) factor
// after the activation (Dropout2d of the FCN head: mask / (1 - p); image = pixel / img_hw over the whole batch).
// y = act(x * scale + shift) * drop, the gn_apply_kernel arithmetic; grid (chunks, n)
__global__ void norm_apply_ex_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                     const float* __restrict__ gamma, const float* __restrict__ beta,
                                     const float* __restrict__ drop, int img_hw, float* __restrict__ out,
                                     __half* __restrict__ planes, int HW, int C, int groups, float eps, int act,
                                     int terms, long long plane, int pix_per_block) {
  extern __shared__ float sm[];  // scale[C], shift[C]
  float* scale = sm;
  float* shift = sm + C;
  const int n = blockIdx.y;
  const int cpg = C / groups;
  const double cnt = (double)HW * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const double s = stats[((long long)n * groups + g) * 2 + 0];
    const double q = stats[((long long)n * groups + g) * 2 + 1];
    const double mean = s / cnt;
    double var = q / cnt - mean * mean;
    if (var < 0) var = 0;
    const float rstd = (float)(1.0 / sqrt(var + (double)eps));
    const float ga = gamma[c] * rstd;
    scale[c] = ga;
    shift[c] = beta[c] - (float)mean * ga;
  }
  __syncthreads();
  const int c8 = C >> 3;
  const long long p_begin = (long long)blockIdx.x * pix_per_block;
  const long long work = (long long)min((long long)pix_per_block, HW - p_begin) * c8;
  const long long ob = ((long long)n * HW + p_begin) * C;
  for (long long i = threadIdx.x; i < work; i += blockDim.x) {
    const int cc = (int)(i % c8);
    const long long o = ob + i * 8;
    const float4 a = __ldg(reinterpret_cast<const float4*>(x + o));
    const float4 b = __ldg(reinterpret_cast<const float4*>(x + o) + 1);
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const float* dr = drop ? drop + (((long long)n * HW + p_begin + i / c8) / img_hw) * C + cc * 8 : nullptr;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = f[e] * scale[cc * 8 + e] + shift[cc * 8 + e];
      if (act == 1) y = y / (1.0f + __expf(-y));
      else if (act == 2) y = y > 0.f ? y : 0.2f * y;
      else if (act == 3) y = y > 0.f ? y : 0.f;
      if (dr) y *= dr[e];
      f[e] = y;
    }
    if (out) {
      reinterpret_cast<float4*>(out + o)[0] = make_float4(f[0], f[1], f[2], f[3]);
      reinterpret_cast<float4*>(out + o)[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    if (planes) {
      H8 hi, lo;
#pragma unroll
      for (int e = 0; e < 8; ++e) split_f16(f[e], hi.v[e], lo.v[e]);
      *reinterpret_cast<H8*>(planes + o) = hi;
      if (terms == 2) *reinterpret_cast<H8*>(planes + plane + o) = lo;
    }
  }
}

// Backward of a ShapeUNet encoder stage's input, [MaxPool2d(2) of] cat([x, e broadcast over H, W]), for the x part:
// dx[n,ih,iw,c] (+)= da[n,ih/2,iw/2,c] at the first maximum (row-major, as torch's max_pool2d) of its 2x2 window,
// 0 elsewhere and on a dropped odd row / column; without pooling dx = da's x channels.  One thread per element of
// dx, so any C; a gather, so no atomics.
__global__ void maxpool2_bcast_dx_kernel(const float* __restrict__ da, int da_ld, const float* __restrict__ x,
                                         float* __restrict__ dx, int accumulate, int H, int W, int C, int pool,
                                         long long total) {
  const int oh_n = pool ? H / 2 : H, ow_n = pool ? W / 2 : W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int iw = (int)(r % W); r /= W;
    const int ih = (int)(r % H);
    const int n = (int)(r / H);
    float g = 0.f;
    if (!pool) {
      g = da[(((long long)n * oh_n + ih) * ow_n + iw) * da_ld + c];
    } else {
      const int oh = ih >> 1, ow = iw >> 1;
      if (oh < oh_n && ow < ow_n) {
        const float* b = x + (((long long)n * H + 2 * oh) * W + 2 * ow) * C + c;
        const float v[4] = {b[0], b[C], b[(long long)W * C], b[(long long)W * C + C]};
        float best = v[0];
        int k = 0;
#pragma unroll
        for (int j = 1; j < 4; ++j)
          if (v[j] > best || isnan(v[j])) { best = v[j]; k = j; }
        if (k == (ih & 1) * 2 + (iw & 1)) g = da[(((long long)n * oh_n + oh) * ow_n + ow) * da_ld + c];
      }
    }
    dx[i] = accumulate ? dx[i] + g : g;
  }
}

// ... and for the broadcast part: partial per-image sums of da's channels [C, C+Ce) over a chunk of pixels, fixed
// order (a thread walks its pixels, the block's lanes are added in lane order) -> ws[n][chunk][Ce]
__global__ void bcast_sum_partial_kernel(const float* __restrict__ da, int da_ld, int C, int Ce, int hw,
                                         int pix_per_chunk, float* __restrict__ ws) {
  extern __shared__ float part[];  // [lanes][Ce]
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int lanes = blockDim.x >= Ce ? blockDim.x / Ce : 1;
  const int lane = threadIdx.x / (blockDim.x >= Ce ? Ce : blockDim.x);
  const int p0 = chunk * pix_per_chunk, p1 = min(hw, p0 + pix_per_chunk);
  if (lane < lanes) {
    for (int j = threadIdx.x % (blockDim.x >= Ce ? Ce : blockDim.x); j < Ce; j += blockDim.x) {
      float s = 0.f;
      for (int p = p0 + lane; p < p1; p += lanes) s += da[((long long)n * hw + p) * da_ld + C + j];
      part[lane * Ce + j] = s;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < Ce; j += blockDim.x) {
    float s = 0.f;
    for (int l = 0; l < lanes; ++l) s += part[l * Ce + j];
    ws[((long long)n * gridDim.x + chunk) * Ce + j] = s;
  }
}

__global__ void bcast_sum_final_kernel(const float* __restrict__ ws, int chunks, int n_img, int Ce,
                                       float* __restrict__ de, int accumulate) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_img * Ce) return;
  const int n = i / Ce, j = i % Ce;
  float s = 0.f;
  for (int k = 0; k < chunks; ++k) s += ws[((long long)n * chunks + k) * Ce + j];
  de[i] = accumulate ? de[i] + s : s;
}

// Adjoint of T2H_CVT_BILINEAR2X (nn.Upsample(x2, bilinear, align_corners=False)) as a gather: input row r receives
// from output rows 2r-1 .. 2r+2 the weights the forward gave it (same source-coordinate arithmetic, border clamps
// included), likewise for columns.  dy [n][2h][2w][c] -> dx [n][h][w][c], c % 4 == 0; fixed summation order.
__device__ __forceinline__ float bilinear_w(int o, int r, int n_in) {
  const float s = fmaxf(0.5f * (o + 0.5f) - 0.5f, 0.f);
  const int i0 = (int)s, i1 = min(i0 + 1, n_in - 1);
  const float l = s - i0;
  return (i0 == r ? 1.f - l : 0.f) + (i1 == r ? l : 0.f);
}

__global__ void bilinear2x_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int H, int W, int C,
                                      long long total) {
  const int c4 = C >> 2;
  const int H2 = 2 * H, W2 = 2 * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c4);
    long long r = i / c4;
    const int s = (int)(r % W); r /= W;
    const int h = (int)(r % H);
    const int n = (int)(r / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int oh = max(2 * h - 1, 0); oh <= min(2 * h + 2, H2 - 1); ++oh) {
      const float wh = bilinear_w(oh, h, H);
      if (wh == 0.f) continue;
      for (int ow = max(2 * s - 1, 0); ow <= min(2 * s + 2, W2 - 1); ++ow) {
        const float ww = bilinear_w(ow, s, W);
        if (ww == 0.f) continue;
        const float wgt = wh * ww;
        const float4 v = __ldg(reinterpret_cast<const float4*>(dy + (((long long)n * H2 + oh) * W2 + ow) * C) + cc);
        acc.x = fmaf(wgt, v.x, acc.x);
        acc.y = fmaf(wgt, v.y, acc.y);
        acc.z = fmaf(wgt, v.z, acc.z);
        acc.w = fmaf(wgt, v.w, acc.w);
      }
    }
    reinterpret_cast<float4*>(dx)[i] = acc;
  }
}

// Pixel cross-entropy (F.cross_entropy(reduction='none', ignore_index) of CrossEntropyLoss, cross_entropy_loss.py)
// over fp32 NHWC logits [pix][c] and int64 labels [pix], one pass: loss[0] += sum over labelled pixels of
// logsumexp(x) - x[label]; planes = fp16 [terms][pix][c_pad] of gscale (softmax(x) - onehot), 0 on ignored pixels
// and pad channels; colsum[c] += column sums of that gradient (conv_seg's bias gradient).  A label outside [0, c)
// contributes nothing (the caller rejects those that are not ignore_index before the launch).
// g = c_pad/8 rounded up to a power of two threads share a pixel (8 channels each) and reduce the row's max and
// sum with shuffles inside their group; blockDim is a multiple of g, so a thread always meets the same channels.
__global__ void ce_logits_kernel(const float* __restrict__ x, const long long* __restrict__ labels, long long npix,
                                 int C, int c_pad, int g, float gscale, double* __restrict__ loss,
                                 __half* __restrict__ planes, int terms, float* __restrict__ colsum) {
  extern __shared__ double cs_sm[];  // [c_pad]
  const int sub = threadIdx.x % g, lane = threadIdx.x / g, lanes = blockDim.x / g;
  const int c0 = sub * 8;
  const unsigned gmask = g == 32 ? 0xffffffffu : (((1u << g) - 1u) << ((threadIdx.x & 31) & ~(g - 1)));
  const long long plane = npix * c_pad;
  for (int c = threadIdx.x; c < c_pad; c += blockDim.x) cs_sm[c] = 0.0;
  __syncthreads();
  float cs[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  double acc = 0.0;
  for (long long p = (long long)blockIdx.x * lanes + lane; p < npix; p += (long long)gridDim.x * lanes) {
    const long long lab = __ldg(labels + p);
    const bool valid = lab >= 0 && lab < C;
    float v[8];
    float m = -INFINITY;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c0 + e;
      v[e] = c < C ? __ldg(x + p * C + c) : -INFINITY;
      m = fmaxf(m, v[e]);
    }
    for (int o = g >> 1; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(gmask, m, o));
    float s = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) s += c0 + e < C ? expf(v[e] - m) : 0.f;
    for (int o = g >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(gmask, s, o);
    if (c0 >= c_pad) continue;  // threads of the group past the padded row (g > c_pad / 8) only help reduce
    H8 hi, lo;
    float part = 0.f;
    const float inv = 1.f / s;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c0 + e;
      float gr = 0.f;
      if (valid && c < C) {
        const bool t = c == (int)lab;
        gr = gscale * (expf(v[e] - m) * inv - (t ? 1.f : 0.f));
        if (t) part -= v[e];
        cs[e] += gr;
      }
      split_f16(gr, hi.v[e], lo.v[e]);
    }
    if (valid && sub == 0) part += m + logf(s);
    acc += (double)part;
    if (planes) {
      *reinterpret_cast<H8*>(planes + p * c_pad + c0) = hi;
      if (terms == 2) *reinterpret_cast<H8*>(planes + plane + p * c_pad + c0) = lo;
    }
  }
  block_add(acc, loss);
  if (colsum) {
    if (c0 < c_pad) {
#pragma unroll
      for (int e = 0; e < 8; ++e) atomicAdd(&cs_sm[c0 + e], (double)cs[e]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&colsum[c], (float)cs_sm[c]);
  }
}

// ShapeAttrEmbedding backward (shape_attr_embedding_arch.py:23-36; LeakyReLU slope 0.01): one CTA walks the images
// in order, recomputes each image's forward exactly as shape_attr_embed_kernel does (pre-activations kept) and
// accumulates every parameter's gradient from d_out[b] into `grad` at the element offsets goff: per attribute i
// (W1_i [dim][cls_i], b1_i, W2_i [dim][dim], b2_i), then (Wf1 [out][n_attr*dim], bf1, Wf2 [out][out], bf2) -- the
// nn.Linear layouts.  A thread owns fixed gradient elements, images are added in order: deterministic, no atomics.
// The one-hot Linear's weight gradient is the column a_i of W1_i.
__global__ void shape_attr_embed_bwd_kernel(const long long* __restrict__ attr, const int* __restrict__ cls_off,
                                            const float* __restrict__ w1t, const float* __restrict__ b1,
                                            const float* __restrict__ w2, const float* __restrict__ b2,
                                            const float* __restrict__ wf1, const float* __restrict__ bf1,
                                            const float* __restrict__ wf2, const float* __restrict__ bf2,
                                            const float* __restrict__ d_out, float* __restrict__ grad,
                                            const long long* __restrict__ goff, int B, int A, int D, int O) {
  extern __shared__ float sm[];
  const int AD = A * D;
  float* p0 = sm;            // [AD] pre-activation of the per-attribute first layers
  float* h1 = p0 + AD;       // [AD] concatenated per-attribute embeddings
  float* pf = h1 + AD;       // [O]  pre-activation of the first fusion layer
  float* d = pf + O;         // [O]  d_out[b]
  float* dpf = d + O;        // [O]  d pf
  float* dh1 = dpf + O;      // [AD] d h1
  float* dp0 = dh1 + AD;     // [AD] d p0
  auto lr = [](float v) { return v >= 0.f ? v : 0.01f * v; };
  auto lrg = [](float v) { return v > 0.f ? 1.f : 0.01f; };
  const long long* gf = goff + 4 * A;
  for (int b = 0; b < B; ++b) {
    for (int t = threadIdx.x; t < AD; t += blockDim.x) {
      const int i = t / D, j = t - i * D;
      const long long a = attr[(long long)b * A + i];
      const int ncls = cls_off[i + 1] - cls_off[i];
      p0[t] = (a >= 0 && a < ncls) ? w1t[(long long)(cls_off[i] + a) * D + j] + b1[t] : 0.f;
    }
    for (int t = threadIdx.x; t < O; t += blockDim.x) d[t] = d_out[(long long)b * O + t];
    __syncthreads();
    for (int t = threadIdx.x; t < AD; t += blockDim.x) {
      const int i = t / D;
      const float* w = w2 + (long long)t * D;
      float s = 0.f;
      for (int k = 0; k < D; ++k) s = fmaf(w[k], lr(p0[i * D + k]), s);
      h1[t] = s + b2[t];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < O; t += blockDim.x) {
      const float* w = wf1 + (long long)t * AD;
      float s = 0.f;
      for (int k = 0; k < AD; ++k) s = fmaf(w[k], h1[k], s);
      pf[t] = s + bf1[t];
    }
    __syncthreads();
    // fusion[2]: dWf2 += d f^T, dbf2 += d; d f = Wf2^T d
    for (int t = threadIdx.x; t < O * O; t += blockDim.x) grad[gf[2] + t] += d[t / O] * lr(pf[t % O]);
    for (int t = threadIdx.x; t < O; t += blockDim.x) {
      grad[gf[3] + t] += d[t];
      float s = 0.f;
      for (int k = 0; k < O; ++k) s = fmaf(wf2[(long long)k * O + t], d[k], s);
      dpf[t] = s * lrg(pf[t]);
    }
    __syncthreads();
    // fusion[0]: dWf1 += dpf h1^T, dbf1 += dpf; d h1 = Wf1^T dpf
    for (int t = threadIdx.x; t < O * AD; t += blockDim.x) grad[gf[0] + t] += dpf[t / AD] * h1[t % AD];
    for (int t = threadIdx.x; t < O; t += blockDim.x) grad[gf[1] + t] += dpf[t];
    for (int t = threadIdx.x; t < AD; t += blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < O; ++k) s = fmaf(wf1[(long long)k * AD + t], dpf[k], s);
      dh1[t] = s;
    }
    __syncthreads();
    // attr_i[2]: dW2_i += dh1_i lrelu(p0_i)^T, db2_i += dh1_i
    for (int t = threadIdx.x; t < AD * D; t += blockDim.x) {
      const int i = t / (D * D), jk = t - i * D * D, j = jk / D, k = jk - j * D;
      grad[goff[4 * i + 2] + jk] += dh1[i * D + j] * lr(p0[i * D + k]);
    }
    for (int t = threadIdx.x; t < AD; t += blockDim.x) grad[goff[4 * (t / D) + 3] + t % D] += dh1[t];
    __syncthreads();
    // d p0_i = (W2_i^T dh1_i) * lrelu'(p0_i); attr_i[0]: column a_i of dW1_i and db1_i
    for (int t = threadIdx.x; t < AD; t += blockDim.x) {
      const int i = t / D, k = t - i * D;
      float s = 0.f;
      for (int j = 0; j < D; ++j) s = fmaf(w2[((long long)i * D + j) * D + k], dh1[i * D + j], s);
      dp0[t] = s * lrg(p0[t]);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < AD; t += blockDim.x) {
      const int i = t / D, j = t - i * D;
      const long long a = attr[(long long)b * A + i];
      const int ncls = cls_off[i + 1] - cls_off[i];
      if (a >= 0 && a < ncls) grad[goff[4 * i] + (long long)j * ncls + a] += dp0[t];
      grad[goff[4 * i + 1] + j] += dp0[t];
    }
    __syncthreads();
  }
}

// ---- routed multi-head cross-entropy (MultiHeadFCNHead + 18 CrossEntropyLoss(ignore_index=-1),
// hierarchy_inference_model.py:227-245): only the head of a position's own texture has a target there, so each
// position computes that one head's logits.  Rows are grouped by head with a stable counting sort; a row tile of
// one head stages that head's weights in shared memory chunk by chunk; the weight / bias gradients are fixed-order
// sums over the head's rows (no floating-point atomics, bitwise reproducible).
constexpr int kRouteMaxBins = 64;   // heads + the bin of rows without a target
constexpr int kRouteThreads = 256;
constexpr int kRouteOut = 2048;     // outputs per CTA (rows x channels, classes x channels): 8 per thread
constexpr int kRouteCls = 32;       // classes per staged weight chunk
constexpr int kRouteRB = 16;        // rows per staged chunk of the weight gradient

__device__ __forceinline__ int route_bin(const long long* __restrict__ tex, const long long* __restrict__ own,
                                         int r, int G, int ncls) {
  const long long k = tex[r], t = own[r];
  return (k >= 0 && k < G && t >= 0 && t < ncls) ? (int)k : G;
}

// stable counting sort of the rows by bin (one CTA of 1024 threads): order[slot] = row, off[b] = first slot of bin
// b (b = G: rows without a target), off[G+1] = M.  Within a 1024-row tile, a row's rank among the rows of its bin
// comes from __match_any_sync and per-warp counts, so rows keep their index order inside each bin.
__global__ void __launch_bounds__(1024) route_sort_kernel(const long long* __restrict__ tex,
                                                          const long long* __restrict__ own, int M, int G, int ncls,
                                                          int* __restrict__ order, int* __restrict__ off) {
  __shared__ int cnt[kRouteMaxBins], base[kRouteMaxBins];
  __shared__ int wc[32][kRouteMaxBins + 1];
  const int nb = G + 1, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int b = threadIdx.x; b < nb; b += blockDim.x) cnt[b] = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < M; r += blockDim.x) atomicAdd(&cnt[route_bin(tex, own, r, G, ncls)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int b = 0; b < nb; ++b) {
      base[b] = off[b] = s;
      s += cnt[b];
    }
    off[nb] = s;
  }
  __syncthreads();
  for (int t0 = 0; t0 < M; t0 += blockDim.x) {
    const int r = t0 + threadIdx.x;
    const int k = r < M ? route_bin(tex, own, r, G, ncls) : nb;  // nb: past the end, never stored
    for (int i = threadIdx.x; i < 32 * (kRouteMaxBins + 1); i += blockDim.x) (&wc[0][0])[i] = 0;
    __syncthreads();
    const unsigned same = __match_any_sync(0xffffffffu, k);
    const int rank = __popc(same & ((1u << lane) - 1u));
    if (rank == 0) wc[warp][k] = __popc(same);
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {  // exclusive scan over the warps, per bin
      int s = 0;
      for (int w = 0; w < 32; ++w) {
        const int c = wc[w][b];
        wc[w][b] = s;
        s += c;
      }
      cnt[b] = s;
    }
    __syncthreads();
    if (r < M) order[base[k] + wc[warp][k] + rank] = r;
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += blockDim.x) base[b] += cnt[b];
    __syncthreads();
  }
}

// One CTA = up to R slots of one bin (R * C <= kRouteOut).  For head k: logits = W_k y + b_k into dl (slot-major
// [M][ncls]), then per row (one warp) loss += logsumexp - logit_t and dl = gscale (softmax - onehot_t), then
// dy[row][k*C..] = dl W_k and every other channel of the row 0.  Bin G rows get an all-zero dy row.
__global__ void __launch_bounds__(kRouteThreads) route_rows_kernel(
    const float* __restrict__ y, const float* __restrict__ w, const float* __restrict__ bias,
    const long long* __restrict__ own, const int* __restrict__ order, const int* __restrict__ off, int G, int C,
    int ncls, int R, float gscale, double* __restrict__ loss, float* __restrict__ dl, float* __restrict__ dy) {
  extern __shared__ float rsm[];
  const int ld = C + 1;              // odd row pitch: a warp reading one channel of 32 classes is conflict-free
  float* ys = rsm;                   // [R][ld]  the tile's rows of the head's C channels
  float* ws = ys + R * ld;           // [kRouteCls][ld]  a chunk of W_k
  float* ds = ws + kRouteCls * ld;   // [R][kRouteCls]   the same chunk of dl
  int t = blockIdx.x, k = -1, s0 = 0, n = 0;
  for (int b = 0; b <= G; ++b) {
    const int nb = off[b + 1] - off[b], tiles = (nb + R - 1) / R;
    if (t < tiles) {
      k = b;
      s0 = off[b] + t * R;
      n = min(R, nb - t * R);
      break;
    }
    t -= tiles;
  }
  if (k < 0) return;  // grid upper bound: no tile left (uniform over the CTA)
  const long long GC = (long long)G * C;
  if (k == G) {
    for (long long i = threadIdx.x; i < n * GC; i += blockDim.x) {
      const int r = (int)(i / GC);
      dy[(long long)order[s0 + r] * GC + (i - r * GC)] = 0.f;
    }
    return;
  }
  const float* wk = w + (long long)k * ncls * C;
  const float* bk = bias + (long long)k * ncls;
  for (int i = threadIdx.x; i < R * C; i += blockDim.x) {
    const int r = i / C, j = i - r * C;
    ys[r * ld + j] = r < n ? y[(long long)order[s0 + r] * GC + (long long)k * C + j] : 0.f;
  }
  for (int c0 = 0; c0 < ncls; c0 += kRouteCls) {
    __syncthreads();
    for (int i = threadIdx.x; i < kRouteCls * C; i += blockDim.x) {
      const int cc = i / C, j = i - cc * C;
      ws[cc * ld + j] = c0 + cc < ncls ? wk[(long long)(c0 + cc) * C + j] : 0.f;
    }
    __syncthreads();
    for (int p = threadIdx.x; p < n * kRouteCls; p += blockDim.x) {
      const int r = p / kRouteCls, cc = p - r * kRouteCls;
      if (c0 + cc >= ncls) continue;
      const float* yr = ys + r * ld;
      const float* wr = ws + cc * ld;
      float s = 0.f;
      for (int j = 0; j < C; ++j) s = fmaf(wr[j], yr[j], s);
      dl[(long long)(s0 + r) * ncls + c0 + cc] = s + bk[c0 + cc];
    }
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  double acc = 0.0;
  for (int r = threadIdx.x >> 5; r < n; r += nw) {
    float* row = dl + (long long)(s0 + r) * ncls;
    const int tgt = (int)own[order[s0 + r]];
    float m = -INFINITY;
    for (int c = lane; c < ncls; c += 32) m = fmaxf(m, row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < ncls; c += 32) s += expf(row[c] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float xt = row[tgt];
    __syncwarp();  // every lane has read the target logit before any lane overwrites the row
    if (lane == 0) acc += (double)(m + logf(s) - xt);
    const float inv = 1.f / s;
    for (int c = lane; c < ncls; c += 32) row[c] = gscale * (expf(row[c] - m) * inv - (c == tgt ? 1.f : 0.f));
  }
  float a[kRouteOut / kRouteThreads];
#pragma unroll
  for (int e = 0; e < kRouteOut / kRouteThreads; ++e) a[e] = 0.f;
  for (int c0 = 0; c0 < ncls; c0 += kRouteCls) {
    __syncthreads();
    for (int i = threadIdx.x; i < kRouteCls * C; i += blockDim.x) {
      const int cc = i / C, j = i - cc * C;
      ws[cc * ld + j] = c0 + cc < ncls ? wk[(long long)(c0 + cc) * C + j] : 0.f;
    }
    for (int i = threadIdx.x; i < R * kRouteCls; i += blockDim.x) {
      const int r = i / kRouteCls, cc = i - r * kRouteCls;
      ds[i] = (r < n && c0 + cc < ncls) ? dl[(long long)(s0 + r) * ncls + c0 + cc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kRouteOut / kRouteThreads; ++e) {
      const int p = threadIdx.x + e * kRouteThreads;
      if (p < R * C) {
        const int r = p / C, j = p - r * C;
        float s = a[e];
        for (int cc = 0; cc < kRouteCls; ++cc) s = fmaf(ds[r * kRouteCls + cc], ws[cc * ld + j], s);
        a[e] = s;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < kRouteOut / kRouteThreads; ++e) {
    const int p = threadIdx.x + e * kRouteThreads;
    if (p < n * C) {
      const int r = p / C, j = p - r * C;
      dy[(long long)order[s0 + r] * GC + (long long)k * C + j] = a[e];
    }
  }
  for (long long i = threadIdx.x; i < n * GC; i += blockDim.x) {
    const int r = (int)(i / GC);
    const long long q = i - r * GC;
    if (q / C != k) dy[(long long)order[s0 + r] * GC + q] = 0.f;
  }
  block_add(acc, loss);
}

// grid (classes / CB, G), CB * C <= kRouteOut: dw[k][c][:] += sum over the head's slots (in slot order) of
// dl[slot][c] y[row][k*C..], db[k][c] += sum of dl[slot][c]; a head without rows adds exact zeros
__global__ void __launch_bounds__(kRouteThreads) route_wgrad_kernel(
    const float* __restrict__ y, const int* __restrict__ order, const int* __restrict__ off,
    const float* __restrict__ dl, int G, int C, int ncls, int CB, float* __restrict__ dw, float* __restrict__ db) {
  extern __shared__ float wsm[];
  float* ds = wsm;                 // [kRouteRB][CB]
  float* ys = ds + kRouteRB * CB;  // [kRouteRB][C]
  const int k = blockIdx.y, c0 = blockIdx.x * CB;
  const int nc = min(CB, ncls - c0);
  const int s_beg = off[k], s_end = off[k + 1];
  const long long GC = (long long)G * C;
  float a[kRouteOut / kRouteThreads];
#pragma unroll
  for (int e = 0; e < kRouteOut / kRouteThreads; ++e) a[e] = 0.f;
  float sb = 0.f;
  for (int s = s_beg; s < s_end; s += kRouteRB) {
    const int nr = min(kRouteRB, s_end - s);
    __syncthreads();
    for (int i = threadIdx.x; i < kRouteRB * CB; i += blockDim.x) {
      const int r = i / CB, cc = i - r * CB;
      ds[i] = (r < nr && cc < nc) ? dl[(long long)(s + r) * ncls + c0 + cc] : 0.f;
    }
    for (int i = threadIdx.x; i < kRouteRB * C; i += blockDim.x) {
      const int r = i / C, j = i - r * C;
      ys[i] = r < nr ? y[(long long)order[s + r] * GC + (long long)k * C + j] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kRouteOut / kRouteThreads; ++e) {
      const int p = threadIdx.x + e * kRouteThreads;
      if (p < CB * C) {
        const int cc = p / C, j = p - cc * C;
        float v = a[e];
#pragma unroll 4
        for (int r = 0; r < kRouteRB; ++r) v = fmaf(ds[r * CB + cc], ys[r * C + j], v);
        a[e] = v;
      }
    }
    if (threadIdx.x < CB) {
      for (int r = 0; r < kRouteRB; ++r) sb += ds[r * CB + threadIdx.x];
    }
  }
#pragma unroll
  for (int e = 0; e < kRouteOut / kRouteThreads; ++e) {
    const int p = threadIdx.x + e * kRouteThreads;
    if (p < nc * C) {
      const int cc = p / C, j = p - cc * C;
      dw[((long long)k * ncls + c0 + cc) * C + j] += a[e];
    }
  }
  if (threadIdx.x < nc) db[(long long)k * ncls + c0 + threadIdx.x] += sb;
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int t2h_norm_bwd(const float* x, const double* stats, const float* gamma, const float* beta, const float* dy,
                 const float* add, float* dx, void* dx_planes, int terms, float* dgamma, float* dbeta, double* ws,
                 int n, int hw, int c, int groups, float eps, int act, float* dx_colsum, int sums_ready,
                 t2h_stream_t stream) {
  return norm_bwd_impl(x, stats, gamma, beta, dy, add, dx, dx_planes, terms, dgamma, dbeta, ws, n, hw, c, groups, eps,
                       act, dx_colsum, sums_ready, nullptr, 1, stream);
}

int t2h_norm_bwd_drop(const float* x, const double* stats, const float* gamma, const float* beta, const float* dy,
                      const float* dy_scale, int img_hw, float* dx, void* dx_planes, int terms, float* dgamma,
                      float* dbeta, double* ws, int n, int hw, int c, int groups, float eps, int act,
                      t2h_stream_t stream) {
  T2H_CHECK_ARG(dy_scale, "norm_bwd_drop: dy_scale is required");
  return norm_bwd_impl(x, stats, gamma, beta, dy, nullptr, dx, dx_planes, terms, dgamma, dbeta, ws, n, hw, c, groups,
                       eps, act, nullptr, 0, dy_scale, img_hw, stream);
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

// ---- parsing-generator training (ParsingGenModel.optimize_parameters, parsing_gen_model.py:80-95)
int t2h_norm_apply_ex(const float* x, const double* stats, const float* gamma, const float* beta, const float* drop,
                      int img_hw, float* out, void* out_planes, int n, int hw, int c, int groups, float eps, int act,
                      int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && stats && gamma && beta && (out || out_planes) && n > 0 && hw > 0, "norm_apply_ex: bad args");
  T2H_CHECK_ARG(c % groups == 0 && c % 8 == 0 && c <= 4096, "norm_apply_ex: C=%d groups=%d unsupported", c, groups);
  T2H_CHECK_ARG(act >= 0 && act <= 3 && (!out_planes || terms == 1 || terms == 2), "norm_apply_ex: act=%d terms=%d",
                act, terms);
  T2H_CHECK_ARG(!drop || (img_hw > 0 && ((long long)n * hw) % img_hw == 0), "norm_apply_ex: img_hw=%d", img_hw);
  int blocks_x = ceil_div(num_sms() * 8, n);
  int ppb = ceil_div(hw, blocks_x);
  if (ppb < 16) ppb = 16;
  blocks_x = ceil_div(hw, ppb);
  norm_apply_ex_kernel<<<dim3(blocks_x, n), 256, 2 * c * sizeof(float), as_stream(stream)>>>(
      x, stats, gamma, beta, drop, img_hw, out, reinterpret_cast<__half*>(out_planes), hw, c, groups, eps, act, terms,
      (long long)n * hw * c, ppb);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_maxpool2_bcast_bwd(const float* da, int da_ld, const float* x, float* dx, int accumulate, float* de,
                           float* ws, int n, int h, int w, int c, int c_e, int pool, t2h_stream_t stream) {
  T2H_CHECK_ARG(da && n > 0 && h > 0 && w > 0 && c >= 0 && c_e >= 0 && da_ld >= c + c_e,
                "maxpool2_bcast_bwd: bad args");
  T2H_CHECK_ARG(!dx || (c > 0 && (x || !pool)), "maxpool2_bcast_bwd: dx needs c > 0 and, pooled, the saved x");
  T2H_CHECK_ARG(!c_e || (de && ws), "maxpool2_bcast_bwd: d_e needs de and ws");
  T2H_CHECK_ARG(!pool || (h >= 2 && w >= 2), "maxpool2_bcast_bwd: pooling needs H, W >= 2");
  cudaStream_t st = as_stream(stream);
  if (dx) {
    const long long total = (long long)n * h * w * c;
    maxpool2_bcast_dx_kernel<<<grid_cap(total, 256), 256, 0, st>>>(da, da_ld, x, dx, accumulate, h, w, c, pool,
                                                                    total);
    T2H_LAUNCH_OK();
  }
  if (c_e) {
    const int hw = (pool ? h / 2 : h) * (pool ? w / 2 : w);
    const int chunks = min(kBcastChunks, ceil_div(hw, 64));
    const int ppc = ceil_div(hw, chunks);
    const int block = 256;
    const int lanes = block >= c_e ? block / c_e : 1;
    const size_t smem = (size_t)lanes * c_e * sizeof(float);
    T2H_CHECK_ARG(smem <= 48 * 1024, "maxpool2_bcast_bwd: c_e=%d too large", c_e);
    bcast_sum_partial_kernel<<<dim3(chunks, n), block, smem, st>>>(da, da_ld, c, c_e, hw, ppc, ws);
    T2H_LAUNCH_OK();
    bcast_sum_final_kernel<<<ceil_div(n * c_e, 128), 128, 0, st>>>(ws, chunks, n, c_e, de, accumulate);
    T2H_LAUNCH_OK();
  }
  return T2H_OK;
}

int t2h_bilinear2x_bwd(const float* dy, float* dx, int n, int h, int w, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(dy && dx && n > 0 && h > 0 && w > 0 && c > 0 && c % 4 == 0, "bilinear2x_bwd: bad args");
  const long long total = (long long)n * h * w * (c / 4);
  bilinear2x_bwd_kernel<<<grid_cap(total, 256), 256, 0, as_stream(stream)>>>(dy, dx, h, w, c, total);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_ce_logits(const float* logits, const int64_t* labels, int n, int h, int w, int c, int c_pad, float gscale,
                  double* loss_sum, void* grad_planes, int terms, float* colsum, t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && labels && loss_sum && n > 0 && h > 0 && w > 0 && c > 0, "ce_logits: bad args");
  T2H_CHECK_ARG(c_pad >= c && c_pad % 8 == 0 && c_pad <= 256, "ce_logits: c=%d c_pad=%d", c, c_pad);
  T2H_CHECK_ARG(!grad_planes || terms == 1 || terms == 2, "ce_logits: terms=%d", terms);
  const long long npix = (long long)n * h * w;
  int g = 1;
  while (g < c_pad / 8) g <<= 1;
  const int block = 256;
  ce_logits_kernel<<<grid_cap(npix, block / g, 4), block, c_pad * sizeof(double), as_stream(stream)>>>(
      logits, reinterpret_cast<const long long*>(labels), npix, c, c_pad, g, gscale, loss_sum,
      reinterpret_cast<__half*>(grad_planes), terms, colsum);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_shape_attr_embed_bwd(const int64_t* attr, const int32_t* cls_off, const float* w1t, const float* b1,
                             const float* w2, const float* b2, const float* wf1, const float* bf1, const float* wf2,
                             const float* bf2, const float* d_out, float* grad, const int64_t* goff, int b,
                             int n_attr, int dim, int out_dim, t2h_stream_t stream) {
  T2H_CHECK_ARG(attr && cls_off && w1t && b1 && w2 && b2 && wf1 && bf1 && wf2 && bf2 && d_out && grad && goff,
                "shape_attr_embed_bwd: null operand");
  T2H_CHECK_ARG(b > 0 && n_attr > 0 && dim > 0 && out_dim > 0, "shape_attr_embed_bwd: bad shape");
  const size_t smem = (size_t)(4 * n_attr * dim + 3 * out_dim) * sizeof(float);
  T2H_CHECK_ARG(smem <= 48 * 1024, "shape_attr_embed_bwd: n_attr*dim=%d, out_dim=%d too large", n_attr * dim,
                out_dim);
  shape_attr_embed_bwd_kernel<<<1, 512, smem, as_stream(stream)>>>(
      reinterpret_cast<const long long*>(attr), cls_off, w1t, b1, w2, b2, wf1, bf1, wf2, bf2, d_out, grad,
      reinterpret_cast<const long long*>(goff), b, n_attr, dim, out_dim);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

// ---- index-prediction training (VQGANTextureAwareSpatialHierarchyInferenceModel.optimize_parameters)
int t2h_routed_head_ce(const float* y, const int64_t* tex, const int64_t* own, const float* w, const float* bias,
                       int64_t m, int g, int c, int ncls, float gscale, double* loss_sum, float* dy, float* dw,
                       float* db, int32_t* order, int32_t* off, float* dl, t2h_stream_t stream) {
  T2H_CHECK_ARG(y && tex && own && w && bias && loss_sum && dy && dw && db && order && off && dl,
                "routed_head_ce: null operand");
  T2H_CHECK_ARG(m > 0 && m <= 0x7fffffffLL && g >= 1 && g < kRouteMaxBins && ncls > 0,
                "routed_head_ce: m=%lld g=%d ncls=%d unsupported", (long long)m, g, ncls);
  T2H_CHECK_ARG(c >= 8 && c % 8 == 0 && c <= 512, "routed_head_ce: c=%d (a multiple of 8, at most 512)", c);
  cudaStream_t st = as_stream(stream);
  const int M = (int)m;
  route_sort_kernel<<<1, 1024, 0, st>>>(reinterpret_cast<const long long*>(tex),
                                        reinterpret_cast<const long long*>(own), M, g, ncls, order, off);
  T2H_LAUNCH_OK();
  const int R = min(64, kRouteOut / c);
  const size_t smem = (size_t)((R + kRouteCls) * (c + 1) + R * kRouteCls) * sizeof(float);
  if (smem > 48 * 1024)
    T2H_CUDA(cudaFuncSetAttribute(route_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  route_rows_kernel<<<(unsigned)(ceil_div64(m, R) + g + 1), kRouteThreads, smem, st>>>(
      y, w, bias, reinterpret_cast<const long long*>(own), order, off, g, c, ncls, R, gscale, loss_sum, dl, dy);
  T2H_LAUNCH_OK();
  const int CB = kRouteOut / c;
  route_wgrad_kernel<<<dim3(ceil_div(ncls, CB), g), kRouteThreads, (size_t)kRouteRB * (CB + c) * sizeof(float),
                       st>>>(y, order, off, dl, g, c, ncls, CB, dw, db);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

}  // extern "C"
