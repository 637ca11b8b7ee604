// Backward / optimiser kernels of the index-prediction transformer's training step
// (TransformerTextureAwareModel._train_loss / optimize_parameters, models/transformer_model.py:232-303).
// Every dense contraction of the backward pass (dgrad, wgrad, attention gradients) runs on the same
// wgmma tap-GEMM as the forward pass; this file holds the HBM-bound pieces around them: operand
// transposes (wgrad contracts over rows, so both operands are needed row-contiguous), GELU / LayerNorm /
// softmax backward, the masked multi-head cross-entropy, embedding scatter-add, column sums (bias
// gradients) and Adam.
#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

// fp32 [G][R][C] -> fp16 planes of scale*x, transposed: out_t[t][g][c][r] (and optionally the untransposed
// planes out_n).  64x64 tiles; 8-byte loads, 4-byte stores when R and C are even (else a scalar tail path).
__global__ void f32_to_planes_t_kernel(const float* __restrict__ x, __half* __restrict__ out_t,
                                       __half* __restrict__ out_n, int R, int C, int terms, long long plane,
                                       float scale) {
  __shared__ float tile[64][65];
  const int g = blockIdx.z;
  const int r0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const float* xg = x + (long long)g * R * C;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  const bool vec_c = (C & 1) == 0, vec_r = (R & 1) == 0;
  for (int i = ty; i < 64; i += 8) {
    const int r = r0 + i, c = c0 + 2 * tx;
    float v0 = 0.f, v1 = 0.f;
    if (r < R) {
      if (vec_c && c + 1 < C) {
        const float2 v = *reinterpret_cast<const float2*>(xg + (long long)r * C + c);
        v0 = v.x * scale;
        v1 = v.y * scale;
      } else {
        if (c < C) v0 = xg[(long long)r * C + c] * scale;
        if (c + 1 < C) v1 = xg[(long long)r * C + c + 1] * scale;
      }
    }
    tile[i][2 * tx] = v0;
    tile[i][2 * tx + 1] = v1;
    if (out_n && r < R && c < C) {
      __half h0, l0, h1, l1;
      split_f16(v0, h0, l0);
      split_f16(v1, h1, l1);
      const long long o = (long long)g * R * C + (long long)r * C + c;
      if (vec_c && c + 1 < C) {
        *reinterpret_cast<__half2*>(out_n + o) = __halves2half2(h0, h1);
        if (terms == 2) *reinterpret_cast<__half2*>(out_n + plane + o) = __halves2half2(l0, l1);
      } else {
        out_n[o] = h0;
        if (terms == 2) out_n[plane + o] = l0;
        if (c + 1 < C) {
          out_n[o + 1] = h1;
          if (terms == 2) out_n[plane + o + 1] = l1;
        }
      }
    }
  }
  if (!out_t) return;  // plain conversion only (uniform across the grid)
  __syncthreads();
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i, r = r0 + 2 * tx;
    if (c < C && r < R) {
      __half h0, l0, h1, l1;
      split_f16(tile[2 * tx][i], h0, l0);
      split_f16(tile[2 * tx + 1][i], h1, l1);
      const long long o = (long long)g * R * C + (long long)c * R + r;
      if (vec_r && r + 1 < R) {
        *reinterpret_cast<__half2*>(out_t + o) = __halves2half2(h0, h1);
        if (terms == 2) *reinterpret_cast<__half2*>(out_t + plane + o) = __halves2half2(l0, l1);
      } else {
        out_t[o] = h0;
        if (terms == 2) out_t[plane + o] = l0;
        if (r + 1 < R) {
          out_t[o + 1] = h1;
          if (terms == 2) out_t[plane + o + 1] = l1;
        }
      }
    }
  }
}

// fp16 planes [T][G][R][C] (row stride ld, column offset applied by the caller) -> [T][G][C][R].
// 64x64 tiles, one plane per blockIdx.z slice; 4-byte accesses when the strides and bases allow it.
__global__ void planes_transpose_kernel(const __half* __restrict__ x, __half* __restrict__ out, int R, int C,
                                        long long ld, long long g_stride, long long in_plane, int G,
                                        long long out_ld, long long out_g_stride, long long out_plane, int vec_in,
                                        int vec_out) {
  __shared__ __half tile[64][66];
  const int t = blockIdx.z / G, g = blockIdx.z - t * G;
  const int r0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  const __half* xg = x + t * in_plane + (long long)g * g_stride;
  __half* og = out + t * out_plane + (long long)g * out_g_stride;
  const __half zero = __float2half(0.f);
  for (int i = ty; i < 64; i += 8) {
    const int r = r0 + i, c = c0 + 2 * tx;
    __half a = zero, b = zero;
    if (r < R) {
      if (vec_in && c + 1 < C) {
        const __half2 v = *reinterpret_cast<const __half2*>(xg + (long long)r * ld + c);
        a = __low2half(v);
        b = __high2half(v);
      } else {
        if (c < C) a = xg[(long long)r * ld + c];
        if (c + 1 < C) b = xg[(long long)r * ld + c + 1];
      }
    }
    *reinterpret_cast<__half2*>(&tile[i][2 * tx]) = __halves2half2(a, b);
  }
  __syncthreads();
  for (int i = ty; i < 64; i += 8) {
    const int c = c0 + i, r = r0 + 2 * tx;
    if (c < C && r < R) {
      const __half a = tile[2 * tx][i], b = tile[2 * tx + 1][i];
      __half* o = og + (long long)c * out_ld + r;
      if (vec_out && r + 1 < R) {
        *reinterpret_cast<__half2*>(o) = __halves2half2(a, b);
      } else {
        o[0] = a;
        if (r + 1 < R) o[1] = b;
      }
    }
  }
}

// out[c] += sum_r x[r][c]
__global__ void colsum_kernel(const float* __restrict__ x, float* __restrict__ out, long long R, int C,
                              int rows_per_block) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = min(R, r0 + rows_per_block);
  float s = 0.f;
  for (long long r = r0; r < r1; ++r) s += x[r * C + c];
  atomicAdd(&out[c], s);
}

// exact-erf GELU: g = gelu(a) -> planes;  backward: da = dg * gelu'(a)
__global__ void gelu_fwd_kernel(const float* __restrict__ a, __half* __restrict__ out, long long n, int terms,
                                long long plane) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    __half hi, lo;
    split_f16(gelu_erf(a[i]), hi, lo);
    out[i] = hi;
    if (terms == 2) out[plane + i] = lo;
  }
}
__global__ void gelu_bwd_kernel(const float* __restrict__ a, const float* __restrict__ dg,
                                float* __restrict__ da, long long n, __half* __restrict__ da_planes, int terms) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float x = a[i];
    const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
    const float pdf = 0.39894228040143267794f * expf(-0.5f * x * x);
    const float g = dg[i] * (cdf + x * pdf);
    da[i] = g;  // fp32 copy for the bias gradient (colsum)
    if (da_planes) {
      __half hi, lo;
      split_f16(g, hi, lo);
      da_planes[i] = hi;
      if (terms == 2) da_planes[n + i] = lo;
    }
  }
}

// LayerNorm backward, one warp per row (C <= 1024): dx = rstd*(g - mean(g) - xhat*mean(g*xhat)), g = dy*gamma;
// dx (+)= into dx_out (accumulate flag), dgamma += dy*xhat, dbeta += dy (atomics)
template <int PER_LANE>
__global__ void layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                     const float* __restrict__ gamma, float* __restrict__ dx,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta, long long rows, int C,
                                     float eps, int accumulate, __half* __restrict__ dx_planes, int terms,
                                     float* __restrict__ dx_colsum) {
  // optional fused outputs: fp16 planes of the updated dx (the operand of the next backward GEMMs) and its
  // column sums (the bias gradient of the linear layer whose output this dx is the gradient of)
  __shared__ float s_dg[PER_LANE * 32], s_db[PER_LANE * 32], s_cs[PER_LANE * 32];
  for (int i = threadIdx.x; i < PER_LANE * 32; i += blockDim.x) {
    s_dg[i] = 0.f;
    s_db[i] = 0.f;
    s_cs[i] = 0.f;
  }
  __syncthreads();
  const int warps = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  float dg_acc[PER_LANE], db_acc[PER_LANE], cs_acc[PER_LANE], gam[PER_LANE];
  const long long plane = rows * C;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    dg_acc[i] = 0.f;
    db_acc[i] = 0.f;
    cs_acc[i] = 0.f;
    gam[i] = c < C ? gamma[c] : 0.f;
  }
  // each warp walks rows with a grid stride and keeps its dgamma/dbeta partial sums in registers
  for (long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5); row < rows;
       row += (long long)gridDim.x * warps) {
    const float* xr = x + row * C;
    const float* dyr = dy + row * C;
    float xv[PER_LANE], gv[PER_LANE];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      xv[i] = c < C ? xr[c] : 0.f;
      sum += xv[i];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      const float d = c < C ? xv[i] - mean : 0.f;
      sq += d * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / C + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      if (c < C) {
        const float xhat = (xv[i] - mean) * rstd;
        const float d = dyr[c];
        xv[i] = xhat;
        gv[i] = d * gam[i];
        s1 += gv[i];
        s2 += gv[i] * xhat;
        dg_acc[i] += d * xhat;
        db_acc[i] += d;
      } else {
        gv[i] = 0.f;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 / C, m2 = s2 / C;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int c = lane + i * 32;
      if (c < C) {
        float v = rstd * (gv[i] - m1 - xv[i] * m2);
        if (accumulate) v += dx[row * C + c];
        dx[row * C + c] = v;
        cs_acc[i] += v;
        if (dx_planes) {
          __half hi, lo;
          split_f16(v, hi, lo);
          dx_planes[row * C + c] = hi;
          if (terms == 2) dx_planes[plane + row * C + c] = lo;
        }
      }
    }
  }
  // warp partials -> block partials in shared memory -> one global atomic per column per block
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    if (c < C) {
      atomicAdd(&s_dg[c], dg_acc[i]);
      atomicAdd(&s_db[c], db_acc[i]);
      if (dx_colsum) atomicAdd(&s_cs[c], cs_acc[i]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(&dgamma[c], s_dg[c]);
    atomicAdd(&dbeta[c], s_db[c]);
    if (dx_colsum) atomicAdd(&dx_colsum[c], s_cs[c]);
  }
}

// softmax backward over the last dim: ds = scale * p * (dp - sum_j dp_j p_j); p given as fp16 planes.
// One warp per row; each lane owns column pairs (4-byte p loads, 8-byte dp/ds accesses); cols must be even.
template <int PAIRS>
__global__ void softmax_bwd_kernel(const __half* __restrict__ p, const float* __restrict__ dp,
                                   float* __restrict__ ds, long long rows, int cols, float scale, int terms,
                                   long long plane, __half* __restrict__ ds_planes, float out_scale) {
  const int warps = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const __half2* ph = reinterpret_cast<const __half2*>(p + row * cols);
  const __half2* pl = reinterpret_cast<const __half2*>(p + plane + row * cols);
  const float2* dpr = reinterpret_cast<const float2*>(dp + row * cols);
  float2* dsr = reinterpret_cast<float2*>(ds + row * cols);
  const int npairs = cols >> 1;
  float2 pv[PAIRS], dv[PAIRS];
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < PAIRS; ++i) {
    const int c = lane + i * 32;
    if (c < npairs) {
      float2 v = __half22float2(ph[c]);
      if (terms == 2) {
        const float2 l = __half22float2(pl[c]);
        v.x += l.x;
        v.y += l.y;
      }
      pv[i] = v;
      dv[i] = dpr[c];
      dot += v.x * dv[i].x + v.y * dv[i].y;
    } else {
      pv[i] = make_float2(0.f, 0.f);
      dv[i] = make_float2(0.f, 0.f);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
#pragma unroll
  for (int i = 0; i < PAIRS; ++i) {
    const int c = lane + i * 32;
    if (c < npairs) {
      const float a = scale * pv[i].x * (dv[i].x - dot), b = scale * pv[i].y * (dv[i].y - dot);
      if (ds_planes) {
        // straight to the fp16 planes (x out_scale) the dQ / dK GEMMs consume: no fp32 round trip
        __half h0, l0, h1, l1;
        split_f16(a * out_scale, h0, l0);
        split_f16(b * out_scale, h1, l1);
        reinterpret_cast<__half2*>(ds_planes + row * cols)[c] = __halves2half2(h0, h1);
        if (terms == 2) reinterpret_cast<__half2*>(ds_planes + plane + row * cols)[c] = __halves2half2(l0, l1);
      } else {
        dsr[c] = make_float2(a, b);
      }
    }
  }
}

// Masked multi-head cross-entropy (transformer_model.py:250-270): row m belongs to head head[m]; its target
// is target[m] (-1 = not masked = ignored).  loss_rows[m] = CE (unweighted), dlogits = w[m] * (softmax - onehot)
// inside the row's own head, 0 in every other head.  One block per row.
__global__ void ce_heads_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                                const long long* __restrict__ head, const float* __restrict__ w,
                                float* __restrict__ loss_rows, float* __restrict__ dlogits, int nh, int ncls) {
  const long long m = blockIdx.x;
  const int tid = threadIdx.x;
  const long long tgt = target[m];
  const int hd = (int)head[m];
  float* drow = dlogits + m * (long long)nh * ncls;
  for (int i = tid; i < nh * ncls; i += blockDim.x) drow[i] = 0.f;
  if (tgt < 0 || hd < 0 || hd >= nh) {
    if (tid == 0) loss_rows[m] = 0.f;
    return;
  }
  __shared__ float red[32];
  const float* lr = logits + m * (long long)nh * ncls + (long long)hd * ncls;
  float mx = -INFINITY;
  for (int i = tid; i < ncls; i += blockDim.x) mx = fmaxf(mx, lr[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = tid; i < ncls; i += blockDim.x) sum += expf(lr[i] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) sum += red[i];
  const float lse = mx + logf(sum);
  const float wm = w[m];
  __syncthreads();  // drow zero-fill above must be complete before the own-head slice is overwritten
  for (int i = tid; i < ncls; i += blockDim.x)
    drow[(long long)hd * ncls + i] = wm * (expf(lr[i] - lse) - (i == tgt ? 1.f : 0.f));
  if (tid == 0) loss_rows[m] = lse - lr[tgt];  // unweighted; the caller forms loss and vb_loss from it
}

// dE[idx[m]] += dx[m]  (embedding backward; also the positional table with idx = m % T)
__global__ void embed_bwd_kernel(const float* __restrict__ dx, const long long* __restrict__ idx,
                                 float* __restrict__ dE, long long rows, int C, int T_mod) {
  const long long m = blockIdx.x;
  if (m >= rows) return;
  const long long e = idx ? idx[m] : (m % T_mod);
  for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(&dE[e * C + c], dx[m * C + c]);
}

// torch.optim.Adam (weight_decay 0, amsgrad off), fp32
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, float lr, float b1, float b2, float eps,
                            float bc1, float bc2_sqrt, float grad_scale) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * grad_scale;
    // a gradient that overflowed the fp16 operand planes of the backward GEMMs (static loss scale) arrives as inf / NaN:
    // leave that element's parameter and moments untouched instead of poisoning them for good
    if (!isfinite(gi)) continue;
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] -= (lr / bc1) * (mi / denom);
  }
}

static inline int grid1d(long long n, int block) {
  long long g = (n + block - 1) / block;
  const long long cap = (long long)num_sms() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int t2h_f32_to_planes_t(const float* x, void* out_t, void* out_n, int g, int r, int c, int terms, float scale,
                        t2h_stream_t stream) {
  T2H_CHECK_ARG(x && (out_t || out_n) && g > 0 && r > 0 && c > 0, "f32_to_planes_t: bad args");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "f32_to_planes_t: terms=%d", terms);
  dim3 grid(ceil_div(r, 64), ceil_div(c, 64), g), block(32, 8);
  f32_to_planes_t_kernel<<<grid, block, 0, as_stream(stream)>>>(
      x, reinterpret_cast<__half*>(out_t), reinterpret_cast<__half*>(out_n), r, c, terms, (long long)g * r * c,
      scale);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_planes_transpose(const void* x, void* out, int g, int r, int c, int64_t ld, int64_t g_stride,
                         int64_t in_plane, int64_t out_ld, int64_t out_g_stride, int64_t out_plane, int terms,
                         t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && g > 0 && r > 0 && c > 0 && ld >= c && out_ld >= r, "planes_transpose: bad args");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "planes_transpose: terms=%d", terms);
  T2H_CHECK_ARG((long long)g * terms <= 65535, "planes_transpose: too many groups");
  dim3 grid(ceil_div(r, 64), ceil_div(c, 64), g * terms), block(32, 8);
  // 4-byte accesses need even strides / offsets everywhere a half2 is formed
  const int vec_in = (reinterpret_cast<uintptr_t>(x) % 4 == 0) && ld % 2 == 0 && g_stride % 2 == 0 && in_plane % 2 == 0;
  const int vec_out = (reinterpret_cast<uintptr_t>(out) % 4 == 0) && out_ld % 2 == 0 && out_g_stride % 2 == 0 &&
                      out_plane % 2 == 0;
  planes_transpose_kernel<<<grid, block, 0, as_stream(stream)>>>(
      reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(out), r, c, ld, g_stride, in_plane, g,
      out_ld, out_g_stride, out_plane, vec_in, vec_out);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_colsum(const float* x, float* out, int64_t rows, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && rows > 0 && c > 0, "colsum: bad args");
  int rpb = 64;  // (tests/test_gpu_row_kernels.py::colsum_route restates this grid)
  if (ceil_div64(rows, rpb) > 16384) rpb = (int)ceil_div64(rows, 16384);  // grid.y limit; conv bias gradients have millions of rows
  dim3 grid(ceil_div(c, 128), (unsigned)ceil_div64(rows, rpb));
  colsum_kernel<<<grid, 128, 0, as_stream(stream)>>>(x, out, rows, c, rpb);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_gelu_fwd(const float* a, void* out, int64_t n, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(a && out && n > 0 && (terms == 1 || terms == 2), "gelu_fwd: bad args");
  gelu_fwd_kernel<<<grid1d(n, 256), 256, 0, as_stream(stream)>>>(a, reinterpret_cast<__half*>(out), n, terms, n);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_gelu_bwd(const float* a, const float* dg, float* da, void* da_planes, int64_t n, int terms,
                 t2h_stream_t stream) {
  T2H_CHECK_ARG(a && dg && da && n > 0 && (!da_planes || terms == 1 || terms == 2), "gelu_bwd: bad args");
  gelu_bwd_kernel<<<grid1d(n, 256), 256, 0, as_stream(stream)>>>(a, dg, da, n, reinterpret_cast<__half*>(da_planes),
                                                                terms);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

static int layernorm_bwd_impl(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                              float* dbeta, int64_t rows, int c, float eps, int accumulate, void* dx_planes, int terms,
                              float* dx_colsum, t2h_stream_t stream);

int t2h_layernorm_bwd(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                      float* dbeta, int64_t rows, int c, float eps, int accumulate, t2h_stream_t stream) {
  return layernorm_bwd_impl(dy, x, gamma, dx, dgamma, dbeta, rows, c, eps, accumulate, nullptr, 1, nullptr, stream);
}

int t2h_layernorm_bwd_fused(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                            float* dbeta, int64_t rows, int c, float eps, int accumulate, void* dx_planes, int terms,
                            float* dx_colsum, t2h_stream_t stream) {
  T2H_CHECK_ARG(!dx_planes || terms == 1 || terms == 2, "layernorm_bwd_fused: terms=%d", terms);
  return layernorm_bwd_impl(dy, x, gamma, dx, dgamma, dbeta, rows, c, eps, accumulate, dx_planes, terms, dx_colsum,
                            stream);
}

static int layernorm_bwd_impl(const float* dy, const float* x, const float* gamma, float* dx, float* dgamma,
                              float* dbeta, int64_t rows, int c, float eps, int accumulate, void* dx_planes, int terms,
                              float* dx_colsum, t2h_stream_t stream) {
  T2H_CHECK_ARG(dy && x && gamma && dx && dgamma && dbeta && rows > 0 && c > 0, "layernorm_bwd: bad args");
  T2H_CHECK_ARG(c <= 1024, "layernorm_bwd: C=%d > 1024 unsupported", c);
  // (tests/test_gpu_row_kernels.py::layernorm_bwd_route restates the grid and the choice of kernel below)
  const int warps = 8;
  long long want = ceil_div64(rows, warps * 2);  // 2 rows per warp, 16 per block: enough warps in flight to
  const int grid = (int)(want < 1 ? 1 : want);   // cover HBM latency, 16x fewer global atomics than per-row
  cudaStream_t st = as_stream(stream);
  if (c <= 512)
    layernorm_bwd_kernel<16><<<grid, warps * 32, 0, st>>>(dy, x, gamma, dx, dgamma, dbeta, rows, c, eps, accumulate,
                                                          reinterpret_cast<__half*>(dx_planes), terms, dx_colsum);
  else
    layernorm_bwd_kernel<32><<<grid, warps * 32, 0, st>>>(dy, x, gamma, dx, dgamma, dbeta, rows, c, eps, accumulate,
                                                          reinterpret_cast<__half*>(dx_planes), terms, dx_colsum);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

static int softmax_bwd_impl(const void* p, const float* dp, float* ds, void* ds_planes, float out_scale, int64_t rows,
                            int cols, float scale, int terms, t2h_stream_t stream);

int t2h_softmax_bwd(const void* p, const float* dp, float* ds, int64_t rows, int cols, float scale, int terms,
                    t2h_stream_t stream) {
  T2H_CHECK_ARG(ds, "softmax_bwd: null output");
  return softmax_bwd_impl(p, dp, ds, nullptr, 1.f, rows, cols, scale, terms, stream);
}

int t2h_softmax_bwd_planes(const void* p, const float* dp, void* ds_planes, int64_t rows, int cols, float scale,
                           int terms, float out_scale, t2h_stream_t stream) {
  T2H_CHECK_ARG(ds_planes, "softmax_bwd_planes: null output");
  return softmax_bwd_impl(p, dp, nullptr, ds_planes, out_scale, rows, cols, scale, terms, stream);
}

static int softmax_bwd_impl(const void* p, const float* dp, float* ds, void* ds_planes, float out_scale, int64_t rows,
                            int cols, float scale, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(p && dp && (ds || ds_planes) && rows > 0 && cols > 0 && cols <= 2048 && cols % 2 == 0,
                "softmax_bwd: bad args (cols must be even and <= 2048)");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "softmax_bwd: terms=%d", terms);
  const int warps = 4;
  const int grid = (int)ceil_div64(rows, warps);
  cudaStream_t st = as_stream(stream);
  const __half* ph = reinterpret_cast<const __half*>(p);
  // (tests/test_gpu_row_kernels.py::softmax_bwd_route restates this choice)
  if (cols <= 512)
    softmax_bwd_kernel<8><<<grid, warps * 32, 0, st>>>(ph, dp, ds, rows, cols, scale, terms, rows * cols,
                                                      reinterpret_cast<__half*>(ds_planes), out_scale);
  else
    softmax_bwd_kernel<32><<<grid, warps * 32, 0, st>>>(ph, dp, ds, rows, cols, scale, terms, rows * cols,
                                                       reinterpret_cast<__half*>(ds_planes), out_scale);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_ce_heads(const float* logits, const int64_t* target, const int64_t* head, const float* w,
                 float* loss_rows, float* dlogits, int64_t rows, int nh, int ncls, t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && target && head && w && loss_rows && dlogits && rows > 0 && nh > 0 && ncls > 0,
                "ce_heads: bad args");
  ce_heads_kernel<<<(unsigned)rows, 256, 0, as_stream(stream)>>>(
      logits, reinterpret_cast<const long long*>(target), reinterpret_cast<const long long*>(head), w, loss_rows,
      dlogits, nh, ncls);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_embed_bwd(const float* dx, const int64_t* idx, float* de, int64_t rows, int c, int t_mod,
                  t2h_stream_t stream) {
  T2H_CHECK_ARG(dx && de && rows > 0 && c > 0 && (idx || t_mod > 0), "embed_bwd: bad args");
  embed_bwd_kernel<<<(unsigned)rows, 128, 0, as_stream(stream)>>>(dx, reinterpret_cast<const long long*>(idx), de,
                                                                rows, c, t_mod);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
             float eps, int step, float grad_scale, t2h_stream_t stream) {
  T2H_CHECK_ARG(p && g && m && v && n > 0 && step >= 1, "adam: bad args");
  // bias corrections in double (as torch does): 1 - beta^step loses ~1e-5 relative in fp32 at small step counts
  const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  const float bc2s = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  adam_kernel<<<grid1d(n, 256), 256, 0, as_stream(stream)>>>(p, g, m, v, n, lr, beta1, beta2, eps, bc1, bc2s,
                                                            grad_scale);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

}  // extern "C"
