// The parts of LPIPS (lpips==0.1.4, net='vgg', version='0.1'; used by models/vqgan_model.py:427,450 and
// models/hierarchy_vqgan_model.py:90,253) that are not VGG16 convolutions: the input ScalingLayer and its
// adjoint, the fused per-slice head (channel-unit normalisation, squared difference, 1x1 "lin" weights, spatial
// mean, and the head's gradient with respect to the xrec features) and the plain ReLU backward inside a slice.
// The 3x3 convolutions of the VGG trunk and their data gradients run on t2h_tapgemm (gemm_tc.cu).
#include <cuda_fp16.h>

#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

namespace {

inline int grid_cap(long long work, int block, int per_sm = 16) {
  long long g = ceil_div64(work, block);
  long long cap = (long long)num_sms() * per_sm;
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}

// warps per block of the head kernel, and the largest channel count a lane's registers hold (16 channels per lane)
constexpr int kHeadWarps = 8;
constexpr int kHeadMaxC = 512;
constexpr int kHeadQ = kHeadMaxC / 128;  // float4 slots per lane

}  // namespace

// (x - shift[c]) / scale[c] of two fp32 NCHW images [b][3][hw] -> planes [terms][2b][hw][8]: images [0,b) from x0,
// [b,2b) from x1, channels 3..7 zero (conv1_1's operand, zero padded after the scaling as nn.Conv2d pads)
__global__ void lpips_scale_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ x1,
                                       const float* __restrict__ shift, const float* __restrict__ scale,
                                       __half* __restrict__ out, int b, long long hw, int terms) {
  const long long total = 2LL * b * hw;
  const float s0 = shift[0], s1 = shift[1], s2 = shift[2];
  const float r0 = 1.f / scale[0], r1 = 1.f / scale[1], r2 = 1.f / scale[2];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hw, p = i % hw;
    const float* x = n < b ? x0 + n * 3 * hw : x1 + (n - b) * 3 * hw;
    const float v[3] = {(__ldg(x + p) - s0) * r0, (__ldg(x + hw + p) - s1) * r1, (__ldg(x + 2 * hw + p) - s2) * r2};
    __align__(16) __half hi[8], lo[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      hi[c] = lo[c] = __float2half_rn(0.f);
      if (c < 3) split_f16(v[c], hi[c], lo[c]);
    }
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(hi);
    if (terms == 2) reinterpret_cast<uint4*>(out)[total + i] = *reinterpret_cast<const uint4*>(lo);
  }
}

// g[n][c][p] += alpha * d[n][p][c] / scale[c] for c < 3: the ScalingLayer's adjoint, d the data gradient of
// conv1_1 (fp32 NHWC, row stride ld)
__global__ void lpips_scale_bwd_kernel(const float* __restrict__ d, int ld, const float* __restrict__ scale,
                                       float alpha, float* __restrict__ g, int b, long long hw) {
  const long long total = 3LL * b * hw;
  const float k0 = alpha / scale[0], k1 = alpha / scale[1], k2 = alpha / scale[2];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % hw, r = i / hw;
    const int c = (int)(r % 3);
    const long long n = r / 3;
    g[i] += (c == 0 ? k0 : (c == 1 ? k1 : k2)) * __ldg(d + (n * hw + p) * ld + c);
  }
}

// One LPIPS head over the slice features f0 (from in0) and f1 (from in1), fp32 NHWC [b][hw][c], one warp per pixel:
//   u = f0 / (|f0| + 1e-10),  v = f1 / (|f1| + 1e-10),  d = sum_c w_c (u_c - v_c)^2
// ws[n][block] = sum over the block's pixels of d, in a fixed order (warps' pixels in order, warps in order).
// With planes: the upstream gradient of the head's spatial mean is the constant gscale, so
//   dd/df1_j = gv_j / (|f1| + eps) - f1_j (sum_c gv_c f1_c) / (|f1| (|f1| + eps)^2),   gv_c = -2 w_c (u_c - v_c)
// and the planes [terms][b][hw][c] get (f1_j > 0) * (gin_j + gscale * dd/df1_j): the gradient at the
// pre-activation of the slice's last conv.  Where f1_j > 0, |f1| > 0, so the masked expression is finite; every
// other element is written 0 (torch's threshold_backward masks the NaN of sqrt's backward at an all-zero pixel).
__global__ void __launch_bounds__(kHeadWarps * 32)
lpips_head_kernel(const float* __restrict__ f0, const float* __restrict__ f1, const float* __restrict__ w,
                  const float* __restrict__ gin, long long hw, int c, float gscale, double* __restrict__ ws,
                  __half* __restrict__ planes, int terms, long long plane) {
  __shared__ double red[kHeadWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.y;
  const int nq = c >> 2;
  float4 wv[kHeadQ];
#pragma unroll
  for (int j = 0; j < kHeadQ; ++j) {
    const int q = lane + 32 * j;
    wv[j] = q < nq ? __ldg(reinterpret_cast<const float4*>(w) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  double acc = 0.0;
  for (long long p = (long long)blockIdx.x * kHeadWarps + warp; p < hw; p += (long long)gridDim.x * kHeadWarps) {
    const long long base = ((long long)n * hw + p) * c;
    float4 a[kHeadQ], v[kHeadQ];
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int j = 0; j < kHeadQ; ++j) {
      const int q = lane + 32 * j;
      a[j] = v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q < nq) {
        a[j] = __ldg(reinterpret_cast<const float4*>(f0 + base) + q);
        v[j] = __ldg(reinterpret_cast<const float4*>(f1 + base) + q);
      }
      s0 += a[j].x * a[j].x + a[j].y * a[j].y + a[j].z * a[j].z + a[j].w * a[j].w;
      s1 += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    const float n1 = sqrtf(s1);
    const float i0 = 1.f / (sqrtf(s0) + 1e-10f), i1 = 1.f / (n1 + 1e-10f);
    float dsum = 0.f, dot = 0.f;
    float4 gv[kHeadQ];
#pragma unroll
    for (int j = 0; j < kHeadQ; ++j) {
      const float ex = a[j].x * i0 - v[j].x * i1, ey = a[j].y * i0 - v[j].y * i1;
      const float ez = a[j].z * i0 - v[j].z * i1, ew = a[j].w * i0 - v[j].w * i1;
      dsum += wv[j].x * ex * ex + wv[j].y * ey * ey + wv[j].z * ez * ez + wv[j].w * ew * ew;
      gv[j] = make_float4(-2.f * wv[j].x * ex, -2.f * wv[j].y * ey, -2.f * wv[j].z * ez, -2.f * wv[j].w * ew);
      dot += gv[j].x * v[j].x + gv[j].y * v[j].y + gv[j].z * v[j].z + gv[j].w * v[j].w;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
    }
    acc += (double)dsum;
    if (planes) {
      const float k2 = n1 > 0.f ? dot * i1 * i1 / n1 : 0.f;
#pragma unroll
      for (int j = 0; j < kHeadQ; ++j) {
        const int q = lane + 32 * j;
        if (q >= nq) continue;
        float4 gi = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gin) gi = __ldg(reinterpret_cast<const float4*>(gin + base) + q);
        const float fv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
        const float gg[4] = {gv[j].x, gv[j].y, gv[j].z, gv[j].w};
        const float gx[4] = {gi.x, gi.y, gi.z, gi.w};
        __align__(8) __half hi[4], lo[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float r = fv[e] > 0.f ? gx[e] + gscale * (gg[e] * i1 - fv[e] * k2) : 0.f;
          split_f16(r, hi[e], lo[e]);
        }
        const long long off = base + 4LL * q;
        *reinterpret_cast<uint2*>(planes + off) = *reinterpret_cast<const uint2*>(hi);
        if (terms == 2) *reinterpret_cast<uint2*>(planes + plane + off) = *reinterpret_cast<const uint2*>(lo);
      }
    }
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < kHeadWarps; ++k) s += red[k];
    ws[(long long)n * gridDim.x + blockIdx.x] = s;
  }
}

// sum[n] += scale * sum_k ws[n][k], k in order (one thread per image)
__global__ void lpips_head_sum_kernel(const double* __restrict__ ws, int chunks, double scale, double* __restrict__ sum,
                                      int b) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= b) return;
  double s = 0.0;
  for (int k = 0; k < chunks; ++k) s += ws[(long long)n * chunks + k];
  sum[n] += s * scale;
}

// planes[t][i] = split(dy[i] * (y[i] > 0)), y = ReLU(pre) given by the hi plane of its fp16 planes (the rule of
// lrelu_bwd_kernel: 0 < y <= 2^-25 rounds to an fp16 0 and passes no gradient).  8 elements per thread.
__global__ void relu_bwd_kernel(const __half* __restrict__ y, const float* __restrict__ dy, __half* __restrict__ out,
                                int terms, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 yv = __ldg(reinterpret_cast<const uint4*>(y) + i);
    const __half* yh = reinterpret_cast<const __half*>(&yv);
    const float4 d0 = __ldg(reinterpret_cast<const float4*>(dy) + 2 * i);
    const float4 d1 = __ldg(reinterpret_cast<const float4*>(dy) + 2 * i + 1);
    const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
    __align__(16) __half hi[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split_f16(__half2float(yh[e]) > 0.f ? dv[e] : 0.f, hi[e], lo[e]);
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(hi);
    if (terms == 2) reinterpret_cast<uint4*>(out)[n8 + i] = *reinterpret_cast<const uint4*>(lo);
  }
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int t2h_lpips_scale_fwd(const float* x0, const float* x1, const float* shift, const float* scale, void* out, int b,
                        int h, int w, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(x0 && x1 && shift && scale && out && b > 0 && h > 0 && w > 0, "lpips_scale_fwd: bad args");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "lpips_scale_fwd: terms=%d", terms);
  const long long hw = (long long)h * w;
  lpips_scale_fwd_kernel<<<grid_cap(2LL * b * hw, 256), 256, 0, as_stream(stream)>>>(
      x0, x1, shift, scale, reinterpret_cast<__half*>(out), b, hw, terms);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_lpips_scale_bwd(const float* d, int ld, const float* scale, float alpha, float* g, int b, int h, int w,
                        t2h_stream_t stream) {
  T2H_CHECK_ARG(d && scale && g && b > 0 && h > 0 && w > 0 && ld >= 3, "lpips_scale_bwd: bad args");
  const long long hw = (long long)h * w;
  lpips_scale_bwd_kernel<<<grid_cap(3LL * b * hw, 256), 256, 0, as_stream(stream)>>>(d, ld, scale, alpha, g, b, hw);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_lpips_head(const float* f0, const float* f1, const float* w, const float* gin, int b, int h, int w_, int c,
                   float inv_hw, float gscale, double* sum, double* ws, void* planes, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(f0 && f1 && w && sum && ws && b > 0 && h > 0 && w_ > 0, "lpips_head: bad args");
  T2H_CHECK_ARG(c % 4 == 0 && c >= 4 && c <= kHeadMaxC, "lpips_head: c=%d (multiple of 4, <= %d)", c, kHeadMaxC);
  T2H_CHECK_ARG(!planes || terms == 1 || terms == 2, "lpips_head: terms=%d", terms);
  T2H_CHECK_ARG(!gin || planes, "lpips_head: gin needs planes");
  const long long hw = (long long)h * w_;
  const int chunks = t2h_lpips_head_chunks(h, w_);
  cudaStream_t st = as_stream(stream);
  lpips_head_kernel<<<dim3(chunks, b), kHeadWarps * 32, 0, st>>>(f0, f1, w, gin, hw, c, gscale, ws,
                                                                  reinterpret_cast<__half*>(planes), terms,
                                                                  (long long)b * hw * c);
  T2H_LAUNCH_OK();
  lpips_head_sum_kernel<<<ceil_div(b, 128), 128, 0, st>>>(ws, chunks, (double)inv_hw, sum, b);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_lpips_head_chunks(int h, int w) {
  const long long hw = (long long)h * w;
  const long long c = ceil_div64(hw, 4 * kHeadWarps);
  return (int)(c < 256 ? (c < 1 ? 1 : c) : 256);
}

int t2h_relu_bwd(const void* y_planes, const float* dy, void* dpre_planes, int terms, int64_t n,
                 t2h_stream_t stream) {
  T2H_CHECK_ARG(y_planes && dy && dpre_planes && n > 0 && n % 8 == 0, "relu_bwd: bad args (n %% 8 == 0)");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "relu_bwd: terms=%d", terms);
  relu_bwd_kernel<<<grid_cap(n / 8, 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const __half*>(y_planes), dy, reinterpret_cast<__half*>(dpre_planes), terms, n / 8);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

}  // extern "C"
