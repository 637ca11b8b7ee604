// HBM-bound kernels around the tensor-core contractions: layout changes,
// fp32 -> fp16-plane splitting, GroupNorm(+swish), LayerNorm, softmax,
// embedding sum.  All are streaming kernels with 128-bit accesses on the
// channel-contiguous (NHWC) side.  Reference call sites are listed in
// include/t2h.h next to each entry point.
#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

// ----------------------------------------------------------------------------
// Tiled transposes between NCHW (pixel-contiguous) and NHWC (channel-contiguous)
// ----------------------------------------------------------------------------
// x: [N][C][HW] fp32  ->  out planes [terms][N][HW][c_pad] fp16
__global__ void nchw_to_planes_kernel(const float* __restrict__ x, __half* __restrict__ out, int C,
                                      int HW, int c_pad, int terms, long long plane) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((long long)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < c_pad) {
      __half hi, lo;
      split_f16(tile[threadIdx.x][i], hi, lo);
      long long o = ((long long)n * HW + p) * c_pad + c;
      out[o] = hi;
      if (terms == 2) out[plane + o] = lo;
    }
  }
}

// x: [N][C][HW] -> out [N][HW][C]   (fp32)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ out, int C,
                                    int HW) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((long long)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < C) out[((long long)n * HW + p) * C + c] = tile[threadIdx.x][i];
  }
}

// x: [N][HW][C] -> out [N][C][HW]   (fp32)
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ out, int C,
                                    int HW) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int p = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? x[((long long)n * HW + p) * C + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    int c = c0 + i, p = p0 + threadIdx.x;
    if (p < HW && c < C) out[((long long)n * C + c) * HW + p] = tile[threadIdx.x][i];
  }
}

// Image write-out packing (save_image in sample_and_refine, sample_model.py:249-253; torchvision:
// mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(uint8)): x fp32 NCHW -> uint8 NHWC, the layout PNG
// encoders take.  `scale`/`shift` let the decoder's [-1,1] output be mapped here ((x+1)/2 -> scale .5, shift .5)
// instead of in a separate pass.  One thread per pixel; C <= 4.
__global__ void pack_u8_kernel(const float* __restrict__ x, unsigned char* __restrict__ out, int C, int HW,
                               long long total, float scale, float shift) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW;
    const int p = (int)(i - n * HW);
    for (int c = 0; c < C; ++c) {
      float v = x[(n * C + c) * HW + p] * scale + shift;
      v = fminf(fmaxf(v, 0.f), 1.f);                       // dec.clamp_(0, 1)
      v = fminf(fmaxf(__fadd_rn(__fmul_rn(v, 255.f), 0.5f), 0.f), 255.f);  // save_image's quantisation (two roundings, no FMA)
      out[i * C + c] = (unsigned char)v;                   // truncation, as .to(torch.uint8)
    }
  }
}

// ----------------------------------------------------------------------------
// fp32 NHWC -> fp16 planes, with optional nearest x2 / space-to-depth
// one thread = 8 channels of one output position (32 B in, 16 B out per plane)
// ----------------------------------------------------------------------------
struct alignas(16) Half8 {
  __half v[8];
};

__device__ __forceinline__ void store_split8(const float (&f)[8], __half* out, long long o,
                                             long long plane, int terms) {
  Half8 hi, lo;
#pragma unroll
  for (int e = 0; e < 8; ++e) split_f16(f[e], hi.v[e], lo.v[e]);
  *reinterpret_cast<Half8*>(out + o) = hi;
  if (terms == 2) *reinterpret_cast<Half8*>(out + plane + o) = lo;
}

__device__ __forceinline__ void load8(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

__global__ void f32_to_planes_kernel(const float* __restrict__ x, __half* __restrict__ out, int N,
                                     int H, int W, int C, int mode, int terms, long long plane) {
  const int c8 = C >> 3;
  int oh_n, ow_n, phases;
  if (mode == T2H_CVT_UP2X || mode == T2H_CVT_BILINEAR2X) { oh_n = 2 * H; ow_n = 2 * W; phases = 1; }
  else if (mode == T2H_CVT_S2D) { oh_n = H / 2; ow_n = W / 2; phases = 4; }
  else if (mode == T2H_CVT_MAXPOOL2) { oh_n = H / 2; ow_n = W / 2; phases = 1; }
  else { oh_n = H; ow_n = W; phases = 1; }
  const long long total = (long long)phases * N * oh_n * ow_n * c8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cc = (int)(i % c8);
    long long r = i / c8;
    const int ow = (int)(r % ow_n); r /= ow_n;
    const int oh = (int)(r % oh_n); r /= oh_n;
    const int n = (int)(r % N);
    const int ph = (int)(r / N);
    if (mode == T2H_CVT_MAXPOOL2) {
      // nn.MaxPool2d(2): window rows 2oh..2oh+1, cols 2ow..2ow+1 (odd trailing row/column dropped)
      const float* b = x + (((long long)n * H + 2 * oh) * W + 2 * ow) * C + cc * 8;
      float f[8], g[8];
      load8(b, f);
      load8(b + C, g);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = fmaxf(f[k], g[k]);
      load8(b + (long long)W * C, g);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = fmaxf(f[k], g[k]);
      load8(b + (long long)W * C + C, g);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = fmaxf(f[k], g[k]);
      store_split8(f, out, i * 8, plane, terms);
      continue;
    }
    if (mode == T2H_CVT_BILINEAR2X) {
      // nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False): src = (dst + 0.5) / 2 - 0.5,
      // clamped at 0; neighbours clamped at the border
      const float sh = fmaxf(0.5f * (oh + 0.5f) - 0.5f, 0.f), sw = fmaxf(0.5f * (ow + 0.5f) - 0.5f, 0.f);
      const int h0 = (int)sh, w0 = (int)sw;
      const int h1 = min(h0 + 1, H - 1), w1 = min(w0 + 1, W - 1);
      const float lh = sh - h0, lw = sw - w0;
      const float* b = x + (long long)n * H * W * C + cc * 8;
      float v00[8], v01[8], v10[8], v11[8], f[8];
      load8(b + ((long long)h0 * W + w0) * C, v00);
      load8(b + ((long long)h0 * W + w1) * C, v01);
      load8(b + ((long long)h1 * W + w0) * C, v10);
      load8(b + ((long long)h1 * W + w1) * C, v11);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        f[k] = (1.f - lh) * ((1.f - lw) * v00[k] + lw * v01[k]) + lh * ((1.f - lw) * v10[k] + lw * v11[k]);
      store_split8(f, out, i * 8, plane, terms);
      continue;
    }
    int ih, iw;
    if (mode == T2H_CVT_UP2X) { ih = oh >> 1; iw = ow >> 1; }
    else if (mode == T2H_CVT_S2D) { ih = 2 * oh + (ph >> 1); iw = 2 * ow + (ph & 1); }
    else { ih = oh; iw = ow; }
    float f[8];
    load8(x + (((long long)n * H + ih) * W + iw) * C + cc * 8, f);
    store_split8(f, out, i * 8, plane, terms);
  }
}

// ----------------------------------------------------------------------------
// GroupNorm statistics: stats[n][g] += (sum, sumsq) in fp64
// grid (chunks, N); a thread owns one float4 channel slot and walks pixels.
// ----------------------------------------------------------------------------
__global__ void gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C,
                                int groups, int pix_per_block) {
  extern __shared__ float sm[];  // [2][groups]
  const int n = blockIdx.y;
  const int c4 = C >> 2;
  const int cpg = C / groups;
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) sm[i] = 0.f;
  __syncthreads();
  const int slots = blockDim.x / c4;  // pixel lanes per block (blockDim multiple of c4)
  const int cs = threadIdx.x % c4;
  const int pl = threadIdx.x / c4;
  const int p_begin = blockIdx.x * pix_per_block;
  const int p_end = min(HW, p_begin + pix_per_block);
  float s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  if (pl < slots) {
    const float* base = x + (long long)n * HW * C + cs * 4;
    for (int p = p_begin + pl; p < p_end; p += slots) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + (long long)p * C));
      s[0] += v.x; ss[0] += v.x * v.x;
      s[1] += v.y; ss[1] += v.y * v.y;
      s[2] += v.z; ss[2] += v.z * v.z;
      s[3] += v.w; ss[3] += v.w * v.w;
    }
    if (cpg % 4 == 0) {  // the float4 lies inside one group; with cpg = 5, 6, 10, ... it can straddle two
      const int g = (cs * 4) / cpg;
      atomicAdd(&sm[g], (s[0] + s[1]) + (s[2] + s[3]));
      atomicAdd(&sm[groups + g], (ss[0] + ss[1]) + (ss[2] + ss[3]));
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int g = (cs * 4 + e) / cpg;
        atomicAdd(&sm[g], s[e]);
        atomicAdd(&sm[groups + g], ss[e]);
      }
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    atomicAdd(&stats[((long long)n * groups + g) * 2 + 0], (double)sm[g]);
    atomicAdd(&stats[((long long)n * groups + g) * 2 + 1], (double)sm[groups + g]);
  }
}

// ----------------------------------------------------------------------------
// GroupNorm apply (+ swish) -> fp16 planes.   grid (chunks, N)
// ----------------------------------------------------------------------------
__global__ void gn_apply_kernel(const float* __restrict__ x, const double* __restrict__ stats,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                __half* __restrict__ out, int HW, int C, int groups, float eps,
                                int swish, int terms, long long plane, int pix_per_block) {
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
  const float* xb = x + ((long long)n * HW + p_begin) * C;
  const long long ob = ((long long)n * HW + p_begin) * C;
  for (long long i = threadIdx.x; i < work; i += blockDim.x) {
    const int cc = (int)(i % c8);
    float f[8];
    load8(xb + i * 8, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = f[e] * scale[cc * 8 + e] + shift[cc * 8 + e];
      if (swish == 1) y = y / (1.0f + __expf(-y));
      else if (swish == 2) y = y > 0.f ? y : 0.2f * y;  // LeakyReLU(0.2) (Discriminator BatchNorm path)
      f[e] = y;
    }
    store_split8(f, out, ob + i * 8, plane, terms);
  }
}

__global__ void add_inplace_kernel(float* __restrict__ x, const float* __restrict__ y, long long n4,
                                   long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 a = reinterpret_cast<float4*>(x)[i];
    const float4 b = __ldg(reinterpret_cast<const float4*>(y) + i);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    reinterpret_cast<float4*>(x)[i] = a;
  }
  if (blockIdx.x == 0)
    for (long long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) x[i] += y[i];
}

// ----------------------------------------------------------------------------
// Row softmax of fp32 [rows][cols] * scale -> fp16 planes.  One warp per row,
// row cached in registers (cols <= 32*64).
// ----------------------------------------------------------------------------
template <int PER_LANE>
__global__ void softmax_rows_kernel(const float* __restrict__ s, __half* __restrict__ out,
                                    long long rows, int cols, float scale, int terms,
                                    long long plane) {
  pdl_launch_dependents();
  pdl_wait();  // before any early return: a grid none of whose CTAs wait could finish before its predecessor
  const int warps = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* src = s + row * cols;
  float v[PER_LANE];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    v[i] = c < cols ? src[c] * scale : -INFINITY;
    m = fmaxf(m, v[i]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    v[i] = expf(v[i] - m);
    sum += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    if (c < cols) {
      __half hi, lo;
      split_f16(v[i] * inv, hi, lo);
      out[row * cols + c] = hi;
      if (terms == 2) out[plane + row * cols + c] = lo;
    }
  }
}

// ----------------------------------------------------------------------------
// LayerNorm over C of fp32 [rows][C] -> fp16 planes.  One warp per row.
// ----------------------------------------------------------------------------
template <int PER_LANE>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, __half* __restrict__ out,
                                 long long rows, int C, float eps, int terms, long long plane,
                                 const long long* __restrict__ row_map) {
  pdl_launch_dependents();
  pdl_wait();  // before any early return: a grid none of whose CTAs wait could finish before its predecessor
  const int warps = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* src = x + row * C;
  const long long orow = row_map ? row_map[row] : row;  // scatter: the grouped-head GEMM wants rows by texture
  float v[PER_LANE];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    v[i] = c < C ? src[c] : 0.f;
    sum += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    const float d = c < C ? v[i] - mean : 0.f;
    sq += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    if (c < C) {
      __half hi, lo;
      split_f16((v[i] - mean) * rstd * gamma[c] + beta[c], hi, lo);
      out[orow * C + c] = hi;
      if (terms == 2) out[plane + orow * C + c] = lo;
    }
  }
}

// Deterministic split-K completion fused with the residual add and the following LayerNorm: one warp per row.
//   x_out = residual + bias + sum_s partials[s]  (s ascending);  ln_out[row_map[row]] = LN(x_out) as fp16 planes
template <int PER_LANE>
__global__ void splitk_reduce_ln_kernel(const float* __restrict__ part, int n_slabs, long long slab,
                                        const float* __restrict__ bias, const float* residual, float* x_out,
                                        const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                        __half* __restrict__ ln_out, int terms, long long plane,
                                        const long long* __restrict__ row_map, long long rows, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int warps = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float v[PER_LANE];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    float a = 0.f;
    if (c < C) {
      a = residual ? residual[row * C + c] : 0.f;
      if (bias) a += bias[c];
      for (int s = 0; s < n_slabs; ++s) a += part[(long long)s * slab + row * C + c];
      x_out[row * C + c] = a;
    }
    v[i] = a;
    sum += a;
  }
  if (!ln_out) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    const float d = c < C ? v[i] - mean : 0.f;
    sq += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  const long long orow = row_map ? row_map[row] : row;
#pragma unroll
  for (int i = 0; i < PER_LANE; ++i) {
    const int c = lane + i * 32;
    if (c < C) {
      __half hi, lo;
      split_f16((v[i] - mean) * rstd * gamma[c] + beta[c], hi, lo);
      ln_out[orow * C + c] = hi;
      if (terms == 2) ln_out[plane + orow * C + c] = lo;
    }
  }
}

// The same pass for C % 4 == 0 with 128-bit accesses: lane l owns columns 4 (l + 32 i) .. +3.  Every load of a row is
// issued before the first store (x_out may alias residual, so stores in the load loop would serialise it into
// one L2 round trip per column group).  x_out is summed in the scalar kernel's order (bit-identical); the LayerNorm
// statistics are reduced in a different, equally fixed, order.
template <int VEC>
__global__ void splitk_reduce_ln_vec_kernel(const float* __restrict__ part, int n_slabs, long long slab,
                                            const float* __restrict__ bias, const float* residual, float* x_out,
                                            const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                            __half* __restrict__ ln_out, int terms, long long plane,
                                            const long long* __restrict__ row_map, long long rows, int C) {
  pdl_launch_dependents();
  pdl_wait();
  const int warps = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nv = C >> 2;
  float4 v[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c4 = lane + i * 32;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < nv && residual) v[i] = *reinterpret_cast<const float4*>(residual + row * C + 4 * c4);
  }
  if (bias) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const int c4 = lane + i * 32;
      if (c4 < nv) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + c4);
        v[i].x += b.x; v[i].y += b.y; v[i].z += b.z; v[i].w += b.w;
      }
    }
  }
  for (int s = 0; s < n_slabs; ++s) {
    const float* ps = part + (long long)s * slab + row * C;
    float4 p[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const int c4 = lane + i * 32;
      p[i] = c4 < nv ? __ldg(reinterpret_cast<const float4*>(ps) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      v[i].x += p[i].x; v[i].y += p[i].y; v[i].z += p[i].z; v[i].w += p[i].w;
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c4 = lane + i * 32;
    if (c4 < nv) {
      *reinterpret_cast<float4*>(x_out + row * C + 4 * c4) = v[i];
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  if (!ln_out) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c4 = lane + i * 32;
    if (c4 < nv) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      sq += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  const long long orow = row_map ? row_map[row] : row;
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    const int c4 = lane + i * 32;
    if (c4 < nv) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + c4);
      __align__(8) __half hi[4];
      __align__(8) __half lo[4];
      split_f16((v[i].x - mean) * rstd * g.x + b.x, hi[0], lo[0]);
      split_f16((v[i].y - mean) * rstd * g.y + b.y, hi[1], lo[1]);
      split_f16((v[i].z - mean) * rstd * g.z + b.z, hi[2], lo[2]);
      split_f16((v[i].w - mean) * rstd * g.w + b.w, hi[3], lo[3]);
      *reinterpret_cast<uint2*>(ln_out + orow * C + 4 * c4) = *reinterpret_cast<uint2*>(hi);
      if (terms == 2) *reinterpret_cast<uint2*>(ln_out + plane + orow * C + 4 * c4) = *reinterpret_cast<uint2*>(lo);
    }
  }
}

// x[b,t,:] = tok[idx] + pos[t] + segm[sg] + tex[tx]
__global__ void embed_sum_kernel(const long long* __restrict__ idx, const long long* __restrict__ segm,
                                 const long long* __restrict__ tex, const float* __restrict__ tok_emb,
                                 const float* __restrict__ pos_emb, const float* __restrict__ segm_emb,
                                 const float* __restrict__ tex_emb, float* __restrict__ x, int T,
                                 int C) {
  pdl_launch_dependents();
  pdl_wait();  // before any early return: a grid none of whose CTAs wait could finish before its predecessor
  const long long row = blockIdx.x;  // b*T + t
  const int t = (int)(row % T);
  const float4* a = reinterpret_cast<const float4*>(tok_emb + idx[row] * C);
  const float4* p = reinterpret_cast<const float4*>(pos_emb + (long long)t * C);
  const float4* s = reinterpret_cast<const float4*>(segm_emb + segm[row] * C);
  const float4* e = reinterpret_cast<const float4*>(tex_emb + tex[row] * C);
  float4* o = reinterpret_cast<float4*>(x + row * C);
  for (int i = threadIdx.x; i < (C >> 2); i += blockDim.x) {
    const float4 va = __ldg(a + i), vp = __ldg(p + i), vs = __ldg(s + i), ve = __ldg(e + i);
    // same association as the reference: ((tok + pos) + segm) + tex
    float4 r;
    r.x = ((va.x + vp.x) + vs.x) + ve.x;
    r.y = ((va.y + vp.y) + vs.y) + ve.y;
    r.z = ((va.z + vp.z) + vs.z) + ve.z;
    r.w = ((va.w + vp.w) + vs.w) + ve.w;
    o[i] = r;
  }
}

// nearest resize of a float id map to int32 ids (src index = floor(dst * in/out))
__global__ void mask_to_ids_kernel(const float* __restrict__ mask, int* __restrict__ ids, int B, int Hs,
                                   int Ws, int Ht, int Wt) {
  const long long total = (long long)B * Ht * Wt;
  const float sh = (float)Hs / (float)Ht, sw = (float)Ws / (float)Wt;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(i % Wt);
    const int y = (int)((i / Wt) % Ht);
    const int b = (int)(i / ((long long)Wt * Ht));
    const int sy = min((int)floorf(y * sh), Hs - 1);
    const int sx = min((int)floorf(x * sw), Ws - 1);
    // the reference selects rows with `segm_map == k` on floats: a non-integer id matches nothing
    const float v = mask[((long long)b * Hs + sy) * Ws + sx];
    ids[i] = (v == floorf(v) && v >= -1.0f && v < 1.0e6f) ? (int)v : -1;
  }
}

// ids [B][HW] (float class ids) -> one-hot fp16 planes [terms][B][HW][c_pad]; the lo plane of an exact
// 0/1 value is zero.  Replaces F.one_hot(...).permute(0,3,1,2).float() (sample_model.py:331-335).
__global__ void onehot_to_planes_kernel(const float* __restrict__ ids, __half* __restrict__ out, long long npix,
                                        int c_pad, int n_classes, int terms, long long plane) {
  const int c8 = c_pad >> 3;
  const long long total = npix * c8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / c8;
    const int c0 = (int)(i % c8) * 8;
    const float v = ids[p];
    const int cls = (v == floorf(v) && v >= 0.f && v < (float)n_classes) ? (int)v : -1;
    Half8 hi, lo;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      hi.v[e] = __float2half_rn((c0 + e) == cls ? 1.f : 0.f);
      lo.v[e] = __float2half_rn(0.f);
    }
    *reinterpret_cast<Half8*>(out + i * 8) = hi;
    if (terms == 2) *reinterpret_cast<Half8*>(out + plane + i * 8) = lo;
  }
}

// Dataset-side preparation (data/segm_attr_dataset.py:120-164) on the device.
// texture mask: mask = attr[group(cls)] + 1 where the parsing class belongs to the upper / lower / outer clothes
// group and that group's fused attribute is not 17 ("NA"), else 0 (:138-151).  cls_group[c] in {-1, 0, 1, 2}.
__global__ void texture_mask_kernel(const float* __restrict__ segm, const int* __restrict__ attrs,
                                    const int* __restrict__ cls_group, int n_cls, float* __restrict__ mask,
                                    long long per_img, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / per_img);
    const float v = segm[i];
    float m = 0.f;
    if (v == floorf(v) && v >= 0.f && v < (float)n_cls) {
      const int g = cls_group[(int)v];
      if (g >= 0) {
        const int a = attrs[b * 3 + g];
        if (a != 17) m = (float)(a + 1);
      }
    }
    mask[i] = m;
  }
}

// uint8 HWC image batch [B][H][W][C] -> fp16 planes NHWC [terms][B][H][W][c_pad] of x*scale + shift
// (image / 127.5 - 1, :154, fused with the split the encoder's conv_in needs) and, optionally, the fp32 NCHW
// tensor the reference's DataLoader would have produced
__global__ void u8_to_planes_kernel(const unsigned char* __restrict__ x, __half* __restrict__ out,
                                    float* __restrict__ nchw, int C, int c_pad, long long HW, long long npix,
                                    float scale, float shift, int terms, long long plane) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < npix;
       p += (long long)gridDim.x * blockDim.x) {
    const long long b = p / HW, q = p - b * HW;
    for (int c = 0; c < c_pad; ++c) {
      float v = 0.f;
      if (c < C) {
        v = __fadd_rn(__fdiv_rn((float)x[p * C + c], scale), shift);   // image / 127.5 - 1: division, then the add
        if (nchw) nchw[(b * C + c) * HW + q] = v;
      }
      __half hi, lo;
      split_f16(v, hi, lo);
      out[p * c_pad + c] = hi;
      if (terms == 2) out[plane + p * c_pad + c] = lo;
    }
  }
}

static inline int grid_for(long long work, int block) {
  long long g = ceil_div64(work, block);
  long long cap = (long long)num_sms() * 16;
  return (int)(g < cap ? (g < 1 ? 1 : g) : cap);
}


// Per-row argmax inside the row's own head (bot_index_prediction, sample_model.py:183-213):
// logits [G][M][ncls]; row m reads head[m]'s slice and returns the lowest index of the maximum (-1 when
// head[m] is outside 0..G-1).  One warp per row.
__global__ void argmax_heads_kernel(const float* __restrict__ logits, const long long* __restrict__ head,
                                    long long* __restrict__ out, long long M, int G, int ncls) {
  const long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (m >= M) return;
  const int lane = threadIdx.x & 31;
  const long long hd = head[m];
  if (hd < 0 || hd >= G) {
    if (lane == 0) out[m] = -1;
    return;
  }
  const float* row = logits + ((long long)hd * M + m) * ncls;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = lane; c < ncls; c += 32) {
    const float v = row[c];
    if (v > best) {  // strictly greater: within a lane the lowest index of the maximum is kept
      best = v;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  if (lane == 0) out[m] = bi == 0x7fffffff ? 0 : bi;
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int t2h_nchw_to_planes(const float* x, void* out, int n, int c, int h, int w, int c_pad, int terms,
                       t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && c > 0 && h > 0 && w > 0, "nchw_to_planes: bad shape");
  T2H_CHECK_ARG(c_pad >= c && c_pad % 8 == 0, "nchw_to_planes: c_pad=%d must be >= c and a multiple of 8",
                c_pad);
  T2H_CHECK_ARG(terms == 1 || terms == 2, "nchw_to_planes: terms=%d", terms);
  const int hw = h * w;
  dim3 grid(ceil_div(hw, 32), ceil_div(c_pad, 32), n), block(32, 8);
  nchw_to_planes_kernel<<<grid, block, 0, as_stream(stream)>>>(
      x, reinterpret_cast<__half*>(out), c, hw, c_pad, terms, (long long)n * hw * c_pad);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_nhwc_to_nchw(const float* x, float* out, int n, int c, int h, int w, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && c > 0 && h > 0 && w > 0, "nhwc_to_nchw: bad shape");
  const int hw = h * w;
  dim3 grid(ceil_div(hw, 32), ceil_div(c, 32), n), block(32, 8);
  nhwc_to_nchw_kernel<<<grid, block, 0, as_stream(stream)>>>(x, out, c, hw);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_nchw_to_nhwc(const float* x, float* out, int n, int c, int h, int w, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && c > 0 && h > 0 && w > 0, "nchw_to_nhwc: bad shape");
  const int hw = h * w;
  dim3 grid(ceil_div(hw, 32), ceil_div(c, 32), n), block(32, 8);
  nchw_to_nhwc_kernel<<<grid, block, 0, as_stream(stream)>>>(x, out, c, hw);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_f32_to_planes(const float* x, void* out, int n, int h, int w, int c, int mode, int terms,
                      t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && h > 0 && w > 0 && c > 0, "f32_to_planes: bad shape");
  T2H_CHECK_ARG(c % 8 == 0, "f32_to_planes: C=%d must be a multiple of 8", c);
  T2H_CHECK_ARG(mode >= 0 && mode <= 4, "f32_to_planes: mode=%d", mode);
  T2H_CHECK_ARG(mode != T2H_CVT_S2D || (h % 2 == 0 && w % 2 == 0), "f32_to_planes: S2D needs even H,W");
  T2H_CHECK_ARG(mode != T2H_CVT_MAXPOOL2 || (h >= 2 && w >= 2), "f32_to_planes: MAXPOOL2 needs H,W >= 2");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "f32_to_planes: terms=%d", terms);
  long long out_elems = (long long)n * h * w * c;
  if (mode == T2H_CVT_UP2X || mode == T2H_CVT_BILINEAR2X) out_elems *= 4;
  if (mode == T2H_CVT_MAXPOOL2) out_elems = (long long)n * (h / 2) * (w / 2) * c;
  const long long work = out_elems / 8;
  f32_to_planes_kernel<<<grid_for(work, 256), 256, 0, as_stream(stream)>>>(
      x, reinterpret_cast<__half*>(out), n, h, w, c, mode, terms, out_elems);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_gn_stats(const float* x, double* stats, int n, int hw, int c, int groups, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && stats && n > 0 && hw > 0, "gn_stats: bad shape");
  T2H_CHECK_ARG(c % groups == 0 && c % 4 == 0 && c <= 4096, "gn_stats: C=%d groups=%d unsupported", c,
                groups);
  const int c4 = c / 4;
  int block = 256;
  if (c4 > block) block = ((c4 + 31) / 32) * 32;
  T2H_CHECK_ARG(block <= 1024, "gn_stats: C=%d too large", c);
  block = (block / c4) * c4;  // whole pixel lanes only
  const int lanes = block / c4;
  // enough blocks to fill the machine, >= 8 pixels per lane
  int blocks_x = ceil_div(num_sms() * 4, n);
  int ppb = ceil_div(hw, blocks_x);
  if (ppb < lanes * 8) ppb = lanes * 8;
  blocks_x = ceil_div(hw, ppb);
  dim3 grid(blocks_x, n);
  gn_stats_kernel<<<grid, block, 2 * groups * sizeof(float), as_stream(stream)>>>(x, stats, hw, c,
                                                                                groups, ppb);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_gn_apply(const float* x, const double* stats, const float* gamma, const float* beta, void* out,
                 int n, int hw, int c, int groups, float eps, int swish, int terms,
                 t2h_stream_t stream) {
  T2H_CHECK_ARG(x && stats && gamma && beta && out && n > 0 && hw > 0, "gn_apply: bad args");
  T2H_CHECK_ARG(c % groups == 0 && c % 8 == 0 && c <= 4096, "gn_apply: C=%d groups=%d unsupported", c,
                groups);
  T2H_CHECK_ARG(terms == 1 || terms == 2, "gn_apply: terms=%d", terms);
  int blocks_x = ceil_div(num_sms() * 8, n);
  int ppb = ceil_div(hw, blocks_x);
  if (ppb < 16) ppb = 16;
  blocks_x = ceil_div(hw, ppb);
  dim3 grid(blocks_x, n);
  gn_apply_kernel<<<grid, 256, 2 * c * sizeof(float), as_stream(stream)>>>(
      x, stats, gamma, beta, reinterpret_cast<__half*>(out), hw, c, groups, eps, swish, terms,
      (long long)n * hw * c, ppb);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_add_inplace(float* x, const float* y, int64_t numel, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && y && numel > 0, "add_inplace: bad args");
  T2H_CHECK_ARG(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(y) % 16 == 0,
                "add_inplace: pointers must be 16-byte aligned");
  const long long n4 = numel / 4;
  add_inplace_kernel<<<grid_for(n4 > 0 ? n4 : 1, 256), 256, 0, as_stream(stream)>>>(x, y, n4, numel);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_softmax_rows(const float* s, void* out, int64_t rows, int cols, float scale, int terms,
                     t2h_stream_t stream) {
  T2H_CHECK_ARG(s && out && rows > 0 && cols > 0, "softmax_rows: bad args");
  T2H_CHECK_ARG(cols <= 2048, "softmax_rows: cols=%d > 2048 unsupported", cols);
  T2H_CHECK_ARG(terms == 1 || terms == 2, "softmax_rows: terms=%d", terms);
  const int warps = 4;
  const int grid = (int)ceil_div64(rows, warps);
  __half* o = reinterpret_cast<__half*>(out);
  const long long plane = rows * cols;
  cudaStream_t st = as_stream(stream);
  if (cols <= 512)
    T2H_CUDA(launch_pdl(softmax_rows_kernel<16>, dim3(grid), dim3(warps * 32), 0, st, s, o, rows, cols, scale, terms, plane));
  else
    T2H_CUDA(launch_pdl(softmax_rows_kernel<64>, dim3(grid), dim3(warps * 32), 0, st, s, o, rows, cols, scale, terms, plane));
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_layernorm(const float* x, const float* gamma, const float* beta, void* out, int64_t rows, int c,
                  float eps, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && gamma && beta && out && rows > 0 && c > 0, "layernorm: bad args");
  T2H_CHECK_ARG(c <= 1024, "layernorm: C=%d > 1024 unsupported", c);
  T2H_CHECK_ARG(terms == 1 || terms == 2, "layernorm: terms=%d", terms);
  const int warps = 4;
  const int grid = (int)ceil_div64(rows, warps);
  __half* o = reinterpret_cast<__half*>(out);
  const long long plane = rows * c;
  cudaStream_t st = as_stream(stream);
  if (c <= 512)
    T2H_CUDA(launch_pdl(layernorm_kernel<16>, dim3(grid), dim3(warps * 32), 0, st, x, gamma, beta, o, rows, c, eps, terms, plane,
                        static_cast<const long long*>(nullptr)));
  else
    T2H_CUDA(launch_pdl(layernorm_kernel<32>, dim3(grid), dim3(warps * 32), 0, st, x, gamma, beta, o, rows, c, eps, terms, plane,
                        static_cast<const long long*>(nullptr)));
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_splitk_reduce_ln(const float* partials, int n_slabs, int64_t slab, const float* bias, const float* residual,
                         float* x_out, const float* gamma, const float* beta, float eps, void* ln_out, int terms,
                         const int64_t* row_map, int64_t ln_rows, int64_t rows, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(partials && x_out && n_slabs >= 1 && rows > 0 && c > 0 && c <= 1024, "splitk_reduce_ln: bad args");
  T2H_CHECK_ARG(!ln_out || (gamma && beta && (terms == 1 || terms == 2) && ln_rows >= (row_map ? 1 : rows)),
                "splitk_reduce_ln: LayerNorm output needs gamma/beta/terms");
  const int warps = 4;
  const int grid = (int)ceil_div64(rows, warps);
  __half* o = reinterpret_cast<__half*>(ln_out);
  const long long plane = (long long)ln_rows * c;
  const long long* rm = reinterpret_cast<const long long*>(row_map);
  cudaStream_t st = as_stream(stream);
  const bool aligned = (c % 4 == 0) && (slab % 4 == 0) && ((reinterpret_cast<uintptr_t>(partials) | reinterpret_cast<uintptr_t>(x_out) |
                                                           reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(bias) |
                                                           reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) % 16 == 0) &&
                       (reinterpret_cast<uintptr_t>(ln_out) % 8 == 0) && (plane % 4 == 0);
  if (aligned && c <= 512)
    T2H_CUDA(launch_pdl(splitk_reduce_ln_vec_kernel<4>, dim3(grid), dim3(warps * 32), 0, st, partials, n_slabs,
                        (long long)slab, bias, residual, x_out, gamma, beta, eps, o, terms, plane, rm, (long long)rows, c));
  else if (aligned)
    T2H_CUDA(launch_pdl(splitk_reduce_ln_vec_kernel<8>, dim3(grid), dim3(warps * 32), 0, st, partials, n_slabs,
                        (long long)slab, bias, residual, x_out, gamma, beta, eps, o, terms, plane, rm, (long long)rows, c));
  else if (c <= 512)
    T2H_CUDA(launch_pdl(splitk_reduce_ln_kernel<16>, dim3(grid), dim3(warps * 32), 0, st, partials, n_slabs,
                        (long long)slab, bias, residual, x_out, gamma, beta, eps, o, terms, plane, rm, (long long)rows, c));
  else
    T2H_CUDA(launch_pdl(splitk_reduce_ln_kernel<32>, dim3(grid), dim3(warps * 32), 0, st, partials, n_slabs,
                        (long long)slab, bias, residual, x_out, gamma, beta, eps, o, terms, plane, rm, (long long)rows, c));
  return T2H_OK;
}

int t2h_embed_sum(const int64_t* idx, const int64_t* segm, const int64_t* tex, const float* tok_emb,
                  const float* pos_emb, const float* segm_emb, const float* tex_emb, float* x, int b,
                  int t, int c, t2h_stream_t stream) {
  T2H_CHECK_ARG(idx && segm && tex && tok_emb && pos_emb && segm_emb && tex_emb && x, "embed_sum: null");
  T2H_CHECK_ARG(b > 0 && t > 0 && c > 0 && c % 4 == 0, "embed_sum: bad shape");
  T2H_CUDA(launch_pdl(embed_sum_kernel, dim3(b * t), dim3(128), 0, as_stream(stream),
                      reinterpret_cast<const long long*>(idx), reinterpret_cast<const long long*>(segm),
                      reinterpret_cast<const long long*>(tex), tok_emb, pos_emb, segm_emb, tex_emb, x, t, c));
  return T2H_OK;
}

int t2h_onehot_to_planes(const float* ids, void* out, int b, int h, int w, int n_classes, int c_pad, int terms,
                         t2h_stream_t stream) {
  T2H_CHECK_ARG(ids && out && b > 0 && h > 0 && w > 0 && n_classes > 0, "onehot_to_planes: bad args");
  T2H_CHECK_ARG(c_pad >= n_classes && c_pad % 8 == 0, "onehot_to_planes: c_pad=%d", c_pad);
  T2H_CHECK_ARG(terms == 1 || terms == 2, "onehot_to_planes: terms=%d", terms);
  const long long npix = (long long)b * h * w;
  onehot_to_planes_kernel<<<grid_for(npix * (c_pad / 8), 256), 256, 0, as_stream(stream)>>>(
      ids, reinterpret_cast<__half*>(out), npix, c_pad, n_classes, terms, npix * c_pad);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_texture_mask(const float* segm, const int32_t* attrs, const int32_t* cls_group, int n_cls, float* mask, int b,
                     int64_t per_img, t2h_stream_t stream) {
  T2H_CHECK_ARG(segm && attrs && cls_group && mask && b > 0 && per_img > 0 && n_cls > 0, "texture_mask: bad args");
  const long long total = (long long)b * per_img;
  texture_mask_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(segm, attrs, cls_group, n_cls, mask,
                                                                          per_img, total);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_u8_to_planes(const uint8_t* x, void* out, float* nchw, int b, int h, int w, int c, int c_pad, float divisor,
                     float shift, int terms, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && b > 0 && h > 0 && w > 0 && c > 0, "u8_to_planes: bad args");
  T2H_CHECK_ARG(c_pad >= c && c_pad % 8 == 0 && (terms == 1 || terms == 2) && divisor != 0.f, "u8_to_planes: c_pad/terms");
  const long long npix = (long long)b * h * w;
  u8_to_planes_kernel<<<grid_for(npix, 256), 256, 0, as_stream(stream)>>>(
      x, reinterpret_cast<__half*>(out), nchw, c, c_pad, (long long)h * w, npix, divisor, shift, terms, npix * c_pad);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_mask_to_ids(const float* mask, int32_t* ids, int b, int hs, int ws, int ht, int wt,
                    t2h_stream_t stream) {
  T2H_CHECK_ARG(mask && ids && b > 0 && hs > 0 && ws > 0 && ht > 0 && wt > 0, "mask_to_ids: bad args");
  const long long total = (long long)b * ht * wt;
  mask_to_ids_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(mask, ids, b, hs, ws, ht, wt);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_argmax_heads(const float* logits, const int64_t* head, int64_t* out, int64_t rows, int n_heads, int ncls,
                     t2h_stream_t stream) {
  T2H_CHECK_ARG(logits && head && out && rows > 0 && n_heads > 0 && ncls > 0, "argmax_heads: bad args");
  const int warps = 8;
  argmax_heads_kernel<<<(unsigned)ceil_div64(rows, warps), warps * 32, 0, as_stream(stream)>>>(
      logits, reinterpret_cast<const long long*>(head), reinterpret_cast<long long*>(out), rows, n_heads, ncls);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_pack_u8(const float* x, uint8_t* out, int n, int c, int h, int w, float scale, float shift,
                t2h_stream_t stream) {
  T2H_CHECK_ARG(x && out && n > 0 && c > 0 && c <= 4 && h > 0 && w > 0, "pack_u8: bad args");
  const long long total = (long long)n * h * w;
  pack_u8_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(x, out, c, h * w, total, scale, shift);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_layernorm_scatter(const float* x, const float* gamma, const float* beta, void* out, int64_t rows, int c,
                          float eps, int terms, const int64_t* row_map, int64_t out_rows, t2h_stream_t stream) {
  T2H_CHECK_ARG(x && gamma && beta && out && row_map && rows > 0 && c > 0 && out_rows >= rows,
                "layernorm_scatter: bad args");
  T2H_CHECK_ARG(c <= 1024 && (terms == 1 || terms == 2), "layernorm_scatter: C=%d terms=%d unsupported", c, terms);
  const int warps = 4;
  const int grid = (int)ceil_div64(rows, warps);
  __half* o = reinterpret_cast<__half*>(out);
  const long long plane = out_rows * c;
  const long long* rm = reinterpret_cast<const long long*>(row_map);
  cudaStream_t st = as_stream(stream);
  if (c <= 512)
    T2H_CUDA(launch_pdl(layernorm_kernel<16>, dim3(grid), dim3(warps * 32), 0, st, x, gamma, beta, o, rows, c, eps,
                        terms, plane, rm));
  else
    T2H_CUDA(launch_pdl(layernorm_kernel<32>, dim3(grid), dim3(warps * 32), 0, st, x, gamma, beta, o, rows, c, eps,
                        terms, plane, rm));
  return T2H_OK;
}

}  // extern "C"
