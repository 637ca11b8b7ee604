// Codebook nearest-neighbour quantizers (VectorQuantizer, VectorQuantizerTexture,
// VectorQuantizerSpatialTextureAware — vqgan_arch.py:79-122, :212-287, :375-461).
//
// One launch replaces the reference's 18-iteration Python loop (each with a
// host sync, boolean-mask gather, sgemm, argmin, embedding lookup and masked
// scatter).  Rows are binned by the codebook their texture id selects, each CTA
// searches one codebook for a tile of 32 rows with fp32 FMA dot products and a
// warp-shuffle argmin, then gathers z_q and writes every output layout.
//
// Arithmetic contract (identical, operation for operation, to oracle/vq_oracle.c
// so indices are bit-reproducible):
//   dot(r,j) = fma chain over d = 0..D-1 ascending, one fp32 accumulator
//   nrm(v)   = 32 interleaved fp32 fma chains (lane l takes d = l, l+32, ...),
//              combined by the xor-butterfly 16,8,4,2,1
//   dist     = (nrm(z) + nrm(e)) - 2*dot        (two roundings, as :246-252)
//   argmin   = lowest index among equal distances (torch.argmin)
//   z_q out  = z + (e - z)                      (straight-through value, :281)
#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

constexpr int kRT = 32;    // rows per CTA
constexpr int kCT = 128;   // codes per smem tile
constexpr int kKC = 32;    // contraction chunk
constexpr int kVqThreads = 256;

struct VqShape {
  int B, Hz, Wz, Cz, ps, Hp, Wp, D, rows, n_books, n_e;
};

__device__ __forceinline__ long long z_offset(const VqShape& s, int row, int d) {
  // row -> (b, ph, pw);  d -> (c, kh, kw) in F.unfold order (vqgan_arch.py:324)
  const int pw = row % s.Wp;
  const int ph = (row / s.Wp) % s.Hp;
  const int b = row / (s.Wp * s.Hp);
  const int pp = s.ps * s.ps;
  const int c = d / pp;
  const int kh = (d / s.ps) % s.ps;
  const int kw = d % s.ps;
  return (((long long)b * s.Hz + ph * s.ps + kh) * s.Wz + pw * s.ps + kw) * s.Cz + c;
}

__device__ __forceinline__ float warp_butterfly_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ee[book*n_e + j] = nrm(codebook row); one warp per code
__global__ void vq_code_norms_kernel(const float* __restrict__ cb, float* __restrict__ ee,
                                     long long n_codes, int D) {
  const long long code = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (code >= n_codes) return;
  const int lane = threadIdx.x & 31;
  const float* e = cb + code * D;
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = e[d];
    acc = __fmaf_rn(v, v, acc);
  }
  acc = warp_butterfly_sum(acc);
  if (lane == 0) ee[code] = acc;
}

// Single-block counting sort of rows by codebook id + tile table (tests/test_gpu_image_kernels.py::vq_bin_route restates it).
// ws layout (int32): [0]=n_tiles, [1..]=tile_book[maxT], tile_start[maxT], tile_cnt[maxT], perm[rows]
__global__ void vq_bin_kernel(const int* __restrict__ book_id, int rows, int n_books, int maxT,
                              int* __restrict__ ws) {
  __shared__ int cnt[64];
  __shared__ int off[65];
  __shared__ int cur[64];
  int* n_tiles = ws;
  int* tile_book = ws + 1;
  int* tile_start = tile_book + maxT;
  int* tile_cnt = tile_start + maxT;
  int* perm = tile_cnt + maxT;
  // bin n_books = "unselected" rows
  for (int i = threadIdx.x; i <= n_books; i += blockDim.x) cnt[i] = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    int k = book_id ? book_id[r] : 0;
    if (k < 0 || k >= n_books) k = n_books;
    atomicAdd(&cnt[k], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0, t = 0;
    for (int k = 0; k <= n_books; ++k) {
      off[k] = acc;
      cur[k] = acc;
      for (int s = 0; s < cnt[k]; s += kRT) {
        tile_book[t] = k;
        tile_start[t] = acc + s;
        tile_cnt[t] = min(kRT, cnt[k] - s);
        ++t;
      }
      acc += cnt[k];
    }
    *n_tiles = t;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < rows; r += blockDim.x) {
    int k = book_id ? book_id[r] : 0;
    if (k < 0 || k >= n_books) k = n_books;
    const int pos = atomicAdd(&cur[k], 1);
    perm[pos] = r;
  }
}

struct VqOut {
  long long* idx;
  long long* idx_cont;
  long long* idx_list;
  float* zq_nhwc;
  float* zq_nchw;
  double* sqerr;
  long long cont_stride;
};

__global__ void __launch_bounds__(kVqThreads)
vq_search_kernel(const float* __restrict__ z, const float* __restrict__ cb, const float* __restrict__ ee,
                 const int* __restrict__ ws, int maxT, VqShape s, VqOut o) {
  const int n_tiles = ws[0];
  if ((int)blockIdx.x >= n_tiles) return;
  const int* tile_book = ws + 1;
  const int* tile_start = tile_book + maxT;
  const int* tile_cnt = tile_start + maxT;
  const int* perm = tile_cnt + maxT;
  const int book = tile_book[blockIdx.x];
  const int start = tile_start[blockIdx.x];
  const int cnt = tile_cnt[blockIdx.x];

  __shared__ int rows_s[kRT];
  __shared__ int best_s[kRT];
  __shared__ float zz_s[kRT];
  __shared__ __align__(16) float zs[kRT][kKC];             // z chunk  [row][k]
  __shared__ __align__(16) float es[kKC / 4][kCT + 1][4];  // code chunk [k/4][code][k%4]
  __shared__ double err_s;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  if (tid < kRT) rows_s[tid] = tid < cnt ? perm[start + tid] : -1;
  if (tid == 0) err_s = 0.0;
  __syncthreads();

  const bool selected = book < s.n_books;
  if (selected) {
    // ---- nrm(z) per row: warp w handles rows w*4 .. w*4+3
    for (int i = 0; i < 4; ++i) {
      const int rl = warp * 4 + i;
      const int row = rows_s[rl];
      float acc = 0.f;
      if (row >= 0)
        for (int d = lane; d < s.D; d += 32) {
          const float v = z[z_offset(s, row, d)];
          acc = __fmaf_rn(v, v, acc);
        }
      acc = warp_butterfly_sum(acc);
      if (lane == 0) zz_s[rl] = acc;
    }

    float best_d[4];
    int best_i[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      best_d[i] = INFINITY;
      best_i[i] = 0x7fffffff;
    }
    const float* cbk = cb + (long long)book * s.n_e * s.D;
    const float* eek = ee + (long long)book * s.n_e;

    for (int c0 = 0; c0 < s.n_e; c0 += kCT) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

      for (int k0 = 0; k0 < s.D; k0 += kKC) {
        __syncthreads();
        // z chunk: kRT*kKC = 1024 floats, 4 per thread
        for (int e = tid; e < kRT * kKC; e += kVqThreads) {
          const int rl = e / kKC, kk = e % kKC;
          const int row = rows_s[rl];
          zs[rl][kk] = (row >= 0 && k0 + kk < s.D) ? z[z_offset(s, row, k0 + kk)] : 0.f;
        }
        // code chunk: kCT codes x kKC/4 float4
        for (int e = tid; e < kCT * (kKC / 4); e += kVqThreads) {
          const int code = e / (kKC / 4), k4 = e % (kKC / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (c0 + code < s.n_e && k0 + k4 * 4 < s.D)
            v = *reinterpret_cast<const float4*>(cbk + (long long)(c0 + code) * s.D + k0 + k4 * 4);
          *reinterpret_cast<float4*>(&es[k4][code][0]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int k4 = 0; k4 < kKC / 4; ++k4) {
          float4 zv[4], ev[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) zv[i] = *reinterpret_cast<const float4*>(&zs[warp * 4 + i][k4 * 4]);
#pragma unroll
          for (int j = 0; j < 4; ++j) ev[j] = *reinterpret_cast<const float4*>(&es[k4][lane + 32 * j][0]);
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float a = acc[i][j];
              a = __fmaf_rn(zv[i].x, ev[j].x, a);
              a = __fmaf_rn(zv[i].y, ev[j].y, a);
              a = __fmaf_rn(zv[i].z, ev[j].z, a);
              a = __fmaf_rn(zv[i].w, ev[j].w, a);
              acc[i][j] = a;
            }
        }
      }
      // distances of this code tile; codes visited in ascending order per thread
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int code = c0 + lane + 32 * j;
        if (code < s.n_e) {
          const float en = eek[code];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float dist =
                __fsub_rn(__fadd_rn(zz_s[warp * 4 + i], en), __fmul_rn(2.0f, acc[i][j]));
            if (dist < best_d[i]) {
              best_d[i] = dist;
              best_i[i] = code;
            }
          }
        }
      }
    }
    // ---- warp-shuffle argmin across the 32 lanes holding a row's candidates
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float bd = best_d[i];
      int bi = best_i[i];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bd, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (od < bd || (od == bd && oi < bi)) {
          bd = od;
          bi = oi;
        }
      }
      // a NaN in z leaves every comparison false: fall back to index 0 (what torch.argmin returns there is an
      // index too) instead of gathering out of bounds
      if (lane == 0) best_s[warp * 4 + i] = bi == 0x7fffffff ? 0 : bi;
    }
  } else {
    if (tid < kRT) best_s[tid] = -1;
  }
  __syncthreads();

  // ---- outputs
  if (tid < cnt) {
    const int row = rows_s[tid];
    const long long bi = best_s[tid];
    if (o.idx) o.idx[row] = bi;
    if (o.idx_cont) o.idx_cont[row] = selected ? bi + o.cont_stride * book : -1;
    if (o.idx_list)
      for (int k = 0; k < s.n_books; ++k) o.idx_list[(long long)k * s.rows + row] = (k == book) ? bi : -1;
  }
  if (o.zq_nhwc || o.zq_nchw || o.sqerr) {
    double err = 0.0;
    const float* cbk = selected ? cb + (long long)book * s.n_e * s.D : nullptr;
    for (int e = tid; e < cnt * s.D; e += kVqThreads) {
      const int rl = e / s.D, d = e % s.D;
      const int row = rows_s[rl];
      const long long zo = z_offset(s, row, d);
      const float zv = z[zo];
      const float qv = selected ? cbk[(long long)best_s[rl] * s.D + d] : 0.f;
      const float diff = __fsub_rn(qv, zv);
      const float outv = __fadd_rn(zv, diff);
      err += (double)diff * (double)diff;
      if (o.zq_nhwc) o.zq_nhwc[zo] = outv;
      if (o.zq_nchw) {
        // zo = ((b*Hz + y)*Wz + x)*Cz + c
        const int c = (int)(zo % s.Cz);
        const long long pix = zo / s.Cz;
        const int x = (int)(pix % s.Wz);
        const int y = (int)((pix / s.Wz) % s.Hz);
        const int b = (int)(pix / ((long long)s.Wz * s.Hz));
        o.zq_nchw[(((long long)b * s.Cz + c) * s.Hz + y) * s.Wz + x] = outv;
      }
    }
    if (o.sqerr) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) err += __shfl_xor_sync(0xffffffffu, err, off);
      if (lane == 0) atomicAdd(&err_s, err);
      __syncthreads();
      if (tid == 0) atomicAdd(o.sqerr, err_s);
    }
  }
}

// get_codebook_entry: plain gather (+ 2x2 fold)
__global__ void vq_gather_kernel(const float* __restrict__ cb, const long long* __restrict__ idx,
                                 const int* __restrict__ book_id, VqShape s, float* __restrict__ zq_nhwc,
                                 float* __restrict__ zq_nchw) {
  const long long total = (long long)s.rows * s.D;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(e / s.D), d = (int)(e % s.D);
    const int book = book_id ? book_id[row] : 0;
    const long long bi = idx[row];
    float v = 0.f;
    if (book >= 0 && book < s.n_books && bi >= 0 && bi < s.n_e)
      v = cb[((long long)book * s.n_e + bi) * s.D + d];
    const long long zo = z_offset(s, row, d);
    if (zq_nhwc) zq_nhwc[zo] = v;
    if (zq_nchw) {
      const int c = (int)(zo % s.Cz);
      const long long pix = zo / s.Cz;
      const int x = (int)(pix % s.Wz);
      const int y = (int)((pix / s.Wz) % s.Hz);
      const int b = (int)(pix / ((long long)s.Wz * s.Hz));
      zq_nchw[(((long long)b * s.Cz + c) * s.Hz + y) * s.Wz + x] = v;
    }
  }
}

// ---- patch quantizer backward (VectorQuantizerSpatialTextureAware.forward :438-454): zq_st = z + (zq - z).detach(),
// loss = mean((zq.detach()-z)^2) + beta*mean((zq - z.detach())^2) over the folded patches:
//   dz = dzq + coef_z * (z - e)                 (e = 0 for rows no codebook selects)
//   dE[book][code] += coef_e * (e - z_patch)    summed over the rows that chose the code, in ascending row order
// The codebook gradient uses no floating-point atomics: rows are sorted by (book, code) with a stable counting sort,
// then one warp reduces each code's segment, so reruns are bitwise equal.
constexpr int kVqSortThreads = 1024;

__device__ __forceinline__ int vq_code_key(const long long* __restrict__ idx, const int* __restrict__ book, int r,
                                           int n_books, int n_e) {
  const int k = book ? book[r] : 0;
  const long long id = idx[r];
  return (k >= 0 && k < n_books && id >= 0 && id < n_e) ? k * n_e + (int)id : n_books * n_e;
}

// One CTA.  off[key] = first slot of key (n_books*n_e keys + the bin of rows without a code), off[nb] = rows;
// order[slot] = row, rows in ascending order inside each key.
__global__ void __launch_bounds__(kVqSortThreads) vq_patch_sort_kernel(const long long* __restrict__ idx,
                                                                       const int* __restrict__ book, int rows,
                                                                       int n_books, int n_e, int* __restrict__ order,
                                                                       int* __restrict__ off) {
  extern __shared__ int cur[];  // [nb]: counts, then write cursors
  __shared__ int wsum[kVqSortThreads / 32];
  const int nb = n_books * n_e + 1;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < nb; i += kVqSortThreads) cur[i] = 0;
  __syncthreads();
  for (int r = tid; r < rows; r += kVqSortThreads) atomicAdd(&cur[vq_code_key(idx, book, r, n_books, n_e)], 1);
  __syncthreads();
  // exclusive scan: thread t owns the contiguous bins [lo, hi)
  const int per = (nb + kVqSortThreads - 1) / kVqSortThreads;
  const int lo = min(nb, tid * per), hi = min(nb, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += cur[i];
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int w = wsum[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= o) wi += v;
    }
    wsum[lane] = wi - w;
  }
  __syncthreads();
  int base = wsum[warp] + incl - s;
  for (int i = lo; i < hi; ++i) {
    const int c = cur[i];
    cur[i] = off[i] = base;
    base += c;
  }
  if (tid == 0) off[nb] = rows;
  __syncthreads();
  // stable scatter by one warp, 32 rows at a time: a row's rank among the equal keys of its 32 comes from
  // __match_any_sync, the lowest such lane advances the key's cursor
  if (warp != 0) return;
  for (int t0 = 0; t0 < rows; t0 += 32) {
    const int r = t0 + lane;
    const int k = r < rows ? vq_code_key(idx, book, r, n_books, n_e) : -1;
    const unsigned same = __match_any_sync(0xffffffffu, k);
    const int rank = __popc(same & ((1u << lane) - 1u));
    const int c = r < rows ? cur[k] : 0;
    __syncwarp();
    if (r < rows) {
      order[c + rank] = r;
      if (rank == 0) cur[k] = c + __popc(same);
    }
    __syncwarp();
  }
}

// dz over the NHWC elements of z (coalesced); the patch row and in-patch index come from the F.unfold order
__global__ void vq_patch_dz_kernel(const float* __restrict__ z, const float* __restrict__ cb,
                                   const long long* __restrict__ idx, const int* __restrict__ book,
                                   const float* __restrict__ dzq, VqShape s, float coef_z, float* __restrict__ dz) {
  const long long total = (long long)s.B * s.Hz * s.Wz * s.Cz;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % s.Cz);
    const long long pix = i / s.Cz;
    const int x = (int)(pix % s.Wz);
    const int y = (int)((pix / s.Wz) % s.Hz);
    const int b = (int)(pix / ((long long)s.Wz * s.Hz));
    const int row = (b * s.Hp + y / s.ps) * s.Wp + x / s.ps;
    const int d = c * s.ps * s.ps + (y % s.ps) * s.ps + x % s.ps;
    const int key = vq_code_key(idx, book, row, s.n_books, s.n_e);
    const float ev = key < s.n_books * s.n_e ? cb[(long long)key * s.D + d] : 0.f;
    dz[i] = (dzq ? dzq[i] : 0.f) + coef_z * (z[i] - ev);
  }
}

// one warp per code: dE[code][d] += coef_e * (e[d] - z_row[d]) for the code's rows in slot (= row) order
__global__ void __launch_bounds__(256) vq_patch_de_kernel(const float* __restrict__ z, const float* __restrict__ cb,
                                                          const int* __restrict__ order, const int* __restrict__ off,
                                                          VqShape s, float coef_e, float* __restrict__ dcb) {
  const int code = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (code >= s.n_books * s.n_e) return;
  const int beg = off[code], end = off[code + 1];
  if (beg == end) return;
  const float* e = cb + (long long)code * s.D;
  float* de = dcb + (long long)code * s.D;
  for (int d = lane; d < s.D; d += 32) {
    const float ev = e[d];
    float acc = de[d];
    for (int i = beg; i < end; ++i)
      acc = __fadd_rn(acc, __fmul_rn(coef_e, __fsub_rn(ev, z[z_offset(s, order[i], d)])));
    de[d] = acc;
  }
}

static int make_shape(VqShape* s, int b, int hz, int wz, int cz, int ps, int n_books, int n_e) {
  T2H_CHECK_ARG(b > 0 && hz > 0 && wz > 0 && cz > 0, "vq: bad z shape");
  T2H_CHECK_ARG(ps == 1 || ps == 2, "vq: patch size %d unsupported", ps);
  T2H_CHECK_ARG(hz % ps == 0 && wz % ps == 0, "vq: z extent not divisible by patch size");
  T2H_CHECK_ARG(n_books >= 1 && n_books <= 63, "vq: n_books=%d unsupported", n_books);
  T2H_CHECK_ARG(n_e >= 1, "vq: n_e=%d", n_e);
  s->B = b; s->Hz = hz; s->Wz = wz; s->Cz = cz; s->ps = ps;
  s->Hp = hz / ps; s->Wp = wz / ps; s->D = cz * ps * ps;
  T2H_CHECK_ARG(s->D % 4 == 0, "vq: D=%d must be a multiple of 4", s->D);
  const long long rows = (long long)b * s->Hp * s->Wp;
  T2H_CHECK_ARG(rows < (1LL << 30), "vq: too many rows");
  s->rows = (int)rows; s->n_books = n_books; s->n_e = n_e;
  return T2H_OK;
}

static inline int vq_max_tiles(long long rows, int n_books) {
  return (int)(rows / kRT + n_books + 2);
}

}  // namespace t2h

using namespace t2h;

extern "C" {

int64_t t2h_vq_workspace_bytes(int64_t rows, int n_books, int n_e) {
  const int64_t maxT = vq_max_tiles(rows, n_books);
  int64_t ints = 1 + 3 * maxT + rows;
  ints = (ints + 3) / 4 * 4;
  return ints * 4 + (int64_t)n_books * n_e * 4 + 64;
}

int t2h_vq_search(const float* z, const float* codebook, const int32_t* book_id, int b, int hz, int wz,
                  int cz, int ps, int n_books, int n_e, int64_t cont_stride, int64_t* idx,
                  int64_t* idx_cont, int64_t* idx_list, float* zq_nhwc, float* zq_nchw, double* sqerr,
                  void* workspace, int64_t workspace_bytes, t2h_stream_t stream) {
  T2H_CHECK_ARG(z && codebook && workspace, "vq_search: null pointer");
  VqShape s;
  int rc = make_shape(&s, b, hz, wz, cz, ps, n_books, n_e);
  if (rc) return rc;
  T2H_CHECK_ARG(workspace_bytes >= t2h_vq_workspace_bytes(s.rows, n_books, n_e),
                "vq_search: workspace too small (%lld < %lld)", (long long)workspace_bytes,
                (long long)t2h_vq_workspace_bytes(s.rows, n_books, n_e));
  T2H_CHECK_ARG(reinterpret_cast<uintptr_t>(codebook) % 16 == 0, "vq_search: codebook must be 16B aligned");
  cudaStream_t st = as_stream(stream);
  const int maxT = vq_max_tiles(s.rows, n_books);
  int* ws = reinterpret_cast<int*>(workspace);
  long long ints = 1 + 3LL * maxT + s.rows;
  ints = (ints + 3) / 4 * 4;
  float* ee = reinterpret_cast<float*>(ws + ints);

  const long long n_codes = (long long)n_books * n_e;
  vq_code_norms_kernel<<<(int)ceil_div64(n_codes, 8), 256, 0, st>>>(codebook, ee, n_codes, s.D);
  T2H_LAUNCH_OK();
  vq_bin_kernel<<<1, 1024, 0, st>>>(book_id, s.rows, n_books, maxT, ws);
  T2H_LAUNCH_OK();
  VqOut o{reinterpret_cast<long long*>(idx), reinterpret_cast<long long*>(idx_cont),
          reinterpret_cast<long long*>(idx_list), zq_nhwc, zq_nchw, sqerr, (long long)cont_stride};
  vq_search_kernel<<<maxT, kVqThreads, 0, st>>>(z, codebook, ee, ws, maxT, s, o);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_vq_gather(const float* codebook, const int64_t* idx, const int32_t* book_id, int b, int hz,
                  int wz, int cz, int ps, int n_books, int n_e, float* zq_nhwc, float* zq_nchw,
                  t2h_stream_t stream) {
  T2H_CHECK_ARG(codebook && idx && (zq_nhwc || zq_nchw), "vq_gather: null pointer");
  VqShape s;
  int rc = make_shape(&s, b, hz, wz, cz, ps, n_books, n_e);
  if (rc) return rc;
  const long long total = (long long)s.rows * s.D;
  long long g = ceil_div64(total, 256);
  if (g > num_sms() * 16LL) g = num_sms() * 16LL;
  vq_gather_kernel<<<(int)g, 256, 0, as_stream(stream)>>>(codebook, reinterpret_cast<const long long*>(idx),
                                                         book_id, s, zq_nhwc, zq_nchw);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

int t2h_vq_bwd_patch(const float* z, const float* codebook, const int64_t* idx, const int32_t* book_id,
                     const float* dzq, float* dz, float* dcodebook, int32_t* order, int32_t* off, int b, int hz, int wz,
                     int cz, int ps, int n_books, int n_e, float coef_z, float coef_e, t2h_stream_t stream) {
  T2H_CHECK_ARG(z && codebook && idx && dz && dcodebook && order && off, "vq_bwd_patch: null pointer");
  VqShape s;
  int rc = make_shape(&s, b, hz, wz, cz, ps, n_books, n_e);
  if (rc) return rc;
  const size_t smem = (size_t)(n_books * n_e + 1) * sizeof(int);
  T2H_CHECK_ARG(smem <= 48 * 1024, "vq_bwd_patch: n_books*n_e=%d codes too many for the sort", n_books * n_e);
  cudaStream_t st = as_stream(stream);
  const long long* id = reinterpret_cast<const long long*>(idx);
  vq_patch_sort_kernel<<<1, kVqSortThreads, smem, st>>>(id, book_id, s.rows, n_books, n_e, order, off);
  T2H_LAUNCH_OK();
  const long long total = (long long)b * hz * wz * cz;
  long long g = ceil_div64(total, 256);
  if (g > num_sms() * 16LL) g = num_sms() * 16LL;
  vq_patch_dz_kernel<<<(int)g, 256, 0, st>>>(z, codebook, id, book_id, dzq, s, coef_z, dz);
  T2H_LAUNCH_OK();
  vq_patch_de_kernel<<<(unsigned)ceil_div64((long long)n_books * n_e, 8), 256, 0, st>>>(z, codebook, order, off, s,
                                                                                         coef_e, dcodebook);
  T2H_LAUNCH_OK();
  return T2H_OK;
}

}  // extern "C"
