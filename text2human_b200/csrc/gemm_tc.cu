// t2h_tapgemm: persistent, warp-specialised wgmma implicit-GEMM for sm_90a.
//
//   warp 0   A producer     cp.async.bulk.tensor 4-D activation "slabs": the rows a tile needs
//                           for all vertical taps of one horizontal shift (zero OOB fill =
//                           conv padding), so a 3x3 conv loads activations 3x, not 9x
//   warp 3   B producer     4-D weight boxes, one per tap (own ring: no head-of-line blocking)
//   warps 4-11 consumers    two warpgroups; each issues wgmma (M=64, N=BN, K=16) for its 64 rows of the
//                           128-row tile on shifted views of the slab, accumulating in registers, then
//                           hands the accumulator to the epilogue through a shared-memory staging array
//                           (one row per thread): alpha/bias/GELU/residual/GroupNorm partial sums ->
//                           swizzled smem staging -> TMA store (residual tiles arrive by TMA load into
//                           smem).  Warps 8-11 join the epilogue only in the plane / plain-fp32 modes,
//                           taking the upper 32 columns of each 64-column unit.
//
// The contraction loop runs over (tap group, 64-channel chunk, tap, product term).  A tap is a
// spatial shift of the activation box (3x3 conv = 9 taps, 1x1/Linear/bmm = 1 tap); taps with the
// same horizontal shift form a group and share one slab.  A product term selects which fp16
// planes feed the MMA so that hi*lo + hi*hi + lo*hi reproduces an fp32 product on the fp16 tensor
// pipe; the hi/lo slabs and weight tiles are each loaded once per (group, chunk[, tap]).
//
// Replaces cuDNN/cuBLAS calls made by the reference modules — see include/t2h.h.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include "t2h_internal.h"
#include "t2h_ptx.cuh"

namespace t2h {

enum { EPI_DIRECT = 0, EPI_TMA_F32 = 1, EPI_TMA_PLANES = 2 };

struct TapGemmDev {
  int n_img, H, W;
  int TW, TH;  // spatial box of one 128-row block
  int tiles_w, tiles_h, n_tiles_n, total_tiles;
  int n_out, C, kchunks, nterms;
  int a_mn, b_mn;  // operand stored contraction-major (rows / columns contiguous): MN-major wgmma descriptors
  int ksplit, kper, total_work;  // split-K: work item = (tile, k-slice); total_work = total_tiles * ksplit
  int a_term_imgs, a_bcast, b_term_g, b_batched, b_batched_h;
  // taps grouped by (dx, img_off): one activation slab per group
  int ngroups, slab_rows;
  int a_slots, b_slots;  // ring depths (A slabs / B tiles)
  int debug;             // T2H_DEBUG bits (16: per-launch trace, see g_t2h_dbg)
  int g_dx[T2H_MAX_TAPS], g_ioff[T2H_MAX_TAPS], g_dy0[T2H_MAX_TAPS], g_ntaps[T2H_MAX_TAPS];
  int g_dyrel[T2H_MAX_TAPS][3], g_btap[T2H_MAX_TAPS][3];
  void* d;
  int d_mode, d_terms, epi_mode, d_term_imgs;
  long long d_plane, d_sn, d_sh, d_sw, d_sc;
  const float* bias;
  long long bias_sn;  // BIAS_COL: elements between the bias vectors of consecutive images (0 = shared)
  int bias_mode, act;
  float alpha;
  const float* residual;
  double* gn_stats;
  int gn_cpg, gn_groups;
  // conv weight-gradient mode (t2h_conv_wgrad): the contraction runs over 64-pixel patches (wg_PW x wg_PH) of the
  // images, both operands are NHWC planes read MN-major, the output "image" index is the tap whose (dy, dx,
  // img_off) shifts the X patch; accum: the epilogue reduce-adds into D even without split-K
  int wg, accum;
  int partials;  // split-K without reduction: k-slice s of a tile is stored to image slot t.img + s of D
  // norm-backward sums in the swapped kernel's epilogue (see t2h_tapgemm_params.nb_sums): `residual` is x
  double* nb_sums;
  const double* nb_stats;
  const float *nb_gamma, *nb_beta;
  float nb_eps;
  int nb_act, nb_groups;
  int n_major;  // tile index = column tile * row tiles + row tile (set with nb_sums; default is row-major)
  int wg_PW, wg_PH, wg_pw, wg_ppi;
  int wg_dy[T2H_MAX_TAPS], wg_dx[T2H_MAX_TAPS], wg_ioff[T2H_MAX_TAPS];
};

// profiling trace (T2H_DEBUG bit 16): CTA 0 of every tap-GEMM / attention launch appends one record of 8 words --
// globaltimer (ns) at {kernel entry, griddepcontrol.wait passed, first operand tile landed, last MMA issued,
// accumulator complete (epilogue woke), CTA done}, then {total work items, contraction chunks per item | kind << 32}
constexpr int kTraceRecords = 2048;
__device__ unsigned long long g_t2h_dbg[kTraceRecords * 8];
__device__ unsigned int g_t2h_dbg_n;
__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

constexpr int kBK = 64;                      // fp16 elements per 128-byte swizzled row
constexpr int kABlockBytes = 128 * 128;      // one 128-row A block of a stage
constexpr int kThreads = 384;  // warps 0-3 producers, warps 4-7 and 8-11 the two consumer warpgroups
constexpr int kEpiBufBytes = 128 * 128;      // one staging tile: 128 rows x 128 bytes
constexpr int kEpiBytes = 4 * kEpiBufBytes;  // 2 output + 2 residual staging tiles

constexpr int kMaxSlots = 8;
constexpr int kDynSmem = 227 * 1024 - 4096;  // opt-in limit minus ~4 KB of static shared memory

// Tiles are 128 rows by BN <= 128 columns: each consumer warpgroup holds a 64 x BN fp32 accumulator
// (BN / 2 registers per thread) and the [128][BN + 4] staging array (the padding spreads a column's rows over the
// shared-memory banks) fits beside the operand rings.
template <int BN>
struct Cfg {
  static_assert(BN <= 128, "sm_90a tiles are 128 x BN, BN <= 128");
  // A ring: slabs of (TH + 2) x TW positions x 128 bytes (TW <= 16 whenever taps share a slab)
  static constexpr int kASlot = kABlockBytes + 4096;
  static constexpr int kBSlot = BN * 128;
  static constexpr int kStageLd = BN + 4;  // fp32 words per staging row
  static constexpr int kStageBytes = 128 * kStageLd * 4;
  static constexpr int kRingBytes = kDynSmem - 1024 - kEpiBytes - kStageBytes;  // A ring + B ring
  static constexpr int kChunk = BN < 32 ? BN : 32;  // columns per staging read in the direct epilogue
};

struct TileCoord {
  int img, h0, w0, n0;
};

__device__ __forceinline__ TileCoord decode_tile(const TapGemmDev& P, int tile, int bn) {
  TileCoord t;
  int n_tile = tile % P.n_tiles_n;
  int m_tile = tile / P.n_tiles_n;
  if (P.n_major) {  // column tile is the slow index: a contiguous tile range stays on one (column block, image)
    const int mt = P.total_tiles / P.n_tiles_n;
    n_tile = tile / mt;
    m_tile = tile - n_tile * mt;
  }
  int per_img = P.tiles_h * P.tiles_w;
  t.img = m_tile / per_img;
  int rem = m_tile - t.img * per_img;
  int ty = rem / P.tiles_w;
  int tx = rem - ty * P.tiles_w;
  t.h0 = ty * P.TH;
  t.w0 = tx * P.TW;
  t.n0 = n_tile * bn;
  return t;
}

// byte offset of 16-byte chunk j of row r inside a 128B-swizzled [128 rows][128 bytes] tile
__device__ __forceinline__ int swz(int r, int j) { return r * 128 + ((j ^ (r & 7)) << 4); }

// Per-warp reduction of 2*NG per-thread partial sums (NG groups x {sum, sumsq}) over the 32 rows
// a warp holds, using a halving butterfly (2*NG-1 + log shuffles), then shared-memory atomics.
template <int NG>
__device__ __forceinline__ void gn_accumulate(const float (&v)[32], bool row_ok, int ncols_valid,
                                              float* gs, int lane) {
  constexpr int W = 32 / NG;
  constexpr int NV = 2 * NG;
  float vals[NV];
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    float s = 0.f, ss = 0.f;
#pragma unroll
    for (int i = 0; i < W; ++i) {
      const int c = g * W + i;
      const float x = (row_ok && c < ncols_valid) ? v[c] : 0.f;
      s += x;
      ss += x * x;
    }
    vals[2 * g] = s;
    vals[2 * g + 1] = ss;
  }
  int idx = 0;
  int step = 0;
#pragma unroll
  for (int n = NV; n > 1; n >>= 1, ++step) {
    const int off = 1 << step;
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float send = upper ? vals[i] : vals[i + n / 2];
      const float recv = __shfl_xor_sync(0xffffffffu, send, off);
      const float keep = upper ? vals[i + n / 2] : vals[i];
      vals[i] = keep + recv;
    }
    idx |= (upper ? 1 : 0) * (n / 2);
  }
#pragma unroll
  for (int off = NV; off < 32; off <<= 1) vals[0] += __shfl_xor_sync(0xffffffffu, vals[0], off);
  if (lane < NV) atomicAdd(&gs[idx], vals[0]);
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
tapgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
               const __grid_constant__ TapGemmDev P) {
  using C = Cfg<BN>;
  pdl_launch_dependents();  // the next kernel may start its prologue once every CTA of this one is running
  const int NA = P.a_slots, NB = P.b_slots;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem =
      reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = smem + NA * C::kASlot;
  uint8_t* out_buf = b_ring + NB * C::kBSlot;     // 2 tiles
  uint8_t* res_buf = out_buf + 2 * kEpiBufBytes;  // 2 tiles
  float* const stage = reinterpret_cast<float*>(res_buf + 2 * kEpiBufBytes);  // [128][kStageLd] accumulator
  constexpr int LD = C::kStageLd;

  __shared__ __align__(8) uint64_t a_full[kMaxSlots];
  __shared__ __align__(8) uint64_t a_empty[kMaxSlots];
  __shared__ __align__(8) uint64_t b_full[kMaxSlots];
  __shared__ __align__(8) uint64_t b_empty[kMaxSlots];
  __shared__ __align__(8) uint64_t res_bar[2];
  __shared__ float gsum[2][2 * 128];  // GroupNorm partial sums of the current / previous tile
  __shared__ __align__(16) float sbias[BN];  // column bias of the current tile (plane epilogue)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // Two epilogue warp groups (warps 4-7: columns 0..31 of every 64-column unit, warps 8-11: columns 32..63) in the
  // modes whose epilogue is pure per-element work; the residual / GroupNorm-statistics / strided paths keep one.
  bool two_groups = false;
  if constexpr (BN >= 64) {
    two_groups = P.epi_mode == EPI_TMA_PLANES ||
                 (P.epi_mode == EPI_TMA_F32 && !P.residual && !P.gn_stats && P.act == T2H_ACT_NONE &&
                  P.bias_mode != T2H_BIAS_ROW);
  }
  const int n_epi = two_groups ? 256 : 128;  // threads at the epilogue's named barriers
  __shared__ unsigned long long* trace_s;  // this launch's trace record (CTA 0, T2H_DEBUG bit 16), else null

  if (warp == 0 && lane == 0) {
    trace_s = nullptr;
    if ((P.debug & 16) && blockIdx.x == 0) {
      trace_s = g_t2h_dbg + (size_t)(atomicAdd(&g_t2h_dbg_n, 1u) % kTraceRecords) * 8;
      trace_s[0] = gtime_ns();
      trace_s[6] = (unsigned long long)P.total_work;
      trace_s[7] = (unsigned long long)min(P.kper, P.kchunks) * P.ngroups;
    }
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (P.epi_mode != EPI_DIRECT) tma_prefetch_desc(&tmD);
    if (P.epi_mode == EPI_TMA_F32 && P.residual) tma_prefetch_desc(&tmR);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < NA; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 256);  // every consumer thread releases a slot
    }
    for (int s = 0; s < NB; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 256);
    }
    for (int s = 0; s < 2; ++s) mbar_init(&res_bar[s], 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < 2 * 2 * 128; i += kThreads) (&gsum[0][0])[i] = 0.f;
  __syncthreads();
  // everything above touched only shared memory and kernel parameters; from here on the previous
  // kernel's results are read (and buffers it may still be reading are overwritten)
  pdl_wait();
  unsigned long long* const trace = trace_s;
  if (trace && threadIdx.x == 0) trace[1] = gtime_ns();

  const int a_planes = (P.nterms == 3) ? 2 : 1;  // slabs per (group, chunk): hi [, lo]
  const int slab_bytes = P.slab_rows * P.TW * 128;
  const int work0 = (int)blockIdx.x;
  const int work_stride = (int)gridDim.x;

  if (warp == 0) {
    // ---------------------------------------------- A producer (activation slabs)
    if (lane == 0) {
      int sa = 0, pa = 0;
      for (int work = work0; work < P.total_work; work += work_stride) {
        const int tile = work % P.total_tiles;
        const int ch0 = (work / P.total_tiles) * P.kper;
        const int ch1 = min(P.kchunks, ch0 + P.kper);
        const TileCoord t = decode_tile(P, tile, BN);
        const int a_img = P.a_bcast ? 0 : t.img;
        for (int g = 0; g < P.ngroups; ++g) {
          for (int ch = ch0; ch < ch1; ++ch) {
            for (int pl = 0; pl < a_planes; ++pl) {  // hi, then lo
              mbar_wait(&a_empty[sa], pa ^ 1);
              if (P.a_mn) {
                // [k][row] storage: two boxes of 64 rows x 64 k per 128-row block
                mbar_expect_tx(&a_full[sa], kABlockBytes);
                int c1 = ch * kBK, c2 = t.h0, c3 = a_img + pl * P.a_term_imgs;
                if (P.wg) {  // chunk = one 64-pixel patch of dY: (channel, x, y, image)
                  const int n = ch / P.wg_ppi, r = ch - n * P.wg_ppi, py = r / P.wg_pw, px = r - py * P.wg_pw;
                  c1 = px * P.wg_PW; c2 = py * P.wg_PH; c3 = n + pl * P.a_term_imgs;
                }
#pragma unroll
                for (int hbox = 0; hbox < 2; ++hbox)
                  tma_load_4d(&tmA, &a_full[sa], a_ring + sa * C::kASlot + hbox * 8192, t.w0 + 64 * hbox,
                              c1, c2, c3);
              } else {
                mbar_expect_tx(&a_full[sa], slab_bytes);
                tma_load_4d(&tmA, &a_full[sa], a_ring + sa * C::kASlot, ch * kBK, t.w0 + P.g_dx[g],
                            t.h0 + P.g_dy0[g], a_img + P.g_ioff[g] + pl * P.a_term_imgs);
              }
              if (++sa == NA) {
                sa = 0;
                pa ^= 1;
              }
            }
          }
        }
      }
    }
  } else if (warp == 3) {
    // ---------------------------------------------- B producer (weight tiles)
    if (lane == 0) {
      int sb = 0, pb = 0;
      const int b_planes = a_planes;
      for (int work = work0; work < P.total_work; work += work_stride) {
        const int tile = work % P.total_tiles;
        const int ch0 = (work / P.total_tiles) * P.kper;
        const int ch1 = min(P.kchunks, ch0 + P.kper);
        const TileCoord t = decode_tile(P, tile, BN);
        const int b_g2 = P.b_batched ? t.img : 0;
        const int b_g = P.b_batched_h ? t.h0 : 0;
        for (int g = 0; g < P.ngroups; ++g) {
          for (int ch = ch0; ch < ch1; ++ch) {
            for (int tp = 0; tp < P.g_ntaps[g]; ++tp) {
              for (int pl = b_planes - 1; pl >= 0; --pl) {  // lo first, then hi (consumption order)
                mbar_wait(&b_empty[sb], pb ^ 1);
                mbar_expect_tx(&b_full[sb], C::kBSlot);
                if (P.b_mn) {
                  // [k][column] storage: one box of 64 columns x 64 k per 64 output columns
                  int c1 = ch * kBK, c2 = b_g + P.g_btap[g][tp] + pl * P.b_term_g, c3 = b_g2;
                  if (P.wg) {  // the same patch of X, shifted by this output tile's tap
                    const int n = ch / P.wg_ppi, r = ch - n * P.wg_ppi, py = r / P.wg_pw, px = r - py * P.wg_pw;
                    c1 = px * P.wg_PW + P.wg_dx[t.img]; c2 = py * P.wg_PH + P.wg_dy[t.img];
                    c3 = n + P.wg_ioff[t.img] + pl * P.b_term_g;
                  }
                  for (int q = 0; q < BN / 64; ++q)
                    tma_load_4d(&tmB, &b_full[sb], b_ring + sb * C::kBSlot + q * 8192, t.n0 + 64 * q, c1, c2, c3);
                } else {
                  tma_load_4d(&tmB, &b_full[sb], b_ring + sb * C::kBSlot, ch * kBK, t.n0,
                              b_g + P.g_btap[g][tp] + pl * P.b_term_g, b_g2);
                }
                if (++sb == NB) {
                  sb = 0;
                  pb ^= 1;
                }
              }
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------ consumers: wgmma, then the epilogue
    const int wg = (warp - 4) >> 2;  // rows 64 wg .. 64 wg + 63 of the tile
    const int wt = threadIdx.x & 127;
    const bool epi = warp < 8 || two_groups;
    const uint64_t a_desc0 = gmma_desc(smem_u32(a_ring) + 8192u * wg, P.a_mn);
    const uint64_t b_desc0 = gmma_desc(smem_u32(b_ring), P.b_mn);
    const uint32_t row16 = (uint32_t)(P.TW * 128) >> 4;  // one slab image row, in 16-byte units
    constexpr uint32_t A16 = C::kASlot >> 4, B16 = C::kBSlot >> 4;
    const int ngroups = P.ngroups;
    int sa = 0, pa = 0, sb = 0, pb = 0;
    // every consumer thread arrives once the warpgroup's MMAs reading the slot have completed (a lane-0 arrival
    // between wgmmas puts them on a divergent path, and ptxas then serialises every MMA)
    auto release = [&](uint64_t* bar) { mbar_arrive(bar); };

    const int grp = (warp - 4) >> 2;  // 0: warps 4-7, 1: warps 8-11
    const int q = warp & 3;           // rows 32 q .. 32 q + 31 of the staging array
    const int row = q * 32 + lane;
    const int th = row / P.TW, tw = row - th * P.TW;
    const bool elected = (threadIdx.x == 128);
    int buf = 0;  // staging buffer toggle (persists across tiles)
    uint32_t res_par = 0;  // bit b: phase of res_bar[b]
    int tile_par = 0;  // gsum buffer of this tile

    for (int work = work0; work < P.total_work; work += work_stride) {
      const int tile = work % P.total_tiles;
      const int ch0 = (work / P.total_tiles) * P.kper;
      const int ch1 = min(P.kchunks, ch0 + P.kper);
      float acc[BN / 2];
      uint32_t accf = 0;
      // D (+)= A_view(dy) * B_tile, complete on return (the caller then releases the slots it read)
      auto batch = [&](uint64_t a, uint64_t b) {
        wgmma_fence();
        if (P.a_mn) {
          if (P.b_mn) wgmma_chunk<1, 1>(acc, a, b, accf);
          else wgmma_chunk<1, 0>(acc, a, b, accf);
        } else {
          if (P.b_mn) wgmma_chunk<0, 1>(acc, a, b, accf);
          else wgmma_chunk<0, 0>(acc, a, b, accf);
        }
        wgmma_commit();
        wgmma_wait<0>();
      };
      for (int g = 0; g < ngroups; ++g) {
        const int nt = P.g_ntaps[g];
        const uint32_t dy0 = P.g_dyrel[g][0] * row16, dy1 = P.g_dyrel[g][1] * row16,
                       dy2 = P.g_dyrel[g][2] * row16;
        for (int ch = ch0; ch < ch1; ++ch) {
          // slab slots of this (group, chunk)
          const int sa_hi = sa, pa_hi = pa;
          if (++sa == NA) { sa = 0; pa ^= 1; }
          const int sa_lo = sa, pa_lo = pa;
          if (a_planes == 2) {
            if (++sa == NA) { sa = 0; pa ^= 1; }
          }
          mbar_wait(&a_full[sa_hi], pa_hi);
          if (trace && threadIdx.x == 128 && work == work0 && g == 0 && ch == ch0) trace[2] = gtime_ns();
          const uint64_t ahi = a_desc0 + sa_hi * A16;
          const uint64_t alo = a_desc0 + sa_lo * A16;
          for (int tp = 0; tp < nt; ++tp) {
            const uint32_t dy = tp == 0 ? dy0 : (tp == 1 ? dy1 : dy2);
            if (a_planes == 1) {
              mbar_wait(&b_full[sb], pb);
              batch(ahi + dy, b_desc0 + sb * B16);
              release(&b_empty[sb]);
              if (++sb == NB) { sb = 0; pb ^= 1; }
            } else {
              mbar_wait(&b_full[sb], pb);  // B lo
              batch(ahi + dy, b_desc0 + sb * B16);  // hi*lo
              release(&b_empty[sb]);
              if (++sb == NB) { sb = 0; pb ^= 1; }
              mbar_wait(&b_full[sb], pb);  // B hi
              const uint64_t bhi = b_desc0 + sb * B16;
              batch(ahi + dy, bhi);  // hi*hi
              if (tp == nt - 1) release(&a_empty[sa_hi]);  // hi slab done
              if (tp == 0) mbar_wait(&a_full[sa_lo], pa_lo);
              batch(alo + dy, bhi);  // lo*hi
              release(&b_empty[sb]);
              if (++sb == NB) { sb = 0; pb ^= 1; }
            }
          }
          release(a_planes == 1 ? &a_empty[sa_hi] : &a_empty[sa_lo]);
        }
      }
      wgmma_fence_regs(acc);
      if (trace && threadIdx.x == 128 && work == work0) trace[3] = gtime_ns();
      named_bar_sync(3, 256);  // the previous tile's epilogue has read the staging array
      acc_store_rows(acc, stage, LD, wg, wt);
      named_bar_sync(3, 256);
      if (!epi) continue;
      const TileCoord t = decode_tile(P, tile, BN);

      const bool plain_f32 = two_groups && P.epi_mode == EPI_TMA_F32;
      if (plain_f32) {
        // ---- fp32 output with nothing but alpha / column bias in the epilogue (split-K slices, weight gradients,
        // plain projections): 64-column units = two 32-column staging tiles, two pairs of them, so that a unit is
        // converted while the previous unit's TMA stores still read theirs -- half the barrier rounds of the
        // general path below
        const int cols_left = P.n_out - t.n0;
        const int nuc = (cols_left >= BN) ? BN / 64 : (cols_left + 63) / 64;
        const bool add_bias = P.bias_mode == T2H_BIAS_COL && ch0 == 0;  // split-K: the first k-slice carries the bias
        if (add_bias) {
          for (int i = threadIdx.x - 128; i < BN; i += 256)
            sbias[i] = (t.n0 + i < P.n_out) ? __ldg(P.bias + t.img * P.bias_sn + t.n0 + i) : 0.f;
        }
        if (trace && elected && work == work0) trace[4] = gtime_ns();
        for (int cc = 0; cc < nuc; ++cc) {
          const int col0 = t.n0 + cc * 64;
          uint8_t* const o0 = buf ? res_buf : out_buf;
          named_bar_sync(1, n_epi);  // this pair is free (elected waited for the stores issued two units ago)
          {
            const int half = grp;
            uint32_t r[32];
            stage_ld<32>(stage, LD, row, cc * 64 + half * 32, r);
            uint8_t* const ob = o0 + half * kEpiBufBytes;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float4 o = make_float4(__uint_as_float(r[4 * j]) * P.alpha, __uint_as_float(r[4 * j + 1]) * P.alpha,
                                     __uint_as_float(r[4 * j + 2]) * P.alpha, __uint_as_float(r[4 * j + 3]) * P.alpha);
              if (add_bias) {
                const float4 b4 = *reinterpret_cast<const float4*>(sbias + cc * 64 + half * 32 + 4 * j);
                o.x += b4.x; o.y += b4.y; o.z += b4.z; o.w += b4.w;
              }
              *reinterpret_cast<float4*>(ob + swz(row, j)) = o;
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(2, n_epi);
          if (elected) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
              const int c0 = col0 + half * 32;
              if (c0 >= P.n_out) break;
              const uint8_t* ob = o0 + half * kEpiBufBytes;
              if (P.partials)  // deterministic split-K: every k-slice owns a slab; a fixed-order pass sums them
                tma_store_4d(&tmD, ob, c0, t.w0, t.h0, t.img + work / P.total_tiles);
              else if (P.ksplit > 1 || P.accum)
                tma_reduce_add_4d(&tmD, ob, c0, t.w0, t.h0, t.img);
              else
                tma_store_4d(&tmD, ob, c0, t.w0, t.h0, t.img);
            }
            tma_store_commit();
            tma_store_wait_read<1>();  // the other pair is free again
          }
          buf ^= 1;
        }
      } else if (P.epi_mode == EPI_TMA_F32) {
        // ---- fp32 NHWC output: 32-column units through swizzled smem + TMA store
        const int cols_left = P.n_out - t.n0;
        const int nuc = (cols_left >= BN) ? BN / 32 : (cols_left + 31) / 32;
        const bool has_res = P.residual != nullptr;
        auto issue_res = [&](int cc, int b) {
          mbar_expect_tx(&res_bar[b], kEpiBufBytes);
          tma_load_4d(&tmR, &res_bar[b], res_buf + b * kEpiBufBytes, t.n0 + cc * 32, t.w0, t.h0, t.img);
        };
        if (has_res && elected) {
          issue_res(0, buf);
          if (nuc > 1) issue_res(1, buf ^ 1);
        }
        if (trace && elected && work == work0) trace[4] = gtime_ns();
        for (int cc = 0; cc < nuc; ++cc) {
          const int col0 = t.n0 + cc * 32;
          const int h = t.h0 + th;
          const int w = t.w0 + tw;
          const bool row_ok = (h < P.H) && (w < P.W);
          uint32_t r[32];
          stage_ld<32>(stage, LD, row, cc * 32, r);
          float v[32];
          const float row_bias =
              (P.bias_mode == T2H_BIAS_ROW && row_ok) ? __ldg(P.bias + h * P.W + w) : 0.f;
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]) * P.alpha + row_bias;
          if (P.bias_mode == T2H_BIAS_COL && ch0 == 0) {  // split-K: the first k-slice carries the bias
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              if (col0 + i < P.n_out) {  // n_out % 4 == 0 in this mode
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(P.bias + t.img * P.bias_sn + col0 + i));
                v[i] += b4.x; v[i + 1] += b4.y; v[i + 2] += b4.z; v[i + 3] += b4.w;
              }
            }
          }
          if (P.act == T2H_ACT_GELU) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
          } else if (P.act == T2H_ACT_RELU) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
          } else if (P.act == T2H_ACT_LRELU) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = v[i] > 0.f ? v[i] : 0.2f * v[i];
          }
          if (has_res) {
            mbar_wait(&res_bar[buf], (res_par >> buf) & 1);
            res_par ^= 1u << buf;
            const uint8_t* rb = res_buf + buf * kEpiBufBytes;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float4 rr = *reinterpret_cast<const float4*>(rb + swz(row, j));
              v[4 * j] += rr.x; v[4 * j + 1] += rr.y; v[4 * j + 2] += rr.z; v[4 * j + 3] += rr.w;
            }
          }
          if (P.gn_stats) {
            float* gs = &gsum[tile_par][0];
            const int ncv = P.n_out - col0;
            switch (P.gn_cpg) {
              case 2: gn_accumulate<16>(v, row_ok, ncv, gs + 2 * (cc * 16), lane); break;
              case 4: gn_accumulate<8>(v, row_ok, ncv, gs + 2 * (cc * 8), lane); break;
              case 8: gn_accumulate<4>(v, row_ok, ncv, gs + 2 * (cc * 4), lane); break;
              case 16: gn_accumulate<2>(v, row_ok, ncv, gs + 2 * (cc * 2), lane); break;
              default: gn_accumulate<1>(v, row_ok, ncv, gs + 2 * ((cc * 32) / P.gn_cpg), lane); break;
            }
          }
          named_bar_sync(1, 128);  // out_buf[buf] is free (elected waited for its previous store)
          uint8_t* ob = out_buf + buf * kEpiBufBytes;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(ob + swz(row, j)) =
                make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          fence_proxy_async_smem();
          named_bar_sync(2, 128);  // staging tile complete; residual tile fully consumed
          if (elected) {
            if (P.partials)  // deterministic split-K: every k-slice owns a slab; a fixed-order pass sums them
              tma_store_4d(&tmD, ob, col0, t.w0, t.h0, t.img + work / P.total_tiles);
            else if (P.ksplit > 1 || P.accum)
              tma_reduce_add_4d(&tmD, ob, col0, t.w0, t.h0, t.img);  // partial sum of a k-slice
            else
              tma_store_4d(&tmD, ob, col0, t.w0, t.h0, t.img);
            tma_store_commit();
            if (has_res && cc + 2 < nuc) issue_res(cc + 2, buf);
            tma_store_wait_read<1>();  // the other staging tile is free again
          }
          buf ^= 1;
        }
        if (P.gn_stats) {
          // all shared atomics of this tile happened before the last named barrier
          const int et = threadIdx.x - 128;
          const int ngt = (BN + P.gn_cpg - 1) / P.gn_cpg;  // groups this tile can touch
          for (int sl = et; sl < 2 * ngt; sl += 128) {
            const int g = t.n0 / P.gn_cpg + (sl >> 1);
            if (g < P.gn_groups)
              atomicAdd(&P.gn_stats[((long long)t.img * P.gn_groups + g) * 2 + (sl & 1)],
                        (double)gsum[tile_par][sl]);
            gsum[tile_par][sl] = 0.f;
          }
          tile_par ^= 1;
        }
      } else if (P.epi_mode == EPI_TMA_PLANES) {
        // ---- fp16 plane output: 64-column units, hi and lo tiles staged side by side
        const int cols_left = P.n_out - t.n0;
        const int nuc = (cols_left >= BN) ? BN / 64 : (cols_left + 63) / 64;
        // the tile's column bias goes to shared memory once per tile (broadcast reads below instead of L2 round trips
        // between every accumulator read and the stores); visible after the first named barrier below
        // (single buffer: whoever gets here has passed the previous tile's last named barrier, which every thread
        // reaches only after its last read of the previous bias)
        float* const sb = sbias;
        if (P.bias_mode == T2H_BIAS_COL) {
          for (int i = threadIdx.x - 128; i < BN; i += n_epi)
            sb[i] = (t.n0 + i < P.n_out) ? __ldg(P.bias + t.img * P.bias_sn + t.n0 + i) : 0.f;
        }
        if (trace && elected && work == work0) trace[4] = gtime_ns();
        for (int cc = 0; cc < nuc; ++cc) {
          const int col0 = t.n0 + cc * 64;
          const int h = t.h0 + th;
          const int w = t.w0 + tw;
          const bool row_ok = (h < P.H) && (w < P.W);
          const float row_bias =
              (P.bias_mode == T2H_BIAS_ROW && row_ok) ? __ldg(P.bias + h * P.W + w) : 0.f;
          // two pairs of staging tiles (the residual tiles are unused in this mode): unit u + 1 is converted while
          // unit u's TMA stores still read theirs
          uint8_t* ohi = buf ? res_buf : out_buf;
          uint8_t* olo = ohi + kEpiBufBytes;
          named_bar_sync(1, n_epi);  // this pair is free (elected waited for the stores issued two units ago)
#pragma unroll
          for (int half = two_groups ? grp : 0; half < (two_groups ? grp + 1 : 2); ++half) {
            uint32_t r[32];
            stage_ld<32>(stage, LD, row, cc * 64 + half * 32, r);
            float v[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]) * P.alpha + row_bias;
            if (P.bias_mode == T2H_BIAS_COL) {
#pragma unroll
              for (int i = 0; i < 32; i += 4) {
                const float4 b4 = *reinterpret_cast<const float4*>(sb + cc * 64 + half * 32 + i);  // broadcast read
                v[i] += b4.x; v[i + 1] += b4.y; v[i + 2] += b4.z; v[i + 3] += b4.w;
              }
            }
            if (P.act == T2H_ACT_GELU) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = gelu_erf(v[i]);
            } else if (P.act == T2H_ACT_RELU) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
            } else if (P.act == T2H_ACT_LRELU) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = v[i] > 0.f ? v[i] : 0.2f * v[i];
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              __align__(16) __half hi[8];
              __align__(16) __half lo[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) split_f16(v[8 * j + e], hi[e], lo[e]);
              *reinterpret_cast<uint4*>(ohi + swz(row, half * 4 + j)) = *reinterpret_cast<uint4*>(hi);
              if (P.d_terms == 2)
                *reinterpret_cast<uint4*>(olo + swz(row, half * 4 + j)) = *reinterpret_cast<uint4*>(lo);
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(2, n_epi);
          if (elected) {
            tma_store_4d(&tmD, ohi, col0, t.w0, t.h0, t.img);
            if (P.d_terms == 2)
              tma_store_4d(&tmD, olo, col0, t.w0, t.h0, t.img + P.d_term_imgs);
            tma_store_commit();
            tma_store_wait_read<1>();  // the other pair of staging tiles is free again
          }
          buf ^= 1;
        }
      } else {
        // ---- direct path: strided / tiny outputs (NCHW conv_out, n_out < 32, unaligned)
        constexpr int CH = C::kChunk;
        if (trace && elected && work == work0) trace[4] = gtime_ns();
        const int h = t.h0 + th;
        const int w = t.w0 + tw;
        const bool row_ok = (h < P.H) && (w < P.W);
        const long long off = (long long)t.img * P.d_sn + (long long)h * P.d_sh + (long long)w * P.d_sw;
        const float row_bias = (P.bias_mode == T2H_BIAS_ROW && row_ok) ? P.bias[h * P.W + w] : 0.f;
#pragma unroll 1
        for (int cc = 0; cc < BN / CH; ++cc) {
          const int col0 = t.n0 + cc * CH;
          if (col0 >= P.n_out) break;  // warp-uniform
          uint32_t r[32];
          stage_ld<CH>(stage, LD, row, cc * CH, r);
          if (!row_ok) continue;
          float v[CH];
#pragma unroll
          for (int i = 0; i < CH; ++i) v[i] = __uint_as_float(r[i]) * P.alpha + row_bias;
          if (P.bias_mode == T2H_BIAS_COL) {
#pragma unroll
            for (int i = 0; i < CH; ++i)
              if (col0 + i < P.n_out) v[i] += __ldg(P.bias + t.img * P.bias_sn + col0 + i);
          }
          if (P.act == T2H_ACT_GELU) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] = gelu_erf(v[i]);
          } else if (P.act == T2H_ACT_RELU) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] = fmaxf(v[i], 0.f);
          } else if (P.act == T2H_ACT_LRELU) {
#pragma unroll
            for (int i = 0; i < CH; ++i) v[i] = v[i] > 0.f ? v[i] : 0.2f * v[i];
          }
          if (P.d_mode == T2H_OUT_F32) {
            float* dst = reinterpret_cast<float*>(P.d);
#pragma unroll
            for (int i = 0; i < CH; ++i) {
              if (col0 + i < P.n_out) {
                const long long o = off + (long long)(col0 + i) * P.d_sc;
                float val = v[i];
                if (P.residual) val += P.residual[o];
                dst[o] = val;
              }
            }
          } else {
            __half* dst = reinterpret_cast<__half*>(P.d);
#pragma unroll
            for (int i = 0; i < CH; ++i) {
              if (col0 + i < P.n_out) {
                const long long o = off + (long long)(col0 + i) * P.d_sc;
                __half hi, lo;
                split_f16(v[i], hi, lo);
                dst[o] = hi;
                if (P.d_terms == 2) dst[P.d_plane + o] = lo;
              }
            }
          }
        }
      }
    }
    if (elected) tma_store_wait_read<0>();
    if (trace && elected) trace[5] = gtime_ns();
  }

}

}  // namespace t2h

#include "gemm_tc_swap.cuh"

namespace t2h {

// ------------------------------------------------------------------ host side
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                        const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                        const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

// elem_bytes: 2 (fp16) or 4 (fp32); strides in elements
static int make_tmap(CUtensorMap* tm, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                     const uint64_t* strides_elems, const uint32_t* box, const char* what,
                     CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_tmapEncodeTiled enc = get_encode_fn();
  if (!enc) return fail(T2H_ECUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t gdim[5], gstr[5];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_elems[i] * elem_bytes;
      if (gstr[i - 1] % 16 != 0)
        return fail(T2H_EINVAL, "%s: stride of dim %d (%llu bytes) is not a multiple of 16", what, i,
                    (unsigned long long)gstr[i - 1]);
    }
  }
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0)
    return fail(T2H_EINVAL, "%s: base pointer not 16-byte aligned", what);
  CUresult r = enc(tm, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                   rank, const_cast<void*>(base), gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(T2H_ECUDA,
                "%s: cuTensorMapEncodeTiled failed (%d) dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]",
                what, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1],
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
  return T2H_OK;
}

template <int BN>
static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                  const CUtensorMap& tmR, const TapGemmDev& P, cudaStream_t stream) {
  using C = Cfg<BN>;
  static bool configured[64] = {};
  int dev = 0;
  T2H_CUDA(cudaGetDevice(&dev));
  if (!configured[dev & 63]) {  // per device: the attribute lives in the device's copy of the function
    T2H_CUDA(cudaFuncSetAttribute(tapgemm_kernel<BN>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, kDynSmem));
    configured[dev & 63] = true;
  }
  // ring depths: enough bytes in flight to cover the TMA round trip at the tile's consumption rate.
  // With the 3-product split both (hi, lo) slabs of a (group, chunk) are live at once.
  TapGemmDev Q = P;
  Q.debug = debug_bits();
  Q.a_slots = 3;
  int nb = (C::kRingBytes - Q.a_slots * C::kASlot) / C::kBSlot;
  Q.b_slots = nb > kMaxSlots ? kMaxSlots : nb;
  if (Q.b_slots < 2) return fail(T2H_EINVAL, "tapgemm: shared-memory rings do not fit");
  int grid = P.total_work < num_sms() ? P.total_work : num_sms();
  // the full dynamic allocation keeps it to one CTA per SM
  T2H_CUDA(launch_pdl(tapgemm_kernel<BN>, dim3(grid), dim3(kThreads), kDynSmem, stream, tmA, tmB, tmD, tmR, Q));
  return T2H_OK;
}

static int launch_swap(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                       const CUtensorMap& tmR, const TapGemmDev& P, cudaStream_t stream) {
  using C = Cfg<128>;
  static bool configured[64] = {};
  int dev = 0;
  T2H_CUDA(cudaGetDevice(&dev));
  if (!configured[dev & 63]) {
    T2H_CUDA(cudaFuncSetAttribute(tapgemm_swap_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDynSmem));
    configured[dev & 63] = true;
  }
  TapGemmDev Q = P;
  // ring depths from what the register epilogue leaves of the shared memory: 4 A slabs load the next chunk's hi and
  // lo slabs during the whole current chunk, the rest holds weight tiles (4: two taps of the 3-product order ahead).
  // The kernel's ring invariant needs a_slots >= 2 and b_slots >= 2.
  Q.a_slots = 4;
  int nb = (kSwapRingBytes - Q.a_slots * C::kASlot) / C::kBSlot;
  Q.b_slots = nb > kMaxSlots ? kMaxSlots : nb;
  if (Q.b_slots < 2) return fail(T2H_EINVAL, "tapgemm: shared-memory rings do not fit");
  int grid = P.total_tiles < num_sms() ? P.total_tiles : num_sms();
  T2H_CUDA(launch_pdl(tapgemm_swap_kernel, dim3(grid), dim3(kSwapThreads), kDynSmem, stream, tmA, tmB, tmD, tmR, Q));
  return T2H_OK;
}

}  // namespace t2h

using namespace t2h;

extern "C" int t2h_debug_read(long long* out, int n) {
  // out[0] = records written so far (the ring keeps the last kTraceRecords), then up to (n - 1) / 8 records
  T2H_CHECK_ARG(out && n >= 1, "debug_read: bad args");
  unsigned int cnt = 0;
  T2H_CUDA(cudaDeviceSynchronize());
  T2H_CUDA(cudaMemcpyFromSymbol(&cnt, g_t2h_dbg_n, sizeof(cnt)));
  out[0] = cnt;
  int words = n - 1;
  if (words > kTraceRecords * 8) words = kTraceRecords * 8;
  if (words > 0) T2H_CUDA(cudaMemcpyFromSymbol(out + 1, g_t2h_dbg, sizeof(long long) * words));
  return T2H_OK;
}

extern "C" int t2h_tapgemm(const t2h_tapgemm_params* p, t2h_stream_t stream) {
  T2H_CHECK_ARG(p && p->a && p->b && p->d, "tapgemm: null operand");
  T2H_CHECK_ARG(p->n_img > 0 && p->H > 0 && p->W > 0 && p->C > 0 && p->n_out > 0,
                "tapgemm: empty problem (n_img=%d H=%d W=%d C=%d n_out=%d)", p->n_img, p->H, p->W, p->C,
                p->n_out);
  T2H_CHECK_ARG(p->ntaps >= 1 && p->ntaps <= T2H_MAX_TAPS, "tapgemm: ntaps=%d", p->ntaps);
  T2H_CHECK_ARG(p->nterms == 1 || p->nterms == 3, "tapgemm: nterms must be 1 or 3 (got %d)", p->nterms);
  T2H_CHECK_ARG(p->nterms == 1 || (p->a_terms == 2 && p->b_terms == 2),
                "tapgemm: nterms=3 needs hi/lo planes on both operands");
  T2H_CHECK_ARG(p->d_mode == T2H_OUT_F32 || p->d_mode == T2H_OUT_PLANES, "tapgemm: d_mode=%d", p->d_mode);
  T2H_CHECK_ARG(p->d_mode == T2H_OUT_F32 || p->d_terms == 1 || p->d_terms == 2, "tapgemm: d_terms=%d",
                p->d_terms);
  T2H_CHECK_ARG(p->d_mode == T2H_OUT_F32 || p->residual == nullptr,
                "tapgemm: residual add needs fp32 output");
  T2H_CHECK_ARG(p->bias_mode == T2H_BIAS_NONE || p->bias != nullptr, "tapgemm: bias_mode without bias");
  T2H_CHECK_ARG(!p->b_batched_h || p->H == 1 || p->tile_rows, "tapgemm: b_batched_h needs row tiles");

  TapGemmDev P;
  memset(&P, 0, sizeof(P));
  P.n_img = p->n_img; P.H = p->H; P.W = p->W;
  P.n_out = p->n_out; P.C = p->C; P.kchunks = (p->C + kBK - 1) / kBK; P.nterms = p->nterms;
  P.a_term_imgs = p->a_term_imgs; P.a_bcast = p->a_bcast;
  P.a_mn = p->a_mn ? 1 : 0; P.b_mn = p->b_mn ? 1 : 0;
  P.b_term_g = p->b_term_g; P.b_batched = p->b_batched; P.b_batched_h = p->b_batched_h;
  P.d = p->d; P.d_mode = p->d_mode; P.d_terms = p->d_terms; P.d_plane = p->d_plane;
  P.d_sn = p->d_sn; P.d_sh = p->d_sh; P.d_sw = p->d_sw; P.d_sc = p->d_sc;
  P.bias = p->bias; P.bias_sn = p->bias_mode == T2H_BIAS_COL ? p->bias_sn : 0; P.bias_mode = p->bias_mode; P.act = p->act; P.alpha = p->alpha;
  P.residual = p->residual; P.gn_stats = p->gn_stats; P.gn_cpg = p->gn_cpg;
  P.nb_sums = p->nb_sums; P.nb_stats = p->nb_stats; P.nb_gamma = p->nb_gamma; P.nb_beta = p->nb_beta;
  P.nb_eps = p->nb_eps; P.nb_act = p->nb_act; P.nb_groups = p->nb_groups;
  P.n_major = p->nb_sums ? 1 : 0;
  P.gn_groups = p->gn_cpg > 0 ? p->n_out / p->gn_cpg : 0;
  P.d_term_imgs = 0;

  // ---- tile shape
  // (tests/test_gpu_tapgemm_paths.py::route restates the selection below, tile shape to epilogue mode, and labels its
  // cases with it: a routing change updates it in the same change)
  // one 128-row block = TH x TW output positions of one image
  int TW, TH;
  if (p->H == 1 || p->tile_rows) {
    TW = 128; TH = 1;
  } else {
    TW = 16;
    while (TW > p->W && TW > 1) TW >>= 1;  // W < 16: narrower, taller boxes
    TH = 128 / TW;
  }
  // Swapped-operand kernel (gemm_tc_swap.cuh): spatial convs with Cout % 128 == 0 and a plain fp32
  // NHWC destination.  The weight tile is the M operand, the 128-pixel tile the N operand.
  const bool rows_mode = (p->H == 1 || p->tile_rows);
  bool swap = !rows_mode && TW <= 16 && p->n_out % 128 == 0 && p->d_mode == T2H_OUT_F32 && p->d_sc == 1 &&
              p->bias_mode != T2H_BIAS_ROW && !p->a_bcast && !p->b_batched && !p->b_batched_h &&
              p->d_sw % 4 == 0 && p->d_sh % 4 == 0 && p->d_sh > 0 && (p->n_img == 1 || (p->d_sn % 4 == 0 && p->d_sn > 0)) &&
              reinterpret_cast<uintptr_t>(p->d) % 16 == 0 &&
              (!p->residual || reinterpret_cast<uintptr_t>(p->residual) % 16 == 0) &&
              (!p->gn_stats || (p->gn_cpg >= 1 && (p->gn_cpg & (p->gn_cpg - 1)) == 0 && p->n_out % p->gn_cpg == 0));
  // ... and with a direct (strided) epilogue for small-Cout convs writing NCHW (conv_out): the weight
  // tile is zero-padded to 128 rows by TMA.
  const bool swap_direct = !swap && !rows_mode && TW <= 16 && p->n_out <= 128 && p->d_mode == T2H_OUT_F32 &&
                           p->d_sc != 1 && p->bias_mode != T2H_BIAS_ROW && !p->a_bcast && !p->b_batched &&
                           !p->b_batched_h && !p->residual && !p->gn_stats && p->act == T2H_ACT_NONE;
  if (swap_direct) swap = true;
  if (p->a_mn || p->b_mn) {
    T2H_CHECK_ARG(rows_mode && p->ntaps == 1 && p->tap_dx[0] == 0 && p->tap_dy[0] == 0,
                  "tapgemm: a_mn / b_mn operands need a row GEMM (H == 1 or tile_rows) with one tap");
    swap = false;
  }
  int BN = 16;
  while (BN < p->n_out && BN < 128) BN <<= 1;
  if (p->b_mn && BN < 64) BN = 64;  // an MN-major B tile is made of whole 64-column boxes
  if (swap) BN = 128;
  P.TW = TW; P.TH = TH;
  // ---- tap groups: taps with the same (dx, img_off) share one activation slab when a vertical
  // shift of the slab view stays 1024-byte aligned (TW*128 bytes per image row, TW >= 8)
  {
    const bool can_share = (TW >= 8) && (TW <= 16);
    P.ngroups = 0;
    int gmin[T2H_MAX_TAPS], gmax[T2H_MAX_TAPS];
    int gt_dy[T2H_MAX_TAPS][3];
    for (int i = 0; i < p->ntaps; ++i) {
      int g = -1;
      if (can_share)
        for (int k = 0; k < P.ngroups; ++k)
          if (P.g_dx[k] == p->tap_dx[i] && P.g_ioff[k] == p->tap_img_off[i] && P.g_ntaps[k] < 3) {
            const int lo = p->tap_dy[i] < gmin[k] ? p->tap_dy[i] : gmin[k];
            const int hi = p->tap_dy[i] > gmax[k] ? p->tap_dy[i] : gmax[k];
            if (hi - lo <= 2) { g = k; gmin[k] = lo; gmax[k] = hi; break; }
          }
      if (g < 0) {
        g = P.ngroups++;
        P.g_dx[g] = p->tap_dx[i]; P.g_ioff[g] = p->tap_img_off[i]; P.g_ntaps[g] = 0;
        gmin[g] = gmax[g] = p->tap_dy[i];
      }
      gt_dy[g][P.g_ntaps[g]] = p->tap_dy[i];
      P.g_btap[g][P.g_ntaps[g]] = p->use_tap_w ? p->tap_w[i] : i;
      P.g_ntaps[g]++;
    }
    int extra = 0;
    for (int g = 0; g < P.ngroups; ++g) {
      P.g_dy0[g] = gmin[g];
      for (int k = 0; k < P.g_ntaps[g]; ++k) P.g_dyrel[g][k] = gt_dy[g][k] - gmin[g];
      if (gmax[g] - gmin[g] > extra) extra = gmax[g] - gmin[g];
    }
    for (int g = P.ngroups; g < T2H_MAX_TAPS; ++g) {
      P.g_dx[g] = P.g_ioff[g] = P.g_dy0[g] = P.g_ntaps[g] = 0;
    }
    P.slab_rows = TH + extra;
  }
  P.tiles_w = ceil_div(p->W, TW);
  P.tiles_h = ceil_div(p->H, TH);
  P.n_tiles_n = ceil_div(p->n_out, BN);
  long long total = (long long)p->n_img * P.tiles_w * P.tiles_h * P.n_tiles_n;
  T2H_CHECK_ARG(total < (1LL << 31), "tapgemm: too many tiles");
  P.total_tiles = (int)total;

  // ---- epilogue mode
  const int esz = (p->d_mode == T2H_OUT_F32) ? 4 : 2;
  const int align_el = 16 / esz;  // elements per 16 bytes
  bool tma_ok = p->d_sc == 1 && p->n_out % (p->d_mode == T2H_OUT_F32 ? 4 : 8) == 0 &&
                p->d_sw % align_el == 0 && (reinterpret_cast<uintptr_t>(p->d) % 16 == 0) &&
                BN >= (p->d_mode == T2H_OUT_F32 ? 32 : 64);
  // strides of the dims the output domain really uses must be TMA-encodable
  if (p->H > 1) tma_ok = tma_ok && p->d_sh % align_el == 0 && p->d_sh > 0;
  if (p->n_img > 1) tma_ok = tma_ok && p->d_sn % align_el == 0 && p->d_sn > 0;
  if (p->d_mode == T2H_OUT_PLANES && p->d_terms == 2) {
    // the lo plane is addressed as extra images: its distance must be a whole number of d_sn
    const long long sn = (p->n_img > 1) ? p->d_sn : p->d_plane;
    tma_ok = tma_ok && sn > 0 && p->d_plane % sn == 0 && p->d_plane % align_el == 0;
  }
  if (p->residual) tma_ok = tma_ok && (reinterpret_cast<uintptr_t>(p->residual) % 16 == 0);
  if (p->bias_mode == T2H_BIAS_COL)
    tma_ok = tma_ok && (reinterpret_cast<uintptr_t>(p->bias) % 16 == 0) && p->bias_sn % 4 == 0;
  P.epi_mode = !tma_ok ? EPI_DIRECT : (p->d_mode == T2H_OUT_F32 ? EPI_TMA_F32 : EPI_TMA_PLANES);
  if (swap) P.epi_mode = swap_direct ? EPI_DIRECT : EPI_TMA_F32;
  if (p->nb_sums) {
    T2H_CHECK_ARG(swap && !swap_direct && p->residual && p->nb_stats && p->nb_gamma && p->nb_beta && !p->gn_stats &&
                      p->act == T2H_ACT_NONE && p->nb_act >= 0 && p->nb_act <= 2 && p->nb_groups > 0 &&
                      p->n_out % p->nb_groups == 0 && p->k_split <= 1 && !p->accumulate && !p->k_partials,
                  "tapgemm: nb_sums needs a swapped-kernel conv (n_out %% 128 == 0, fp32 NHWC output), x in `residual`, "
                  "statistics / gamma / beta, and no other epilogue work");
  }
  // ---- split-K: k-slices of one tile go to different CTAs and are reduce-added into a zeroed output
  P.ksplit = 1;
  P.kper = P.kchunks;
  if (p->k_partials > 1) {
    T2H_CHECK_ARG(!swap && P.epi_mode == EPI_TMA_F32 && !p->residual && p->bias_mode == T2H_BIAS_NONE &&
                      p->act == T2H_ACT_NONE && !p->gn_stats && p->n_img == 1 && p->k_split <= 1 &&
                      p->d_slab > 0 && p->d_slab % 4 == 0,
                  "tapgemm: k_partials needs a plain single-image fp32 GEMM output and an aligned slab stride");
    int ks = p->k_partials < P.kchunks ? p->k_partials : P.kchunks;
    P.kper = ceil_div(P.kchunks, ks);
    P.ksplit = ceil_div(P.kchunks, P.kper);
    P.partials = 1;
  } else if (p->k_split > 1 && !swap && P.epi_mode == EPI_TMA_F32 && !p->residual && p->bias_mode != T2H_BIAS_ROW &&
      p->act == T2H_ACT_NONE && !p->gn_stats) {
    int ks = p->k_split < P.kchunks ? p->k_split : P.kchunks;
    P.kper = ceil_div(P.kchunks, ks);
    P.ksplit = ceil_div(P.kchunks, P.kper);
  } else {
    T2H_CHECK_ARG(p->k_split <= 1, "tapgemm: k_split needs an aligned fp32 output and no row bias/act/residual");
  }
  T2H_CHECK_ARG((long long)P.total_tiles * P.ksplit < (1LL << 31), "tapgemm: too many work items");
  P.total_work = P.total_tiles * P.ksplit;
  if (p->accumulate) {
    T2H_CHECK_ARG(!swap && P.epi_mode == EPI_TMA_F32 && !p->residual && p->bias_mode != T2H_BIAS_ROW &&
                      p->act == T2H_ACT_NONE && !p->gn_stats,
                  "tapgemm: accumulate needs an aligned fp32 output and no row bias/act/residual");
    P.accum = 1;
  }
  if (p->gn_stats && !swap) {
    T2H_CHECK_ARG(P.epi_mode == EPI_TMA_F32, "tapgemm: gn_stats needs an aligned fp32 NHWC output");
    T2H_CHECK_ARG(p->gn_cpg >= 2 && (p->gn_cpg & (p->gn_cpg - 1)) == 0 && p->n_out % p->gn_cpg == 0,
                  "tapgemm: gn_cpg=%d must be a power of two >= 2 dividing n_out", p->gn_cpg);
    T2H_CHECK_ARG(BN % p->gn_cpg == 0 || p->n_out <= BN, "tapgemm: group straddles column tiles");
  }

  // ---- tensor maps
  CUtensorMap tmA, tmB, tmD, tmR;
  {
    uint64_t dims[4] = {(uint64_t)p->C, (uint64_t)p->a_W, (uint64_t)p->a_H, (uint64_t)p->a_imgs};
    uint64_t str[4] = {1, (uint64_t)p->a_sw, (uint64_t)p->a_sh, (uint64_t)p->a_sn};
    uint32_t box[4] = {(uint32_t)kBK, (uint32_t)TW, (uint32_t)P.slab_rows, 1};
    if (p->a_mn) {  // (row, k, h, img): rows contiguous, a_sw = distance between consecutive k
      dims[0] = (uint64_t)p->a_W; dims[1] = (uint64_t)p->C;
      box[0] = 64; box[1] = (uint32_t)kBK; box[2] = 1;
    }
    int rc = make_tmap(&tmA, p->a, 2, 4, dims, str, box, "tapgemm A");
    if (rc) return rc;
  }
  {
    const int g2 = p->b_groups2 > 0 ? p->b_groups2 : 1;
    uint64_t dims[4] = {(uint64_t)p->C, (uint64_t)p->n_out, (uint64_t)p->b_groups, (uint64_t)g2};
    uint64_t str[4] = {1, (uint64_t)p->b_sn, (uint64_t)p->b_sg,
                       (uint64_t)(g2 > 1 ? p->b_sg2 : p->b_sg)};
    uint32_t box[4] = {(uint32_t)kBK, (uint32_t)BN, 1, 1};
    if (p->b_mn) {  // (n, k, g, g2): output columns contiguous, b_sn = distance between consecutive k
      dims[0] = (uint64_t)p->n_out; dims[1] = (uint64_t)p->C;
      box[0] = 64; box[1] = (uint32_t)kBK;
    }
    int rc = make_tmap(&tmB, p->b, 2, 4, dims, str, box, "tapgemm B");
    if (rc) return rc;
  }
  tmD = tmA;
  tmR = tmA;
  if (P.epi_mode != EPI_DIRECT) {
    // dims the output domain does not use get a harmless, 16-byte-aligned stride
    const uint64_t sw = (uint64_t)p->d_sw;
    const uint64_t sh = (p->H > 1) ? (uint64_t)p->d_sh : sw * (uint64_t)p->W;
    uint64_t sn = (p->n_img > 1) ? (uint64_t)p->d_sn : sh * (uint64_t)p->H;
    uint64_t imgs = (uint64_t)p->n_img;
    if (P.partials) {  // one slab per k-slice, addressed through the image dim
      sn = (uint64_t)p->d_slab;
      imgs = (uint64_t)P.ksplit;
    }
    if (P.epi_mode == EPI_TMA_PLANES && p->d_terms == 2) {
      if (p->n_img == 1) sn = (uint64_t)p->d_plane;
      P.d_term_imgs = (int)(p->d_plane / (long long)sn);
      imgs = (uint64_t)P.d_term_imgs + (uint64_t)p->n_img;
    }
    uint64_t dims[4] = {(uint64_t)p->n_out, (uint64_t)p->W, (uint64_t)p->H, imgs};
    uint64_t str[4] = {1, sw, sh, sn};
    uint32_t box[4] = {(uint32_t)(esz == 4 ? 32 : 64), (uint32_t)TW, (uint32_t)TH, 1};
    CUtensorMapSwizzle sw_mode = CU_TENSOR_MAP_SWIZZLE_128B;
    if (swap) {  // one box of a swapped-kernel warp: 16 channels (64 bytes) x 32 pixels
      box[0] = 16;
      box[2] = (uint32_t)(32 / TW);
      sw_mode = CU_TENSOR_MAP_SWIZZLE_64B;
    }
    int rc = make_tmap(&tmD, p->d, esz, 4, dims, str, box, "tapgemm D", sw_mode);
    if (rc) return rc;
    if (p->residual) {
      uint64_t rdims[4] = {(uint64_t)p->n_out, (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->n_img};
      rc = make_tmap(&tmR, p->residual, 4, 4, rdims, str, box, "tapgemm residual", sw_mode);
      if (rc) return rc;
    }
  }

  cudaStream_t s = as_stream(stream);
  if (swap) return launch_swap(tmA, tmB, tmD, tmR, P, s);
  switch (BN) {
    case 16: return launch<16>(tmA, tmB, tmD, tmR, P, s);
    case 32: return launch<32>(tmA, tmB, tmD, tmR, P, s);
    case 64: return launch<64>(tmA, tmB, tmD, tmR, P, s);
    default: return launch<128>(tmA, tmB, tmD, tmR, P, s);
  }
}

// ---------------------------------------------------------------------------------------------------------
// t2h_conv_wgrad: dW[tap][co][ci] += alpha * sum_{n,h,w} dY[n,h,w,co] * X[n + ioff(tap), h + dy(tap), w + dx(tap), ci]
// on the same wgmma kernel: both operands are NHWC fp16 planes consumed MN-major (the contraction index -- the
// pixel -- is the outer dimension of both), the K loop walks 64-pixel patches (one TMA box {64 ch, PW, PH, 1}
// per operand and patch; the tap is a coordinate shift of the X box, zero-filled outside the image = the conv's
// padding), one output tile per (tap, 128 couts, BN cins), patches split over the SMs and TMA-reduce-added.
// ---------------------------------------------------------------------------------------------------------
extern "C" int t2h_conv_wgrad(const t2h_conv_wgrad_params* p, t2h_stream_t stream) {
  T2H_CHECK_ARG(p && p->dy && p->x && p->dw, "conv_wgrad: null operand");
  T2H_CHECK_ARG(p->n_img > 0 && p->H > 0 && p->W > 0 && p->cout > 0 && p->cin > 0, "conv_wgrad: empty problem");
  T2H_CHECK_ARG(p->ntaps >= 1 && p->ntaps <= T2H_MAX_TAPS, "conv_wgrad: ntaps=%d", p->ntaps);
  T2H_CHECK_ARG(p->nterms == 1 || (p->nterms == 3 && p->dy_terms == 2 && p->x_terms == 2),
                "conv_wgrad: nterms=%d needs hi/lo planes on both operands", p->nterms);
  T2H_CHECK_ARG(p->cin % 4 == 0 && p->dw_ld % 4 == 0 && p->dw_tap_stride % 4 == 0 &&
                    reinterpret_cast<uintptr_t>(p->dw) % 16 == 0,
                "conv_wgrad: dW needs cin %% 4 == 0 and 16-byte aligned rows (cin=%d ld=%lld)", p->cin,
                (long long)p->dw_ld);
  TapGemmDev P;
  memset(&P, 0, sizeof(P));
  int PW = 16;
  while (PW > 1 && PW / 2 >= p->W) PW >>= 1;  // narrow images: taller patches
  const int PH = 64 / PW;
  P.wg = 1; P.accum = 1;
  P.wg_PW = PW; P.wg_PH = PH;
  P.wg_pw = ceil_div(p->W, PW);
  P.wg_ppi = P.wg_pw * ceil_div(p->H, PH);
  for (int i = 0; i < p->ntaps; ++i) {
    P.wg_dy[i] = p->tap_dy[i]; P.wg_dx[i] = p->tap_dx[i]; P.wg_ioff[i] = p->tap_img_off[i];
  }
  const long long chunks = (long long)p->n_img * P.wg_ppi;
  T2H_CHECK_ARG(chunks < (1LL << 24), "conv_wgrad: too many pixel patches");
  P.n_img = p->ntaps; P.H = 1; P.W = p->cout;
  P.n_out = p->cin; P.kchunks = (int)chunks; P.C = P.kchunks * kBK; P.nterms = p->nterms;
  P.a_term_imgs = p->dy_term_imgs; P.b_term_g = p->x_term_imgs;
  P.a_mn = 1; P.b_mn = 1;
  P.d = p->dw; P.d_mode = T2H_OUT_F32; P.alpha = p->alpha;
  P.bias_mode = T2H_BIAS_NONE; P.act = T2H_ACT_NONE;
  P.TW = 128; P.TH = 1;
  P.ngroups = 1; P.g_ntaps[0] = 1; P.slab_rows = 1;
  const int BN = p->cin <= 64 ? 64 : 128;
  P.tiles_w = ceil_div(p->cout, 128); P.tiles_h = 1;
  P.n_tiles_n = ceil_div(p->cin, BN);
  P.total_tiles = P.n_img * P.tiles_w * P.n_tiles_n;
  P.epi_mode = EPI_TMA_F32;
  int ks = p->k_split > 0 ? p->k_split : num_sms() / P.total_tiles;
  if (ks < 1) ks = 1;
  if (ks > P.kchunks) ks = P.kchunks;
  P.kper = ceil_div(P.kchunks, ks);
  P.ksplit = ceil_div(P.kchunks, P.kper);
  T2H_CHECK_ARG((long long)P.total_tiles * P.ksplit < (1LL << 31), "conv_wgrad: too many work items");
  P.total_work = P.total_tiles * P.ksplit;

  CUtensorMap tmA, tmB, tmD, tmR;
  {
    uint64_t dims[4] = {(uint64_t)p->cout, (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->dy_imgs};
    uint64_t str[4] = {1, (uint64_t)p->dy_sw, (uint64_t)p->dy_sh, (uint64_t)p->dy_sn};
    uint32_t box[4] = {64, (uint32_t)PW, (uint32_t)PH, 1};
    int rc = make_tmap(&tmA, p->dy, 2, 4, dims, str, box, "conv_wgrad dY");
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)p->cin, (uint64_t)p->x_W, (uint64_t)p->x_H, (uint64_t)p->x_imgs};
    uint64_t str[4] = {1, (uint64_t)p->x_sw, (uint64_t)p->x_sh, (uint64_t)p->x_sn};
    uint32_t box[4] = {64, (uint32_t)PW, (uint32_t)PH, 1};
    int rc = make_tmap(&tmB, p->x, 2, 4, dims, str, box, "conv_wgrad X");
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)p->cin, (uint64_t)p->cout, 1, (uint64_t)p->ntaps};
    uint64_t str[4] = {1, (uint64_t)p->dw_ld, (uint64_t)p->dw_ld * (uint64_t)p->cout, (uint64_t)p->dw_tap_stride};
    uint32_t box[4] = {32, 128, 1, 1};
    int rc = make_tmap(&tmD, p->dw, 4, 4, dims, str, box, "conv_wgrad dW");
    if (rc) return rc;
  }
  tmR = tmA;
  cudaStream_t s = as_stream(stream);
  return BN == 64 ? launch<64>(tmA, tmB, tmD, tmR, P, s) : launch<128>(tmA, tmB, tmD, tmR, P, s);
}

#include "attn_fused.cuh"
