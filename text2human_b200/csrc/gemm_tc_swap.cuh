// Transposed ("swapped-operand") variant of the tap-GEMM for spatial convolutions whose output
// channel count is a multiple of 128.
//
// The weight tile is the M=128 operand (each consumer warpgroup issues wgmma M=64 for its 64 output
// channels) and the activation slab view (128 consecutive slab rows = 128 output pixels) is the N=128
// operand, so D^T[cout, pixel] accumulates with one output channel per accumulator row.  That is the
// layout the per-channel epilogue wants: bias, GroupNorm sums and norm-backward sums are per lane.
//
// Mainloop: one MMA group (four K=16 steps of one (weight tile, slab view) product) stays in flight while the next
// is issued; the ring slots a group read last are released once the following group has been issued and the
// group itself has completed (wgmma.wait_group 1).
//
// Epilogue, straight from the accumulator registers: thread t of warpgroup wg holds output channels
// 64 wg + 16 (t / 32) + (t % 32) / 4 and that + 8, at pixels 8 j + 2 (t % 4) + {0, 1} of every 8-pixel block j, so
// each consumer warp owns 16 channels x 128 pixels and finishes them alone (no block or warpgroup barrier):
// +bias (two registers) -> activation -> +residual (its own TMA-loaded boxes) -> GroupNorm / norm-backward partial
// sums (per thread, reduced over the four lanes of a channel and the channels of a group) -> st.shared into its own
// 64-byte-swizzled [32 pixels][16 channels] boxes -> TMA store.
#pragma once

namespace t2h {

constexpr int kSwapThreads = 384;  // 4 producer warps + 8 consumer warps (two warpgroups of 64 output channels)
constexpr int kSwapBox = 32 * 16 * 4;         // one TMA box of the epilogue: 32 pixels x 16 fp32 channels
constexpr int kSwapWarpBuf = 4 * kSwapBox;    // a consumer warp's 128 pixels: residual in, output out, in place
static_assert(8 * kSwapWarpBuf == kEpiBytes, "epilogue boxes");
constexpr int kSwapRingBytes = kDynSmem - 1024 - kEpiBytes;  // A ring + B ring
// Register split (setmaxnreg): the producer warpgroup only issues TMA and waits on barriers; the consumers hold a
// 64-register accumulator plus the epilogue's values.  The split redistributes what the CTA was launched with, 384
// threads x 168 registers (the __launch_bounds__ ceiling): 128 x 40 + 256 x 232.
constexpr int kSwapProducerRegs = 40;
constexpr int kSwapConsumerRegs = 232;
static_assert(128 * kSwapProducerRegs + 256 * kSwapConsumerRegs <= kSwapThreads * 168,
              "register split exceeds the CTA's registers");

// byte offset of fp32 channel c (0..15) of pixel i (0..31) in a [32][16] box TMA wrote with the 64-byte swizzle
// (address bits [4,6) ^= bits [7,9))
__device__ __forceinline__ int swz64(int i, int c) {
  const int o = i * 64 + c * 4;
  return o ^ ((o >> 3) & 0x30);
}

// norm-backward: add a thread's per-channel sums (channels c and c + 8) to nb_sums, after reducing them over the
// four lanes that hold the same channel
__device__ __forceinline__ void nb_flush(const TapGemmDev& P, int img, int c, int lane, float s1a, float s1b, float s2a,
                                         float s2b) {
#pragma unroll
  for (int off = 1; off < 4; off <<= 1) {
    s1a += __shfl_xor_sync(0xffffffffu, s1a, off);
    s1b += __shfl_xor_sync(0xffffffffu, s1b, off);
    s2a += __shfl_xor_sync(0xffffffffu, s2a, off);
    s2b += __shfl_xor_sync(0xffffffffu, s2b, off);
  }
  if ((lane & 3) == 0) {
    if (c < P.n_out) {
      double* dst = P.nb_sums + ((long long)img * P.n_out + c) * 2;
      atomicAdd(dst, (double)s1a);
      atomicAdd(dst + 1, (double)s2a);
    }
    if (c + 8 < P.n_out) {
      double* dst = P.nb_sums + ((long long)img * P.n_out + c + 8) * 2;
      atomicAdd(dst, (double)s1b);
      atomicAdd(dst + 1, (double)s2b);
    }
  }
}

// Ring invariant: no group waits on a slot whose release is deferred behind it.  When a group's operands are waited
// for, every slot whose last reader is two or more groups back has been released.  Each group reads one B tile and
// the B index advances by at most one per group, so the tile a group needs reuses a slot released two groups back
// whenever b_slots >= 2.  A slabs (3-product order hi.lo, hi.hi, lo.hi per tap): the next chunk's hi slab reuses the
// slot of the current chunk's hi slab (last read by the hi.hi group before the chunk's final group) when
// a_slots >= 2.  1-product: one slab per chunk, a_slots >= 2.
__global__ void __launch_bounds__(kSwapThreads, 1)
tapgemm_swap_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                    const __grid_constant__ TapGemmDev P) {
  using C = Cfg<128>;
  pdl_launch_dependents();  // the next kernel may start its prologue once every CTA of this one is running
  const int NA = P.a_slots, NB = P.b_slots;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem =
      reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = smem + NA * C::kASlot;
  uint8_t* epi_buf = b_ring + NB * C::kBSlot;  // 8 consumer warps x kSwapWarpBuf

  __shared__ __align__(8) uint64_t a_full[kMaxSlots];
  __shared__ __align__(8) uint64_t a_empty[kMaxSlots];
  __shared__ __align__(8) uint64_t b_full[kMaxSlots];
  __shared__ __align__(8) uint64_t b_empty[kMaxSlots];
  __shared__ __align__(8) uint64_t res_bar[8];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (P.epi_mode != EPI_DIRECT) tma_prefetch_desc(&tmD);
    if (P.residual) tma_prefetch_desc(&tmR);
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
    for (int s = 0; s < 8; ++s) mbar_init(&res_bar[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  // everything above touched only shared memory and kernel parameters; from here on the previous
  // kernel's results are read (and buffers it may still be reading are overwritten)
  pdl_wait();
  // tile schedule: round-robin over the CTAs, or -- when the epilogue accumulates per-image sums (nb_sums) -- one
  // contiguous range per CTA, so that a CTA stays inside one image and flushes its sums once or twice per launch
  // instead of once per tile (round-robin put ~1000 double atomics per launch on every (image, channel) address)
  const bool contig = P.nb_sums != nullptr;
  const int tile_first = contig ? (int)((long long)blockIdx.x * P.total_tiles / gridDim.x) : (int)blockIdx.x;
  const int tile_end = contig ? (int)((long long)(blockIdx.x + 1) * P.total_tiles / gridDim.x) : P.total_tiles;
  const int tile_step = contig ? 1 : (int)gridDim.x;

  const int a_planes = (P.nterms == 3) ? 2 : 1;
  const int slab_bytes = P.slab_rows * P.TW * 128;

  if (warp < 4) {
    // (each role's setmaxnreg sits inside its branch: ptxas ignores a reallocation that code needing more registers
    // can follow)
    setmaxnreg_dec<kSwapProducerRegs>();
    if (warp == 0) {
      // ---------------------------------------------- activation slab producer
      if (lane == 0) {
        int sa = 0, pa = 0;
        for (int tile = tile_first; tile < tile_end; tile += tile_step) {
          const TileCoord t = decode_tile(P, tile, 128);
          for (int g = 0; g < P.ngroups; ++g)
            for (int ch = 0; ch < P.kchunks; ++ch)
              for (int pl = 0; pl < a_planes; ++pl) {
                mbar_wait(&a_empty[sa], pa ^ 1);
                mbar_expect_tx(&a_full[sa], slab_bytes);
                tma_load_4d(&tmA, &a_full[sa], a_ring + sa * C::kASlot, ch * kBK, t.w0 + P.g_dx[g],
                            t.h0 + P.g_dy0[g], t.img + P.g_ioff[g] + pl * P.a_term_imgs);
                if (++sa == NA) {
                  sa = 0;
                  pa ^= 1;
                }
              }
        }
      }
    } else if (warp == 3) {
      // ---------------------------------------------- weight tile producer (128 couts x 64 k)
      if (lane == 0) {
        int sb = 0, pb = 0;
        for (int tile = tile_first; tile < tile_end; tile += tile_step) {
          const TileCoord t = decode_tile(P, tile, 128);
          for (int g = 0; g < P.ngroups; ++g)
            for (int ch = 0; ch < P.kchunks; ++ch)
              for (int tp = 0; tp < P.g_ntaps[g]; ++tp)
                for (int pl = a_planes - 1; pl >= 0; --pl) {  // lo first, then hi
                  mbar_wait(&b_empty[sb], pb ^ 1);
                  mbar_expect_tx(&b_full[sb], C::kBSlot);
                  tma_load_4d(&tmB, &b_full[sb], b_ring + sb * C::kBSlot, ch * kBK, t.n0,
                              P.g_btap[g][tp] + pl * P.b_term_g, 0);
                  if (++sb == NB) {
                    sb = 0;
                    pb ^= 1;
                  }
                }
        }
      }
    }
  } else {
    // ---------------------------------------------- consumers: D^T[cout, pixel] += W * slab^T, then the epilogue
    setmaxnreg_inc<kSwapConsumerRegs>();
    const int wg = (warp - 4) >> 2;  // output channels 64 wg .. 64 wg + 63 of the tile
    const uint32_t row16 = (uint32_t)(P.TW * 128) >> 4;  // one slab image row, in 16-byte units
    const uint64_t x_desc0 = gmma_desc(smem_u32(a_ring));
    const uint64_t w_desc0 = gmma_desc(smem_u32(b_ring) + 8192u * wg);
    constexpr uint32_t A16 = C::kASlot >> 4, B16 = C::kBSlot >> 4;
    const int ngroups = P.ngroups, kchunks = P.kchunks;
    int sa = 0, pa = 0, sb = 0, pb = 0;
    const int e = warp - 4;  // 0..7
    uint8_t* my_buf = epi_buf + e * kSwapWarpBuf;
    const uint32_t buf_s = smem_u32(my_buf);
    const bool has_res = P.residual != nullptr;
    const int tw_shift = 31 - __clz(P.TW);      // TW is a power of two <= 16
    const int rows_per_box = 32 >> tw_shift;    // image rows covered by 32 pixels
    const int m2 = 2 * (lane & 3);              // pixel offset of this thread inside each 8-pixel block
    uint32_t res_par = 0;
    const int cpg = P.gn_cpg;
    const int red = 4 * (cpg < 8 ? cpg : 8);  // lanes holding one GroupNorm group's (channel, pixel) partial sums
    // norm-backward sums: the "residual" tile is x and is not added
    const bool nb = P.nb_sums != nullptr;
    // per thread: channel c (index 0) and c + 8 (index 1); the sums run on across consecutive tiles of the same
    // (image, channel block) and are flushed when that changes
    float nb_mean[2] = {0.f, 0.f}, nb_rstd[2] = {0.f, 0.f}, nb_ga[2] = {0.f, 0.f}, nb_be[2] = {0.f, 0.f};
    float nb_s1[2] = {0.f, 0.f}, nb_s2[2] = {0.f, 0.f};
    int nb_img = -1, nb_c = -1;

    for (int tile = tile_first; tile < tile_end; tile += tile_step) {
      const TileCoord t = decode_tile(P, tile, 128);
      const int c0 = t.n0 + 16 * e;       // this warp's 16 output channels
      const int ca = c0 + (lane >> 2);    // this thread's channels: ca and ca + 8
      if (has_res && lane == 0) {
        // the tile's residual (or x) boxes load while its MMAs run, into the boxes the previous tile's output
        // stores read from
        tma_store_wait_read<0>();
        mbar_expect_tx(&res_bar[e], kSwapWarpBuf);
        for (int k = 0; k < 4; ++k)
          tma_load_4d(&tmR, &res_bar[e], my_buf + k * kSwapBox, c0, t.w0, t.h0 + k * rows_per_box, t.img);
        if (nb && tile + tile_step < tile_end) {
          // the NEXT tile's x boxes go to L2 now, so that its loads above are L2 hits
          const TileCoord tn = decode_tile(P, tile + tile_step, 128);
          for (int k = 0; k < 4; ++k)
            tma_prefetch_4d(&tmR, tn.n0 + 16 * e, tn.w0, tn.h0 + k * rows_per_box, tn.img);
        }
      }
      float acc[64];
      {
        uint32_t accf = 0;
        int rel_b = -1, rel_a = -1;  // the slots the group in flight is the last reader of (-1: none)
        // every consumer thread arrives (a lane-0 arrival between wgmmas puts them on a divergent path, and ptxas
        // then serialises every MMA); the arrivals are for the previous group, which wait_group 1 has completed
        auto group = [&](uint64_t w, uint64_t x, int last_b, int last_a) {
          wgmma_fence();
          wgmma_chunk<0, 0>(acc, w, x, accf);
          wgmma_commit();
          wgmma_wait<1>();
          if (rel_b >= 0) mbar_arrive(&b_empty[rel_b]);
          if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
          rel_b = last_b;
          rel_a = last_a;
        };
        for (int g = 0; g < ngroups; ++g) {
          const int nt = P.g_ntaps[g];
          const uint32_t dy0 = P.g_dyrel[g][0] * row16, dy1 = P.g_dyrel[g][1] * row16,
                         dy2 = P.g_dyrel[g][2] * row16;
          for (int ch = 0; ch < kchunks; ++ch) {
            const int sa_hi = sa, pa_hi = pa;
            if (++sa == NA) { sa = 0; pa ^= 1; }
            const int sa_lo = sa, pa_lo = pa;
            if (a_planes == 2) {
              if (++sa == NA) { sa = 0; pa ^= 1; }
            }
            mbar_wait(&a_full[sa_hi], pa_hi);
            const uint64_t xhi = x_desc0 + sa_hi * A16;
            const uint64_t xlo = x_desc0 + sa_lo * A16;
            for (int tp = 0; tp < nt; ++tp) {
              const uint32_t dy = tp == 0 ? dy0 : (tp == 1 ? dy1 : dy2);
              const bool last = tp == nt - 1;
              if (a_planes == 1) {
                mbar_wait(&b_full[sb], pb);
                group(w_desc0 + sb * B16, xhi + dy, sb, last ? sa_hi : -1);
                if (++sb == NB) { sb = 0; pb ^= 1; }
              } else {
                mbar_wait(&b_full[sb], pb);  // w_lo
                group(w_desc0 + sb * B16, xhi + dy, sb, -1);  // x_hi*w_lo
                if (++sb == NB) { sb = 0; pb ^= 1; }
                mbar_wait(&b_full[sb], pb);  // w_hi
                const uint64_t whi = w_desc0 + sb * B16;
                group(whi, xhi + dy, -1, last ? sa_hi : -1);  // x_hi*w_hi
                if (tp == 0) mbar_wait(&a_full[sa_lo], pa_lo);
                group(whi, xlo + dy, sb, last ? sa_lo : -1);  // x_lo*w_hi
                if (++sb == NB) { sb = 0; pb ^= 1; }
              }
            }
          }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (rel_b >= 0) mbar_arrive(&b_empty[rel_b]);
        if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
      }
      // accumulator element i: channel ca + 8 ((i >> 1) & 1), pixel 8 (i >> 2) + m2 + (i & 1); in-box pixel and
      // channel of the [32][16] box i >> 4
      auto box_off = [&](int i) { return (i >> 4) * kSwapBox + swz64(8 * ((i >> 2) & 3) + m2 + (i & 1), (lane >> 2) + 8 * ((i >> 1) & 1)); };
      auto pix_ok = [&](int i) {
        const int p = 8 * (i >> 2) + m2 + (i & 1);
        return (t.h0 + (p >> tw_shift) < P.H) && (t.w0 + (p & (P.TW - 1)) < P.W);
      };
      // interior tiles need no per-pixel validity test for the GroupNorm / norm-backward sums
      const bool interior = (t.h0 + P.TH <= P.H) && (t.w0 + P.TW <= P.W);
      {
        float bias2[2] = {0.f, 0.f};
        if (P.bias_mode == T2H_BIAS_COL) {
          if (ca < P.n_out) bias2[0] = __ldg(P.bias + t.img * P.bias_sn + ca);
          if (ca + 8 < P.n_out) bias2[1] = __ldg(P.bias + t.img * P.bias_sn + ca + 8);
        }
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = acc[i] * P.alpha + bias2[(i >> 1) & 1];
      }
      if (P.act == T2H_ACT_GELU) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = gelu_erf(acc[i]);
      } else if (P.act == T2H_ACT_RELU) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = fmaxf(acc[i], 0.f);
      } else if (P.act == T2H_ACT_LRELU) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = acc[i] > 0.f ? acc[i] : 0.2f * acc[i];
      }
      if (has_res) {
        mbar_wait(&res_bar[e], res_par);
        res_par ^= 1;
        if (nb) {
          // norm-backward constants of this thread's two channels in image t.img (mean, rstd from the forward
          // statistics); the previous (image, channel block)'s sums are flushed first
          if (t.img != nb_img || c0 != nb_c) {
            if (nb_img >= 0) nb_flush(P, nb_img, nb_c + (lane >> 2), lane, nb_s1[0], nb_s1[1], nb_s2[0], nb_s2[1]);
            nb_img = t.img;
            nb_c = c0;
            const int ncpg = P.n_out / P.nb_groups;
            const double cnt = (double)P.H * P.W * ncpg;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              nb_s1[h] = 0.f;
              nb_s2[h] = 0.f;
              const int c = min(ca + 8 * h, P.n_out - 1);
              const double* st = P.nb_stats + ((long long)t.img * P.nb_groups + c / ncpg) * 2;
              const double m = st[0] / cnt;
              double var = st[1] / cnt - m * m;
              if (var < 0) var = 0;
              nb_mean[h] = (float)m;
              nb_rstd[h] = (float)(1.0 / sqrt(var + (double)P.nb_eps));
              nb_ga[h] = __ldg(P.nb_gamma + c);
              nb_be[h] = __ldg(P.nb_beta + c);
            }
          }
          // acc = dL/d act(norm(x)); accumulate pass 1 of the norm backward: sum du, sum du*xhat over the pixels.
          // Pixels outside the image are zeroed up front (their x boxes are zero-filled), the activation is chosen
          // outside the element loop.
          if (!interior) {
#pragma unroll
            for (int i = 0; i < 64; ++i)
              if (!pix_ok(i)) acc[i] = 0.f;
          }
          if (P.nb_act == 1) {
#pragma unroll
            for (int i = 0; i < 64; ++i) {
              const int h = (i >> 1) & 1;
              const float xh = (lds_f32(buf_s + box_off(i)) - nb_mean[h]) * nb_rstd[h];
              const float du = acc[i] * act_grad_fast(fmaf(xh, nb_ga[h], nb_be[h]), 1);
              nb_s1[h] += du;
              nb_s2[h] = fmaf(du, xh, nb_s2[h]);
            }
          } else {
            const int a = P.nb_act;
#pragma unroll
            for (int i = 0; i < 64; ++i) {
              const int h = (i >> 1) & 1;
              const float xh = (lds_f32(buf_s + box_off(i)) - nb_mean[h]) * nb_rstd[h];
              const float du = acc[i] * ((a == 2 && fmaf(xh, nb_ga[h], nb_be[h]) <= 0.f) ? 0.2f : 1.0f);
              nb_s1[h] += du;
              nb_s2[h] = fmaf(du, xh, nb_s2[h]);
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[i] += lds_f32(buf_s + box_off(i));
        }
      }
      if (P.gn_stats) {
        float gs[2] = {0.f, 0.f}, gss[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const float x = (interior || pix_ok(i)) ? acc[i] : 0.f;
          gs[(i >> 1) & 1] += x;
          gss[(i >> 1) & 1] = fmaf(x, x, gss[(i >> 1) & 1]);
        }
        // lanes 4c .. 4c + 3 hold channel c's pixels; the channels of a group are consecutive lane quads
        for (int off = 1; off < red; off <<= 1) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            gs[h] += __shfl_xor_sync(0xffffffffu, gs[h], off);
            gss[h] += __shfl_xor_sync(0xffffffffu, gss[h], off);
          }
        }
        if (cpg >= 16) {  // channels ca and ca + 8 are in the same group
          gs[0] += gs[1];
          gss[0] += gss[1];
        }
        if ((lane & (red - 1)) == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (h == 1 && cpg >= 16) break;
            double* dst = P.gn_stats + ((long long)t.img * P.gn_groups + (ca + 8 * h) / cpg) * 2;
            atomicAdd(dst, (double)gs[h]);
            atomicAdd(dst + 1, (double)gss[h]);
          }
        }
      }
      if (P.epi_mode == EPI_DIRECT) {
        // strided destination (NCHW conv_out, Cout < 128): the threads of valid channels store their pixels
        float* dst = reinterpret_cast<float*>(P.d) + (long long)t.img * P.d_sn;
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int c = ca + 8 * ((i >> 1) & 1);
          const int p = 8 * (i >> 2) + m2 + (i & 1);
          const int h = t.h0 + (p >> tw_shift), w = t.w0 + (p & (P.TW - 1));
          if (c < P.n_out && h < P.H && w < P.W) dst[(long long)c * P.d_sc + (long long)h * P.d_sh + (long long)w * P.d_sw] = acc[i];
        }
        continue;
      }
      // Output boxes, written in place of the residual boxes they were added from.  Per st.shared the 32 lanes
      // write 8 channels x 4 pixels of one pixel parity; the 64-byte swizzle puts them on 16 banks, 2 lanes each:
      // 2-way bank conflicts.
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!has_res) {
          if (lane == 0) tma_store_wait_read<3>();  // the store that last read this box (4 commits ago) is done
          __syncwarp();
        }
#pragma unroll
        for (int i = 16 * k; i < 16 * k + 16; ++i) sts_f32(buf_s + box_off(i), acc[i]);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_4d(&tmD, my_buf + k * kSwapBox, c0, t.w0, t.h0 + k * rows_per_box, t.img);
          tma_store_commit();
        }
      }
    }
    if (nb && nb_img >= 0) nb_flush(P, nb_img, nb_c + (lane >> 2), lane, nb_s1[0], nb_s1[1], nb_s2[0], nb_s2[1]);
    if (lane == 0) tma_store_wait_read<0>();
  }
}

}  // namespace t2h
