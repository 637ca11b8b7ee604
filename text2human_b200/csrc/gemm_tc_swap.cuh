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
// Paired mode (kPair): a work item is two vertically adjacent tiles (rows h0 and h0 + TH, same image and 128-channel
// block).  One slab of 2 TH + extra rows serves both tiles: the second tile's view starts TH TW 128 = 16 KB after the
// first's (a multiple of the 1024-byte swizzle period), so the two views are one 256-row K-major operand.  Warpgroup
// wg computes channels 64 wg .. 64 wg + 63 of both tiles with one m64n256k16 wgmma per K step, into one 128-register
// accumulator (registers 64 h .. 64 h + 63: tile h).  Each weight tile feeds 256 output pixels, so the weight bytes
// per pixel halve, and a K step reads 2 KB of weights + 8 KB of slab from shared memory per 128 tensor-pipe clocks
// (80 B/clk of the SM's 128; two m64n128k16 on 128-pixel views read 96).  Per output element the MMA sequence is the
// unpaired one, so outputs are bit-identical; only the order of the fp64 sum atomics differs.
// The second tile of a pair may lie partly or wholly below the image: TMA zero-fills its slab rows and residual boxes,
// clips its stores, and pix_ok keeps it out of the sums.
//
// A warpgroup whose 64 channels all lie at or beyond n_out (warpgroup 1 of a column block with n0 + 64 >= n_out: the
// 3-channel conv_out) has nothing to compute: it issues no wgmma and runs no epilogue for the item, and only keeps
// the rings' barrier protocol (it waits on every fill and releases every slot, in the same order).
//
// Epilogue, straight from the accumulator registers: thread t of a warpgroup holds channels 16 (t / 32) + (t % 32) / 4
// and that + 8 of the warpgroup's 64, at pixels 8 j + 2 (t % 4) + {0, 1} of every 8-pixel block j of each tile, so
// each consumer warp owns 16 channels x 128 pixels per tile and finishes them alone (no block or warpgroup barrier):
// +bias (two registers) -> activation -> +residual (its own TMA-loaded boxes) -> GroupNorm / norm-backward partial
// sums (per thread, reduced over the four lanes of a channel and the channels of a group) -> st.shared into its own
// 64-byte-swizzled [32 pixels][16 channels] boxes -> TMA store.  In paired mode a warp runs this twice through the
// same boxes, once per tile, and reduces the GroupNorm sums of both tiles together.
#pragma once

#include <type_traits>

namespace t2h {

constexpr int kSwapThreads = 384;  // 4 producer warps + 8 consumer warps (two warpgroups of 64 output channels)
constexpr int kSwapBox = 32 * 16 * 4;         // one TMA box of the epilogue: 32 pixels x 16 fp32 channels
constexpr int kSwapWarpBuf = 4 * kSwapBox;    // a consumer warp's 128 pixels: residual in, output out, in place
static_assert(8 * kSwapWarpBuf == kEpiBytes, "epilogue boxes");
constexpr int kSwapRingBytes = kDynSmem - 1024 - kEpiBytes;  // A ring + B ring
// a paired-mode slab: 2 TH + 2 rows of TW positions (TH TW = 128, TW <= 16) x 128 bytes
constexpr int kSwapPairASlot = (2 * 128 + 2 * 16) * 128;
static_assert(kSwapPairASlot % 1024 == 0, "slab slots keep the 128-byte swizzle phase");
// Register split (setmaxnreg): the producer warpgroup only issues TMA and waits on barriers; the consumers hold a
// 64-register (paired: 128-register) accumulator plus the epilogue's values.  The split redistributes what the CTA was launched with, 384
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

// work item -> its (first) tile; in paired mode tiles_h counts pairs of tile rows
template <bool kPair>
__device__ __forceinline__ TileCoord decode_item(const TapGemmDev& P, int item) {
  TileCoord t = decode_tile(P, item, 128);
  if (kPair) t.h0 *= 2;
  return t;
}

// Ring invariant (both modes; tests/test_swap_ring_model.py replays it).  Within one warpgroup, no group waits on a
// slot whose release is deferred behind it: when a group's operands are waited for, every slot whose last reader is
// two or more groups back has been released.  Each group reads one B tile and the B index advances by at most one
// per group, so the tile a group needs reuses a slot released two groups back whenever b_slots >= 2.  A slabs
// (3-product order hi.lo, hi.hi, lo.hi per tap): the next chunk's hi slab reuses the slot of the current chunk's hi
// slab (last read by the hi.hi group before the chunk's final group) when a_slots >= 2.  1-product: one slab per
// chunk, a_slots >= 2.
// Across the two warpgroups: both read every slot (one 64-row half of each weight tile and the same slab view, 128
// rows unpaired and 256 paired; a paired group is still one group on the same slots, and a warpgroup with no valid
// channel reads nothing but waits and releases alike), every slot's empty barrier counts all 256 consumer threads,
// and both warpgroups wait on the fills in the same order.  So the warpgroup that is further behind never
// waits on the other: every fill it waits for reuses a slot it has released itself (the invariant above) and the
// other warpgroup, having passed that point, has released too.  The lag between the two is bounded by the ring
// depth, and the leader simply waits for the fills the laggard's releases allow.
template <bool kPair>
__global__ void __launch_bounds__(kSwapThreads, 1)
tapgemm_swap_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmR,
                    const __grid_constant__ TapGemmDev P) {
  using C = Cfg<128>;
  constexpr int kASlot = kPair ? kSwapPairASlot : C::kASlot;
  constexpr int NT = kPair ? 2 : 1;  // tiles of a work item: a consumer warpgroup computes 64 channels of each
  pdl_launch_dependents();  // the next kernel may start its prologue once every CTA of this one is running
  const int NA = P.a_slots, NB = P.b_slots;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem =
      reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_ring = smem;
  uint8_t* b_ring = smem + NA * kASlot;
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
  // work schedule (items: tiles, or pairs of tiles): round-robin over the CTAs, or -- when the epilogue accumulates
  // per-image sums (nb_sums) -- one contiguous range per CTA, so that a CTA stays inside one image and flushes its sums
  // once or twice per launch instead of once per item (round-robin put ~1000 double atomics per launch on every
  // (image, channel) address)
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
          const TileCoord t = decode_item<kPair>(P, tile);
          for (int g = 0; g < P.ngroups; ++g)
            for (int ch = 0; ch < P.kchunks; ++ch)
              for (int pl = 0; pl < a_planes; ++pl) {
                mbar_wait(&a_empty[sa], pa ^ 1);
                mbar_expect_tx(&a_full[sa], slab_bytes);
                tma_load_4d(&tmA, &a_full[sa], a_ring + sa * kASlot, ch * kBK, t.w0 + P.g_dx[g],
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
          const TileCoord t = decode_item<kPair>(P, tile);
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
    const int wg = (warp - 4) >> 2;  // output channels 64 wg .. 64 wg + 63 of the item's tile(s)
    const int q = (warp - 4) & 3;    // warp of the warpgroup: channels 16 q .. 16 q + 15 of those 64
    const uint32_t row16 = (uint32_t)(P.TW * 128) >> 4;  // one slab image row, in 16-byte units
    const uint64_t x_desc0 = gmma_desc(smem_u32(a_ring));  // paired: both tiles' views, 256 rows
    const uint64_t w_desc0 = gmma_desc(smem_u32(b_ring) + 8192u * wg);
    constexpr uint32_t A16 = kASlot >> 4, B16 = C::kBSlot >> 4;
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
    // first of the 16 channels this warp finishes in the column block at n0
    auto chan0 = [&](int n0) { return n0 + 64 * wg + 16 * q; };
    // norm-backward sums: the "residual" tile is x and is not added
    const bool nb = P.nb_sums != nullptr;
    // per thread: channel c (index 0) and c + 8 (index 1); the sums run on across consecutive items of the same
    // (image, channel block) and are flushed when that changes.  Their GroupNorm constants are derived again for
    // every tile: held across items, they would cost the paired accumulator registers.
    float nb_s1[2] = {0.f, 0.f}, nb_s2[2] = {0.f, 0.f};
    int nb_img = -1, nb_n0 = -1;
    // residual (or x) boxes of this warp's channels of the tile at row h0, into the boxes the previous stores read from
    auto load_res = [&](const TileCoord& t, int h0) {
      tma_store_wait_read<0>();
      mbar_expect_tx(&res_bar[e], kSwapWarpBuf);
      for (int k = 0; k < 4; ++k)
        tma_load_4d(&tmR, &res_bar[e], my_buf + k * kSwapBox, chan0(t.n0), t.w0, h0 + k * rows_per_box, t.img);
    };

    for (int tile = tile_first; tile < tile_end; tile += tile_step) {
      const TileCoord t = decode_item<kPair>(P, tile);
      // none of this warpgroup's 64 channels exists: keep the rings' barrier protocol and do nothing else
      const bool idle = t.n0 + 64 * wg >= P.n_out;
      if (has_res && !idle && lane == 0) {
        // the first tile's boxes load while the MMAs run; the second's go to L2 now, so that its load is an L2 hit
        load_res(t, t.h0);
#pragma unroll
        for (int h = 1; h < NT; ++h)
          for (int k = 0; k < 4; ++k)
            tma_prefetch_4d(&tmR, chan0(t.n0), t.w0, t.h0 + h * P.TH + k * rows_per_box, t.img);
        if (nb && tile + tile_step < tile_end) {
          // the NEXT item's x boxes go to L2 now, so that its loads above are L2 hits
          const TileCoord tn = decode_item<kPair>(P, tile + tile_step);
#pragma unroll
          for (int h = 0; h < NT; ++h)
            for (int k = 0; k < 4; ++k)
              tma_prefetch_4d(&tmR, chan0(tn.n0), tn.w0, tn.h0 + h * P.TH + k * rows_per_box, tn.img);
        }
      }
      float acc[64 * NT];
      // the item's MMA groups; kIdle: the same waits and releases without the MMAs
      auto mainloop = [&](auto kIdle) {
        uint32_t accf = 0;
        int rel_b = -1, rel_a = -1;  // the slots the group in flight is the last reader of (-1: none)
        // every consumer thread arrives (a lane-0 arrival between wgmmas puts them on a divergent path, and ptxas
        // then serialises every MMA); the arrivals are for the previous group, which wait_group 1 has completed
        auto group = [&](uint64_t w, uint64_t x, int last_b, int last_a) {
          if constexpr (!decltype(kIdle)::value) {
            wgmma_fence();
            wgmma_chunk<0, 0>(acc, w, x, accf);
            wgmma_commit();
            wgmma_wait<1>();
          }
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
        if constexpr (!decltype(kIdle)::value) {
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
        }
        if (rel_b >= 0) mbar_arrive(&b_empty[rel_b]);
        if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
      };
      if (idle) {
        mainloop(std::true_type{});
        continue;
      }
      mainloop(std::false_type{});
      if (nb && (t.img != nb_img || t.n0 != nb_n0)) {  // the previous (image, channel block)'s sums are flushed
        if (nb_img >= 0)
          nb_flush(P, nb_img, chan0(nb_n0) + (lane >> 2), lane, nb_s1[0], nb_s1[1], nb_s2[0], nb_s2[1]);
#pragma unroll
        for (int k = 0; k < 2; ++k) nb_s1[k] = nb_s2[k] = 0.f;
        nb_img = t.img;
        nb_n0 = t.n0;
      }
      const int c0 = chan0(t.n0);       // this warp's 16 output channels
      const int ca = c0 + (lane >> 2);  // this thread's channels, in every tile of the item: ca and ca + 8
      float bias2[2] = {0.f, 0.f};
      if (P.bias_mode == T2H_BIAS_COL) {
        if (ca < P.n_out) bias2[0] = __ldg(P.bias + t.img * P.bias_sn + ca);
        if (ca + 8 < P.n_out) bias2[1] = __ldg(P.bias + t.img * P.bias_sn + ca + 8);
      }
      float gs[2] = {0.f, 0.f}, gss[2] = {0.f, 0.f};  // GroupNorm partial sums over the item's tiles
#pragma unroll
      for (int h = 0; h < NT; ++h) {
        float* a = acc + 64 * h;
        const int th0 = t.h0 + h * P.TH;  // first image row of tile h
        if (h > 0 && has_res && lane == 0) load_res(t, th0);
        // interior tiles need no per-pixel validity test for the GroupNorm / norm-backward sums
        const bool interior = (th0 + P.TH <= P.H) && (t.w0 + P.TW <= P.W);
        // bit 2 j + b: this thread's pixel 8 j + m2 + b of the tile lies inside the image
        uint32_t ok_mask = ~0u;
        if (!interior) {
          ok_mask = 0;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const int p = 8 * (j >> 1) + m2 + (j & 1);
            if ((th0 + (p >> tw_shift) < P.H) && (t.w0 + (p & (P.TW - 1)) < P.W)) ok_mask |= 1u << j;
          }
        }
        auto pix_ok = [&](int i) { return ((ok_mask >> (2 * (i >> 2) + (i & 1))) & 1u) != 0; };
        // accumulator element i: channel ca + 8 ((i >> 1) & 1), pixel 8 (i >> 2) + m2 + (i & 1); in-box pixel and
        // channel of the [32][16] box i >> 4
        auto box_off = [&](int i) { return (i >> 4) * kSwapBox + swz64(8 * ((i >> 2) & 3) + m2 + (i & 1), (lane >> 2) + 8 * ((i >> 1) & 1)); };
#pragma unroll
        for (int i = 0; i < 64; ++i) a[i] = a[i] * P.alpha + bias2[(i >> 1) & 1];
        apply_act<64>(a, P.act);
        if (has_res) {
          mbar_wait(&res_bar[e], res_par);
          res_par ^= 1;
          if (nb) {
            // norm-backward constants of this thread's two channels in image t.img (mean, rstd from the forward
            // statistics)
            float nb_mean[2], nb_rstd[2], nb_ga[2], nb_be[2];
            const int ncpg = P.n_out / P.nb_groups;
            const double cnt = (double)P.H * P.W * ncpg;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const int c = min(ca + 8 * k, P.n_out - 1);
              const double* st = P.nb_stats + ((long long)t.img * P.nb_groups + c / ncpg) * 2;
              const double m = st[0] / cnt;
              double var = st[1] / cnt - m * m;
              if (var < 0) var = 0;
              nb_mean[k] = (float)m;
              nb_rstd[k] = (float)(1.0 / sqrt(var + (double)P.nb_eps));
              nb_ga[k] = __ldg(P.nb_gamma + c);
              nb_be[k] = __ldg(P.nb_beta + c);
            }
            // acc = dL/d act(norm(x)); accumulate pass 1 of the norm backward: sum du, sum du*xhat over the pixels.
            // Pixels outside the image are zeroed up front (their x boxes are zero-filled), the activation is chosen
            // outside the element loop.
            if (!interior) {
#pragma unroll
              for (int i = 0; i < 64; ++i)
                if (!pix_ok(i)) a[i] = 0.f;
            }
            if (P.nb_act == 1) {
#pragma unroll
              for (int i = 0; i < 64; ++i) {
                const int k = (i >> 1) & 1;
                const float xh = (lds_f32(buf_s + box_off(i)) - nb_mean[k]) * nb_rstd[k];
                const float du = a[i] * act_grad_fast(fmaf(xh, nb_ga[k], nb_be[k]), 1);
                nb_s1[k] += du;
                nb_s2[k] = fmaf(du, xh, nb_s2[k]);
              }
            } else {
              const int an = P.nb_act;
#pragma unroll
              for (int i = 0; i < 64; ++i) {
                const int k = (i >> 1) & 1;
                const float xh = (lds_f32(buf_s + box_off(i)) - nb_mean[k]) * nb_rstd[k];
                const float du = a[i] * ((an == 2 && fmaf(xh, nb_ga[k], nb_be[k]) <= 0.f) ? 0.2f : 1.0f);
                nb_s1[k] += du;
                nb_s2[k] = fmaf(du, xh, nb_s2[k]);
              }
            }
          } else {
#pragma unroll
            for (int i = 0; i < 64; ++i) a[i] += lds_f32(buf_s + box_off(i));
          }
        }
        if (P.gn_stats) {
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const float x = (interior || pix_ok(i)) ? a[i] : 0.f;
            gs[(i >> 1) & 1] += x;
            gss[(i >> 1) & 1] = fmaf(x, x, gss[(i >> 1) & 1]);
          }
        }
        if (P.epi_mode == EPI_DIRECT) {
          // strided destination (NCHW conv_out, Cout < 128): the threads of valid channels store their pixels
          float* dst = reinterpret_cast<float*>(P.d) + (long long)t.img * P.d_sn;
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const int c = ca + 8 * ((i >> 1) & 1);
            const int p = 8 * (i >> 2) + m2 + (i & 1);
            const int hh = th0 + (p >> tw_shift), w = t.w0 + (p & (P.TW - 1));
            if (c < P.n_out && hh < P.H && w < P.W) dst[(long long)c * P.d_sc + (long long)hh * P.d_sh + (long long)w * P.d_sw] = a[i];
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
          for (int i = 16 * k; i < 16 * k + 16; ++i) sts_f32(buf_s + box_off(i), a[i]);
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            tma_store_4d(&tmD, my_buf + k * kSwapBox, c0, t.w0, th0 + k * rows_per_box, t.img);
            tma_store_commit();
          }
        }
      }
      if (P.gn_stats) {
        // lanes 4c .. 4c + 3 hold channel c's pixels; the channels of a group are consecutive lane quads
        for (int off = 1; off < red; off <<= 1) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            gs[k] += __shfl_xor_sync(0xffffffffu, gs[k], off);
            gss[k] += __shfl_xor_sync(0xffffffffu, gss[k], off);
          }
        }
        if (cpg >= 16) {  // channels ca and ca + 8 are in the same group
          gs[0] += gs[1];
          gss[0] += gss[1];
        }
        if ((lane & (red - 1)) == 0) {
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (k == 1 && cpg >= 16) break;
            double* dst = P.gn_stats + ((long long)t.img * P.gn_groups + (ca + 8 * k) / cpg) * 2;
            atomicAdd(dst, (double)gs[k]);
            atomicAdd(dst + 1, (double)gss[k]);
          }
        }
      }
    }
    if (nb && nb_img >= 0)
      nb_flush(P, nb_img, chan0(nb_n0) + (lane >> 2), lane, nb_s1[0], nb_s1[1], nb_s2[0], nb_s2[1]);
    if (lane == 0) tma_store_wait_read<0>();
  }
}

}  // namespace t2h
