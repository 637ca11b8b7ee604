// t2h_attn_fwd: softmax(q k^T * scale) v of the index-prediction transformer's multi-head attention as ONE
// kernel per layer (reference: models/archs/transformer_arch.py:37-71, CausalSelfAttention.forward with
// causal=False) -- replaces the q k^T tap-GEMM, the softmax kernel and the p v tap-GEMM and their [B, nh, T, T]
// round trips through HBM.  Included by gemm_tc.cu (shares its tensor-map helper).
//
// One CTA per (sequence, head, block of 128 queries); head_dim = 64, T = 128 .. 512 keys (a multiple of 128):
//
//   warp 0     TMA producer   the Q block, then 64-key chunks of the fused q|k|v projection (fp16 hi / lo planes)
//                             through a ring: K chunks for pass 1, then (K, V) chunk pairs for pass 2
//   warps 4-11 consumers      two warpgroups, 64 query rows each, accumulators in registers:
//                             pass 1  S_j = Q K_j^T (3 products hi*lo + hi*hi + lo*hi in parity mode) -> row max
//                             pass 2  S_j again -> e = 2^((s - max) * scale * log2 e), row sums, split into fp16
//                                     hi / lo register operands -> O += P_j V_j (V consumed MN-major, i.e.
//                                     token-major as the projection wrote it)
//                             finally O / sum(e) -> fp16 planes, heads side by side
// Recomputing S in pass 2 keeps the softmax exactly two-pass (max over the whole key range first) while only one
// 64-key chunk of S is ever live.
#pragma once

namespace t2h {

struct AttnDev {
  int tokens, heads, qblocks, nchunks;  // nchunks = tokens / 64
  int terms;                            // 1: single fp16 plane, 2: hi + lo planes (3 tensor-core products)
  int q_col, k_col, v_col;
  float kfac;  // scale * log2(e)
  int debug;   // T2H_DEBUG (bit 16: timeline record, see g_t2h_dbg)
  __half* out;
  long long out_plane, ld_out;
};

constexpr int kAttnThreads = 384;
constexpr int kAttnQPlane = 128 * 128;   // 128 query rows x 64 fp16
constexpr int kAttnSlot = 4 * 64 * 128;  // one ring slot: K hi, K lo, V hi, V lo of 64 keys
constexpr int kAttnSlots = 4;
constexpr int kAttnSmem = 2 * kAttnQPlane + kAttnSlots * kAttnSlot + 1024;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(__half a, __half b) {
  return static_cast<uint32_t>(__half_as_ushort(a)) | (static_cast<uint32_t>(__half_as_ushort(b)) << 16);
}

__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fused_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ AttnDev P) {
  pdl_launch_dependents();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* qs = smem;                    // [plane][128 rows][128 B]
  uint8_t* ring = qs + 2 * kAttnQPlane;  // [slot][K hi, K lo, V hi, V lo][64 rows][128 B]

  __shared__ __align__(8) uint64_t kv_full[kAttnSlots], kv_empty[kAttnSlots];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  __shared__ unsigned long long* trace_s;
  if (warp == 0 && lane == 0) {
    trace_s = nullptr;
    if ((P.debug & 16) && blockIdx.x == 0) {
      trace_s = g_t2h_dbg + (size_t)(atomicAdd(&g_t2h_dbg_n, 1u) % kTraceRecords) * 8;
      trace_s[0] = gtime_ns();
      trace_s[6] = gridDim.x;
      trace_s[7] = (1ull << 32) | (unsigned long long)P.nchunks;
    }
    tma_prefetch_desc(&tmX);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kAttnSlots; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 8);  // every consumer warp releases a slot
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  unsigned long long* const trace = trace_s;
  if (trace && threadIdx.x == 0) trace[1] = gtime_ns();

  const int qb = (int)blockIdx.x % P.qblocks;
  const int hb = (int)blockIdx.x / P.qblocks;
  const int head = hb % P.heads;
  const int seq = hb / P.heads;
  const int row0 = seq * P.tokens;    // first row of this sequence in the [rows][ld] projection
  const int qrow0 = row0 + qb * 128;  // first query row of this CTA
  const int NC = P.nchunks;
  const int T2 = P.terms;

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      for (int i = 0; i < 2 * NC; ++i) {  // ring item i: K chunk i (pass 1), then K and V chunk i - NC (pass 2)
        const int s = i % kAttnSlots;
        const bool pass2 = i >= NC;
        const int c = pass2 ? i - NC : i;
        mbar_wait(&kv_empty[s], ((i / kAttnSlots) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], (uint32_t)(8192 * T2 * (pass2 ? 2 : 1) + (i == 0 ? kAttnQPlane * T2 : 0)));
        if (i == 0) {
          for (int pl = 0; pl < T2; ++pl)
            for (int hbox = 0; hbox < 2; ++hbox)
              tma_load_3d(&tmX, &kv_full[0], qs + pl * kAttnQPlane + hbox * 8192, P.q_col + head * 64,
                          qrow0 + 64 * hbox, pl);
        }
        uint8_t* slot = ring + s * kAttnSlot;
        for (int pl = 0; pl < T2; ++pl) {
          tma_load_3d(&tmX, &kv_full[s], slot + pl * 8192, P.k_col + head * 64, row0 + 64 * c, pl);
          if (pass2)
            tma_load_3d(&tmX, &kv_full[s], slot + 16384 + pl * 8192, P.v_col + head * 64, row0 + 64 * c, pl);
        }
      }
    }
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ consumers, 64 query rows per warpgroup
    const int wg = (warp - 4) >> 2;
    const int wt = threadIdx.x & 127;
    const uint64_t q_desc = gmma_desc(smem_u32(qs) + 8192u * wg);
    const uint64_t ring_desc = gmma_desc(smem_u32(ring));
    const uint64_t v_desc0 = gmma_desc(smem_u32(ring) + 16384u, true);
    constexpr uint32_t QPL = kAttnQPlane >> 4, PL = 8192 >> 4, SLOT = kAttnSlot >> 4;
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    // S = Q K_c^T of ring item i for this warpgroup's rows (thread: rows r, r + 8, 16 columns each)
    auto scores = [&](int i, float (&sc)[32]) {
      const int s = i % kAttnSlots;
      mbar_wait(&kv_full[s], (i / kAttnSlots) & 1);
      if (trace && threadIdx.x == 128 && i == 0) trace[2] = gtime_ns();
      const uint64_t kb = ring_desc + s * SLOT;
      uint32_t acc = 0;
      wgmma_fence();
      if (T2 == 2) {
        wgmma_chunk<0, 0>(sc, q_desc, kb + PL, acc);   // hi * lo
        wgmma_chunk<0, 0>(sc, q_desc, kb, acc);        // hi * hi
        wgmma_chunk<0, 0>(sc, q_desc + QPL, kb, acc);  // lo * hi
      } else {
        wgmma_chunk<0, 0>(sc, q_desc, kb, acc);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
    };
    float m0 = -INFINITY, m1 = -INFINITY;  // rows r, r + 8
    for (int c = 0; c < NC; ++c) {
      float sc[32];
      scores(c, sc);
      release(&kv_empty[c % kAttnSlots]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        m0 = fmaxf(m0, fmaxf(sc[4 * j], sc[4 * j + 1]));
        m1 = fmaxf(m1, fmaxf(sc[4 * j + 2], sc[4 * j + 3]));
      }
    }
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {  // the four lanes of a row
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, off));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, off));
    }
    // (s - m) * kfac as one fma: the rounding of m * kfac is common to the row and cancels in e / sum(e)
    const float mk0 = m0 * P.kfac, mk1 = m1 * P.kfac;
    float sum0 = 0.f, sum1 = 0.f;
    float o[32];
    uint32_t acc_o = 0;
    for (int c = 0; c < NC; ++c) {
      const int i = NC + c, s = i % kAttnSlots;
      float sc[32];
      scores(i, sc);
      // e in the register layout of the A operand: k-step kk covers keys 16 kk .. 16 kk + 15, i.e. the 8-column
      // blocks 2 kk (registers 0, 1) and 2 kk + 1 (registers 2, 3); even registers row r, odd ones row r + 8
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        __half h[4], l[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float ev = ex2_approx(fmaf(sc[4 * j + e], P.kfac, e < 2 ? -mk0 : -mk1));
          if (e < 2) sum0 += ev; else sum1 += ev;
          split_f16(ev, h[e], l[e]);
        }
        ahi[j >> 1][(j & 1) * 2] = pack_half2(h[0], h[1]);
        ahi[j >> 1][(j & 1) * 2 + 1] = pack_half2(h[2], h[3]);
        alo[j >> 1][(j & 1) * 2] = pack_half2(l[0], l[1]);
        alo[j >> 1][(j & 1) * 2 + 1] = pack_half2(l[2], l[3]);
      }
      const uint64_t vb = v_desc0 + s * SLOT;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint64_t v = vb + kk * kGmmaStepMN;
        if (T2 == 2) {
          wgmma_rs<1>(o, ahi[kk], v + PL, acc_o);  // hi * lo
          acc_o = 1;
          wgmma_rs<1>(o, ahi[kk], v, acc_o);       // hi * hi
          wgmma_rs<1>(o, alo[kk], v, acc_o);       // lo * hi
        } else {
          wgmma_rs<1>(o, ahi[kk], v, acc_o);
          acc_o = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      release(&kv_empty[s]);
    }
    if (trace && threadIdx.x == 128) trace[3] = trace[4] = gtime_ns();
#pragma unroll
    for (int off = 1; off < 4; off <<= 1) {
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, off);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, off);
    }
    const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
    const int r = qrow0 + 64 * wg + 16 * (wt >> 5) + ((wt & 31) >> 2);
    __half* o0 = P.out + (long long)r * P.ld_out + head * 64 + 2 * (wt & 3);
    __half* o1 = o0 + 8 * P.ld_out;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      __half h[4], l[4];
      split_f16(o[4 * j] * inv0, h[0], l[0]);
      split_f16(o[4 * j + 1] * inv0, h[1], l[1]);
      split_f16(o[4 * j + 2] * inv1, h[2], l[2]);
      split_f16(o[4 * j + 3] * inv1, h[3], l[3]);
      *reinterpret_cast<uint32_t*>(o0 + 8 * j) = pack_half2(h[0], h[1]);
      *reinterpret_cast<uint32_t*>(o1 + 8 * j) = pack_half2(h[2], h[3]);
      if (T2 == 2) {
        *reinterpret_cast<uint32_t*>(o0 + P.out_plane + 8 * j) = pack_half2(l[0], l[1]);
        *reinterpret_cast<uint32_t*>(o1 + P.out_plane + 8 * j) = pack_half2(l[2], l[3]);
      }
    }
    if (trace && threadIdx.x == 128) trace[5] = gtime_ns();
  }
}

}  // namespace t2h

extern "C" int t2h_attn_fwd(const void* qkv, int terms, int64_t plane, int64_t ld, int64_t rows, int q_col, int k_col,
                            int v_col, int batch, int tokens, int heads, int head_dim, float scale, void* out,
                            int64_t out_plane, int64_t ld_out, t2h_stream_t stream) {
  using namespace t2h;
  T2H_CHECK_ARG(qkv && out && batch > 0 && heads > 0, "attn_fwd: bad args");
  T2H_CHECK_ARG(terms == 1 || terms == 2, "attn_fwd: terms=%d", terms);
  T2H_CHECK_ARG(head_dim == 64, "attn_fwd: head_dim=%d (only 64 is built; use the q k^T / softmax / p v launches)", head_dim);
  T2H_CHECK_ARG(tokens >= 128 && tokens <= 512 && tokens % 128 == 0,
                "attn_fwd: tokens=%d (need a multiple of 128 in 128..512)", tokens);
  T2H_CHECK_ARG(rows >= (int64_t)batch * tokens, "attn_fwd: rows=%lld < batch*tokens", (long long)rows);
  T2H_CHECK_ARG(q_col >= 0 && k_col >= 0 && v_col >= 0 && q_col % 8 == 0 && k_col % 8 == 0 && v_col % 8 == 0 &&
                    q_col + heads * 64 <= ld && k_col + heads * 64 <= ld && v_col + heads * 64 <= ld,
                "attn_fwd: q/k/v columns outside the projection (ld=%lld)", (long long)ld);
  T2H_CHECK_ARG(ld_out % 8 == 0 && out_plane % 8 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0 &&
                    ld_out >= heads * 64,
                "attn_fwd: output planes need 16-byte aligned rows");
  CUtensorMap tmX;
  const uint64_t dims[3] = {(uint64_t)ld, (uint64_t)rows, (uint64_t)terms};
  const uint64_t strides[3] = {1, (uint64_t)ld, (uint64_t)(terms == 2 ? plane : rows * ld)};
  const uint32_t box[3] = {64, 64, 1};
  int rc = make_tmap(&tmX, qkv, 2, 3, dims, strides, box, "attn_fwd qkv");
  if (rc != T2H_OK) return rc;
  static bool configured[64] = {};
  int dev = 0;
  T2H_CUDA(cudaGetDevice(&dev));
  if (!configured[dev & 63]) {
    T2H_CUDA(cudaFuncSetAttribute(attn_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kAttnSmem));
    configured[dev & 63] = true;
  }
  AttnDev P;
  memset(&P, 0, sizeof(P));
  P.tokens = tokens;
  P.heads = heads;
  P.qblocks = tokens / 128;  // (tests/test_gpu_row_kernels.py::attn_route restates the grid)
  P.nchunks = tokens / 64;
  P.terms = terms;
  P.q_col = q_col;
  P.k_col = k_col;
  P.v_col = v_col;
  P.kfac = scale * 1.4426950408889634f;
  P.out = reinterpret_cast<__half*>(out);
  P.out_plane = out_plane;
  P.ld_out = ld_out;
  P.debug = debug_bits();
  const int grid = batch * heads * P.qblocks;
  T2H_CUDA(launch_pdl(attn_fused_kernel, dim3(grid), dim3(kAttnThreads), kAttnSmem, as_stream(stream), tmX, P));
  T2H_LAUNCH_OK();
  return T2H_OK;
}
