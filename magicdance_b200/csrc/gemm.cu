// wgmma GEMM / 3x3 implicit-GEMM convolution for sm_90a.
//
//   D[M,N] = epilogue(A[M,K] * B[N,K]^T), fp16 operands, fp32 accumulation in registers.
//
// One CTA computes one 128 x BN output tile (optionally one K-split of it).  Warp roles:
//   warp 8     TMA producer   — streams 128x64 A tiles and BNx64 B tiles (128B-swizzled) through a
//                               kStages-deep smem ring; completion on `full` mbarriers.  In conv
//                               mode the A tile of tap (kh,kw) is a 4-D TMA box over the NHWC
//                               activation shifted by (kw-1, kh-1): out-of-bounds rows/cols are
//                               zero-filled by TMA, which IS the pad-1 halo — no im2col buffer.
//   warps 0-7  two warpgroups, 64 rows each: wgmma (M=64, N=BN, K=16) x4 per stage straight from the
//                               swizzled smem tiles, one stage in flight while the next is issued; a
//                               stage is handed back (`empty`) once the MMAs reading it have retired.
//                               Then the fp32 tile is parked in the idle operand ring and the same
//                               threads run the epilogue one row per thread: bias / per-batch bias
//                               (timestep embedding) / residual / GEGLU, fp16 stores.
// Tiles up to 128 wide with a 3-stage ring fit twice per SM (<= 97 KB smem, <= 112 registers a thread), so one
// CTA's epilogue overlaps the other's main loop; deep rings and 256-wide tiles run one CTA per SM.
#include <stdlib.h>

#include "common.cuh"

namespace mdb {

constexpr int kBM = 128;
constexpr int kBK = 64;  // 64 halves = 128 B = one swizzle row

struct GemmKParams {
  CUtensorMap tmA;
  CUtensorMap tmA2;
  CUtensorMap tmB;
  __half* d;
  long long ldd;
  const float* bias;
  long long bias_batch_stride;
  const __half* residual;
  long long ldr;
  float* ws;
  int rows_per_batch;
  int m, n;
  int k_chunks;        // total K / 64
  int k1_chunks;       // chunks taken from tmA (plain mode); rest from tmA2
  int chunks_per_split;
  int splits;
  int conv;            // conv mode
  int chunks_per_tap;  // c / 64
  int w, hw;           // conv geometry of the OUTPUT (== input for stride 1)
  int cs;              // conv stride (1 | 2): input pixel = cs * output pixel + tap - 1
  int cluster_reduce;  // split-K partners form a cluster (1,1,splits) and reduce through distributed smem
  // LayerNorm folded into this GEMM (gemm_tc_kernel only): D = rstd_r (A W'^T - mean_r u) + bias with W' = W diag(gamma),
  // u[n] = sum_k W'[n][k]; the epilogue warps compute (mean_r, rstd_r) of their A rows from the staged tiles
  const float* ln_u;
  float ln_eps;
};

// STAGES = 3: <=109 KB, two CTAs per SM (large grids: the co-resident CTA hides the TMA round trip).
// STAGES = 6 (8 for 80-wide tiles): one CTA per SM with a ring deep enough to cover the TMA latency on
// its own — used when the grid has at most one CTA per SM anyway and the K loop is long.
// BN = 256, STAGES = 4 (the large grids, see mdb_gemm_f16): one CTA per SM; half the L2 -> SM bytes per flop of two
// 128-wide tiles.
template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kTotal = STAGES * kStageBytes + 1024;  // + alignment slack
  static constexpr int kCtasPerSm = (kTotal <= 113 * 1024 && BN <= 128) ? 2 : 1;
};

__device__ __forceinline__ void epi_store_chunk(const GemmKParams& p, long long row, int col0, int ncols,
                                                float (&v)[32], const float* bias_chunk) {
  // v holds columns col0 .. col0+31 of `row` (fp32 accumulators); bias + residual, then fp16 store.
  // Whole groups of 8 columns go through 16-byte accesses, a ragged tail (N = 77) is scalar.
  // bias_chunk: this chunk's 32 bias values (shared or global memory) or nullptr.
  const __half* rp = (p.residual != nullptr) ? p.residual + row * p.ldr + col0 : nullptr;
  __half* dp = p.d + row * p.ldd + col0;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (q * 8 + 8 <= ncols) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = v[q * 8 + e];
      if (bias_chunk != nullptr) {
        const float4 b0 = *reinterpret_cast<const float4*>(bias_chunk + q * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(bias_chunk + q * 8 + 4);
        o[0] += b0.x; o[1] += b0.y; o[2] += b0.z; o[3] += b0.w;
        o[4] += b1.x; o[5] += b1.y; o[6] += b1.z; o[7] += b1.w;
      }
      if (rp != nullptr) {
        const uint4 r4 = *reinterpret_cast<const uint4*>(rp + q * 8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&r4);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h2[e]);
          o[2 * e] += f.x;
          o[2 * e + 1] += f.y;
        }
      }
      uint4 o4;
      o4.x = pack_half2(o[0], o[1]);
      o4.y = pack_half2(o[2], o[3]);
      o4.z = pack_half2(o[4], o[5]);
      o4.w = pack_half2(o[6], o[7]);
      *reinterpret_cast<uint4*>(dp + q * 8) = o4;
    } else if (q * 8 < ncols) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = q * 8 + e;
        if (j < ncols) {
          float x = v[j];
          if (bias_chunk != nullptr) x += bias_chunk[j];
          if (rp != nullptr) x += __half2float(rp[j]);
          dp[j] = __float2half_rn(x);
        }
      }
    }
  }
}

// IM2COL: the 3x3 conv's A tiles come from TMA im2col loads (tmap_nhwc_im2col), which walk 128 consecutive output
// pixels across row and image boundaries: any latent size, one or two sources split along the channels (k1_chunks of
// the chunks_per_tap chunks of a tap from tmA, the rest from tmA2).  The tiles are the ones the 4-D boxes give at sizes
// that tile, so everything after the producer is shared.
template <int BN, bool GEGLU, int kStages, bool IM2COL>
__device__ __forceinline__ void gemm_tc_body(const GemmKParams& p) {
  using S = GemmSmem<BN, kStages>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kStages];
  __shared__ __align__(8) uint64_t empty_bar[kStages];
  __shared__ __align__(16) float s_bias[BN];  // this N tile's bias row (when one row serves all batches)
  __shared__ __align__(16) float s_lnu[BN];   // this N tile's u (LayerNorm folded into the GEMM)
  __shared__ float2 s_ln[kBM];                // (mean, rstd) of each row of the tile (LayerNorm fusion)

  uint8_t* smem = align1024(smem_raw);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * kBM;
  const int n0 = blockIdx.y * BN;
  const int split = blockIdx.z;
  const int kc_begin = split * p.chunks_per_split;
  const int kc_end = min(p.k_chunks, kc_begin + p.chunks_per_split);
  const int n_iter = kc_end - kc_begin;
  constexpr int kRedLd = BN + 4;  // fp32 row pitch of the accumulator tile parked in shared memory
  static_assert(kBM * kRedLd * 4 <= kStages * S::kStageBytes, "the accumulator tile must fit in the operand ring");
  const bool ln = p.ln_u != nullptr;

  pdl_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&p.tmA);
    if constexpr (IM2COL) tma_prefetch_desc(&p.tmA2);
    tma_prefetch_desc(&p.tmB);
    ring_init<kStages>(full_bar, empty_bar, 1);
    fence_barrier_init();
  }
  // a bias row that serves all batches is a constant weight: stage it before the PDL wait (overlaps the
  // previous kernel's tail).  Per-batch biases (timestep embedding) are produced upstream and are read later.
  const bool bias_in_smem = (p.bias != nullptr) && (p.bias_batch_stride == 0) && !p.cluster_reduce;
  if (bias_in_smem && warp < kProducerWarp) {
    for (int j = threadIdx.x; j < BN; j += kConsumers) s_bias[j] = (n0 + j < p.n) ? p.bias[n0 + j] : 0.f;
  }
  if (ln && warp < kProducerWarp) {  // a constant of the weights, like the bias
    for (int j = threadIdx.x; j < BN; j += kConsumers) s_lnu[j] = (n0 + j < p.n) ? p.ln_u[n0 + j] : 0.f;
  }
  __syncthreads();
  pdl_wait();  // everything above overlapped the previous kernel's tail; global memory from here on

  if (warp == kProducerWarp) {
    if (lane == 0 && n_iter > 0) {
      // conv geometry of this M tile
      int b0 = 0, y0 = 0, x0 = 0;
      if constexpr (IM2COL) {  // the first output pixel of this M tile; the tile may run on into later rows and images
        b0 = m0 / p.hw;
        y0 = (m0 - b0 * p.hw) / p.w;
        x0 = (m0 - b0 * p.hw) - y0 * p.w;
      } else if (p.conv) {
        b0 = m0 / p.hw;
        y0 = (p.hw >= kBM) ? (m0 % p.hw) / p.w : 0;
        x0 = (p.hw >= kBM) ? (m0 % p.hw) % p.w : 0;  // != 0 only for rows wider than the 128-pixel tile
      }
      for (int it = 0; it < n_iter; ++it) {
        const int s = ring_acquire<kStages>(empty_bar, it);
        uint8_t* sa = smem + s * S::kStageBytes;
        uint8_t* sb = sa + S::kABytes;
        const int kc = kc_begin + it;
        mbar_expect_tx(&full_bar[s], S::kStageBytes);
        if constexpr (IM2COL) {
          const int tap = kc / p.chunks_per_tap;
          const int cc = kc - tap * p.chunks_per_tap;
          const int kh = tap / 3, kw = tap - kh * 3;
          const int xs = p.cs * x0 - 1, ys = p.cs * y0 - 1;  // the first window's corner; the tap is the offset
          if (cc < p.k1_chunks) tma_load_im2col_4d(sa, &p.tmA, &full_bar[s], cc * kBK, xs, ys, b0, kw, kh);
          else tma_load_im2col_4d(sa, &p.tmA2, &full_bar[s], (cc - p.k1_chunks) * kBK, xs, ys, b0, kw, kh);
        } else if (p.conv) {
          const int tap = kc / p.chunks_per_tap;
          const int cc = kc - tap * p.chunks_per_tap;
          const int kh = tap / 3, kw = tap - kh * 3;
          tma_load_4d(sa, &p.tmA, &full_bar[s], cc * kBK, p.cs * x0 + kw - 1, p.cs * y0 + kh - 1, b0);
        } else if (kc < p.k1_chunks) {
          tma_load_2d(sa, &p.tmA, &full_bar[s], kc * kBK, m0);
        } else {
          tma_load_2d(sa, &p.tmA2, &full_bar[s], (kc - p.k1_chunks) * kBK, m0);
        }
        tma_load_2d(sb, &p.tmB, &full_bar[s], kc * kBK, n0);
      }
    }
  } else {
    // ---------------- warpgroups 0, 1: main loop on wgmma, then the epilogue ----------------
    const int wg = warp >> 2;          // this warpgroup's 64 rows of the tile
    const int tid = threadIdx.x;       // 0 .. kConsumers-1
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // LayerNorm folded into the GEMM: statistics of the A rows (pivot-shifted sums, biased variance as nn.LayerNorm),
    // taken from the A tiles AS THEY PASS THROUGH SHARED MEMORY on their way to the tensor core, while the wgmma of
    // the stage runs: two threads per row, each summing half of the 64 columns.  No extra global or L2 traffic.
    const int ln_row = tid >> 1, ln_half = tid & 1;
    float pivot = 0.f, ls0 = 0.f, ls1 = 0.f, lq0 = 0.f, lq1 = 0.f;
    for (int it = 0; it < n_iter; ++it) {
      const int s = ring_wait_full<kStages>(full_bar, it);
      const uint32_t a_addr = smem_u32(smem + s * S::kStageBytes);
      const uint64_t da = wgmma_desc_k_sw128(a_addr + wg * (64 * 128));
      const uint64_t db = wgmma_desc_k_sw128(a_addr + S::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, 1u);
      wgmma_commit();
      if (ln) {
        const uint32_t arow = a_addr + (ln_row >> 3) * 1024 + (ln_row & 7) * 128;
        if (it == 0) {  // every thread of the row pair takes the row's first element as the pivot
          uint32_t w0;
          asm volatile("ld.shared.b32 %0, [%1];" : "=r"(w0) : "r"(arow + ((0 ^ (ln_row & 7)) << 4)));
          pivot = __low2float(*reinterpret_cast<const __half2*>(&w0));
        }
#pragma unroll
        for (int l = ln_half * 4; l < ln_half * 4 + 4; ++l) {  // logical 16-byte chunk l sits at l ^ (row & 7)
          uint4 u4;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(u4.x), "=r"(u4.y), "=r"(u4.z), "=r"(u4.w)
                       : "r"(arow + ((l ^ (ln_row & 7)) << 4)));
          const __half2* h2 = reinterpret_cast<const __half2*>(&u4);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h2[e]);
            const float d0 = f.x - pivot, d1 = f.y - pivot;
            ls0 += d0; lq0 = fmaf(d0, d0, lq0);
            ls1 += d1; lq1 = fmaf(d1, d1, lq1);
          }
        }
      }
      wgmma_wait<1>();  // the previous stage's MMAs have finished reading it
      wgmma_fence_regs(acc);
      if (it > 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (ln) {
      float s_ = ls0 + ls1, q_ = lq0 + lq1;
      s_ += __shfl_xor_sync(0xffffffffu, s_, 1);
      q_ += __shfl_xor_sync(0xffffffffu, q_, 1);
      const float inv_k = 1.0f / static_cast<float>(p.k_chunks * kBK);
      const float ms = s_ * inv_k;
      if (ln_half == 0) s_ln[ln_row] = make_float2(pivot + ms, rsqrtf(fmaxf(fmaf(-ms, ms, q_ * inv_k), 0.f) + p.ln_eps));
    }
    // Both warpgroups' MMAs are complete, so the operand ring is idle: park the fp32 tile in it, [128][kRedLd]
    // (the layout the split-K cluster reduction reads), and run the epilogue with one thread per row.
    named_bar_sync(1, kConsumers);
    float* red = reinterpret_cast<float*>(smem);
    {
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN / 2; j += 2) {
        const int row_t = r0 + 8 * ((j >> 1) & 1);
        const int col = 8 * (j >> 2) + 2 * (lane & 3);
        *reinterpret_cast<float2*>(red + row_t * kRedLd + col) = make_float2(acc[j], acc[j + 1]);
      }
    }
    named_bar_sync(1, kConsumers);

    const int rt = tid & (kBM - 1);   // row inside the tile
    const int half = tid / kBM;       // which of the tile's column chunks this thread takes (alternating)
    const long long row = static_cast<long long>(m0) + rt;
    const bool row_ok = row < p.m;
    const float* rrow = red + rt * kRedLd;
    if constexpr (!GEGLU) {
      if (!p.cluster_reduce) {
        const float2 lnst = ln ? s_ln[rt] : make_float2(0.f, 1.f);
#pragma unroll 1
        for (int ch = half; ch < (BN + 31) / 32; ch += 2) {
          const int col0 = n0 + ch * 32;
          if (col0 >= p.n) break;
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            if (ch * 32 + j < BN) {
              const float4 f = *reinterpret_cast<const float4*>(rrow + ch * 32 + j);
              v[j] = f.x; v[j + 1] = f.y; v[j + 2] = f.z; v[j + 3] = f.w;
            } else {
              v[j] = v[j + 1] = v[j + 2] = v[j + 3] = 0.f;
            }
          }
          if (ln) {  // rstd_r (acc - mean_r u[n]); the bias row carries W beta (+ the layer's own bias)
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (ch * 32 + j < BN) v[j] = lnst.y * fmaf(-lnst.x, s_lnu[ch * 32 + j], v[j]);
          }
          const int ncols = min(min(32, BN - ch * 32), p.n - col0);
          if (p.splits > 1) {
            // split-K through global memory: this split's fp32 partial goes to its own workspace slab
            // (plain vector stores); splitk_finalize_kernel sums the slabs in a fixed order.
            if (row_ok) {
              float* wp = p.ws + (static_cast<long long>(split) * p.m + row) * p.n + col0;
#pragma unroll
              for (int j = 0; j < 32; j += 4) {
                if (j + 4 <= ncols && (p.n & 3) == 0) {
                  *reinterpret_cast<float4*>(wp + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                } else {
#pragma unroll
                  for (int e = 0; e < 4; ++e)
                    if (j + e < ncols) wp[j + e] = v[j + e];
                }
              }
            }
          } else if (row_ok) {
            const float* bias_chunk = nullptr;
            if (bias_in_smem) {
              bias_chunk = s_bias + ch * 32;
            } else if (p.bias != nullptr) {
              const long long brow = (p.bias_batch_stride != 0) ? (row / p.rows_per_batch) : 0;
              bias_chunk = p.bias + brow * p.bias_batch_stride + col0;
            }
            epi_store_chunk(p, row, col0, ncols, v, bias_chunk);
          }
        }
      }
    } else {
      // GEGLU: chunk pairs (value, gate); output column = n0/2 + pair*32 + j
      const long long brow = (p.bias_batch_stride != 0) ? (row / p.rows_per_batch) : 0;
#pragma unroll 1
      for (int pr = half; pr < BN / 64; pr += 2) {
        const int col0 = n0 + pr * 64;
        if (col0 >= p.n) break;
        if (row_ok) {
          const float* bp = bias_in_smem ? (s_bias + pr * 64)
                                         : ((p.bias != nullptr) ? p.bias + brow * p.bias_batch_stride + col0 : nullptr);
          const float* rv = rrow + pr * 64;
          uint4* d4 = reinterpret_cast<uint4*>(p.d + row * p.ldd + (col0 >> 1));
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float o[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int j = q * 8 + e;
              float a = rv[j];
              float gt = rv[32 + j];
              if (bp != nullptr) {
                a += bp[j];
                gt += bp[32 + j];
              }
              o[e] = a * gelu_erf_f(gt);
            }
            uint4 o4;
            o4.x = pack_half2(o[0], o[1]);
            o4.y = pack_half2(o[2], o[3]);
            o4.z = pack_half2(o[4], o[5]);
            o4.w = pack_half2(o[6], o[7]);
            d4[q] = o4;
          }
        }
      }
    }
  }

  if constexpr (!GEGLU) {
    if (p.cluster_reduce) {
      // ---- split-K reduction across the cluster through distributed shared memory ----
      // cluster = the `splits` CTAs of this output tile (2 ... 8).  CTA r owns rows [r*128/S, (r+1)*128/S) of the
      // tile: it sums that slice over all partners' parked partials in split order (ld.shared::cluster), applies the
      // epilogue and stores fp16.  No global workspace, no second kernel.
      const int S_ = p.splits;
      const uint32_t crank = cluster_ctarank();
      const int r_begin = static_cast<int>(crank) * kBM / S_;
      const int R = (static_cast<int>(crank) + 1) * kBM / S_ - r_begin;
      const int groups = BN / 8;
      // this thread's share of the residual is known up front: fetch it before the cluster barrier
      constexpr int kMaxItems = 4;
      uint4 rpre[kMaxItems];
      if (p.residual != nullptr) {
#pragma unroll
        for (int q = 0; q < kMaxItems; ++q) {
          const int item = threadIdx.x + q * kWsThreads;
          if (item < R * groups) {
            const int rl = item / groups, cgp = item - rl * groups;
            const long long row = static_cast<long long>(m0) + r_begin + rl;
            const int col0 = n0 + cgp * 8;
            if (row < p.m && col0 + 8 <= p.n) rpre[q] = *reinterpret_cast<const uint4*>(p.residual + row * p.ldr + col0);
          }
        }
      }
      cluster_sync_all();
      const uint32_t red_base = smem_u32(smem);
#pragma unroll 1
      for (int it_ = 0; it_ * kWsThreads < R * groups; ++it_) {
        const int item = threadIdx.x + it_ * kWsThreads;
        if (item >= R * groups) break;
        const int rl = item / groups, cgp = item - rl * groups;
        const int rt = r_begin + rl;  // row inside the tile
        const long long row = static_cast<long long>(m0) + rt;
        const int col0 = n0 + cgp * 8;
        if (row >= p.m || col0 >= p.n) continue;
        const uint32_t off = red_base + static_cast<uint32_t>((rt * kRedLd + cgp * 8) * 4);
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = 0.f;
        for (int pr = 0; pr < S_; ++pr) {
          const uint32_t ra = dsmem_map(off, static_cast<uint32_t>(pr));
          const float4 a = dsmem_ld_f4(ra), b = dsmem_ld_f4(ra + 16);
          o[0] += a.x; o[1] += a.y; o[2] += a.z; o[3] += a.w;
          o[4] += b.x; o[5] += b.y; o[6] += b.z; o[7] += b.w;
        }
        const int ncols = min(8, p.n - col0);
        const long long brow = (p.bias_batch_stride != 0) ? (row / p.rows_per_batch) : 0;
        if (p.bias != nullptr) {
          const float* bp = p.bias + brow * p.bias_batch_stride + col0;
          for (int e = 0; e < ncols; ++e) o[e] += bp[e];
        }
        if (ncols == 8) {
          if (p.residual != nullptr) {
            uint4 r4 = make_uint4(0, 0, 0, 0);
            if (it_ < kMaxItems) {
#pragma unroll
              for (int q = 0; q < kMaxItems; ++q)
                if (q == it_) r4 = rpre[q];
            } else {
              r4 = *reinterpret_cast<const uint4*>(p.residual + row * p.ldr + col0);
            }
            const __half2* h2 = reinterpret_cast<const __half2*>(&r4);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f = __half22float2(h2[e]);
              o[2 * e] += f.x;
              o[2 * e + 1] += f.y;
            }
          }
          uint4 o4;
          o4.x = pack_half2(o[0], o[1]);
          o4.y = pack_half2(o[2], o[3]);
          o4.z = pack_half2(o[4], o[5]);
          o4.w = pack_half2(o[6], o[7]);
          *reinterpret_cast<uint4*>(p.d + row * p.ldd + col0) = o4;
        } else {
          for (int e = 0; e < ncols; ++e) {
            float x = o[e];
            if (p.residual != nullptr) x += __half2float(p.residual[row * p.ldr + col0 + e]);
            p.d[row * p.ldd + col0 + e] = __float2half_rn(x);
          }
        }
      }
      cluster_sync_all();  // nobody leaves while a partner may still read its shared memory
    }
  }
}

template <int BN, bool GEGLU, int kStages>
__global__ void __launch_bounds__(kWsThreads, (GemmSmem<BN, kStages>::kCtasPerSm))
    gemm_tc_kernel(const __grid_constant__ GemmKParams p) {
  gemm_tc_body<BN, GEGLU, kStages, false>(p);
}

template <int BN, int kStages>
__global__ void __launch_bounds__(kWsThreads, (GemmSmem<BN, kStages>::kCtasPerSm))
    gemm_igemm_kernel(const __grid_constant__ GemmKParams p) {
  gemm_tc_body<BN, false, kStages, true>(p);
}

// split-K second pass: sum of the fp32 partial slabs ws[splits][M][N] -> bias/residual -> fp16 D
__global__ void splitk_finalize_kernel(GemmKParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const long long slab = static_cast<long long>(p.m) * p.n;
  if ((p.n & 3) == 0) {
    const long long total4 = slab >> 2;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
      const long long e = i << 2;
      const long long row = e / p.n;
      const int col = static_cast<int>(e - row * p.n);
      float4 a = *reinterpret_cast<const float4*>(p.ws + e);
      for (int s = 1; s < p.splits; ++s) {
        const float4 b = *reinterpret_cast<const float4*>(p.ws + s * slab + e);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      if (p.bias != nullptr) {
        const long long brow = (p.bias_batch_stride != 0) ? (row / p.rows_per_batch) : 0;
        const float* bp = p.bias + brow * p.bias_batch_stride + col;
        a.x += bp[0]; a.y += bp[1]; a.z += bp[2]; a.w += bp[3];
      }
      if (p.residual != nullptr) {
        const __half2* rp = reinterpret_cast<const __half2*>(p.residual + row * p.ldr + col);
        const float2 r0 = __half22float2(rp[0]), r1 = __half22float2(rp[1]);
        a.x += r0.x; a.y += r0.y; a.z += r1.x; a.w += r1.y;
      }
      uint2 o;
      o.x = pack_half2(a.x, a.y);
      o.y = pack_half2(a.z, a.w);
      *reinterpret_cast<uint2*>(p.d + row * p.ldd + col) = o;
    }
    return;
  }
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < slab;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / p.n;
    const int col = static_cast<int>(i - row * p.n);
    float v = 0.f;
    for (int s = 0; s < p.splits; ++s) v += p.ws[s * slab + i];
    if (p.bias != nullptr) {
      const long long brow = (p.bias_batch_stride != 0) ? (row / p.rows_per_batch) : 0;
      v += p.bias[brow * p.bias_batch_stride + col];
    }
    if (p.residual != nullptr) v += __half2float(p.residual[row * p.ldr + col]);
    p.d[row * p.ldd + col] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int pixel_box(int ho, int wo, int cs, int rows, bool fwd, uint32_t box[4]) {
  const int hw = ho * wo;
  if (fwd ? wo > rows : wo >= rows) {
    // rows as wide as the tile or wider (the VAE's 256- and 512-pixel levels): `rows` consecutive pixels of ONE row
    if (wo % rows || (fwd && cs != 1)) return kBoxWideRows;
    box[1] = cs * rows; box[2] = 1; box[3] = 1;
  } else if (hw >= rows) {
    if (rows % wo || hw % rows) return kBoxRowsPerTile;
    box[1] = cs * wo; box[2] = cs * (rows / wo); box[3] = 1;
  } else {
    if (rows % hw) return kBoxImagesPerTile;
    box[1] = cs * wo; box[2] = cs * ho; box[3] = rows / hw;
  }
  box[0] = 64;
  return box[1] <= 256 && box[2] <= 256 ? kBoxOk : kBoxTooLarge;
}

// launch heuristics (mdb_set_tuning)
static int g_pair_min_tiles = 128;  // smallest grid, in 128-row tile equivalents, that goes to the 256-wide tiles
static int g_bn80_below = 100;      // N % 160 == 0 layers with fewer 160-wide CTAs than this use 80-wide tiles
static int g_skinny_ctas = 96;      // long-K grids of at most half this many tiles split K up to this many CTAs (0: off)
static int g_split_min_chunks = 8;  // ... keeping at least this many K chunks per split
constexpr int kLongKChunks = 64;    // ... unless K >= 4096 (automatic split-K): then 160-wide tiles and split K

template <auto kern, int BN, int STAGES>
static int launch_kernel(const GemmKParams& kp, dim3 grid, cudaStream_t st) {
  const unsigned cluster_z = kp.cluster_reduce ? static_cast<unsigned>(kp.splits) : 1u;
  constexpr int kSmem = GemmSmem<BN, STAGES>::kTotal;
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
  if (int rc = set_max_dyn_smem<kern>(kSmem)) return rc;
  MDB_CHECK_CUDA(launch_pdl_cluster(kern, grid, dim3(kWsThreads), kSmem, st, cluster_z, kp));
  count_launch();
  return MDB_OK;
}
// IM2COL: the conv at any size (gemm_igemm_kernel, never with GEGLU), else gemm_tc_kernel
template <int BN, bool GEGLU, int STAGES, bool IM2COL>
static int launch_gemm(const GemmKParams& kp, dim3 grid, cudaStream_t st) {
  if constexpr (IM2COL) {
    static_assert(!GEGLU, "the im2col conv has no GEGLU epilogue");
    return launch_kernel<gemm_igemm_kernel<BN, STAGES>, BN, STAGES>(kp, grid, st);
  } else {
    return launch_kernel<gemm_tc_kernel<BN, GEGLU, STAGES>, BN, STAGES>(kp, grid, st);
  }
}

static int* gemm_tuning_slot(int key) {
  switch (key) {
    case MDB_TUNE_GEMM_PAIR_MIN_TILES: return &g_pair_min_tiles;
    case MDB_TUNE_GEMM_SKINNY_CTAS: return &g_skinny_ctas;
    case MDB_TUNE_GEMM_SPLIT_MIN_CHUNKS: return &g_split_min_chunks;
    default: return &g_bn80_below;
  }
}
int get_gemm_tuning(int key) { return *gemm_tuning_slot(key); }
void set_gemm_tuning(int key, int value) { *gemm_tuning_slot(key) = value; }

// tile width, split-K and kernel choice for a descriptor validated and A-mapped by the caller: the same rules for the
// GEMM, the box-path conv and (IM2COL) the conv at any size
template <bool IM2COL>
static int dispatch(const char* fn, const mdb_gemm_desc* g, GemmKParams& kp, bool geglu, cudaStream_t st) {
  int rc;
  // ---- which kernel ----
  // Large grids (>= g_pair_min_tiles 128-row tile equivalents, no split-K, at least two M tiles): 128 x 256 tiles
  // (N % 256 == 0) or 128 x 160 / 128 x 128 tiles with deep rings, one CTA per SM — widest first: fewest L2 -> SM
  // bytes per flop.
  const int m_tiles = (g->m + kBM - 1) / kBM;
  bool pair = g->splits <= 1 && m_tiles >= 2 && g->n % 8 == 0 && g->ln_u == nullptr;
  int bn = 0;
  if (pair) {
    if (geglu) bn = (g->n % 256 == 0) ? 256 : 0;
    else if (g->n % 256 == 0) bn = 256;
    else if (g->n % 160 == 0) bn = 160;
    else bn = 128;
    // ... and enough work per launch: only a large grid AND a K loop that is not a handful of chunks pays for the
    // single-CTA-per-SM tiles
    const long long eq = (long long)m_tiles * ((g->n + bn - 1) / (bn ? bn : 1));
    if (bn == 0 || eq < (long long)g_pair_min_tiles || eq * kp.k_chunks < 16ll * g_pair_min_tiles) pair = false;
  }
  if (pair) {
    // bn chosen above
  } else if (geglu) {
    MDB_REQUIRE(g->n % 128 == 0, "%s: GEGLU needs N %% 128 == 0 (N=%d)", fn, g->n);
    bn = 128;
  } else if (g->n % 160 == 0) {
    // 160-wide tiles unless that leaves most of the SMs idle; then (short K) halve the tile width, or (long K:
    // the weight-streaming 3x3 convs of the 8x8 ... 32x32 levels at one frame) keep the wide tile and split K —
    // see the automatic split-K below (scripts/gpu_microbench.py times the tile width x split-K choices).  Under the
    // skinny plan the narrow tile always comes first: it doubles the CTAs that stream distinct weight rows.
    const long long tiles160 = (long long)m_tiles * (g->n / 160) * (g->splits > 1 ? g->splits : 1);
    const bool skinny80 = g->splits == 0 && g_skinny_ctas > 0 && kp.k_chunks >= kLongKChunks && tiles160 * 4 <= g_skinny_ctas;
    const bool wide_split = g->splits == 0 && !skinny80 && kp.k_chunks >= kLongKChunks && tiles160 * 2 <= kNumSms;
    bn = (tiles160 < g_bn80_below && !wide_split) ? 80 : 160;
  } else {
    bn = 128;
  }
  rc = tmap_rows(&kp.tmB, g->b, g->k, g->n, g->ldb, kBK, bn);
  if (rc) return rc;

  int splits = g->splits > 1 ? g->splits : 1;
  if (g->ln_u != nullptr) splits = 1;  // the correction is applied by the CTA that holds the whole K range
  if (g->splits == 0 && !geglu && !pair && g->ln_u == nullptr) {
    const long long tiles = (long long)m_tiles * ((g->n + bn - 1) / bn);
    if (g_skinny_ctas > 0 && kp.k_chunks >= kLongKChunks && tiles * 2 <= g_skinny_ctas) {
      // skinny plan (the 3x3 convs and ff out of the deep levels of a one-frame step, M = 64 ... 512): too few flops
      // per weight byte to be compute-bound, so what counts is how many SMs stream the weights.  Split K into any
      // count up to 8 (one cluster, reduced through DSMEM) that keeps the grid within g_skinny_ctas CTAs and every
      // split at g_split_min_chunks or more.  On H100 (scripts/gpu_microbench.py skinny) 96 CTAs beat 128: clusters
      // of one-CTA-per-SM tiles do not all fit into the GPCs at once beyond that.  Short K (< 64 chunks) keeps the
      // plan below: there the fixed cost of a launch dominates and more splits only add reduction work.
      for (int c = 8; c >= 2; --c)
        if (tiles * c <= g_skinny_ctas && kp.k_chunks / c >= g_split_min_chunks) {
          splits = c;
          break;
        }
    } else if (tiles < 100) {
      // compute-bound plan: a power of two up to 8 that brings the grid to about one CTA per SM while every split
      // keeps at least 16 K chunks
      for (int c = 8; c >= 2; c >>= 1)
        if (tiles * c <= kNumSms && kp.k_chunks / c >= 16) {
          splits = c;
          break;
        }
    }
  }
  if (splits > kp.k_chunks) splits = kp.k_chunks;
  if (geglu || pair) splits = 1;
  kp.chunks_per_split = (kp.k_chunks + splits - 1) / splits;
  splits = (kp.k_chunks + kp.chunks_per_split - 1) / kp.chunks_per_split;  // no empty splits
  kp.splits = splits;
  kp.ws = g->splitk_ws;
  // 2 ... 8 splits (a portable cluster size): the partners form a thread-block cluster and reduce through DSMEM (one
  // kernel); more go through the global fp32 workspace + finalize kernel.
  kp.cluster_reduce = (!geglu && splits >= 2 && splits <= 8) ? 1 : 0;
  if (splits > 1 && !kp.cluster_reduce) {
    MDB_REQUIRE(g->splitk_ws != nullptr, "%s: splits > 1 needs splitk_ws", fn);
  }

  dim3 grid(m_tiles, (g->n + bn - 1) / bn, splits);
  const bool deep = (long long)grid.x * grid.y * grid.z <= kNumSms && kp.chunks_per_split >= 12;
  if constexpr (!IM2COL) {
    if (geglu) return pair ? launch_gemm<256, true, 4, false>(kp, grid, st) : launch_gemm<128, true, 3, false>(kp, grid, st);
  }
  if (pair) {
    if (bn == 256) rc = launch_gemm<256, false, 4, IM2COL>(kp, grid, st);
    else if (bn == 160) rc = launch_gemm<160, false, 6, IM2COL>(kp, grid, st);
    else rc = launch_gemm<128, false, 6, IM2COL>(kp, grid, st);
    return rc;
  }
  if (bn == 160) rc = deep ? launch_gemm<160, false, 6, IM2COL>(kp, grid, st) : launch_gemm<160, false, 3, IM2COL>(kp, grid, st);
  else if (bn == 80) rc = deep ? launch_gemm<80, false, 8, IM2COL>(kp, grid, st) : launch_gemm<80, false, 3, IM2COL>(kp, grid, st);
  else rc = deep ? launch_gemm<128, false, 6, IM2COL>(kp, grid, st) : launch_gemm<128, false, 3, IM2COL>(kp, grid, st);
  if (rc) return rc;
  if (splits > 1 && !kp.cluster_reduce) {
    const long long total = ((long long)g->m * g->n + 3) / 4;
    int blocks = (int)((total + 255) / 256);
    if (blocks > kNumSms * 8) blocks = kNumSms * 8;
    MDB_CHECK_CUDA(launch_pdl(splitk_finalize_kernel, dim3(blocks), dim3(256), 0, st, kp));
    count_launch();
  }
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

extern "C" int mdb_gemm_f16(const mdb_gemm_desc* g, mdb_stream_t stream) {
  MDB_REQUIRE(g != nullptr, "mdb_gemm_f16: null descriptor");
  MDB_REQUIRE(g->m > 0 && g->n > 0 && g->k > 0, "mdb_gemm_f16: bad shape m=%d n=%d k=%d", g->m, g->n, g->k);
  MDB_REQUIRE(g->k % kBK == 0, "mdb_gemm_f16: K=%d must be a multiple of 64", g->k);
  MDB_REQUIRE(g->a && g->b && g->d, "mdb_gemm_f16: null operand");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool geglu = g->epilogue == MDB_EPI_GEGLU;
  GemmKParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.d = static_cast<__half*>(g->d);
  kp.ldd = g->ldd;
  kp.bias = g->bias;
  kp.bias_batch_stride = g->bias_batch_stride;
  kp.rows_per_batch = g->rows_per_batch > 0 ? g->rows_per_batch : 1;
  kp.residual = static_cast<const __half*>(g->residual);
  kp.ldr = g->ldr;
  kp.m = g->m;
  kp.n = g->n;
  kp.k_chunks = g->k / kBK;
  kp.conv = g->conv;
  MDB_REQUIRE(g->ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(g->d) & 15) == 0,
              "mdb_gemm_f16: D must be 16B aligned with ldd %% 8 == 0 (ldd=%lld)", (long long)g->ldd);
  if (g->bias) {
    MDB_REQUIRE((reinterpret_cast<uintptr_t>(g->bias) & 15) == 0 && g->bias_batch_stride % 4 == 0,
                "mdb_gemm_f16: bias must be 16B aligned with bias_batch_stride %% 4 == 0");
  }
  if (g->residual) {
    MDB_REQUIRE(g->ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(g->residual) & 15) == 0,
                "mdb_gemm_f16: residual must be 16B aligned with ldr %% 8 == 0");
    MDB_REQUIRE(!geglu, "mdb_gemm_f16: residual is not supported with the GEGLU epilogue");
  }

  if (g->ln_u != nullptr) {
    MDB_REQUIRE(!geglu, "mdb_gemm_f16: LayerNorm fusion is not available with the GEGLU epilogue (N / 128 CTAs per row "
                        "block would each recompute the row statistics: measured slower than the LayerNorm kernel)");
    MDB_REQUIRE(!g->conv && g->a2 == nullptr && (reinterpret_cast<uintptr_t>(g->ln_u) & 15) == 0,
                "mdb_gemm_f16: LayerNorm fusion needs a plain single-source A whose K is the normalised width");
    kp.ln_u = g->ln_u;
    kp.ln_eps = g->ln_eps;
  }
  int rc;
  if (g->conv) {
    MDB_REQUIRE(g->a2 == nullptr, "mdb_gemm_f16: conv mode takes a single source");
    MDB_REQUIRE(g->c % kBK == 0 && g->k == 9 * g->c, "mdb_gemm_f16: conv needs c %% 64 == 0 and k == 9c (c=%d k=%d)",
                g->c, g->k);
    // conv == 1: stride 1; conv == 2: stride 2 (Downsample.op, openaimodel.py:175): the output pixel (y, x) reads input
    // (2y + kh - 1, 2x + kw - 1) — the same shifted boxes with TMA element strides of 2 along w and h, no im2col buffer
    const int cs = g->conv == 2 ? 2 : 1;
    const int ho = (g->h - 1) / cs + 1, wo = (g->w - 1) / cs + 1;
    MDB_REQUIRE(g->m == g->nb * ho * wo, "mdb_gemm_f16: conv m != nb*ho*wo");
    const int hw = ho * wo;  // OUTPUT pixels per image: tiles are cut over these
    uint32_t box[4];
    const int why = pixel_box(ho, wo, cs, kBM, true, box);
    MDB_REQUIRE(why != kBoxWideRows, "mdb_gemm_f16: conv rows wider than 128 pixels need 128 | w and stride 1 (w=%d)", g->w);
    MDB_REQUIRE(why != kBoxRowsPerTile, "mdb_gemm_f16: conv tile needs w | 128 and 128 | h*w (output h=%d w=%d)", ho, wo);
    MDB_REQUIRE(why != kBoxImagesPerTile, "mdb_gemm_f16: conv tile needs h*w | 128 (output h=%d w=%d)", ho, wo);
    MDB_REQUIRE(why != kBoxTooLarge, "mdb_gemm_f16: conv TMA box too large");
    rc = tmap_nhwc(&kp.tmA, g->a, g->c, g->w, g->h, g->nb, g->c, box, cs);
    if (rc) return rc;
    kp.chunks_per_tap = g->c / kBK;
    kp.w = wo;
    kp.hw = hw;
    kp.cs = cs;
    kp.k1_chunks = kp.k_chunks;
  } else {
    const int k1 = g->a2 ? g->k1 : g->k;
    MDB_REQUIRE(k1 % kBK == 0 && k1 > 0 && k1 <= g->k, "mdb_gemm_f16: k1=%d must be a multiple of 64 within K", k1);
    rc = tmap_rows(&kp.tmA, g->a, k1, g->m, g->lda, kBK, kBM);
    if (rc) return rc;
    if (g->a2) {
      rc = tmap_rows(&kp.tmA2, g->a2, g->k - k1, g->m, g->lda2, kBK, kBM);
      if (rc) return rc;
    }
    kp.k1_chunks = k1 / kBK;
  }

  return dispatch<false>("mdb_gemm_f16", g, kp, geglu, st);
}

extern "C" int mdb_conv3x3_igemm_f16(const mdb_gemm_desc* g, mdb_stream_t stream) {
  const char* fn = "mdb_conv3x3_igemm_f16";
  MDB_REQUIRE(g != nullptr, "%s: null descriptor", fn);
  MDB_REQUIRE(g->conv == 1 || g->conv == 2, "%s: conv must be the stride, 1 or 2 (got %d)", fn, g->conv);
  MDB_REQUIRE(g->a && g->b && g->d, "%s: null operand", fn);
  MDB_REQUIRE(g->nb > 0 && g->h > 0 && g->w > 0 && g->c > 0 && g->c % kBK == 0 && g->k == 9 * g->c,
              "%s: needs nb, h, w > 0, c %% 64 == 0 and k == 9c (nb=%d h=%d w=%d c=%d k=%d)", fn, g->nb, g->h, g->w, g->c,
              g->k);
  const int cs = g->conv;
  const int ho = (g->h - 1) / cs + 1, wo = (g->w - 1) / cs + 1;
  MDB_REQUIRE(g->m == g->nb * ho * wo && g->n > 0, "%s: m=%d must be nb*ho*wo=%d and n=%d > 0", fn, g->m,
              g->nb * ho * wo, g->n);
  MDB_REQUIRE(g->epilogue == MDB_EPI_NONE && g->ln_u == nullptr, "%s: no GEGLU epilogue or folded LayerNorm", fn);
  // two sources: channels [0, k1) of every pixel from a, [k1, c) from a2 (a fused torch.cat along channels)
  const int c1 = g->a2 ? g->k1 : g->c;
  MDB_REQUIRE(c1 > 0 && c1 % kBK == 0 && (g->a2 ? c1 < g->c : c1 == g->c),
              "%s: with a2, k1 (the channels taken from a) must be a multiple of 64 below c (k1=%d c=%d)", fn, c1, g->c);
  const long long lda = g->lda > 0 ? g->lda : c1, lda2 = g->lda2 > 0 ? g->lda2 : g->c - c1;
  MDB_REQUIRE(lda >= c1 && lda % 8 == 0 && (!g->a2 || (lda2 >= g->c - c1 && lda2 % 8 == 0)),
              "%s: the pixel strides lda / lda2 must cover their channels and be multiples of 8 (lda=%lld lda2=%lld)", fn,
              lda, lda2);
  MDB_REQUIRE(g->ldd >= g->n && g->ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(g->d) & 15) == 0,
              "%s: D must be 16B aligned with ldd %% 8 == 0 and ldd >= n (ldd=%lld)", fn, (long long)g->ldd);
  if (g->bias) {
    MDB_REQUIRE((reinterpret_cast<uintptr_t>(g->bias) & 15) == 0 && g->bias_batch_stride % 4 == 0,
                "%s: bias must be 16B aligned with bias_batch_stride %% 4 == 0", fn);
  }
  if (g->residual) {
    MDB_REQUIRE(g->ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(g->residual) & 15) == 0,
                "%s: residual must be 16B aligned with ldr %% 8 == 0", fn);
  }
  GemmKParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.d = static_cast<__half*>(g->d);
  kp.ldd = g->ldd;
  kp.bias = g->bias;
  kp.bias_batch_stride = g->bias_batch_stride;
  kp.rows_per_batch = g->rows_per_batch > 0 ? g->rows_per_batch : 1;
  kp.residual = static_cast<const __half*>(g->residual);
  kp.ldr = g->ldr;
  kp.m = g->m;
  kp.n = g->n;
  kp.k_chunks = g->k / kBK;
  kp.conv = 1;
  kp.chunks_per_tap = g->c / kBK;
  kp.k1_chunks = c1 / kBK;
  kp.w = wo;
  kp.hw = ho * wo;
  kp.cs = cs;
  int rc = tmap_nhwc_im2col(&kp.tmA, g->a, c1, g->w, g->h, g->nb, lda, kBM, cs);
  if (rc) return rc;
  if (g->a2 && (rc = tmap_nhwc_im2col(&kp.tmA2, g->a2, g->c - c1, g->w, g->h, g->nb, lda2, kBM, cs))) return rc;
  return dispatch<true>(fn, g, kp, false, static_cast<cudaStream_t>(stream));
}
