// Backward of the two-source attention of attention.cu, for sm_90a:
//   out = softmax([Q K0^T | Q K1^T] * scale) [V0 ; V1]   ->   dQ, dK0, dV0, dK1, dV1 from dOut.
// FlashAttention-2's recompute scheme: the forward stores only the row log-sum-exp (mdb_attention_lse_f16); here
//   P = exp(S - LSE),  D = rowsum(dO o O),  dP = dO V^T,  dS = P o (dP - D),
//   dV = P^T dO,  dQ = scale dS K,  dK = scale dS^T Q.
// Like the forward, both kernels walk source 0's key tiles and then source 1's (the appearance bank, only for batch
// elements b < bank_batches): no concatenated K/V buffer exists.
//
// Deterministic, no atomics: every gradient element is owned by exactly one CTA, which accumulates it in a fixed order.
//   attn_bwd_dq_kernel    one CTA per (128 queries, head, batch element): D for its rows (also written to the
//                         workspace), then dQ over all key tiles of both sources.
//   attn_bwd_dkdv_kernel  one CTA per (128 keys of one source, head, batch element): dK and dV over that batch
//                         element's query tiles; it reads D from the workspace, so it runs after the dQ kernel.
// Shared sources (kv*_batches == 1 with batch > 1) would need a reduction across batch elements and are rejected.
//
// Warp roles as in the forward: warp 8 is the TMA producer, warps 0-7 are two warpgroups of 64 rows each (queries in
// the dQ kernel, keys in the dK/dV kernel).  Every product is a wgmma with fp32 register accumulators; P and dS are
// rounded to fp16 in registers in the register-A fragment layout.  Products that reduce over tokens read dO, Q and K
// MN-major (wgmma trans = 1) straight from the same 128-byte-swizzled TMA tiles, and dP = dO V^T reads V from its
// transposed V^T tile MN-major, so no operand is ever transposed in memory.
//
// d = 160 is the register-pressure case: the dK/dV kernel then runs twice, once for dV and once for dK, so that
// each pass holds one 64 x 160 accumulator per warpgroup (no instantiation spills).
#include "common.cuh"

namespace mdb {

int attention_check_desc(const mdb_attn_desc* a);

constexpr int kBwdRows = 128;  // queries per dQ CTA, keys per dK/dV CTA
constexpr int kBwdStep = 64;   // keys per dQ step, queries per dK/dV step: one 128-byte swizzle row of V^T
constexpr float kLog2e = 1.4426950408889634f;

template <int D>
struct BwdCfg {
  static constexpr int kDkChunks = (D + 63) / 64;       // 64-column chunks of a [rows][d] tile (zero-filled past d)
  static constexpr int kDV = (D + 15) / 16 * 16;        // N of the d-wide products, K-steps * 16 of the d-reductions
  static constexpr int kKSteps = kDV / 16;
  static constexpr int kChunk64 = kBwdStep * 128;       // one 64-column chunk of a 64-row tile
  static constexpr int kChunk128 = kBwdRows * 128;      // ... of a 128-row tile
  static constexpr int kTile64 = kDkChunks * kChunk64;  // [64][d] K-major tile
  static constexpr int kTile128 = kDkChunks * kChunk128;
  static constexpr int kVtBytes = kDV * 128;            // V^T tile [kDV channels][64 keys]
  static constexpr int kStages = D == 160 ? 2 : 4;
  // dQ kernel: Q and dO once, then a ring of (K tile, V^T tile)
  static constexpr int kDqStage = kTile64 + kVtBytes;
  static constexpr int kDqSmem = 2 * kTile128 + kStages * kDqStage + 1024;
  // dK/dV kernel: K and V^T of the CTA's 128 keys once, then a ring of (Q tile, dO tile)
  static constexpr int kKvStage = 2 * kTile64;
  static constexpr int kKvSmem = kTile128 + 2 * kVtBytes + kStages * kKvStage + 1024;
  static_assert(kVtBytes % 1024 == 0 && kTile64 % 1024 == 0, "tiles start on swizzle-atom boundaries");
  static_assert(kDqSmem <= 227 * 1024 && kKvSmem <= 227 * 1024, "shared memory");
};

struct AttnBwdKParams {
  CUtensorMap tmQ, tmDO, tmK0, tmV0, tmK1, tmV1;  // [64 rows] x [64 columns] boxes; V^T: [kDV rows] x [64 keys]
  const __half* out;
  const __half* dout;
  long long ldo, lddo;
  const float* lse;  // [batch][heads][nq], natural log
  float* dsum;       // D, [batch][heads][nq]
  __half* dq;
  long long lddq;
  __half* dk[2];
  long long lddk[2];
  __half* dvt[2];
  long long lddvt[2];
  int nq, n[2], ldv_batch[2];
  int bank_batches;
  float scale, scale_log2;
};

// ------------------------------------------------------------------------------------------------------------------
// dQ (and D): one CTA per 128 queries x head x batch element
// ------------------------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kWsThreads, 1) attn_bwd_dq_kernel(const __grid_constant__ AttnBwdKParams p) {
  using C = BwdCfg<D>;
  constexpr int STAGES = C::kStages;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_bar;
  __shared__ __align__(8) uint64_t kv_full[STAGES], kv_empty[STAGES];

  uint8_t* sQ = align1024(smem_raw);
  uint8_t* sDO = sQ + C::kTile128;
  uint8_t* sKV = sDO + C::kTile128;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kBwdRows;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int t0 = (p.n[0] + kBwdStep - 1) / kBwdStep;
  const int t1 = (b < p.bank_batches && p.n[1] > 0) ? (p.n[1] + kBwdStep - 1) / kBwdStep : 0;
  const int n_tiles = t0 + t1;

  pdl_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    mbar_init(&q_bar, 1);
    ring_init<STAGES>(kv_full, kv_empty, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_expect_tx(&q_bar, 2 * C::kTile128);
      for (int dc = 0; dc < C::kDkChunks; ++dc)
        for (int half = 0; half < 2; ++half) {
          const int row = b * p.nq + q0 + half * kBwdStep;
          tma_load_3d(sQ + dc * C::kChunk128 + half * C::kChunk64, &p.tmQ, &q_bar, dc * 64, head, row);
          tma_load_3d(sDO + dc * C::kChunk128 + half * C::kChunk64, &p.tmDO, &q_bar, dc * 64, head, row);
        }
      for (int j = 0; j < n_tiles; ++j) {
        const int src = j >= t0 ? 1 : 0;
        const int key0 = (src ? j - t0 : j) * kBwdStep;
        const int s = ring_acquire<STAGES>(kv_empty, j);
        mbar_expect_tx(&kv_full[s], C::kDqStage);
        uint8_t* sk = sKV + s * C::kDqStage;
        for (int dc = 0; dc < C::kDkChunks; ++dc)
          tma_load_4d(sk + dc * C::kChunk64, src ? &p.tmK1 : &p.tmK0, &kv_full[s], dc * 64, head, key0, b);
        tma_load_3d(sk + C::kTile64, src ? &p.tmV1 : &p.tmV0, &kv_full[s], key0, b, head * D);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int cq = 2 * (lane & 3);
  const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows r and r + 8 of the CTA's 128
  const long long stat0 = (static_cast<long long>(b) * gridDim.y + head) * p.nq;

  // row statistics: LSE (log2 domain) and D = rowsum(dO o O) over the four threads that share a row
  float lse2[2], dsum[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + r + 8 * h;
    float acc = 0.f;
    lse2[h] = INFINITY;  // rows past nq: P = exp2(-inf) = 0
    if (q < p.nq) {
      lse2[h] = p.lse[stat0 + q] * kLog2e;
      const __half* op = p.out + (static_cast<long long>(b) * p.nq + q) * p.ldo + head * D + cq;
      const __half* gp = p.dout + (static_cast<long long>(b) * p.nq + q) * p.lddo + head * D + cq;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8) {
        const float2 o = __half22float2(*reinterpret_cast<const __half2*>(op + 8 * c8));
        const float2 g = __half22float2(*reinterpret_cast<const __half2*>(gp + 8 * c8));
        acc = fmaf(o.x, g.x, acc);
        acc = fmaf(o.y, g.y, acc);
      }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    dsum[h] = acc;
    if (q < p.nq && (lane & 3) == 0) p.dsum[stat0 + q] = acc;
  }

  const uint32_t q_addr = smem_u32(sQ) + wg * C::kChunk64;  // this warpgroup's 64 rows of each 128-row chunk
  const uint32_t do_addr = smem_u32(sDO) + wg * C::kChunk64;
  const uint32_t kv_base = smem_u32(sKV);
  float dq[C::kDV / 2];
#pragma unroll
  for (int i = 0; i < C::kDV / 2; ++i) dq[i] = 0.f;
  mbar_wait(&q_bar, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int src = j >= t0 ? 1 : 0;
    const int valid = min(kBwdStep, p.n[src] - (src ? j - t0 : j) * kBwdStep);
    const int s = ring_wait_full<STAGES>(kv_full, j);
    const uint32_t k_addr = kv_base + s * C::kDqStage;
    const uint32_t vt_addr = k_addr + C::kTile64;

    // S = Q K^T and dP = dO V^T (V^T tile read MN-major), one commit group
    float sc[kBwdStep / 2], dp[kBwdStep / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < C::kKSteps; ++ks) {
      const int dc = ks >> 2, kk = ks & 3;
      wgmma_ss<kBwdStep>(sc, wgmma_desc_k_sw128(q_addr + dc * C::kChunk128) + 2 * kk,
                         wgmma_desc_k_sw128(k_addr + dc * C::kChunk64) + 2 * kk, ks != 0 ? 1u : 0u);
    }
#pragma unroll
    for (int ks = 0; ks < C::kKSteps; ++ks) {
      const int dc = ks >> 2, kk = ks & 3;
      wgmma_ss<kBwdStep, 0, 1>(dp, wgmma_desc_k_sw128(do_addr + dc * C::kChunk128) + 2 * kk,
                               wgmma_desc_mn_sw128(vt_addr + ks * 2048, 0), ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    wgmma_fence_regs(dp);

    // sc[i], dp[i]: row r + 8 ((i >> 1) & 1), key 8 (i >> 2) + cq + (i & 1); keys past the source's end get P = 0
    uint32_t ds[kBwdStep / 16][4];
#pragma unroll
    for (int i = 0; i < kBwdStep / 2; i += 2) {
      const int h = (i >> 1) & 1;
      const int key = 8 * (i >> 2) + cq;
      const float p0 = key < valid ? ex2_approx(fmaf(sc[i], p.scale_log2, -lse2[h])) : 0.f;
      const float p1 = key + 1 < valid ? ex2_approx(fmaf(sc[i + 1], p.scale_log2, -lse2[h])) : 0.f;
      ds[i >> 3][(i >> 1) & 3] = pack_half2(p0 * (dp[i] - dsum[h]), p1 * (dp[i + 1] - dsum[h]));
    }

    // dQ += dS K: K tile read MN-major (N = channels, 64-channel chunks kChunk64 apart)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBwdStep / 16; ++kk)
      wgmma_rs<C::kDV, 1>(dq, ds[kk], wgmma_desc_mn_sw128(k_addr + kk * 2048, C::kChunk64), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(dq);
    mbar_arrive(&kv_empty[s]);
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + r + 8 * h;
    if (q < p.nq) {
      __half* dst = p.dq + (static_cast<long long>(b) * p.nq + q) * p.lddq + head * D + cq;
#pragma unroll
      for (int c8 = 0; c8 < D / 8; ++c8)
        *reinterpret_cast<uint32_t*>(dst + 8 * c8) =
            pack_half2(dq[4 * c8 + 2 * h] * p.scale, dq[4 * c8 + 2 * h + 1] * p.scale);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// dK / dV: one CTA per 128 keys of one source x head x batch element.  MODE bit 0: dV, bit 1: dK.
// ------------------------------------------------------------------------------------------------------------------
template <int D, int MODE>
__global__ void __launch_bounds__(kWsThreads, 1) attn_bwd_dkdv_kernel(const __grid_constant__ AttnBwdKParams p) {
  using C = BwdCfg<D>;
  constexpr int STAGES = C::kStages;
  constexpr bool kDV_ = (MODE & 1) != 0, kDK = (MODE & 2) != 0;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t kv_bar;
  __shared__ __align__(8) uint64_t q_full[STAGES], q_empty[STAGES];
  __shared__ float s_lse2[STAGES][kBwdStep], s_dsum[STAGES][kBwdStep];

  uint8_t* sK = align1024(smem_raw);
  uint8_t* sVt = sK + C::kTile128;
  uint8_t* sQD = sVt + 2 * C::kVtBytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int t0 = (p.n[0] + kBwdRows - 1) / kBwdRows;
  const int src = static_cast<int>(blockIdx.x) >= t0 ? 1 : 0;
  if (src == 1 && b >= p.bank_batches) return;  // no bank for this batch element: nothing reads these keys
  const int key0 = (src ? blockIdx.x - t0 : blockIdx.x) * kBwdRows;
  const int nsrc = p.n[src];
  const int n_qt = (p.nq + kBwdStep - 1) / kBwdStep;
  const long long stat0 = (static_cast<long long>(b) * gridDim.y + head) * p.nq;

  pdl_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    mbar_init(&kv_bar, 1);
    ring_init<STAGES>(q_full, q_empty, 32);  // every producer lane arrives on q_full after writing its LSE / D entries
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_expect_tx(&kv_bar, C::kTile128 + (kDK ? 2 * C::kVtBytes : 0));
      for (int dc = 0; dc < C::kDkChunks; ++dc)
        for (int half = 0; half < 2; ++half)
          tma_load_4d(sK + dc * C::kChunk128 + half * C::kChunk64, src ? &p.tmK1 : &p.tmK0, &kv_bar, dc * 64, head,
                      key0 + half * kBwdStep, b);
      if (kDK)
        for (int half = 0; half < 2; ++half)
          tma_load_3d(sVt + half * C::kVtBytes, src ? &p.tmV1 : &p.tmV0, &kv_bar, key0 + half * kBwdStep, b,
                      head * D);
    }
    for (int j = 0; j < n_qt; ++j) {
      const int s = ring_acquire<STAGES>(q_empty, j);
      for (int c = lane; c < kBwdStep; c += 32) {
        const int q = j * kBwdStep + c;
        s_lse2[s][c] = q < p.nq ? p.lse[stat0 + q] * kLog2e : INFINITY;  // queries past nq: P = 0
        s_dsum[s][c] = q < p.nq ? p.dsum[stat0 + q] : 0.f;
      }
      if (lane == 0) {
        mbar_expect_tx(&q_full[s], C::kKvStage);
        uint8_t* sq = sQD + s * C::kKvStage;
        for (int dc = 0; dc < C::kDkChunks; ++dc) {
          tma_load_3d(sq + dc * C::kChunk64, &p.tmQ, &q_full[s], dc * 64, head, b * p.nq + j * kBwdStep);
          tma_load_3d(sq + C::kTile64 + dc * C::kChunk64, &p.tmDO, &q_full[s], dc * 64, head, b * p.nq + j * kBwdStep);
        }
      } else {
        mbar_arrive(&q_full[s]);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int cq = 2 * (lane & 3);
  const uint32_t k_base = smem_u32(sK) + wg * C::kChunk64;  // this warpgroup's 64 keys of each 128-row chunk
  const uint32_t vt_base = smem_u32(sVt) + wg * C::kVtBytes;
  const uint32_t qd_base = smem_u32(sQD);
  float dv[kDV_ ? C::kDV / 2 : 1], dk[kDK ? C::kDV / 2 : 1];
#pragma unroll
  for (int i = 0; i < (kDV_ ? C::kDV / 2 : 1); ++i) dv[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (kDK ? C::kDV / 2 : 1); ++i) dk[i] = 0.f;
  mbar_wait(&kv_bar, 0);

  for (int j = 0; j < n_qt; ++j) {
    const int s = ring_wait_full<STAGES>(q_full, j);
    const uint32_t q_addr = qd_base + s * C::kKvStage;
    // opaque per step: otherwise the loop-invariant K and V^T descriptors of every K step are hoisted out of the
    // loop and held in registers, which spills the d = 160 dK pass
    uint32_t k_addr = k_base, vt_addr = vt_base;
    asm volatile("" : "+r"(k_addr), "+r"(vt_addr));
    const uint32_t do_addr = q_addr + C::kTile64;

    // S^T = K Q^T; P^T is rounded to fp16 at once, so that S^T and dP^T are never live together (the accumulators
    // of the 288-thread CTA have 168 registers per thread)
    float st[kBwdStep / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < C::kKSteps; ++ks) {
      const int dc = ks >> 2, kk = ks & 3;
      wgmma_ss<kBwdStep>(st, wgmma_desc_k_sw128(k_addr + dc * C::kChunk128) + 2 * kk,
                         wgmma_desc_k_sw128(q_addr + dc * C::kChunk64) + 2 * kk, ks != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(st);

    // st[i]: key row r + 8 ((i >> 1) & 1), query column 8 (i >> 2) + cq + (i & 1)
    uint32_t pa[kBwdStep / 16][4];
#pragma unroll
    for (int i = 0; i < kBwdStep / 2; i += 2) {
      const int c = 8 * (i >> 2) + cq;
      pa[i >> 3][(i >> 1) & 3] = pack_half2(ex2_approx(fmaf(st[i], p.scale_log2, -s_lse2[s][c])),
                                            ex2_approx(fmaf(st[i + 1], p.scale_log2, -s_lse2[s][c + 1])));
    }

    // dV += P^T dO (dO tile read MN-major, N = channels)
    if constexpr (kDV_) {
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBwdStep / 16; ++kk)
        wgmma_rs<C::kDV, 1>(dv, pa[kk], wgmma_desc_mn_sw128(do_addr + kk * 2048, C::kChunk64), 1u);
      wgmma_commit();
    }

    if constexpr (kDK) {
      // dP^T = V dO^T (V read MN-major from its V^T tile)
      float dpt[kBwdStep / 2];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < C::kKSteps; ++ks) {
        const int dc = ks >> 2, kk = ks & 3;
        wgmma_ss<kBwdStep, 1, 0>(dpt, wgmma_desc_mn_sw128(vt_addr + ks * 2048, 0),
                                 wgmma_desc_k_sw128(do_addr + dc * C::kChunk64) + 2 * kk, ks != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dpt);
      // dS^T = P^T o (dP^T - D), in place of P^T (the dV product has completed)
#pragma unroll
      for (int i = 0; i < kBwdStep / 2; i += 2) {
        const int c = 8 * (i >> 2) + cq;
        uint32_t& frag = pa[i >> 3][(i >> 1) & 3];
        const float2 pp = __half22float2(*reinterpret_cast<const __half2*>(&frag));
        frag = pack_half2(pp.x * (dpt[i] - s_dsum[s][c]), pp.y * (dpt[i + 1] - s_dsum[s][c + 1]));
      }
      // dK += dS^T Q (Q tile read MN-major)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBwdStep / 16; ++kk)
        wgmma_rs<C::kDV, 1>(dk, pa[kk], wgmma_desc_mn_sw128(q_addr + kk * 2048, C::kChunk64), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(dk);
    } else {
      wgmma_wait<0>();
    }
    if constexpr (kDV_) wgmma_fence_regs(dv);
    mbar_arrive(&q_empty[s]);
  }

  const int rk = (warp & 3) * 16 + (lane >> 2);  // this thread's key rows rk and rk + 8 of the warpgroup's 64
  if constexpr (kDV_) {
    // dV^T[channel][key]: the accumulator's row is the key, so the store is transposed (once per CTA)
    __half* dvt = p.dvt[src] + static_cast<long long>(head) * D * p.lddvt[src] + b * p.ldv_batch[src];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = key0 + wg * 64 + rk + 8 * h;
      if (key < nsrc) {
#pragma unroll
        for (int i = 2 * h; i < D / 2; i += 4) {
          const int c = 8 * (i >> 2) + cq;
          dvt[static_cast<long long>(c) * p.lddvt[src] + key] = __float2half_rn(dv[i]);
          dvt[static_cast<long long>(c + 1) * p.lddvt[src] + key] = __float2half_rn(dv[i + 1]);
        }
      }
    }
  }
  if constexpr (kDK) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int key = key0 + wg * 64 + rk + 8 * h;
      if (key < nsrc) {
        __half* dst = p.dk[src] + (static_cast<long long>(b) * nsrc + key) * p.lddk[src] + head * D + cq;
#pragma unroll
        for (int c8 = 0; c8 < D / 8; ++c8)
          *reinterpret_cast<uint32_t*>(dst + 8 * c8) =
              pack_half2(dk[4 * c8 + 2 * h] * p.scale, dk[4 * c8 + 2 * h + 1] * p.scale);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------
template <int D>
static int bwd_launch(const mdb_attn_bwd_desc* a, cudaStream_t st) {
  using C = BwdCfg<D>;
  const mdb_attn_desc* f = &a->fwd;
  AttnBwdKParams kp;
  memset(&kp, 0, sizeof(kp));
  const int hd = f->heads * D;
  int rc;
  // the forward's head slices (attention.cu), 64 tokens per box
  auto mk_rows = [&](CUtensorMap* m, const void* base, long long ld, long long rows) -> int {
    return tmap_heads(m, base, D, f->heads, rows, ld, kBwdStep);
  };
  // K per sample: keys past n are zero-filled rather than the next sample's rows.  dQ = dS K reduces over keys, and
  // dS = 0 there does not cancel a NaN or Inf in bank rows of samples >= bank_batches, which are never read
  auto mk_k = [&](CUtensorMap* m, const void* base, long long ld, int n, int nb) -> int {
    return tmap_heads_per_sample(m, base, D, f->heads, n, nb, ld, kBwdStep);
  };
  // kDV rows from row head * d: rows past d (d = 40 -> 48) are the next head's or zero-filled; they meet only the
  // zero-filled channels d..47 of the dO tile.  Keys past n are zero-filled (tmap_vt): dS = P (dP - D) is 0 there
  // only if dP is finite
  auto mk_vt = [&](CUtensorMap* m, const void* base, long long ld, int n, int nb, int ldvb) -> int {
    return tmap_vt(m, base, n, nb, ldvb, hd, ld, C::kDV);
  };
  if ((rc = mk_rows(&kp.tmQ, f->q, f->ldq, (long long)f->batch * f->nq))) return rc;
  if ((rc = mk_rows(&kp.tmDO, a->dout, a->lddout, (long long)f->batch * f->nq))) return rc;
  if ((rc = mk_k(&kp.tmK0, f->k0, f->ldk0, f->n0, f->kv0_batches))) return rc;
  if ((rc = mk_vt(&kp.tmV0, f->vt0, f->ldvt0, f->n0, f->kv0_batches, f->ldv0_batch))) return rc;
  const bool bank = f->n1 > 0 && f->bank_batches > 0;
  if (bank) {
    if ((rc = mk_k(&kp.tmK1, f->k1, f->ldk1, f->n1, f->kv1_batches))) return rc;
    if ((rc = mk_vt(&kp.tmV1, f->vt1, f->ldvt1, f->n1, f->kv1_batches, f->ldv1_batch))) return rc;
  }
  kp.out = static_cast<const __half*>(f->out);
  kp.ldo = f->ldo;
  kp.dout = static_cast<const __half*>(a->dout);
  kp.lddo = a->lddout;
  kp.lse = a->lse;
  kp.dsum = a->ws;
  kp.dq = static_cast<__half*>(a->dq);
  kp.lddq = a->lddq;
  kp.dk[0] = static_cast<__half*>(a->dk0);
  kp.lddk[0] = a->lddk0;
  kp.dvt[0] = static_cast<__half*>(a->dvt0);
  kp.lddvt[0] = a->lddvt0;
  kp.dk[1] = static_cast<__half*>(a->dk1);
  kp.lddk[1] = a->lddk1;
  kp.dvt[1] = static_cast<__half*>(a->dvt1);
  kp.lddvt[1] = a->lddvt1;
  kp.nq = f->nq;
  kp.n[0] = f->n0;
  kp.n[1] = bank ? f->n1 : 0;
  kp.ldv_batch[0] = f->ldv0_batch;
  kp.ldv_batch[1] = f->ldv1_batch;
  kp.bank_batches = bank ? f->bank_batches : 0;
  kp.scale = f->scale;
  kp.scale_log2 = f->scale * kLog2e;

  if ((rc = set_max_dyn_smem<attn_bwd_dq_kernel<D>>(C::kDqSmem))) return rc;
  const dim3 gq((f->nq + kBwdRows - 1) / kBwdRows, f->heads, f->batch);
  MDB_CHECK_CUDA(launch_pdl(attn_bwd_dq_kernel<D>, gq, dim3(kWsThreads), C::kDqSmem, st, kp));
  count_launch();

  const int tiles = (f->n0 + kBwdRows - 1) / kBwdRows + (bank ? (f->n1 + kBwdRows - 1) / kBwdRows : 0);
  const dim3 gk(tiles, f->heads, f->batch);
  if constexpr (D == 160) {  // one 64 x 160 accumulator per warpgroup per pass: dV, then dK
    if ((rc = set_max_dyn_smem<attn_bwd_dkdv_kernel<D, 1>>(C::kKvSmem))) return rc;
    if ((rc = set_max_dyn_smem<attn_bwd_dkdv_kernel<D, 2>>(C::kKvSmem))) return rc;
    MDB_CHECK_CUDA(launch_pdl(attn_bwd_dkdv_kernel<D, 1>, gk, dim3(kWsThreads), C::kKvSmem, st, kp));
    MDB_CHECK_CUDA(launch_pdl(attn_bwd_dkdv_kernel<D, 2>, gk, dim3(kWsThreads), C::kKvSmem, st, kp));
    count_launch(2);
  } else {
    if ((rc = set_max_dyn_smem<attn_bwd_dkdv_kernel<D, 3>>(C::kKvSmem))) return rc;
    MDB_CHECK_CUDA(launch_pdl(attn_bwd_dkdv_kernel<D, 3>, gk, dim3(kWsThreads), C::kKvSmem, st, kp));
    count_launch();
  }
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

extern "C" int64_t mdb_attention_bwd_ws_floats(int32_t batch, int32_t heads, int32_t nq) {
  if (batch <= 0 || heads <= 0 || nq <= 0) return 0;
  return static_cast<int64_t>(batch) * heads * nq;
}

extern "C" int mdb_attention_bwd_f16(const mdb_attn_bwd_desc* a, mdb_stream_t stream) {
  MDB_REQUIRE(a != nullptr, "mdb_attention_bwd_f16: null descriptor");
  const int rc = attention_check_desc(&a->fwd);
  if (rc) return rc;
  const mdb_attn_desc* f = &a->fwd;
  MDB_REQUIRE(f->batch == 1 || f->kv0_batches == f->batch,
              "mdb_attention_bwd_f16: shared source 0 (kv0_batches == 1 with batch %d) is not supported: its gradient "
              "would need a reduction across batch elements", f->batch);
  MDB_REQUIRE(f->n1 == 0 || f->bank_batches == 0 || f->batch == 1 || f->kv1_batches > 1,
              "mdb_attention_bwd_f16: shared source 1 (kv1_batches == 1 with batch %d) is not supported: its gradient "
              "would need a reduction across batch elements", f->batch);
  MDB_REQUIRE(a->dout && a->lse && a->dq && a->dk0 && a->dvt0 && a->ws, "mdb_attention_bwd_f16: null operand");
  MDB_REQUIRE(f->n1 == 0 || f->bank_batches == 0 || (a->dk1 && a->dvt1), "mdb_attention_bwd_f16: n1 > 0 needs dk1/dvt1");
  MDB_REQUIRE(a->lddout % 8 == 0 && (reinterpret_cast<uintptr_t>(a->dout) & 15) == 0,
              "mdb_attention_bwd_f16: dout alignment");
  MDB_REQUIRE(a->lddq % 2 == 0 && a->lddk0 % 2 == 0 && a->lddk1 % 2 == 0 &&
                  (reinterpret_cast<uintptr_t>(a->dq) & 3) == 0 && (reinterpret_cast<uintptr_t>(a->dk0) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->dk1) & 3) == 0,
              "mdb_attention_bwd_f16: dq / dk rows must be 4-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (f->d) {
    case 40:
      return bwd_launch<40>(a, st);
    case 80:
      return bwd_launch<80>(a, st);
    case 160:
      return bwd_launch<160>(a, st);
    default:
      set_error("mdb_attention_bwd_f16: head dim %d not supported (40, 80, 160)", f->d);
      return MDB_ERR_UNSUPPORTED;
  }
}
