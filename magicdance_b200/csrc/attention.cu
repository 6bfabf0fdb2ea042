// Fused attention for sm_90a: softmax([Q K0^T | Q K1^T] * scale) [V0 ; V1], FlashAttention-style
// online softmax, both GEMMs on wgmma with register accumulators, operands fed by TMA.
//
// The two key/value sources are the layer's own tokens (source 0) and the appearance bank
// (source 1): the reference concatenates them with torch.cat before to_k/to_v
// (ldm/modules/attention.py:303-307); here the tile loop simply walks source 0's tiles and then
// source 1's, so no concatenated K/V buffer ever exists.
//
// One CTA = 128 queries x 1 head x 1 batch element.  Warp roles:
//   warp 8     TMA producer: Q once; K tile [BKV][d] and V^T tile [d][BKV] per step, STAGES-deep ring.
//              Head slices are cut out of the [tokens][heads*d] activations by a 3-D tensor map
//              (d, heads, tokens) whose innermost extent is d, so the 64-wide box is zero-filled
//              beyond d — that is the K-dim padding 40->48 / 80->80 / 160->192 for free.  V^T is read
//              through a (key, sample, channel) map whose key extent is the source's n: the keys past n
//              of a ragged last tile arrive as zeros.  P = 0 masks them, and 0 * NaN would not.
//   warps 0-7  two warpgroups of 64 query rows each.  Per key tile: S = Q K^T (wgmma, M=64, N=BKV, both
//              operands in shared memory) into registers; running max / sum in the log2 domain over the
//              four threads that share a row; P = exp2(S - max) is rounded to fp16 IN REGISTERS, in exactly
//              the fragment layout the register-A form of wgmma takes, and O += P V^T (N = d rounded up to
//              16) accumulates in registers.  O / l -> fp16 at the end.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

namespace mdb {

constexpr int kBQ = 128;

template <int D, int BKV, int STAGES>
struct AttnCfg {
  static constexpr int kDkChunks = (D + 63) / 64;
  static constexpr int kDV = (D + 15) / 16 * 16;  // PV N and number of QK K-steps * 16
  static constexpr int kKSteps = kDV / 16;
  static constexpr int kQBytes = kDkChunks * kBQ * 128;
  static constexpr int kKBytes = kDkChunks * BKV * 128;
  static constexpr int kVBytes = kDV * 128;         // one 64-key chunk of V^T: [kDV rows][64 keys]
  static constexpr int kStageBytes = kKBytes + kVBytes;
  static constexpr int kSmem = kQBytes + STAGES * kStageBytes + 1024;
  static_assert(BKV == 64, "one 128-byte swizzle row of keys per V^T tile");
  static_assert(kVBytes % 1024 == 0 && kKBytes % 1024 == 0, "stage tiles start on swizzle-atom boundaries");
};

struct AttnKParams {
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1;
  __half* out;
  long long ldo;
  int nq, n0, n1;
  int kv0_batches, kv1_batches;
  int bank_batches;
  float scale_log2;
};
// the forward that also stores the softmax statistics for the backward (attention_bwd.cu)
struct AttnLseKParams : AttnKParams {
  float* lse;  // fp32 [batch][heads][nq]: natural-log log-sum-exp of the row's scaled scores
};

// MINB = 2 caps the registers so that two CTAs (four MMA warpgroups) share an SM.  LSE: also store the row
// log-sum-exp (then the parameters are an AttnLseKParams); without it the kernel is exactly the inference one.
template <int D, int BKV, int STAGES, int MINB, bool LSE = false>
__global__ void __launch_bounds__(kWsThreads, MINB)
    attn_wg_kernel(const __grid_constant__ std::conditional_t<LSE, AttnLseKParams, AttnKParams> p) {
  using C = AttnCfg<D, BKV, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t q_bar;
  __shared__ __align__(8) uint64_t kv_full[STAGES], kv_empty[STAGES];

  uint8_t* sQ = align1024(smem_raw);
  uint8_t* sKV = sQ + C::kQBytes;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kBQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int t0 = (p.n0 + BKV - 1) / BKV;
  const int t1 = (b < p.bank_batches && p.n1 > 0) ? (p.n1 + BKV - 1) / BKV : 0;
  const int n_tiles = t0 + t1;

  pdl_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&p.tmQ);
    tma_prefetch_desc(&p.tmK0);
    tma_prefetch_desc(&p.tmV0);
    mbar_init(&q_bar, 1);
    ring_init<STAGES>(kv_full, kv_empty, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      mbar_expect_tx(&q_bar, C::kQBytes);
      for (int dc = 0; dc < C::kDkChunks; ++dc)
        tma_load_3d(sQ + dc * (kBQ * 128), &p.tmQ, &q_bar, dc * 64, head, b * p.nq + q0);
      for (int j = 0; j < n_tiles; ++j) {
        const bool src1 = j >= t0;
        const int key0 = (src1 ? (j - t0) : j) * BKV;
        const CUtensorMap* tk = src1 ? &p.tmK1 : &p.tmK0;
        const CUtensorMap* tv = src1 ? &p.tmV1 : &p.tmV0;
        const int nsrc = src1 ? p.n1 : p.n0;
        const int kvb = src1 ? (p.kv1_batches > 1 ? b : 0) : (p.kv0_batches > 1 ? b : 0);
        const int s = ring_acquire<STAGES>(kv_empty, j);
        mbar_expect_tx(&kv_full[s], C::kStageBytes);
        uint8_t* sk = sKV + s * C::kStageBytes;
        uint8_t* sv = sk + C::kKBytes;
        for (int dc = 0; dc < C::kDkChunks; ++dc)
          tma_load_3d(sk + dc * (BKV * 128), tk, &kv_full[s], dc * 64, head, kvb * nsrc + key0);
        tma_load_3d(sv, tv, &kv_full[s], key0, kvb, head * D);
      }
    }
  } else {
    // ---------------- warpgroups 0, 1: S, softmax, O ----------------
    const int wg = warp >> 2;
    const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);  // this warpgroup's 64 query rows of each Q chunk
    const int cq = 2 * (lane & 3);                           // this thread's first column inside an 8-column block
    float o[C::kDV / 2];
#pragma unroll
    for (int i = 0; i < C::kDV / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY};  // rows r and r + 8 of this thread, log2 domain
    float l_run[2] = {0.f, 0.f};              // this thread's share of the row sums
    mbar_wait(&q_bar, 0);

    for (int j = 0; j < n_tiles; ++j) {
      const bool src1 = j >= t0;
      const int key0 = (src1 ? (j - t0) : j) * BKV;
      const int valid = min(BKV, (src1 ? p.n1 : p.n0) - key0);
      const int s = ring_wait_full<STAGES>(kv_full, j);
      const uint32_t k_addr = smem_u32(sKV + s * C::kStageBytes);
      const uint32_t v_addr = k_addr + C::kKBytes;

      float sc[BKV / 2];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < C::kKSteps; ++ks) {
        const int dc = ks >> 2, kk = ks & 3;
        const uint64_t da = wgmma_desc_k_sw128(q_addr + dc * (kBQ * 128)) + 2 * kk;
        const uint64_t db = wgmma_desc_k_sw128(k_addr + dc * (BKV * 128)) + 2 * kk;
        wgmma_ss<BKV>(sc, da, db, ks != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);

      // sc[i]: row r + 8 ((i >> 1) & 1), key 8 (i >> 2) + cq + (i & 1)
      if (valid < BKV) {
#pragma unroll
        for (int i = 0; i < BKV / 2; ++i)
          if (8 * (i >> 2) + cq + (i & 1) >= valid) sc[i] = -INFINITY;
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < BKV / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
      float alpha[2], neg_m[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        const float m_new = fmaxf(m_run[h], mx[h] * p.scale_log2);  // a tile holds at least one valid key
        alpha[h] = ex2_approx(m_run[h] - m_new);                   // m_run = -inf on the first tile -> 0
        m_run[h] = m_new;
        neg_m[h] = -m_new;
      }
      float ls[2] = {0.f, 0.f};
      uint32_t pa[BKV / 16][4];
#pragma unroll
      for (int i = 0; i < BKV / 2; i += 2) {
        const int h = (i >> 1) & 1;
        const float e0 = ex2_approx(fmaf(sc[i], p.scale_log2, neg_m[h]));      // masked keys: exp2(-inf) = 0
        const float e1 = ex2_approx(fmaf(sc[i + 1], p.scale_log2, neg_m[h]));
        ls[h] += e0 + e1;
        pa[i >> 3][(i >> 1) & 3] = pack_half2(e0, e1);  // m16n8k16 A fragment of key slice i / 8
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l_run[h] = fmaf(l_run[h], alpha[h], ls[h]);
#pragma unroll
      for (int i = 0; i < C::kDV / 2; ++i) o[i] *= alpha[(i >> 1) & 1];

      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk)
        wgmma_rs<C::kDV>(o, pa[kk], wgmma_desc_k_sw128(v_addr) + 2 * kk, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      mbar_arrive(&kv_empty[s]);  // this thread's reads of stage s (through its warpgroup's MMAs) are done
    }

    float inv_l[2], l_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv_l[h] = 1.0f / l;
      l_row[h] = l;
    }
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    if constexpr (LSE) {
      // log-sum-exp of the scaled scores: m and l are in the log2 domain, the stored value in the natural one
      if ((lane & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int q = q0 + r + 8 * h;
          if (q < p.nq)
            p.lse[(static_cast<long long>(b) * gridDim.y + head) * p.nq + q] =
                (m_run[h] + log2f(l_row[h])) * 0.6931471805599453f;
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + r + 8 * h;
      if (q < p.nq) {
        __half* op = p.out + (static_cast<long long>(b) * p.nq + q) * p.ldo + head * D + cq;
#pragma unroll
        for (int c8 = 0; c8 < D / 8; ++c8)
          *reinterpret_cast<uint32_t*>(op + 8 * c8) =
              pack_half2(o[4 * c8 + 2 * h] * inv_l[h], o[4 * c8 + 2 * h + 1] * inv_l[h]);
      }
    }
  }
}

// d = 40: grids of at least this many 128-row CTAs take the register-capped variant, which runs two CTAs (four MMA
// warpgroups) per SM; smaller grids keep the uncapped one-CTA-per-SM variant with a deeper ring.  (At d = 80 the
// capped variant spills: one CTA per SM.)  `scripts/gpu_microbench.py attn` compares the two at self + bank attention
// of 4096 queries: on an H100 80GB HBM3 (400 W power limit) the capped variant took 335 us against 448 us at 512 CTAs
// (one frame's cond | uncond batch) and 2.68 ms against 3.68 ms at 4096 (eight frames); grids below 512 CTAs were
// not measured and keep the uncapped variant.
// mdb_set_tuning(MDB_TUNE_ATTN40_2Q_MIN_CTAS).
static int g_attn40_2q_min_ctas = 512;
int get_attn_tuning() { return g_attn40_2q_min_ctas; }
void set_attn_tuning(int v) { g_attn40_2q_min_ctas = v; }

template <int D, int BKV, int STAGES, int MINB, bool LSE = false, typename P>
static int launch_attn(const P& kp, dim3 grid, cudaStream_t st) {
  using C = AttnCfg<D, BKV, STAGES>;
  static_assert(MINB == 1 || C::kSmem <= 113 * 1024, "two CTAs per SM must fit");
  constexpr auto kern = attn_wg_kernel<D, BKV, STAGES, MINB, LSE>;
  if (int rc = set_max_dyn_smem<kern>(C::kSmem)) return rc;
  MDB_CHECK_CUDA(launch_pdl(kern, grid, dim3(kWsThreads), C::kSmem, st, kp));
  count_launch();
  return MDB_OK;
}

// lse != nullptr: the LSE-storing variants, with the same variant choice (and so the same `out`) as without
template <int D, int BKV>
static int build_and_launch(const mdb_attn_desc* a, float* lse, cudaStream_t st) {
  constexpr int kDV = AttnCfg<D, BKV, 1>::kDV;
  AttnKParams kp;
  memset(&kp, 0, sizeof(kp));
  const int hd = a->heads * a->d;
  int rc;
  if ((rc = tmap_heads(&kp.tmQ, a->q, a->d, a->heads, (uint64_t)a->batch * a->nq, a->ldq, kBQ))) return rc;
  auto mk_kv = [&](const void* k, long long ldk, const void* vt, long long ldvt, int n, int nb, int ldvb,
                   CUtensorMap* tk, CUtensorMap* tv) -> int {
    int r = tmap_heads(tk, k, a->d, a->heads, (uint64_t)nb * n, ldk, BKV);
    if (r) return r;
    // kDV rows from row head * d: rows past d (d = 40 -> 48) are the next head's or zero-filled, and only feed
    // output columns >= d, which are never stored
    return tmap_vt(tv, vt, n, nb, ldvb, hd, ldvt, kDV);
  };
  if ((rc = mk_kv(a->k0, a->ldk0, a->vt0, a->ldvt0, a->n0, a->kv0_batches, a->ldv0_batch, &kp.tmK0, &kp.tmV0))) return rc;
  if (a->n1 > 0) {
    if ((rc = mk_kv(a->k1, a->ldk1, a->vt1, a->ldvt1, a->n1, a->kv1_batches, a->ldv1_batch, &kp.tmK1, &kp.tmV1)))
      return rc;
  }
  kp.out = static_cast<__half*>(a->out);
  kp.ldo = a->ldo;
  kp.nq = a->nq;
  kp.n0 = a->n0;
  kp.n1 = a->n1;
  kp.kv0_batches = a->kv0_batches;
  kp.kv1_batches = a->kv1_batches;
  kp.bank_batches = a->n1 > 0 ? a->bank_batches : 0;
  kp.scale_log2 = a->scale * 1.4426950408889634f;
  dim3 grid((a->nq + kBQ - 1) / kBQ, a->heads, a->batch);
  if (lse != nullptr) {
    AttnLseKParams lp;
    memset(&lp, 0, sizeof(lp));
    static_cast<AttnKParams&>(lp) = kp;
    lp.lse = lse;
    if constexpr (D == 40) {
      const long long ctas = (long long)grid.x * grid.y * grid.z;
      if (ctas >= (long long)g_attn40_2q_min_ctas) return launch_attn<D, BKV, 3, 2, true>(lp, grid, st);
    }
    return launch_attn<D, BKV, (D == 160 ? 2 : 4), 1, true>(lp, grid, st);
  }
  if constexpr (D == 40) {
    const long long ctas = (long long)grid.x * grid.y * grid.z;
    if (ctas >= (long long)g_attn40_2q_min_ctas) return launch_attn<D, BKV, 3, 2>(kp, grid, st);
  }
  return launch_attn<D, BKV, (D == 160 ? 2 : 4), 1>(kp, grid, st);
}

static int attention_entry(const mdb_attn_desc* a, float* lse, cudaStream_t st) {
  switch (a->d) {
    case 40:
      return build_and_launch<40, 64>(a, lse, st);
    case 80:
      return build_and_launch<80, 64>(a, lse, st);
    case 160:
      return build_and_launch<160, 64>(a, lse, st);
    default:
      set_error("mdb_attention_f16: head dim %d not supported (40, 80, 160)", a->d);
      return MDB_ERR_UNSUPPORTED;
  }
}

// the forward's operand checks, shared by mdb_attention_f16, mdb_attention_lse_f16 and mdb_attention_bwd_f16
int attention_check_desc(const mdb_attn_desc* a) {
  MDB_REQUIRE(a != nullptr, "mdb_attention_f16: null descriptor");
  MDB_REQUIRE(a->q && a->k0 && a->vt0 && a->out, "mdb_attention_f16: null operand");
  MDB_REQUIRE(a->batch > 0 && a->heads > 0 && a->nq > 0 && a->n0 > 0 && a->n1 >= 0,
              "mdb_attention_f16: bad shape");
  MDB_REQUIRE(a->n1 == 0 || (a->k1 && a->vt1), "mdb_attention_f16: n1 > 0 needs k1/vt1");
  MDB_REQUIRE(a->kv0_batches == 1 || a->kv0_batches == a->batch, "mdb_attention_f16: kv0_batches must be 1 or batch");
  MDB_REQUIRE(a->n1 == 0 || a->kv1_batches == 1 || a->kv1_batches >= a->bank_batches,
              "mdb_attention_f16: kv1_batches must be 1 or cover bank_batches");
  MDB_REQUIRE(a->ldv0_batch >= a->n0 && a->ldv0_batch % 8 == 0, "mdb_attention_f16: ldv0_batch must be >= n0 and %% 8");
  MDB_REQUIRE(a->n1 == 0 || (a->ldv1_batch >= a->n1 && a->ldv1_batch % 8 == 0),
              "mdb_attention_f16: ldv1_batch must be >= n1 and %% 8");
  MDB_REQUIRE(a->ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0, "mdb_attention_f16: out alignment");
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

extern "C" int mdb_attention_f16(const mdb_attn_desc* a, mdb_stream_t stream) {
  const int rc = attention_check_desc(a);
  if (rc) return rc;
  return attention_entry(a, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int mdb_attention_lse_f16(const mdb_attn_desc* a, float* lse, mdb_stream_t stream) {
  const int rc = attention_check_desc(a);
  if (rc) return rc;
  MDB_REQUIRE(lse != nullptr, "mdb_attention_lse_f16: null lse");
  return attention_entry(a, lse, static_cast<cudaStream_t>(stream));
}
