// GroupNorm(32) [+SiLU] and LayerNorm over channels-last fp16 activations (HBM/L2-bound kernels).
//
// GroupNorm32 / Normalize (util.py:252-254, attention.py:89-90): fp32 statistics, two eps values.  Both paths below
// are DETERMINISTIC (no atomics on data: fixed-order warp-shuffle / shared-memory / DSMEM reductions) and use
// PIVOT-SHIFTED sums: with K = x[b, pixel 0, first channel of the group] every partial accumulates
// S = sum(x - K), Q = sum((x - K)^2); mean = K + S/n, var = Q/n - (S/n)^2.  K is a sample of the data, so
// |mean - K| is of the order of the standard deviation and the subtraction loses a few bits at most — unlike
// E[x^2] - mean^2, which cancels catastrophically for activations whose mean is large against their spread.
//
//   gn_cluster_kernel   ONE launch (every layer but the 320-channel ones at more than two samples): a thread-block
//                       cluster per (batch element, group) splits the pixels, warp shuffles -> shared memory ->
//                       DSMEM exchange of (S, Q), second pass from L1/L2.
//   gn_stats_kernel     coalesced full-row reads, per-CTA (S, Q) partials to a workspace, the LAST CTA of a batch
//                       element (ticket) folds them in slot order -> (mean, var)
//   gn_apply_kernel     y = x * a_c + b_c [+ SiLU], 8 channels per thread.
// The input may be the channel concatenation of two tensors, which is how torch.cat([h, skip], 1) (cldm.py:104)
// disappears: the normalised copy is the only concatenated buffer.
#include "norm.cuh"

namespace mdb {

constexpr int kGnFinalThreads = 256;  // threads of the last CTA that fold the partials (4 slices x 64 entries)

// ws layout (floats): [kGnMaxBatch] tickets (uint, zero at first use, self-resetting; a FIXED region so that calls
//                     with different batch sizes can share one workspace) | [batch][64] final (mean, var) per group |
//                     [batch][gridDim.x][64] partials (S_0..S_31, Q_0..Q_31)
// rows_per_cta is chosen by the launcher so that ~2 waves of CTAs cover the tensor and every thread
// owns at most a handful of rows (loads of one thread are independent and unrolled).
__global__ void gn_stats_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2,
                                float* __restrict__ ws, int batch, int hw, int rows_per_cta) {
  extern __shared__ float sh[];  // [2][rstride][c] per-thread channel sums, reused as [4][64] by the final fold
  __shared__ int s_last;
  pdl_launch_dependents();
  const int c = c1 + c2;
  const int cg = c / 32;
  const int b = blockIdx.y;
  const int row0 = blockIdx.x * rows_per_cta;
  const int rows = min(rows_per_cta, hw - row0);
  const int vecs = c / 8;
  const int v = threadIdx.x % vecs;
  const int rphase = threadIdx.x / vecs;
  const int rstride = blockDim.x / vecs;
  unsigned* ticket = reinterpret_cast<unsigned*>(ws) + b;
  float* stats = ws + kGnMaxBatch + static_cast<long long>(b) * 64;
  float* pbase = ws + kGnMaxBatch + static_cast<long long>(batch) * 64;
  float* partial = pbase + (static_cast<long long>(b) * gridDim.x + blockIdx.x) * 64;
  pdl_wait();
  // this thread's 8 channels lie in at most two groups (cg >= 8, or cg == 4 where a vector is two whole groups)
  const int g_first = (v * 8) / cg;
  const float ka = gn_pivot(x1, c1, x2, c2, b, hw, g_first * cg);
  const float kb = (g_first + 1 < 32) ? gn_pivot(x1, c1, x2, c2, b, hw, (g_first + 1) * cg) : 0.f;
  float piv[8], s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    piv[i] = ((v * 8 + i) / cg == g_first) ? ka : kb;
    s[i] = q[i] = 0.f;
  }
#pragma unroll 4
  for (int r = rphase; r < rows; r += rstride) {
    const long long row = static_cast<long long>(b) * hw + row0 + r;
    uint4 u = *gn_src(x1, c1, x2, c2, row, v * 8);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = __half22float2(h2[e]);
      const float d0 = f.x - piv[2 * e], d1 = f.y - piv[2 * e + 1];
      s[2 * e] += d0; q[2 * e] = fmaf(d0, d0, q[2 * e]);
      s[2 * e + 1] += d1; q[2 * e + 1] = fmaf(d1, d1, q[2 * e + 1]);
    }
  }
  // per-thread channel sums -> shared memory, then thread (g, which) folds its group in a fixed order
  float* sh_s = sh;
  float* sh_q = sh + rstride * c;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sh_s[rphase * c + v * 8 + i] = s[i];
    sh_q[rphase * c + v * 8 + i] = q[i];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x & 31;
    const float* src = (threadIdx.x < 32) ? sh_s : sh_q;
    float acc = 0.f;
    for (int r = 0; r < rstride; ++r)
      for (int j = 0; j < cg; ++j) acc += src[r * c + g * cg + j];
    partial[threadIdx.x] = acc;
  }
  // ---- ticket: the last CTA of this batch element folds all partials in slot order ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pall = pbase + static_cast<long long>(b) * gridDim.x * 64;
  const int nblk = gridDim.x;
  if (threadIdx.x < kGnFinalThreads) {
    const int e = threadIdx.x & 63, sl = threadIdx.x >> 6;
    const int per = (nblk + 3) / 4;
    const int i0 = sl * per, i1 = min(nblk, i0 + per);
    float acc = 0.f;
    for (int i = i0; i < i1; ++i) acc += __ldcg(pall + static_cast<long long>(i) * 64 + e);
    sh[sl * 64 + e] = acc;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int g = threadIdx.x;
    const float S = ((sh[g] + sh[64 + g]) + sh[128 + g]) + sh[192 + g];
    const float Q = ((sh[32 + g] + sh[96 + g]) + sh[160 + g]) + sh[224 + g];
    const float inv_n = 1.0f / (static_cast<float>(cg) * hw);
    const float k = gn_pivot(x1, c1, x2, c2, b, hw, g * cg);
    const float ms = S * inv_n;
    stats[2 * g] = k + ms;
    stats[2 * g + 1] = fmaxf(fmaf(-ms, ms, Q * inv_n), 0.f);
  }
  if (threadIdx.x == 0) *ticket = 0u;  // self-resetting: the next call on this workspace starts from zero
}

// apply: every CTA first turns the 32 group statistics of its batch element into per-channel
// (scale, shift) pairs in shared memory — y = x * a_c + b_c with a_c = rstd_g * gamma_c and
// b_c = beta_c - mean_g * a_c — and then streams its rows with one FMA (+ SiLU) per element.
__global__ void gn_apply_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                const float* __restrict__ stats, __half* __restrict__ y, int hw, int rows_per_cta,
                                float eps, int silu) {
  extern __shared__ float s_ab[];  // [2][c]
  pdl_launch_dependents();
  const int c = c1 + c2;
  const int cg = c / 32;
  const int vecs = c / 8;
  const int b = blockIdx.y;
  // gamma / beta are constants: park them in shared memory before the PDL wait, combine with the statistics after
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    s_ab[ch] = gamma[ch];
    s_ab[c + ch] = beta[ch];
  }
  pdl_wait();
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {  // same thread owns the same channels: no sync needed
    const int g = ch / cg;
    const float mean = stats[(b * 32 + g) * 2];
    const float var = stats[(b * 32 + g) * 2 + 1];
    const float a = rsqrtf(var + eps) * s_ab[ch];
    s_ab[ch] = a;
    s_ab[c + ch] = s_ab[c + ch] - mean * a;
  }
  __syncthreads();
  const int row0 = blockIdx.x * rows_per_cta;
  const int rows = min(rows_per_cta, hw - row0);
  const int total = rows * vecs;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const int r = i / vecs;
    const int v = i - r * vecs;
    const long long row = static_cast<long long>(b) * hw + row0 + r;
    uint4 u = *gn_src(x1, c1, x2, c2, row, v * 8);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
    float f[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 t = __half22float2(h2[e]);
      f[2 * e] = t.x; f[2 * e + 1] = t.y;
    }
    const float4 a0 = *reinterpret_cast<const float4*>(&s_ab[v * 8]);
    const float4 a1 = *reinterpret_cast<const float4*>(&s_ab[v * 8 + 4]);
    const float4 b0 = *reinterpret_cast<const float4*>(&s_ab[c + v * 8]);
    const float4 b1 = *reinterpret_cast<const float4*>(&s_ab[c + v * 8 + 4]);
    f[0] = fmaf(f[0], a0.x, b0.x); f[1] = fmaf(f[1], a0.y, b0.y); f[2] = fmaf(f[2], a0.z, b0.z); f[3] = fmaf(f[3], a0.w, b0.w);
    f[4] = fmaf(f[4], a1.x, b1.x); f[5] = fmaf(f[5], a1.y, b1.y); f[6] = fmaf(f[6], a1.z, b1.z); f[7] = fmaf(f[7], a1.w, b1.w);
    if (silu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = silu_f(f[e]);
    }
    uint4 o4;
    o4.x = pack_half2(f[0], f[1]); o4.y = pack_half2(f[2], f[3]);
    o4.z = pack_half2(f[4], f[5]); o4.w = pack_half2(f[6], f[7]);
    *reinterpret_cast<uint4*>(y + row * c + v * 8) = o4;
  }
}

// ------------------------------------------------------------------------------------------------
// Single-launch GroupNorm for small batches.  At one frame a stats -> apply pair costs two dependent launches
// (~7 + ~9 us, 88 pairs per step) for tensors of 0.1 ... 8 MB.  Here one CLUSTER owns one (batch element, group):
// its CTAs split the pixels, each reads its hw/CS x cg slice twice (the second pass hits L1/L2), the partial
// (S, Q) pairs are exchanged through distributed shared memory — no atomics, no workspace, no second kernel.
// Thread layout: a group is cg = C/32 consecutive channels = cg/2 half2 words per pixel; thread t owns word
// t % (cg/2) of pixels t / (cg/2), + rows_per_iter, ... so a warp reads whole pixels' slices back to back and
// there is no division in the loops.
// ------------------------------------------------------------------------------------------------
constexpr int kGnFusedThreads = 512;

__global__ void __launch_bounds__(kGnFusedThreads) gn_cluster_kernel(const __half* __restrict__ x1, int c1,
                                                                      const __half* __restrict__ x2, int c2,
                                                                      const float* __restrict__ gamma,
                                                                      const float* __restrict__ beta, __half* __restrict__ y,
                                                                      int hw, float eps, int silu) {
  __shared__ float s_warp[2][kGnFusedThreads / 32];
  __shared__ __align__(8) float s_part[2];  // this CTA's (S, Q): read by the cluster partners
  pdl_launch_dependents();
  const int c = c1 + c2;
  const int cg = c / 32;
  const int wpp = cg >> 1;  // half2 words per pixel in one group
  const int g = blockIdx.x, b = blockIdx.y;
  const int cs = gridDim.z;          // cluster = (1, 1, cs): the CTAs that share this (batch element, group)
  const int part = blockIdx.z;
  const int tid = threadIdx.x;
  const int rows_per_iter = kGnFusedThreads / wpp;
  const int w = tid % wpp, r0 = tid / wpp;
  const bool active = r0 < rows_per_iter;
  const int ch = g * cg + 2 * w;  // this thread's channel pair (c1 is even: a pair never straddles the sources)
  const __half* src;
  long long pitch;
  if (ch < c1) { src = x1 + ch; pitch = c1; } else { src = x2 + (ch - c1); pitch = c2; }
  src += static_cast<long long>(b) * hw * pitch;
  __half* dst = y + static_cast<long long>(b) * hw * c + ch;
  // pixels [p_begin, p_end) belong to this CTA
  const int per = (hw + cs - 1) / cs;
  const int p_begin = part * per;
  const int p_end = min(hw, p_begin + per);
  const float ga0 = gamma[ch], ga1 = gamma[ch + 1], be0 = beta[ch], be1 = beta[ch + 1];  // constants: before the wait
  pdl_wait();
  const float piv = gn_pivot(x1, c1, x2, c2, b, hw, g * cg);  // the same value in every CTA of the cluster

  float s = 0.f, q = 0.f;
  if (active) {
#pragma unroll 8
    for (int pix = p_begin + r0; pix < p_end; pix += rows_per_iter) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(src + static_cast<long long>(pix) * pitch));
      const float d0 = f.x - piv, d1 = f.y - piv;
      s += d0 + d1;
      q = fmaf(d0, d0, fmaf(d1, d1, q));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((tid & 31) == 0) {
    s_warp[0][tid >> 5] = s;
    s_warp[1][tid >> 5] = q;
  }
  __syncthreads();
  if (tid < 32) {
    float ss = (tid < kGnFusedThreads / 32) ? s_warp[0][tid] : 0.f;
    float qq = (tid < kGnFusedThreads / 32) ? s_warp[1][tid] : 0.f;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      ss += __shfl_xor_sync(0xffffffffu, ss, o);
      qq += __shfl_xor_sync(0xffffffffu, qq, o);
    }
    if (tid == 0) {
      s_part[0] = ss;
      s_part[1] = qq;
    }
  }
  float tot_s, tot_q;
  if (cs > 1) {
    cluster_sync_all();  // every partner's partial is written (release) and visible (acquire)
    tot_s = tot_q = 0.f;
    const uint32_t a = smem_u32(&s_part[0]);
    for (int r = 0; r < cs; ++r) {  // same order in every CTA: identical statistics across the cluster
      const uint32_t ra = dsmem_map(a, static_cast<uint32_t>(r));
      float ps, pq;
      asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(ps), "=f"(pq) : "r"(ra));
      tot_s += ps;
      tot_q += pq;
    }
  } else {
    __syncthreads();
    tot_s = s_part[0];
    tot_q = s_part[1];
  }
  const float inv_n = 1.0f / (static_cast<float>(cg) * hw);
  const float ms = tot_s * inv_n;
  const float mean = piv + ms;
  const float var = fmaxf(fmaf(-ms, ms, tot_q * inv_n), 0.f);
  const float rstd = rsqrtf(var + eps);
  const float a0 = rstd * ga0, a1 = rstd * ga1;
  const float b0 = be0 - mean * a0, b1 = be1 - mean * a1;
  if (active) {
#pragma unroll 8
    for (int pix = p_begin + r0; pix < p_end; pix += rows_per_iter) {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(src + static_cast<long long>(pix) * pitch));
      float o0 = fmaf(f.x, a0, b0), o1 = fmaf(f.y, a1, b1);
      if (silu) {
        o0 = silu_f(o0);
        o1 = silu_f(o1);
      }
      *reinterpret_cast<__half2*>(dst + static_cast<long long>(pix) * c) = __floats2half2_rn(o0, o1);
    }
  }
  if (cs > 1) cluster_sync_all();  // nobody leaves while a partner may still read its shared memory
}

// LayerNorm: one warp per row, row cached in registers (c <= 1280 -> <= 40 values per lane)
template <int VPL>  // half2 pairs per lane
__global__ void layernorm_kernel(const __half* __restrict__ x, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, __half* __restrict__ y, long long rows, int c,
                                 float eps) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const __half2* xr = reinterpret_cast<const __half2*>(x + static_cast<long long>(warp) * c);
  float2 v[VPL];
  float mean, rstd;
  ln_row_stats<VPL>(xr, lane, c, eps, v, mean, rstd);
  __half2* yr = reinterpret_cast<__half2*>(y + static_cast<long long>(warp) * c);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int ch = (lane + i * 32) * 2;
    const float a = (v[i].x - mean) * rstd * gamma[ch] + beta[ch];
    const float bb = (v[i].y - mean) * rstd * gamma[ch + 1] + beta[ch + 1];
    yr[lane + i * 32] = __floats2half2_rn(a, bb);
  }
}

// rows per stats CTA / stats grid: ~296 CTAs (2 per SM) in total, whole multiples of the row-phase count,
// at most 8 rows per thread
void gn_stats_geometry(int c, int batch, int hw, int* threads_out, int* rows_per_cta_out, int* nblk_out) {
  const int vecs = c / 8;
  int threads = ((512 / vecs) * vecs);  // whole number of row phases
  if (threads < vecs) threads = vecs;
  const int rstride = threads / vecs;
  int per = (batch * hw + 295) / 296;
  int rows_per_cta = ((per + rstride - 1) / rstride) * rstride;
  if (rows_per_cta > 8 * rstride) rows_per_cta = 8 * rstride;
  if (rows_per_cta < rstride) rows_per_cta = rstride;
  *threads_out = threads;
  *rows_per_cta_out = rows_per_cta;
  *nblk_out = (hw + rows_per_cta - 1) / rows_per_cta;
}

int launch_gn_stats(const __half* x1, int c1, const __half* x2, int c2, float* ws, int batch, int hw,
                    cudaStream_t st) {
  const int c = c1 + c2;
  int threads, rows_per_cta, nblk;
  gn_stats_geometry(c, batch, hw, &threads, &rows_per_cta, &nblk);
  const int rstride = threads / (c / 8);
  size_t smem_stats = static_cast<size_t>(2) * rstride * c * sizeof(float);
  if (smem_stats < 256 * sizeof(float)) smem_stats = 256 * sizeof(float);
  MDB_REQUIRE(threads >= kGnFinalThreads && smem_stats <= 48 * 1024, "mdb_groupnorm_f16: unsupported width %d", c);
  MDB_REQUIRE(batch <= kGnMaxBatch, "mdb_groupnorm_f16: batch %d > %d", batch, kGnMaxBatch);
  MDB_CHECK_CUDA(launch_pdl(gn_stats_kernel, dim3(nblk, batch), dim3(threads), smem_stats, st, x1, c1, x2, c2, ws,
                            batch, hw, rows_per_cta));
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

// floats of workspace mdb_groupnorm_f16 needs for the two-kernel path (0 when the call takes the single-launch
// cluster path).  The workspace must be ZERO when first used (tickets); the kernels leave it reusable.
extern "C" int64_t mdb_groupnorm_ws_floats(int32_t c, int32_t batch, int32_t hw) {
  if (c <= 0 || batch <= 0 || hw <= 0 || c % 8 != 0) return 0;
  int threads, rows_per_cta, nblk;
  gn_stats_geometry(c, batch, hw, &threads, &rows_per_cta, &nblk);
  return kGnMaxBatch + static_cast<int64_t>(batch) * 64 + static_cast<int64_t>(batch) * nblk * 64;
}

// single-launch cluster path: needs even channels per group.  Automatic choice (scripts/gpu_microbench.py gn compares
// the two paths): the cluster kernel is taken once a group is >= 20 channels wide (>= 40 bytes per pixel: whole
// sectors); with 10-channel groups (the 320-channel layers of the 64x64 level) its 20-byte slivers waste half of every
// sector, so it is taken only while the launch count dominates (batch <= 2).
// mode: 0 = automatic, 1 = force the two-kernel path, 2 = force the cluster path (tests)
static bool gn_use_cluster(int c, int c1, int c2, int batch, int mode) {
  const bool ok = (c % 64 == 0) && (c1 % 2 == 0) && (c2 % 2 == 0) && (c / 64 <= kGnFusedThreads);
  if (mode == 1 || !ok) return false;
  if (mode == 2) return true;
  return (c / 32 >= 20) || batch <= 2;
}

extern "C" int mdb_groupnorm_f16(const void* x1, int32_t c1, const void* x2, int32_t c2, const float* gamma,
                                 const float* beta, void* y, float* ws, int32_t batch, int32_t hw, float eps,
                                 int32_t silu, int32_t mode, mdb_stream_t stream) {
  const int c = c1 + (x2 ? c2 : 0);
  if (!x2) c2 = 0;
  MDB_REQUIRE(x1 && y && gamma && beta, "mdb_groupnorm_f16: null pointer");
  MDB_REQUIRE(batch > 0 && hw > 0 && batch <= 65535, "mdb_groupnorm_f16: bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (gn_use_cluster(c, c1, c2, batch, mode)) {
    // cluster size: enough CTAs to cover the SMs about twice, at least ~64 pixels per CTA, at most 8 (portable)
    int cs = 1;
    while (cs < 8 && 32 * batch * cs * 2 <= 2 * kNumSms && hw / (cs * 2) >= 64) cs *= 2;
    MDB_CHECK_CUDA(launch_pdl_cluster(gn_cluster_kernel, dim3(32, batch, cs), dim3(kGnFusedThreads), 0, st,
                                      static_cast<unsigned>(cs), static_cast<const __half*>(x1), c1,
                                      static_cast<const __half*>(x2), c2, gamma, beta, static_cast<__half*>(y), hw, eps,
                                      silu));
    count_launch(1);
    return MDB_OK;
  }
  MDB_REQUIRE(ws != nullptr, "mdb_groupnorm_f16: the two-kernel path needs a workspace (mdb_groupnorm_ws_floats)");
  // a thread's 8-channel vector may straddle at most two groups: 8 or more channels per group, or exactly 4
  // (the first-stage VAE's 128-channel level), where every vector is exactly two whole groups
  MDB_REQUIRE(c % 32 == 0 && c1 % 8 == 0 && c2 % 8 == 0 && (c / 32 >= 8 || c / 32 == 4),
              "mdb_groupnorm_f16: channels must be multiples of 8, c %% 32 == 0 and c/32 >= 8 or == 4 (c1=%d c2=%d)", c1, c2);
  MDB_REQUIRE(c / 8 <= 512, "mdb_groupnorm_f16: too many channels (%d)", c);
  const int rc = launch_gn_stats(static_cast<const __half*>(x1), c1, static_cast<const __half*>(x2), c2, ws, batch, hw,
                                 st);
  if (rc) return rc;
  {
    // ~2-4 CTAs per SM; each CTA pays a c-element (scale, shift) setup, so rows per CTA grow with c
    int rows_apply = (batch * hw + 443) / 444;
    const int min_rows = (c >= 1280) ? 2 : 4;  // few rows per CTA when hw is small: parallelism beats setup reuse
    if (rows_apply < min_rows) rows_apply = min_rows;
    if (rows_apply > 64) rows_apply = 64;
    dim3 agrid((hw + rows_apply - 1) / rows_apply, batch);
    MDB_CHECK_CUDA(launch_pdl(gn_apply_kernel, agrid, dim3(256), 2 * c * sizeof(float), st,
                              static_cast<const __half*>(x1), c1, static_cast<const __half*>(x2), c2, gamma, beta,
                              static_cast<const float*>(ws + kGnMaxBatch), static_cast<__half*>(y), hw, rows_apply, eps,
                              silu));
  }
  count_launch(2);
  return MDB_OK;
}

extern "C" int mdb_layernorm_f16(const void* x, const float* gamma, const float* beta, void* y, int64_t rows,
                                 int32_t c, float eps, mdb_stream_t stream) {
  MDB_REQUIRE(x && y && gamma && beta, "mdb_layernorm_f16: null pointer");
  MDB_REQUIRE(c % 64 == 0 && c <= 1280, "mdb_layernorm_f16: c must be a multiple of 64 and <= 1280 (c=%d)", c);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int vpl = c / 64;
  const int threads = 256;
  const int blocks = static_cast<int>((rows * 32 + threads - 1) / threads);
  const __half* xp = static_cast<const __half*>(x);
  __half* yp = static_cast<__half*>(y);
#define MDB_LN_CASE(V)                                                                                       \
  case V:                                                                                                    \
    MDB_CHECK_CUDA(launch_pdl(layernorm_kernel<V>, dim3(blocks), dim3(threads), 0, st, xp, gamma, beta, yp,  \
                              static_cast<long long>(rows), c, eps));                                        \
    break;
  switch (vpl) {
    MDB_LN_CASE(5)
    MDB_LN_CASE(10)
    MDB_LN_CASE(20)
    default:
      set_error("mdb_layernorm_f16: unsupported width %d (320, 640, 1280)", c);
      return MDB_ERR_UNSUPPORTED;
  }
#undef MDB_LN_CASE
  count_launch();
  return MDB_OK;
}
