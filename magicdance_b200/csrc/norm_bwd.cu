// Backward of GroupNorm(32) [+SiLU] and LayerNorm (norm.cu), and the GEGLU activation in the projection's own row
// order, over channels-last fp16 activations (HBM/L2-bound kernels).
//
// GroupNorm, per (batch element b, group g) with n = (c/32) hw, xhat = (x - mean) rstd, z = gamma xhat + beta,
// dz = dy silu'(z) (or dy):
//   gn_stats_kernel (norm.cu)  the forward's pivot-shifted statistics, recomputed into the workspace
//   gn_bwd_reduce_kernel       per CTA of rows: A_bc = sum dz, B_bc = sum dz xhat over its rows -> fp32 slabs
//   colsum_finalize_kernel     (gemm_bwd.cu) the slabs summed in CTA order -> A, B [2][batch][c]; dbeta / dgamma are
//                              the same kernel over the batch elements, in batch order
//   gn_bwd_apply_kernel        the per-group sums S_A = sum_{c in g} gamma_c A_bc, S_B likewise, in its prologue, then
//                              dx = a_c dz - rstd (S_A + xhat S_B) / n with a_c = rstd gamma_c
// Both data passes use gn_stats_kernel's thread layout: thread t owns the 8-channel vector t % (c/8) of rows
// t / (c/8), + rstride, ...; its 8 channels lie in at most two groups (groups are >= 10 channels wide).
// LayerNorm: one warp per row with the row in registers, statistics by the forward's code (ln_row_stats); the
// per-warp column partials of dgamma / dbeta stay in registers and are folded in warp order in shared memory into
// one fp32 slab per CTA, which colsum_finalize_kernel sums in CTA order.
// Deterministic throughout: fixed-order reductions, no atomics on data (the statistics kernel's ticket only).
#include "norm.cuh"

namespace mdb {

constexpr int kGnBwdThreads = 512;  // bound of gn_stats_geometry's block size, which both passes use
constexpr int kLnBwdWarps = 8;      // rows of one LayerNorm CTA in flight

// the per-channel constants of channels [ch0, ch0 + 8) of batch element b: the group's mean and rstd, and the
// forward's scale and shift (z = x a + s, as gn_apply_kernel computes them)
struct GnChan {
  float mean[8], rstd[8], a[8], s[8];
};

__device__ __forceinline__ void gn_chan(const float* stats, const float* gamma, const float* beta, int b, int ch0,
                                        int cg, float eps, GnChan& k) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (ch0 + i) / cg;
    const float mean = stats[(b * 32 + g) * 2];
    const float var = stats[(b * 32 + g) * 2 + 1];
    const float a = rsqrtf(var + eps) * gamma[ch0 + i];
    k.mean[i] = mean;
    k.rstd[i] = rsqrtf(var + eps);
    k.a[i] = a;
    k.s[i] = beta[ch0 + i] - mean * a;
  }
}

// one 8-channel vector of a row: x, dy -> xhat, dz
__device__ __forceinline__ void gn_load8(const __half* x1, int c1, const __half* x2, int c2, const __half* dy,
                                         long long row, int ch0, const GnChan& k, int silu, float (&xh)[8],
                                         float (&dz)[8]) {
  const uint4 u = *gn_src(x1, c1, x2, c2, row, ch0);
  const uint4 du = *reinterpret_cast<const uint4*>(dy + row * (c1 + c2) + ch0);
  const __half2* x2h = reinterpret_cast<const __half2*>(&u);
  const __half2* d2h = reinterpret_cast<const __half2*>(&du);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 xf = __half22float2(x2h[e]);
    const float2 df = __half22float2(d2h[e]);
    const float xv[2] = {xf.x, xf.y}, dv[2] = {df.x, df.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int i = 2 * e + j;
      xh[i] = (xv[j] - k.mean[i]) * k.rstd[i];
      dz[i] = silu ? dv[j] * dsilu(fmaf(xv[j], k.a[i], k.s[i])) : dv[j];
    }
  }
}

// A and B partial sums of rows [blockIdx.x * rows_per_cta, ...) of batch element blockIdx.y -> slabs
// part[2][batch][gridDim.x][c]
__global__ void __launch_bounds__(kGnBwdThreads) gn_bwd_reduce_kernel(
    const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2, const __half* __restrict__ dy,
    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
    float* __restrict__ part, int hw, int rows_per_cta, float eps, int silu) {
  extern __shared__ float sh[];  // [2][rstride][c] per-thread channel sums
  pdl_launch_dependents();
  const int c = c1 + c2;
  const int cg = c / 32;
  const int vecs = c / 8;
  const int b = blockIdx.y;
  const int row0 = blockIdx.x * rows_per_cta;
  const int rows = min(rows_per_cta, hw - row0);
  const int v = threadIdx.x % vecs;
  const int rphase = threadIdx.x / vecs;
  const int rstride = blockDim.x / vecs;
  pdl_wait();
  GnChan k;
  gn_chan(stats, gamma, beta, b, v * 8, cg, eps, k);
  float sa[8], sb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sa[i] = sb[i] = 0.f;
#pragma unroll 2
  for (int r = rphase; r < rows; r += rstride) {
    float xh[8], dz[8];
    gn_load8(x1, c1, x2, c2, dy, static_cast<long long>(b) * hw + row0 + r, v * 8, k, silu, xh, dz);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      sa[i] += dz[i];
      sb[i] = fmaf(dz[i], xh[i], sb[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sh[rphase * c + v * 8 + i] = sa[i];
    sh[(rstride + rphase) * c + v * 8 + i] = sb[i];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 2 * c; e += blockDim.x) {  // each entry sums its row phases in order
    const int which = e / c, ch = e - which * c;
    float acc = 0.f;
    for (int r = 0; r < rstride; ++r) acc += sh[(which * rstride + r) * c + ch];
    part[((static_cast<long long>(which) * gridDim.y + b) * gridDim.x + blockIdx.x) * c + ch] = acc;
  }
}

// dx of rows [blockIdx.x * rows_per_cta, ...) of batch element blockIdx.y from ab = [A | B] as [2][batch][c]
__global__ void __launch_bounds__(kGnBwdThreads) gn_bwd_apply_kernel(
    const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2, const __half* __restrict__ dy,
    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
    const float* __restrict__ ab, GbOut dx1, GbOut dx2, int hw, int rows_per_cta, float eps, int silu) {
  __shared__ float s_grp[64];  // per group: S_A / n, then S_B / n
  pdl_launch_dependents();
  const int c = c1 + c2;
  const int cg = c / 32;
  const int vecs = c / 8;
  const int b = blockIdx.y;
  const int row0 = blockIdx.x * rows_per_cta;
  const int rows = min(rows_per_cta, hw - row0);
  const int v = threadIdx.x % vecs;
  const int rphase = threadIdx.x / vecs;
  const int rstride = blockDim.x / vecs;
  pdl_wait();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x & 31, which = threadIdx.x >> 5;
    const float* src = ab + (static_cast<long long>(which) * gridDim.y + b) * c + g * cg;
    float acc = 0.f;
    for (int j = 0; j < cg; ++j) acc = fmaf(gamma[g * cg + j], src[j], acc);
    s_grp[threadIdx.x] = acc / (static_cast<float>(cg) * hw);
  }
  __syncthreads();
  GnChan k;
  gn_chan(stats, gamma, beta, b, v * 8, cg, eps, k);
  float p[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int g = (v * 8 + i) / cg;
    p[i] = k.rstd[i] * s_grp[g];
    q[i] = k.rstd[i] * s_grp[32 + g];
  }
  const bool first = v * 8 < c1;  // c1 % 8 == 0: a vector never straddles the two sources
  const GbOut o = first ? dx1 : dx2;
  const int col0 = first ? v * 8 : v * 8 - c1;
#pragma unroll 2
  for (int r = rphase; r < rows; r += rstride) {
    const long long row = static_cast<long long>(b) * hw + row0 + r;
    float xh[8], dz[8];
    gn_load8(x1, c1, x2, c2, dy, row, v * 8, k, silu, xh, dz);
#pragma unroll
    for (int e = 0; e < 4; ++e)
      gb_store2(o, row, col0 + 2 * e, fmaf(k.a[2 * e], dz[2 * e], -fmaf(q[2 * e], xh[2 * e], p[2 * e])),
                fmaf(k.a[2 * e + 1], dz[2 * e + 1], -fmaf(q[2 * e + 1], xh[2 * e + 1], p[2 * e + 1])));
  }
}

// LayerNorm backward: warp w of CTA blk takes rows [(blk * kLnBwdWarps + w) * rows_per_warp, ... + rows_per_warp).
// params != 0: the CTA's dgamma / dbeta column partials -> part[2][gridDim.x][c]
template <int VPL>  // half2 pairs per lane
__global__ void __launch_bounds__(kLnBwdWarps * 32) layernorm_bwd_kernel(
    const __half* __restrict__ x, const float* __restrict__ gamma, const __half* __restrict__ dy, GbOut dx,
    float* __restrict__ part, long long rows, int c, float eps, int rows_per_warp, int params) {
  __shared__ float s_par[2][VPL * 64];
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long r0 = (static_cast<long long>(blockIdx.x) * kLnBwdWarps + warp) * rows_per_warp;
  float pg[2 * VPL], pb[2 * VPL];
#pragma unroll
  for (int i = 0; i < 2 * VPL; ++i) pg[i] = pb[i] = 0.f;
  for (int rr = 0; rr < rows_per_warp; ++rr) {
    const long long row = r0 + rr;
    if (row >= rows) break;
    float2 v[VPL];  // x, then xhat
    float mean, rstd;
    ln_row_stats<VPL>(reinterpret_cast<const __half2*>(x + row * c), lane, c, eps, v, mean, rstd);
    const __half2* dr = reinterpret_cast<const __half2*>(dy + row * c);
    float2 g[VPL];  // dxhat = dy gamma
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int ch = (lane + i * 32) * 2;
      const float2 d = __half22float2(dr[lane + i * 32]);
      v[i].x = (v[i].x - mean) * rstd;
      v[i].y = (v[i].y - mean) * rstd;
      if (params) {
        pg[2 * i] = fmaf(d.x, v[i].x, pg[2 * i]);
        pg[2 * i + 1] = fmaf(d.y, v[i].y, pg[2 * i + 1]);
        pb[2 * i] += d.x;
        pb[2 * i + 1] += d.y;
      }
      g[i].x = d.x * gamma[ch];
      g[i].y = d.y * gamma[ch + 1];
      s1 += g[i].x + g[i].y;
      s2 = fmaf(g[i].x, v[i].x, fmaf(g[i].y, v[i].y, s2));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 / c, m2 = s2 / c;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
      gb_store2(dx, row, (lane + i * 32) * 2, rstd * (g[i].x - m1 - v[i].x * m2), rstd * (g[i].y - m1 - v[i].y * m2));
  }
  if (!params) return;
  for (int w = 0; w < kLnBwdWarps; ++w) {  // the warps' partials, added in warp order
    if (warp == w) {
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int ch = (lane + i * 32) * 2;
        s_par[0][ch] = (w ? s_par[0][ch] : 0.f) + pg[2 * i];
        s_par[0][ch + 1] = (w ? s_par[0][ch + 1] : 0.f) + pg[2 * i + 1];
        s_par[1][ch] = (w ? s_par[1][ch] : 0.f) + pb[2 * i];
        s_par[1][ch + 1] = (w ? s_par[1][ch + 1] : 0.f) + pb[2 * i + 1];
      }
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < 2 * c; e += blockDim.x) {
    const int which = e / c, ch = e - which * c;
    part[(static_cast<long long>(which) * gridDim.x + blockIdx.x) * c + ch] = s_par[which][ch];
  }
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(h2[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_half2(f[0], f[1]);
  o.y = pack_half2(f[2], f[3]);
  o.z = pack_half2(f[4], f[5]);
  o.w = pack_half2(f[6], f[7]);
  return o;
}

// GEGLU forward: out[r][j] = h[r][j] * gelu_erf(h[r][n + j]), 8 columns per thread
__global__ void geglu_kernel(const __half* __restrict__ h, long long ldh, __half* __restrict__ out, long long ldo,
                             long long m, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = n / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < m * vecs;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vecs;
    const int col = static_cast<int>(i - r * vecs) * 8;
    float v[8], g[8];
    unpack8(*reinterpret_cast<const uint4*>(h + r * ldh + col), v);
    unpack8(*reinterpret_cast<const uint4*>(h + r * ldh + n + col), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] *= gelu_erf_f(g[e]);
    *reinterpret_cast<uint4*>(out + r * ldo + col) = pack8(v);
  }
}

// GEGLU backward: dh[r][j] = dout gelu_erf(g), dh[r][n + j] = dout v gelu_erf'(g)
__global__ void geglu_bwd_kernel(const __half* __restrict__ h, long long ldh, const __half* __restrict__ dout,
                                 long long lddout, __half* __restrict__ dh, long long lddh, long long m, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = n / 8;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < m * vecs;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / vecs;
    const int col = static_cast<int>(i - r * vecs) * 8;
    float v[8], g[8], d[8], dv[8], dg[8];
    unpack8(*reinterpret_cast<const uint4*>(h + r * ldh + col), v);
    unpack8(*reinterpret_cast<const uint4*>(h + r * ldh + n + col), g);
    unpack8(*reinterpret_cast<const uint4*>(dout + r * lddout + col), d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      dv[e] = d[e] * gelu_erf_f(g[e]);
      dg[e] = d[e] * v[e] * dgelu_erf(g[e]);
    }
    *reinterpret_cast<uint4*>(dh + r * lddh + col) = pack8(dv);
    *reinterpret_cast<uint4*>(dh + r * lddh + n + col) = pack8(dg);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------
static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static bool dtype_ok(int dtype) { return dtype == MDB_DTYPE_F16 || dtype == MDB_DTYPE_F32; }

struct GnBwdPlan {
  int c, threads, rows_per_cta, nblk;
  long long ab, part, ws_floats;  // workspace: [statistics kernel's region][A, B: 2 batch c][slabs: 2 batch nblk c]
};

static int plan_gn_bwd(const mdb_groupnorm_bwd_desc* d, GnBwdPlan* pl) {
  MDB_REQUIRE(d != nullptr, "mdb_groupnorm_bwd_f16: null descriptor");
  MDB_REQUIRE(d->x1 && d->gamma && d->beta && d->dy, "mdb_groupnorm_bwd_f16: null pointer (x1, gamma, beta, dy)");
  MDB_REQUIRE((d->x2 != nullptr) == (d->c2 > 0), "mdb_groupnorm_bwd_f16: x2 and c2 > 0 go together (c2=%d)", d->c2);
  const int c = d->c1 + d->c2;
  MDB_REQUIRE(d->c1 > 0 && d->c2 >= 0 && d->c1 % 8 == 0 && d->c2 % 8 == 0 && c % 32 == 0,
              "mdb_groupnorm_bwd_f16: channels must be multiples of 8 with c %% 32 == 0 (c1=%d c2=%d)", d->c1, d->c2);
  MDB_REQUIRE(c / 32 >= 10,
              "mdb_groupnorm_bwd_f16: %d-channel groups have no backward (groups of 10 channels or more; the "
              "first-stage VAE runs without gradient)", c / 32);
  MDB_REQUIRE(c <= 2560, "mdb_groupnorm_bwd_f16: unsupported width %d (320 ... 2560 channels)", c);
  MDB_REQUIRE(d->batch > 0 && d->batch <= kGnMaxBatch && d->hw > 0, "mdb_groupnorm_bwd_f16: bad shape batch=%d hw=%d",
              d->batch, d->hw);
  MDB_REQUIRE(d->eps > 0.f, "mdb_groupnorm_bwd_f16: eps must be positive");
  MDB_REQUIRE(al16(d->x1) && al16(d->x2) && al16(d->dy), "mdb_groupnorm_bwd_f16: x1, x2 and dy must be 16B aligned");
  if (d->dx1)
    MDB_REQUIRE(al16(d->dx1) && dtype_ok(d->dx1_dtype), "mdb_groupnorm_bwd_f16: dx1 must be 16B aligned, dtype 0|1");
  if (d->dx2) {
    MDB_REQUIRE(d->x2 != nullptr, "mdb_groupnorm_bwd_f16: dx2 without a second source");
    MDB_REQUIRE(al16(d->dx2) && dtype_ok(d->dx2_dtype), "mdb_groupnorm_bwd_f16: dx2 must be 16B aligned, dtype 0|1");
  }
  pl->c = c;
  gn_stats_geometry(c, d->batch, d->hw, &pl->threads, &pl->rows_per_cta, &pl->nblk);
  const long long batch = d->batch;
  pl->ab = kGnMaxBatch + batch * 64 + batch * pl->nblk * 64;  // mdb_groupnorm_ws_floats: a multiple of 4
  pl->part = pl->ab + 2 * batch * c;
  pl->ws_floats = pl->part + 2 * batch * pl->nblk * c;
  return MDB_OK;
}

struct LnBwdPlan {
  int rows_per_warp, nblk;
  long long ws_floats;  // slabs [2][nblk][c] when dgamma or dbeta is wanted
};

static int plan_ln_bwd(const mdb_layernorm_bwd_desc* d, LnBwdPlan* pl) {
  MDB_REQUIRE(d != nullptr, "mdb_layernorm_bwd_f16: null descriptor");
  MDB_REQUIRE(d->x && d->gamma && d->dy, "mdb_layernorm_bwd_f16: null pointer (x, gamma, dy)");
  MDB_REQUIRE(d->c == 320 || d->c == 640 || d->c == 1280, "mdb_layernorm_bwd_f16: unsupported width %d (320, 640, 1280)",
              d->c);
  MDB_REQUIRE(d->rows > 0, "mdb_layernorm_bwd_f16: bad shape rows=%lld", (long long)d->rows);
  MDB_REQUIRE(d->eps > 0.f, "mdb_layernorm_bwd_f16: eps must be positive");
  MDB_REQUIRE(al16(d->x) && al16(d->dy), "mdb_layernorm_bwd_f16: x and dy must be 16B aligned");
  if (d->dx)
    MDB_REQUIRE(al16(d->dx) && dtype_ok(d->dx_dtype), "mdb_layernorm_bwd_f16: dx must be 16B aligned, dtype 0|1");
  // about two CTAs of kLnBwdWarps warps per SM; each CTA contributes one slab to the column sums
  const long long warps = 2LL * kNumSms * kLnBwdWarps;
  pl->rows_per_warp = static_cast<int>((d->rows + warps - 1) / warps);
  const long long rows_per_cta = static_cast<long long>(pl->rows_per_warp) * kLnBwdWarps;
  pl->nblk = static_cast<int>((d->rows + rows_per_cta - 1) / rows_per_cta);
  pl->ws_floats = (d->dgamma || d->dbeta) ? 2LL * pl->nblk * d->c : 0;
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

extern "C" int64_t mdb_groupnorm_bwd_ws_floats(const mdb_groupnorm_bwd_desc* d) {
  GnBwdPlan pl;
  const int rc = plan_gn_bwd(d, &pl);
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_groupnorm_bwd_f16(const mdb_groupnorm_bwd_desc* d, mdb_stream_t stream) {
  GnBwdPlan pl;
  int rc = plan_gn_bwd(d, &pl);
  if (rc) return rc;
  MDB_REQUIRE(d->ws != nullptr && al16(d->ws),
              "mdb_groupnorm_bwd_f16: needs a 16B-aligned, initially zero workspace of mdb_groupnorm_bwd_ws_floats() = "
              "%lld floats", (long long)pl.ws_floats);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __half* x1 = static_cast<const __half*>(d->x1);
  const __half* x2 = static_cast<const __half*>(d->x2);
  const __half* dy = static_cast<const __half*>(d->dy);
  const int c = pl.c, batch = d->batch;
  if ((rc = launch_gn_stats(x1, d->c1, x2, d->c2, d->ws, batch, d->hw, st))) return rc;
  count_launch();
  const float* stats = d->ws + kGnMaxBatch;
  float* ab = d->ws + pl.ab;
  float* part = d->ws + pl.part;
  const int rstride = pl.threads / (c / 8);
  const dim3 grid(pl.nblk, batch);
  MDB_CHECK_CUDA(launch_pdl(gn_bwd_reduce_kernel, grid, dim3(pl.threads), 2 * rstride * c * sizeof(float), st, x1,
                            d->c1, x2, d->c2, dy, d->gamma, d->beta, stats, part, d->hw, pl.rows_per_cta, d->eps,
                            d->silu));
  count_launch();
  if ((rc = launch_colsum_finalize(part, c, 2 * batch, pl.nblk, ab, c, 0, st))) return rc;
  if (d->dx1 || d->dx2) {
    MDB_CHECK_CUDA(launch_pdl(gn_bwd_apply_kernel, grid, dim3(pl.threads), 0, st, x1, d->c1, x2, d->c2, dy, d->gamma,
                              d->beta, stats, static_cast<const float*>(ab),
                              gb_out(d->dx1, d->c1, d->dx1_dtype, d->dx1_accumulate),
                              gb_out(d->dx2, d->c2, d->dx2_dtype, d->dx2_accumulate), d->hw, pl.rows_per_cta, d->eps,
                              d->silu));
    count_launch();
  }
  if (d->dbeta && (rc = launch_colsum_finalize(ab, c, 1, batch, d->dbeta, 0, d->dbeta_accumulate, st))) return rc;
  if (d->dgamma &&
      (rc = launch_colsum_finalize(ab + static_cast<long long>(batch) * c, c, 1, batch, d->dgamma, 0,
                                   d->dgamma_accumulate, st)))
    return rc;
  return MDB_OK;
}

extern "C" int64_t mdb_layernorm_bwd_ws_floats(const mdb_layernorm_bwd_desc* d) {
  LnBwdPlan pl;
  const int rc = plan_ln_bwd(d, &pl);
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_layernorm_bwd_f16(const mdb_layernorm_bwd_desc* d, mdb_stream_t stream) {
  LnBwdPlan pl;
  int rc = plan_ln_bwd(d, &pl);
  if (rc) return rc;
  MDB_REQUIRE(pl.ws_floats == 0 || (d->ws != nullptr && al16(d->ws)),
              "mdb_layernorm_bwd_f16: needs a 16B-aligned workspace of mdb_layernorm_bwd_ws_floats() = %lld floats",
              (long long)pl.ws_floats);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __half* x = static_cast<const __half*>(d->x);
  const __half* dy = static_cast<const __half*>(d->dy);
  const GbOut dx = gb_out(d->dx, d->c, d->dx_dtype, d->dx_accumulate);
  const int params = pl.ws_floats > 0;
  const long long rows = d->rows;
#define MDB_LNB_CASE(V)                                                                                              \
  case V:                                                                                                            \
    MDB_CHECK_CUDA(launch_pdl(layernorm_bwd_kernel<V>, dim3(pl.nblk), dim3(kLnBwdWarps * 32), 0, st, x, d->gamma, dy, \
                              dx, d->ws, rows, d->c, d->eps, pl.rows_per_warp, params));                             \
    break;
  switch (d->c / 64) {
    MDB_LNB_CASE(5)
    MDB_LNB_CASE(10)
    MDB_LNB_CASE(20)
  }
#undef MDB_LNB_CASE
  count_launch();
  const long long slab = static_cast<long long>(pl.nblk) * d->c;
  if (d->dgamma && (rc = launch_colsum_finalize(d->ws, d->c, 1, pl.nblk, d->dgamma, 0, d->dgamma_accumulate, st)))
    return rc;
  if (d->dbeta && (rc = launch_colsum_finalize(d->ws + slab, d->c, 1, pl.nblk, d->dbeta, 0, d->dbeta_accumulate, st)))
    return rc;
  return MDB_OK;
}

static int geglu_check(const char* what, const void* h, int64_t ldh, int64_t m, int32_t n) {
  MDB_REQUIRE(h != nullptr && al16(h), "%s: h must be a 16B-aligned pointer", what);
  MDB_REQUIRE(m > 0 && n > 0 && n % 8 == 0 && ldh % 8 == 0 && ldh >= 2LL * n,
              "%s: needs m > 0, n %% 8 == 0 and ldh %% 8 == 0 with ldh >= 2n (m=%lld n=%d ldh=%lld)", what,
              (long long)m, n, (long long)ldh);
  return MDB_OK;
}

static unsigned geglu_blocks(int64_t m, int32_t n) {
  const long long total = m * (n / 8);
  return static_cast<unsigned>(min((total + 255) / 256, static_cast<long long>(kNumSms) * 16));
}

extern "C" int mdb_geglu_f16(const void* h, int64_t ldh, void* out, int64_t ldo, int64_t m, int32_t n,
                             mdb_stream_t stream) {
  int rc = geglu_check("mdb_geglu_f16", h, ldh, m, n);
  if (rc) return rc;
  MDB_REQUIRE(out != nullptr && al16(out) && ldo % 8 == 0 && ldo >= n,
              "mdb_geglu_f16: out must be 16B aligned with ldo %% 8 == 0 and ldo >= n");
  MDB_CHECK_CUDA(launch_pdl(geglu_kernel, dim3(geglu_blocks(m, n)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                            static_cast<const __half*>(h), (long long)ldh, static_cast<__half*>(out), (long long)ldo,
                            (long long)m, n));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_geglu_bwd_f16(const void* h, int64_t ldh, const void* dout, int64_t lddout, void* dh,
                                 int64_t lddh, int64_t m, int32_t n, mdb_stream_t stream) {
  int rc = geglu_check("mdb_geglu_bwd_f16", h, ldh, m, n);
  if (rc) return rc;
  MDB_REQUIRE(dout != nullptr && al16(dout) && lddout % 8 == 0 && lddout >= n,
              "mdb_geglu_bwd_f16: dout must be 16B aligned with lddout %% 8 == 0 and lddout >= n");
  MDB_REQUIRE(dh != nullptr && al16(dh) && lddh % 8 == 0 && lddh >= 2LL * n,
              "mdb_geglu_bwd_f16: dh must be 16B aligned with lddh %% 8 == 0 and lddh >= 2n");
  MDB_CHECK_CUDA(launch_pdl(geglu_bwd_kernel, dim3(geglu_blocks(m, n)), dim3(256), 0,
                            static_cast<cudaStream_t>(stream), static_cast<const __half*>(h), (long long)ldh,
                            static_cast<const __half*>(dout), (long long)lddout, static_cast<__half*>(dh),
                            (long long)lddh, (long long)m, n));
  count_launch();
  return MDB_OK;
}
