// Backward of the direct 3x3 convolutions (misc.cu: the ControlNet hint encoder, the 4->320 input conv and the 320->4
// output conv), of the skinny timestep Linear, and of the nearest x2 upsample.  HBM / CUDA-core kernels.
//
// Direct conv, y = act(z) + residual with z = conv(x, W) + bias, dz = dy silu'(z) (or dy):
//   recompute      z by the unchanged forward kernel (silu = 0, no residual) into the workspace, then dz in place
//   dx, stride 1   the forward kernel itself on dz with the flipped, transposed weight [I][2-kh][2-kw][O] (the caller's
//                  wt_t), which the forward dispatch sends to the generic, small-cin or small-cout kernel
//   dx, stride 2   conv3x3_s2_dx_kernel: a gather over the 1, 2 or 4 taps an input pixel's parity allows
//   dW, dbias      conv3x3_dw_kernel: per-CTA fp32 slabs over a fixed run of 8x8 output tiles, then
//                  colsum_finalize_kernel (gemm_bwd.cu) sums the slabs in CTA order; dW lands in OIHW order
// Skinny Linear, out[r][n] = sum_k f(x[r][k]) W[n][k] + bias[n], f = SiLU when silu_in:
//   dX             skinny_bwd_dx_kernel: fp32 slabs over fixed chunks of n; skinny_bwd_dx_finalize_kernel sums them in
//                  chunk order and applies silu'(x)
//   dW, dbias      skinny_bwd_dw_kernel: the rows summed in row order (taller inputs: row chunks accumulate in order)
// Upsample: dx = the 2x2 block sum of dy, in a fixed order.
// Deterministic throughout: fixed-order reductions, no atomics.
#include "common.cuh"

namespace mdb {

constexpr int kDwTile = 8;         // output tile edge of the dW kernel (8x8 pixels)
constexpr int kDwCout = 32;        // output channels of one dW CTA
constexpr int kDwCin = 16;         // input channels of one dW CTA
constexpr int kDwThreads = 288;    // 9 taps (one per warp) x 8 cout quads x 4 cin quads
constexpr int kDxCin = 32;         // input channels of one stride-2 dx CTA
constexpr int kDxCout = 16;        // output-channel slice staged per step
constexpr int kDxPatch = 5;        // dz rows / columns a tile of 8 input pixels reaches at stride 2
constexpr int kDxPitch = kDxCout + 1;  // padded pixel pitch of the staged dz patch (no bank conflicts)
constexpr int kSkThreads = 64;     // skinny backward: column quads per CTA
constexpr int kSkDwRows = 32;      // skinny dW: n rows per CTA

// dz = dy silu'(z) over n elements, in place over z
__global__ void silu_grad_kernel(const __half* __restrict__ dy, __half* z, long long n) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    z[i] = __float2half_rn(__half2float(dy[i]) * dsilu(__half2float(z[i])));
}

// dW / dbias partials of output channels [co0, co0 + 32) x input channels [ci0, ci0 + 16) over output tiles
// [blockIdx.x * tiles_per_cta, ...): wpart[blockIdx.x][cout][cin][3][3], bpart[blockIdx.x][cout] (ci block 0 only)
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads) conv3x3_dw_kernel(
    const __half* __restrict__ x, const __half* __restrict__ dz, float* __restrict__ wpart, float* __restrict__ bpart,
    int h, int w, int cin, int cout, int ho, int wo, int tiles, int tiles_per_cta, int want_w) {
  constexpr int PH = (kDwTile - 1) * STRIDE + 3;
  __shared__ __align__(16) float s_in[PH * PH * kDwCin];
  __shared__ __align__(16) float s_dz[kDwTile * kDwTile * kDwCout];
  pdl_launch_dependents();
  const int tid = threadIdx.x;
  const int cq = tid & 3;         // input-channel quad
  const int oq = (tid >> 2) & 7;  // output-channel quad
  const int t = tid >> 5;         // tap, one per warp
  const int kh = t / 3, kw = t % 3;
  const int co0 = blockIdx.y * kDwCout, ci0 = blockIdx.z * kDwCin;
  const int tiles_x = (wo + kDwTile - 1) / kDwTile;
  const int tiles_img = tiles_x * ((ho + kDwTile - 1) / kDwTile);
  const bool bias_thread = bpart != nullptr && blockIdx.z == 0 && t == 0 && cq == 0;
  float acc[4][4], bacc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    bacc[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  pdl_wait();
  const int tile1 = min(tiles, (blockIdx.x + 1) * tiles_per_cta);
  for (int tile = blockIdx.x * tiles_per_cta; tile < tile1; ++tile) {
    const int b = tile / tiles_img, r = tile - b * tiles_img;
    const int oy0 = (r / tiles_x) * kDwTile, ox0 = (r % tiles_x) * kDwTile;
    const int iy0 = oy0 * STRIDE - 1, ix0 = ox0 * STRIDE - 1;
    if (want_w) {
      for (int i = tid; i < PH * PH * kDwCin; i += kDwThreads) {
        const int ci = i % kDwCin, pp = i / kDwCin;
        const int yy = iy0 + pp / PH, xx = ix0 + pp % PH;
        float v = 0.f;
        if (ci0 + ci < cin && yy >= 0 && yy < h && xx >= 0 && xx < w)
          v = __half2float(x[((static_cast<long long>(b) * h + yy) * w + xx) * cin + ci0 + ci]);
        s_in[i] = v;
      }
    }
    for (int i = tid; i < kDwTile * kDwTile * kDwCout; i += kDwThreads) {
      const int co = i % kDwCout, p = i / kDwCout;
      const int oy = oy0 + p / kDwTile, ox = ox0 + p % kDwTile;
      float v = 0.f;
      if (co0 + co < cout && oy < ho && ox < wo)
        v = __half2float(dz[((static_cast<long long>(b) * ho + oy) * wo + ox) * cout + co0 + co]);
      s_dz[i] = v;
    }
    __syncthreads();
    if (want_w) {
#pragma unroll 4
      for (int p = 0; p < kDwTile * kDwTile; ++p) {
        const float4 d = *reinterpret_cast<const float4*>(&s_dz[p * kDwCout + oq * 4]);
        const float4 xv = *reinterpret_cast<const float4*>(
            &s_in[(((p / kDwTile) * STRIDE + kh) * PH + (p % kDwTile) * STRIDE + kw) * kDwCin + cq * 4]);
        const float dv[4] = {d.x, d.y, d.z, d.w}, xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(dv[i], xa[j], acc[i][j]);
      }
    }
    if (bias_thread) {
      for (int p = 0; p < kDwTile * kDwTile; ++p)
#pragma unroll
        for (int i = 0; i < 4; ++i) bacc[i] += s_dz[p * kDwCout + oq * 4 + i];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + oq * 4 + i;
    if (co >= cout) continue;
    if (want_w) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ci = ci0 + cq * 4 + j;
        if (ci < cin) wpart[((static_cast<long long>(blockIdx.x) * cout + co) * cin + ci) * 9 + t] = acc[i][j];
      }
    }
    if (bias_thread) bpart[static_cast<long long>(blockIdx.x) * cout + co] = bacc[i];
  }
}

// dx of a stride-2 conv.  CTA: 8x8 input pixels x 32 input channels; thread: one pixel x 8 channels.  Input pixel
// (iy, ix) receives dz(oy, ox) W[kh][kw] for oy = (iy + 1 - kh) / 2 with kh of iy + 1's parity: kh = 1 for even iy,
// kh = 0, 2 for odd iy (likewise along x).  Threads are ordered by pixel parity class, so the 32 lanes of a warp share
// their taps.
__global__ void __launch_bounds__(256) conv3x3_s2_dx_kernel(const __half* __restrict__ dz, const __half* __restrict__ wt,
                                                            __half* __restrict__ dx, int h, int w, int cin, int cout,
                                                            int ho, int wo) {
  __shared__ float s_dz[kDxPatch * kDxPatch * kDxPitch];              // [pixel][co]
  __shared__ __align__(16) float s_w[9 * kDxCout * kDxCin];           // [tap][co][ci]
  pdl_launch_dependents();
  const int idx = threadIdx.x & 15, cg = (threadIdx.x >> 4) & 3, cls = threadIdx.x >> 6;
  const int pyl = (cls >> 1) + 2 * (idx >> 2), pxl = (cls & 1) + 2 * (idx & 3);  // pixel within the tile
  const int tiles_x = (w + 7) / 8;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x % tiles_x;
  const int b = blockIdx.z;
  const int ci0 = blockIdx.y * kDxCin;
  const int iy = ty * 8 + pyl, ix = tx * 8 + pxl;
  const int oy0 = ty * 4, ox0 = tx * 4;  // first dz row / column of the patch
  const int nkh = (pyl & 1) ? 2 : 1, nkw = (pxl & 1) ? 2 : 1;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  pdl_wait();
  for (int c0 = 0; c0 < cout; c0 += kDxCout) {
    for (int i = threadIdx.x; i < kDxPatch * kDxPatch * kDxCout; i += blockDim.x) {
      const int co = i % kDxCout, pp = i / kDxCout;
      const int oy = oy0 + pp / kDxPatch, ox = ox0 + pp % kDxPatch;
      float v = 0.f;
      if (c0 + co < cout && oy < ho && ox < wo)
        v = __half2float(dz[((static_cast<long long>(b) * ho + oy) * wo + ox) * cout + c0 + co]);
      s_dz[pp * kDxPitch + co] = v;
    }
    for (int i = threadIdx.x; i < 9 * kDxCout * kDxCin; i += blockDim.x) {
      const int ci = i % kDxCin, co = (i / kDxCin) % kDxCout, t = i / (kDxCin * kDxCout);
      float v = 0.f;
      if (c0 + co < cout && ci0 + ci < cin)
        v = __half2float(wt[(static_cast<long long>(c0 + co) * 9 + t) * cin + ci0 + ci]);
      s_w[i] = v;
    }
    __syncthreads();
    for (int a = 0; a < nkh; ++a) {
      const int kh = (pyl & 1) ? 2 * a : 1;
      const int row = (pyl + 1 - kh) / 2;
      for (int e = 0; e < nkw; ++e) {
        const int kw = (pxl & 1) ? 2 * e : 1;
        const int col = (pxl + 1 - kw) / 2;
        const float* dp = &s_dz[(row * kDxPatch + col) * kDxPitch];
        const float* wp = &s_w[(kh * 3 + kw) * kDxCout * kDxCin + cg * 8];
#pragma unroll 4
        for (int co = 0; co < kDxCout; ++co) {
          const float d = dp[co];
          const float4 w0 = *reinterpret_cast<const float4*>(wp + co * kDxCin);
          const float4 w1 = *reinterpret_cast<const float4*>(wp + co * kDxCin + 4);
          acc[0] = fmaf(d, w0.x, acc[0]);
          acc[1] = fmaf(d, w0.y, acc[1]);
          acc[2] = fmaf(d, w0.z, acc[2]);
          acc[3] = fmaf(d, w0.w, acc[3]);
          acc[4] = fmaf(d, w1.x, acc[4]);
          acc[5] = fmaf(d, w1.y, acc[5]);
          acc[6] = fmaf(d, w1.z, acc[6]);
          acc[7] = fmaf(d, w1.w, acc[7]);
        }
      }
    }
    __syncthreads();
  }
  if (iy < h && ix < w) {
    __half* o = dx + ((static_cast<long long>(b) * h + iy) * w + ix) * cin;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ci = ci0 + cg * 8 + j;
      if (ci < cin) o[ci] = __float2half_rn(acc[j]);
    }
  }
}

// partial dX of the skinny Linear over n in [blockIdx.y * chunk, ...): part[blockIdx.y][r][k] = sum_n dy[r][n] W[n][k]
template <int ROWS>
__global__ void __launch_bounds__(kSkThreads) skinny_bwd_dx_kernel(const float* __restrict__ dy,
                                                                   const __half* __restrict__ w,
                                                                   float* __restrict__ part, int rows, int n, int k,
                                                                   int chunk) {
  pdl_launch_dependents();
  pdl_wait();
  const int col = (blockIdx.x * kSkThreads + threadIdx.x) * 4;
  if (col >= k) return;
  const int n0 = blockIdx.y * chunk, n1 = min(n, n0 + chunk);
  float acc[ROWS][4];
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
#pragma unroll 4
  for (int nn = n0; nn < n1; ++nn) {
    const uint2 u = *reinterpret_cast<const uint2*>(w + static_cast<long long>(nn) * k + col);
    const float2 w01 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 w23 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      if (r < rows) {
        const float d = dy[static_cast<long long>(r) * n + nn];
        acc[r][0] = fmaf(d, w01.x, acc[r][0]);
        acc[r][1] = fmaf(d, w01.y, acc[r][1]);
        acc[r][2] = fmaf(d, w23.x, acc[r][2]);
        acc[r][3] = fmaf(d, w23.y, acc[r][3]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
    if (r < rows)
      *reinterpret_cast<float4*>(part + (static_cast<long long>(blockIdx.y) * rows + r) * k + col) =
          make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
}

// dx[r][k] (+)= (sum over the parts, in order) * silu'(x[r][k]) when silu_in
__global__ void skinny_bwd_dx_finalize_kernel(const float* __restrict__ part, int parts, const float* __restrict__ x,
                                              float* dx, int rows, int k, int silu_in, int acc) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(rows) * k;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < parts; ++q) s += part[q * total + i];
    if (silu_in) s *= dsilu(x[i]);
    dx[i] = acc ? dx[i] + s : s;
  }
}

// dW[n][k] (+)= sum_r dy[r][n] f(x[r][k]) and dbias[n] (+)= sum_r dy[r][n], rows in order.  CTA: kSkDwRows rows of n x
// kSkThreads column quads; f(x) of the thread's four columns stays in registers.
template <int ROWS>
__global__ void __launch_bounds__(kSkThreads) skinny_bwd_dw_kernel(const float* __restrict__ x,
                                                                   const float* __restrict__ dy, float* dw,
                                                                   float* dbias, int rows, int n, int k, int silu_in,
                                                                   int dw_acc, int db_acc) {
  pdl_launch_dependents();
  pdl_wait();
  const int col = (blockIdx.x * kSkThreads + threadIdx.x) * 4;
  const bool mine = dw != nullptr && col < k;
  const bool bias = dbias != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (!mine && !bias) return;
  float fx[ROWS][4];
#pragma unroll
  for (int r = 0; r < ROWS; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = 0.f;
      if (mine && r < rows) {
        v = x[static_cast<long long>(r) * k + col + j];
        if (silu_in) v = silu_f(v);
      }
      fx[r][j] = v;
    }
  const int n1 = min(n, (blockIdx.y + 1) * kSkDwRows);
  for (int nn = blockIdx.y * kSkDwRows; nn < n1; ++nn) {
    float d[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) d[r] = r < rows ? dy[static_cast<long long>(r) * n + nn] : 0.f;
    if (mine) {
      float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int r = 0; r < ROWS; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = fmaf(d[r], fx[r][j], o[j]);
      float4* p = reinterpret_cast<float4*>(dw + static_cast<long long>(nn) * k + col);
      if (dw_acc) {
        const float4 old = *p;
        o[0] += old.x;
        o[1] += old.y;
        o[2] += old.z;
        o[3] += old.w;
      }
      *p = make_float4(o[0], o[1], o[2], o[3]);
    }
    if (bias) {
      float s = 0.f;
#pragma unroll
      for (int r = 0; r < ROWS; ++r) s += d[r];
      dbias[nn] = db_acc ? dbias[nn] + s : s;
    }
  }
}

// dx[b][y][x] = dy[2y][2x] + dy[2y][2x+1] + dy[2y+1][2x] + dy[2y+1][2x+1], 8 channels per thread
__global__ void upsample2x_bwd_kernel(const __half* __restrict__ dy, GbOut dx, int batch, int h, int w, int c) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = c / 8;
  const long long total = static_cast<long long>(batch) * h * w * vecs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % vecs);
    const long long r = i / vecs;  // input pixel
    const int xx = static_cast<int>(r % w), yy = static_cast<int>((r / w) % h);
    const long long b = r / (static_cast<long long>(w) * h);
    float s[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const long long o = ((b * 2 * h + 2 * yy + (q >> 1)) * 2 * w + 2 * xx + (q & 1)) * c + v * 8;
      const uint4 u = *reinterpret_cast<const uint4*>(dy + o);
      const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        s[2 * e] += f.x;
        s[2 * e + 1] += f.y;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) gb_store2(dx, r, v * 8 + 2 * e, s[2 * e], s[2 * e + 1]);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------
static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static long long up4(long long v) { return (v + 3) / 4 * 4; }

static int grid_cap(long long total, int threads = 256) {
  const long long b = (total + threads - 1) / threads;
  return static_cast<int>(b < 1 ? 1 : (b > kNumSms * 16 ? kNumSms * 16 : b));
}

struct DcBwdPlan {
  int ho, wo, tiles, tiles_per_cta, nsplit, co_blocks, ci_blocks;
  long long z, wpart, bpart, ws_floats;  // workspace: [z / dz fp16 (silu)][dW slabs][dbias slabs]
};

static int plan_dc_bwd(const mdb_conv3x3_bwd_desc* d, DcBwdPlan* pl) {
  MDB_REQUIRE(d != nullptr, "mdb_conv3x3_direct_bwd_f16: null descriptor");
  MDB_REQUIRE(d->x && d->wt && d->dy, "mdb_conv3x3_direct_bwd_f16: null pointer (x, wt, dy)");
  MDB_REQUIRE(d->stride == 1 || d->stride == 2, "mdb_conv3x3_direct_bwd_f16: stride must be 1 or 2 (got %d)",
              d->stride);
  MDB_REQUIRE(d->batch > 0 && d->h > 0 && d->w > 0 && d->cin > 0 && d->cout > 0 && d->cin <= 4096 &&
                  d->cout <= 4096 && d->batch <= 65535,
              "mdb_conv3x3_direct_bwd_f16: bad shape batch=%d h=%d w=%d cin=%d cout=%d", d->batch, d->h, d->w, d->cin,
              d->cout);
  MDB_REQUIRE(d->dx || d->dw || d->dbias, "mdb_conv3x3_direct_bwd_f16: no gradient requested (dx, dw, dbias all NULL)");
  MDB_REQUIRE(al16(d->x) && al16(d->wt) && al16(d->dy), "mdb_conv3x3_direct_bwd_f16: x, wt and dy must be 16B aligned");
  if (d->dx) {
    MDB_REQUIRE(al16(d->dx), "mdb_conv3x3_direct_bwd_f16: dx must be 16B aligned");
    if (d->stride == 1)
      MDB_REQUIRE(d->wt_t != nullptr && al16(d->wt_t),
                  "mdb_conv3x3_direct_bwd_f16: stride-1 dx needs the flipped weight wt_t [cin][3][3][cout], 16B "
                  "aligned");
  }
  pl->ho = (d->h - 1) / d->stride + 1;
  pl->wo = (d->w - 1) / d->stride + 1;
  pl->co_blocks = (d->cout + kDwCout - 1) / kDwCout;
  pl->ci_blocks = d->dw ? (d->cin + kDwCin - 1) / kDwCin : 1;
  pl->tiles = d->batch * ((pl->ho + kDwTile - 1) / kDwTile) * ((pl->wo + kDwTile - 1) / kDwTile);
  // about two CTAs per SM; each contributes one slab that the finalize pass sums in CTA order
  const int want = max(1, 2 * kNumSms / (pl->co_blocks * pl->ci_blocks));
  pl->tiles_per_cta = (pl->tiles + want - 1) / want;
  pl->nsplit = (pl->tiles + pl->tiles_per_cta - 1) / pl->tiles_per_cta;
  const long long zhalves = d->silu ? static_cast<long long>(d->batch) * pl->ho * pl->wo * d->cout : 0;
  pl->z = 0;
  pl->wpart = up4((zhalves + 1) / 2);
  pl->bpart = pl->wpart + (d->dw ? up4(static_cast<long long>(pl->nsplit) * d->cout * 9 * d->cin) : 0);
  pl->ws_floats = pl->bpart + (d->dbias ? up4(static_cast<long long>(pl->nsplit) * d->cout) : 0);
  return MDB_OK;
}

struct SkBwdPlan {
  int chunk, nsplit, gx;
  long long ws_floats;  // dX slabs [nsplit][rows][k]
};

static int plan_sk_bwd(const mdb_skinny_linear_bwd_desc* d, SkBwdPlan* pl) {
  MDB_REQUIRE(d != nullptr, "mdb_skinny_linear_bwd_f32: null descriptor");
  MDB_REQUIRE(d->x && d->w && d->dy, "mdb_skinny_linear_bwd_f32: null pointer (x, w, dy)");
  MDB_REQUIRE(d->rows >= 1 && d->rows <= 16 && d->n > 0 && d->k > 0 && d->k % 8 == 0,
              "mdb_skinny_linear_bwd_f32: bad shape rows=%d n=%d k=%d (rows 1..16, k %% 8 == 0)", d->rows, d->n, d->k);
  MDB_REQUIRE(d->dx || d->dw || d->dbias, "mdb_skinny_linear_bwd_f32: no gradient requested (dx, dw, dbias all NULL)");
  MDB_REQUIRE(al16(d->x) && al16(d->w) && al16(d->dy) && al16(d->dx) && al16(d->dw),
              "mdb_skinny_linear_bwd_f32: x, w, dy, dx and dw must be 16B aligned");
  pl->gx = (d->k / 4 + kSkThreads - 1) / kSkThreads;
  // about four 64-thread CTAs per SM stream W; each contributes one slab summed in chunk order
  const int want = max(1, 4 * kNumSms / pl->gx);
  pl->chunk = (d->n + want - 1) / want;
  pl->nsplit = (d->n + pl->chunk - 1) / pl->chunk;
  pl->ws_floats = d->dx ? static_cast<long long>(pl->nsplit) * d->rows * d->k : 0;
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

extern "C" int64_t mdb_conv3x3_direct_bwd_ws_floats(const mdb_conv3x3_bwd_desc* d) {
  DcBwdPlan pl;
  const int rc = plan_dc_bwd(d, &pl);
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_conv3x3_direct_bwd_f16(const mdb_conv3x3_bwd_desc* d, mdb_stream_t stream) {
  DcBwdPlan pl;
  int rc = plan_dc_bwd(d, &pl);
  if (rc) return rc;
  MDB_REQUIRE(pl.ws_floats == 0 || (d->ws != nullptr && al16(d->ws)),
              "mdb_conv3x3_direct_bwd_f16: needs a 16B-aligned workspace of mdb_conv3x3_direct_bwd_ws_floats() = "
              "%lld floats", (long long)pl.ws_floats);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __half* dz = static_cast<const __half*>(d->dy);
  if (d->silu) {  // z by the unchanged forward (no SiLU, no residual), then dz = dy silu'(z) in place
    __half* z = reinterpret_cast<__half*>(d->ws + pl.z);
    if ((rc = mdb_conv3x3_direct_f16(d->x, d->wt, d->bias, nullptr, z, d->batch, d->h, d->w, d->cin, d->cout,
                                     d->stride, 0, stream)))
      return rc;
    const long long n = static_cast<long long>(d->batch) * pl.ho * pl.wo * d->cout;
    MDB_CHECK_CUDA(launch_pdl(silu_grad_kernel, dim3(grid_cap(n)), dim3(256), 0, st, dz, z, n));
    count_launch();
    dz = z;
  }
  if (d->dx) {
    if (d->stride == 1) {  // the forward on dz with the flipped, transposed weight
      if ((rc = mdb_conv3x3_direct_f16(dz, d->wt_t, nullptr, nullptr, d->dx, d->batch, d->h, d->w, d->cout, d->cin, 1,
                                       0, stream)))
        return rc;
    } else {
      const dim3 grid(((d->w + 7) / 8) * ((d->h + 7) / 8), (d->cin + kDxCin - 1) / kDxCin, d->batch);
      MDB_CHECK_CUDA(launch_pdl(conv3x3_s2_dx_kernel, grid, dim3(256), 0, st, dz, static_cast<const __half*>(d->wt),
                                static_cast<__half*>(d->dx), d->h, d->w, d->cin, d->cout, pl.ho, pl.wo));
      count_launch();
    }
  }
  if (d->dw || d->dbias) {
    const dim3 grid(pl.nsplit, pl.co_blocks, pl.ci_blocks);
    float* wpart = d->dw ? d->ws + pl.wpart : nullptr;
    float* bpart = d->dbias ? d->ws + pl.bpart : nullptr;
    const __half* x = static_cast<const __half*>(d->x);
    if (d->stride == 1)
      MDB_CHECK_CUDA(launch_pdl(conv3x3_dw_kernel<1>, grid, dim3(kDwThreads), 0, st, x, dz, wpart, bpart, d->h, d->w,
                                d->cin, d->cout, pl.ho, pl.wo, pl.tiles, pl.tiles_per_cta, d->dw != nullptr ? 1 : 0));
    else
      MDB_CHECK_CUDA(launch_pdl(conv3x3_dw_kernel<2>, grid, dim3(kDwThreads), 0, st, x, dz, wpart, bpart, d->h, d->w,
                                d->cin, d->cout, pl.ho, pl.wo, pl.tiles, pl.tiles_per_cta, d->dw != nullptr ? 1 : 0));
    count_launch();
    if (d->dw &&
        (rc = launch_colsum_finalize(wpart, d->cout * 9 * d->cin, 1, pl.nsplit, d->dw, 0, d->dw_accumulate, st)))
      return rc;
    if (d->dbias && (rc = launch_colsum_finalize(bpart, d->cout, 1, pl.nsplit, d->dbias, 0, d->dbias_accumulate, st)))
      return rc;
  }
  return MDB_OK;
}

extern "C" int64_t mdb_skinny_linear_bwd_ws_floats(const mdb_skinny_linear_bwd_desc* d) {
  SkBwdPlan pl;
  const int rc = plan_sk_bwd(d, &pl);
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_skinny_linear_bwd_f32(const mdb_skinny_linear_bwd_desc* d, mdb_stream_t stream) {
  SkBwdPlan pl;
  int rc = plan_sk_bwd(d, &pl);
  if (rc) return rc;
  MDB_REQUIRE(pl.ws_floats == 0 || (d->ws != nullptr && al16(d->ws)),
              "mdb_skinny_linear_bwd_f32: needs a 16B-aligned workspace of mdb_skinny_linear_bwd_ws_floats() = %lld "
              "floats", (long long)pl.ws_floats);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const __half* w = static_cast<const __half*>(d->w);
  const int rows = d->rows, n = d->n, k = d->k;
  if (d->dx) {
    const dim3 grid(pl.gx, pl.nsplit);
    if (rows <= 2)
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dx_kernel<2>, grid, dim3(kSkThreads), 0, st, d->dy, w, d->ws, rows, n, k,
                                pl.chunk));
    else if (rows <= 8)
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dx_kernel<8>, grid, dim3(kSkThreads), 0, st, d->dy, w, d->ws, rows, n, k,
                                pl.chunk));
    else
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dx_kernel<16>, grid, dim3(kSkThreads), 0, st, d->dy, w, d->ws, rows, n, k,
                                pl.chunk));
    count_launch();
    MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dx_finalize_kernel, dim3(grid_cap(static_cast<long long>(rows) * k)),
                              dim3(256), 0, st, static_cast<const float*>(d->ws), pl.nsplit, d->x, d->dx, rows, k,
                              d->silu_in, d->dx_accumulate));
    count_launch();
  }
  if (d->dw || d->dbias) {
    const dim3 grid(d->dw ? pl.gx : 1, (n + kSkDwRows - 1) / kSkDwRows);
    if (rows <= 2)
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dw_kernel<2>, grid, dim3(kSkThreads), 0, st, d->x, d->dy, d->dw, d->dbias,
                                rows, n, k, d->silu_in, d->dw_accumulate, d->dbias_accumulate));
    else if (rows <= 8)
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dw_kernel<8>, grid, dim3(kSkThreads), 0, st, d->x, d->dy, d->dw, d->dbias,
                                rows, n, k, d->silu_in, d->dw_accumulate, d->dbias_accumulate));
    else
      MDB_CHECK_CUDA(launch_pdl(skinny_bwd_dw_kernel<16>, grid, dim3(kSkThreads), 0, st, d->x, d->dy, d->dw, d->dbias,
                                rows, n, k, d->silu_in, d->dw_accumulate, d->dbias_accumulate));
    count_launch();
  }
  return MDB_OK;
}

extern "C" int mdb_upsample2x_bwd_f16(const void* dy, void* dx, int32_t dx_dtype, int32_t accumulate, int32_t batch,
                                      int32_t h, int32_t w, int32_t c, mdb_stream_t stream) {
  MDB_REQUIRE(dy && dx, "mdb_upsample2x_bwd_f16: null pointer (dy, dx)");
  MDB_REQUIRE(batch > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0,
              "mdb_upsample2x_bwd_f16: bad shape batch=%d h=%d w=%d c=%d (c %% 8 == 0)", batch, h, w, c);
  MDB_REQUIRE(al16(dy) && al16(dx), "mdb_upsample2x_bwd_f16: dy and dx must be 16B aligned");
  MDB_REQUIRE(dx_dtype == MDB_DTYPE_F16 || dx_dtype == MDB_DTYPE_F32, "mdb_upsample2x_bwd_f16: dx_dtype must be 0|1");
  const long long total = static_cast<long long>(batch) * h * w * (c / 8);
  MDB_CHECK_CUDA(launch_pdl(upsample2x_bwd_kernel, dim3(grid_cap(total)), dim3(256), 0,
                            static_cast<cudaStream_t>(stream), static_cast<const __half*>(dy),
                            gb_out(dx, c, dx_dtype, accumulate), batch, h, w, c));
  count_launch();
  return MDB_OK;
}
