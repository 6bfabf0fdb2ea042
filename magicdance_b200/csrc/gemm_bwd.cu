// Backward of the wgmma GEMM / 3x3 implicit-GEMM convolution of gemm.cu, for sm_90a.
//
//   forward  D[M,N] = A[M,K] B[N,K]^T (+ bias + residual)
//   dA = dD B      [M,K], reduces over N     (conv: dD shifted by (1-kw, 1-kh) per tap: the transposed convolution)
//   dB = dD^T A    [N,K], reduces over M     (conv: the forward's shifted 4-D TMA boxes of the input, per tap)
//   dbias          column sums of dD, per segment of rows_per_batch rows for a per-batch bias
//
// gemm_bwd_kernel<TA> computes one 128 x 128 tile of either product, optionally one split of its reduction.  Warp
// roles as in gemm_tc_kernel: warp 8 is the TMA producer, warps 0-7 two warpgroups of 64 output rows each.  A stage is
// 64 steps of the reduction: the A-side tile (dD) and two 64-column chunks of the B-side tile, all 128B-swizzled.
//   TA = 0 (dA): A-side = dD [128 rows][64 of N], K-major as in the forward; B-side = the forward's B read MN-major
//                (its rows are the reduction), so no transposed copy of a weight is made.
//   TA = 1 (dB): A-side = dD [64 of M][128 of N] and B-side = the forward's A [64 of M][128 of K], both MN-major.
// The B-side chunks of dB are loaded one 64-column chunk at a time, so a chunk may come from a2 (dual source) or from
// another tap (conv) than its neighbour.  TMA zero-fill handles ragged M / N and the conv halo on both operands.
//
// Deterministic, no atomics: a tile's reduction runs in one CTA (fixed order), or in `splits` CTAs that write fp32
// slabs which gemm_bwd_finalize_kernel sums in split order.  Stride-2 dA and latents whose pixels do not form the
// TMA boxes go through an fp32 column buffer [M_out][9c] and col2im_gather_kernel (each input pixel sums its taps in
// a fixed order, no scatter-add); dB for such latents through im2col + the plain path.
#include "common.cuh"

namespace mdb {

constexpr int kGbM = 128;  // output rows per CTA
constexpr int kGbN = 128;  // output columns per CTA
constexpr int kGbK = 64;   // reduction step per stage: one 128-byte swizzle row
constexpr int kGbStages = 3;
constexpr int kGbABytes = kGbM * kGbK * 2;    // 16 KB
constexpr int kGbChunk = 64 * kGbK * 2;       // 8 KB: 64 output rows or columns x 64 reduction steps
constexpr int kGbStageBytes = kGbABytes + (kGbN / 64) * kGbChunk;
constexpr int kGbSmem = kGbStages * kGbStageBytes + 1024;  // two CTAs per SM
constexpr int kBiasRows = 256;  // rows per partial column sum

struct GemmBwdKParams {
  CUtensorMap tmD;   // dD: TA = 0 [128 x 64] boxes (4-D pixel boxes in conv mode); TA = 1 [64 x 64] boxes
  CUtensorMap tmB;   // TA = 0: the forward's B, [64 x 64] boxes; TA = 1: the forward's A (4-D pixel boxes in conv mode)
  CUtensorMap tmB2;  // TA = 1: the forward's a2
  GbOut out[2];      // output columns < split_col go to out[0], the others to out[1] at column - split_col
  int split_col;
  float* ws;         // splits > 1: fp32 slabs [splits][rows][cols]
  int rows, cols;    // output extent (cols is a multiple of 64)
  int chunks, chunks_per_split, splits;
  int conv;          // implicit convolution
  int chunks_per_tap;  // TA = 0 conv: 64-wide chunks of N per tap
  int c;             // conv: input channels (the column width of one tap)
  int w, hw, cs;     // conv pixel geometry: TA = 0 the row tiles (stride 1), TA = 1 the forward's output pixels
  int k1;            // TA = 1 plain: columns taken from tmB, the rest from tmB2
};

__device__ __forceinline__ void gb_put(const GemmBwdKParams& p, long long row, int col, float v0, float v1) {
  if (col < p.split_col) gb_store2(p.out[0], row, col, v0, v1);
  else gb_store2(p.out[1], row, col - p.split_col, v0, v1);
}

// IM2COL (conv only, any latent size): the pixel operands come from TMA im2col loads (tmap_nhwc_im2col) that walk the
// tile's pixels across row and image boundaries.  TA = 0: 128 input pixels of dD per load (stride 1), the window corner
// (x - 1, y - 1) with offsets (2 - kw, 2 - kh), i.e. output pixel (y + 1 - kh, x + 1 - kw).  TA = 1: 64 output pixels
// of the forward's A per load, offsets (kw, kh) as in the forward, channels [0, k1) from tmB and the rest from tmB2.
template <int TA, bool IM2COL>
__device__ __forceinline__ void gemm_bwd_body(const GemmBwdKParams& p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kGbStages];
  __shared__ __align__(8) uint64_t empty_bar[kGbStages];
  uint8_t* smem = align1024(smem_raw);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * kGbM;
  const int c0 = blockIdx.y * kGbN;
  const int split = blockIdx.z;
  const int kc_begin = split * p.chunks_per_split;
  const int n_iter = min(p.chunks, kc_begin + p.chunks_per_split) - kc_begin;
  // chunks wholly past the last output row / column are not loaded: they feed only accumulators that are not stored
  const int a_bytes = TA == 0 ? kGbABytes : min(2, (p.rows - r0 + 63) / 64) * kGbChunk;
  const int b_chunks = min(kGbN / 64, (p.cols - c0) / 64);

  pdl_launch_dependents();
  if (warp == kProducerWarp && lane == 0) {
    ring_init<kGbStages>(full_bar, empty_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kProducerWarp) {
    if (lane == 0 && n_iter > 0) {
      int b0 = 0, y0 = 0, x0 = 0;  // TA = 0 conv: the first pixel of this row tile
      if (TA == 0 && p.conv) {
        b0 = r0 / p.hw;
        y0 = (r0 - b0 * p.hw) / p.w;
        x0 = (r0 - b0 * p.hw) - y0 * p.w;
      }
      for (int it = 0; it < n_iter; ++it) {
        const int s = ring_acquire<kGbStages>(empty_bar, it);
        uint8_t* sa = smem + s * kGbStageBytes;
        uint8_t* sb = sa + kGbABytes;
        const int kc = kc_begin + it;
        mbar_expect_tx(&full_bar[s], a_bytes + b_chunks * kGbChunk);
        if constexpr (TA == 0) {
          int tap = 0, nc = kc;
          if (p.conv) {
            // input pixel (y, x) receives output pixel (y + 1 - kh, x + 1 - kw) through tap (kh, kw)
            tap = kc / p.chunks_per_tap;
            nc = kc - tap * p.chunks_per_tap;
            const int kh = tap / 3, kw = tap - kh * 3;
            if constexpr (IM2COL) tma_load_im2col_4d(sa, &p.tmD, &full_bar[s], nc * 64, x0 - 1, y0 - 1, b0, 2 - kw, 2 - kh);
            else tma_load_4d(sa, &p.tmD, &full_bar[s], nc * 64, x0 + 1 - kw, y0 + 1 - kh, b0);
          } else {
            tma_load_2d(sa, &p.tmD, &full_bar[s], kc * 64, r0);
          }
          for (int j = 0; j < b_chunks; ++j)
            tma_load_2d(sb + j * kGbChunk, &p.tmB, &full_bar[s], tap * p.c + c0 + j * 64, nc * 64);
        } else {
          for (int h = 0; h * kGbChunk < a_bytes; ++h)
            tma_load_2d(sa + h * kGbChunk, &p.tmD, &full_bar[s], r0 + h * 64, kc * 64);
          const int m = kc * 64;  // first row of the forward's A in this stage (conv: output pixel)
          for (int j = 0; j < b_chunks; ++j) {
            const int col = c0 + j * 64;
            if (p.conv) {
              const int tap = col / p.c, cc = col - tap * p.c;
              const int kh = tap / 3, kw = tap - kh * 3;
              const int bb = m / p.hw, rem = m - bb * p.hw;
              const int yy = rem / p.w, xx = rem - yy * p.w;
              if constexpr (IM2COL) {
                if (cc < p.k1)
                  tma_load_im2col_4d(sb + j * kGbChunk, &p.tmB, &full_bar[s], cc, p.cs * xx - 1, p.cs * yy - 1, bb, kw, kh);
                else
                  tma_load_im2col_4d(sb + j * kGbChunk, &p.tmB2, &full_bar[s], cc - p.k1, p.cs * xx - 1, p.cs * yy - 1, bb,
                                     kw, kh);
              } else {
                tma_load_4d(sb + j * kGbChunk, &p.tmB, &full_bar[s], cc, p.cs * xx + kw - 1, p.cs * yy + kh - 1, bb);
              }
            } else if (col < p.k1) {
              tma_load_2d(sb + j * kGbChunk, &p.tmB, &full_bar[s], col, m);
            } else {
              tma_load_2d(sb + j * kGbChunk, &p.tmB2, &full_bar[s], col - p.k1, m);
            }
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float acc[kGbN / 2];
#pragma unroll
  for (int i = 0; i < kGbN / 2; ++i) acc[i] = 0.f;
  for (int it = 0; it < n_iter; ++it) {
    const int s = ring_wait_full<kGbStages>(full_bar, it);
    const uint32_t a_addr = smem_u32(smem + s * kGbStageBytes) + wg * kGbChunk;  // this warpgroup's 64 rows
    const uint32_t b_addr = smem_u32(smem + s * kGbStageBytes) + kGbABytes;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kGbK / 16; ++k) {
      if constexpr (TA == 0)
        wgmma_ss<kGbN, 0, 1>(acc, wgmma_desc_k_sw128(a_addr) + 2 * k, wgmma_desc_mn_sw128(b_addr + k * 2048, kGbChunk),
                             1u);
      else
        wgmma_ss<kGbN, 1, 1>(acc, wgmma_desc_mn_sw128(a_addr + k * 2048, kGbChunk),
                             wgmma_desc_mn_sw128(b_addr + k * 2048, kGbChunk), 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous stage's MMAs have finished reading it
    wgmma_fence_regs(acc);
    if (it > 0) mbar_arrive(&empty_bar[(it - 1) % kGbStages]);
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  // acc[j]: row 16 (warp & 3) + lane / 4 + 8 ((j / 2) & 1) of the warpgroup's 64, column 8 (j / 4) + 2 (lane & 3)
  const int row0 = r0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < kGbN / 2; j += 2) {
    const long long row = row0 + 8 * ((j >> 1) & 1);
    const int col = c0 + 8 * (j >> 2) + 2 * (lane & 3);
    if (row < p.rows && col < p.cols) {
      if (p.splits > 1)
        *reinterpret_cast<float2*>(p.ws + (static_cast<long long>(split) * p.rows + row) * p.cols + col) =
            make_float2(acc[j], acc[j + 1]);
      else
        gb_put(p, row, col, acc[j], acc[j + 1]);
    }
  }
}

template <int TA>
__global__ void __launch_bounds__(kWsThreads, 2) gemm_bwd_kernel(const __grid_constant__ GemmBwdKParams p) {
  gemm_bwd_body<TA, false>(p);
}

template <int TA>
__global__ void __launch_bounds__(kWsThreads, 2) gemm_bwd_igemm_kernel(const __grid_constant__ GemmBwdKParams p) {
  gemm_bwd_body<TA, true>(p);
}

// the split reduction's second pass: slabs summed in split order, then the destination's dtype / accumulate
__global__ void gemm_bwd_finalize_kernel(const __grid_constant__ GemmBwdKParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const long long slab = static_cast<long long>(p.rows) * p.cols;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 2; i < slab;
       i += static_cast<long long>(gridDim.x) * blockDim.x * 2) {
    float2 v = *reinterpret_cast<const float2*>(p.ws + i);
    for (int s = 1; s < p.splits; ++s) {
      const float2 b = *reinterpret_cast<const float2*>(p.ws + s * slab + i);
      v.x += b.x;
      v.y += b.y;
    }
    const long long row = i / p.cols;
    gb_put(p, row, static_cast<int>(i - row * p.cols), v.x, v.y);
  }
}

// dA of a 3x3 pad-1 conv from the column gradient col[M_out][9c] (fp32, K order (kh, kw, c)): input pixel (y, x)
// sums, over the taps in (kh, kw) order, the output pixel (y + 1 - kh, x + 1 - kw) / stride where that is one
__global__ void col2im_gather_kernel(const float* col, GbOut out, int batch, int h, int w, int c, int stride, int ho,
                                     int wo) {
  pdl_launch_dependents();
  pdl_wait();
  const int pairs = c / 2;
  const long long total = static_cast<long long>(batch) * h * w * pairs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(i % pairs) * 2;
    const long long pix = i / pairs;
    const int x = static_cast<int>(pix % w);
    const int y = static_cast<int>((pix / w) % h);
    const int b = static_cast<int>(pix / (static_cast<long long>(w) * h));
    float2 s = make_float2(0.f, 0.f);
    for (int kh = 0; kh < 3; ++kh) {
      const int ys = y + 1 - kh;
      if (ys < 0 || ys % stride != 0 || ys / stride >= ho) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int xs = x + 1 - kw;
        if (xs < 0 || xs % stride != 0 || xs / stride >= wo) continue;
        const long long orow = (static_cast<long long>(b) * ho + ys / stride) * wo + xs / stride;
        const float2 v = *reinterpret_cast<const float2*>(col + orow * 9 * c + (kh * 3 + kw) * c + ch);
        s.x += v.x;
        s.y += v.y;
      }
    }
    gb_store2(out, pix, ch, s.x, s.y);
  }
}

// dbias, first pass: block (32, 8) sums rows [seg * rpb + part * kBiasRows, ...) of 32 columns in a fixed order
__global__ void colsum_partial_kernel(const __half* dd, long long ldd, int m, int n, int rpb, int parts, float* ws) {
  __shared__ float red[8][33];
  pdl_launch_dependents();
  pdl_wait();
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int seg = blockIdx.y / parts, part = blockIdx.y - seg * parts;
  const long long seg_end = min(static_cast<long long>(seg + 1) * rpb, static_cast<long long>(m));
  const long long r_begin = static_cast<long long>(seg) * rpb + static_cast<long long>(part) * kBiasRows;
  const long long r_end = min(r_begin + kBiasRows, seg_end);
  float s = 0.f;
  if (col < n)
    for (long long r = r_begin + threadIdx.y; r < r_end; r += 8) s += __half2float(dd[r * ldd + col]);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < n) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    ws[static_cast<long long>(blockIdx.y) * n + col] = t;
  }
}

// dbias, second pass: each (segment, column) sums its parts in order
__global__ void colsum_finalize_kernel(const float* ws, int n, int segs, int parts, float* dbias, long long stride,
                                       int acc) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < static_cast<long long>(segs) * n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int seg = static_cast<int>(i / n), col = static_cast<int>(i - static_cast<long long>(seg) * n);
    float t = 0.f;
    for (int q = 0; q < parts; ++q) t += ws[(static_cast<long long>(seg) * parts + q) * n + col];
    float* d = dbias + seg * stride + col;
    *d = acc ? *d + t : t;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------------
struct GbPlan {
  bool da, db, dbias;
  int m, cs, ho, wo;
  bool da_col;           // conv dA through the fp32 column buffer + col2im_gather_kernel
  bool db_col;           // conv dB through im2col
  int da_splits, da_cps, db_splits, db_cps;
  long long da_col_floats, db_col_floats;
  int bias_segs, bias_rpb, bias_parts;
  long long ws_floats;
};

static void pick_splits(int requested, long long tiles, int chunks, int* splits, int* cps) {
  int s = requested;
  if (s <= 0) {  // automatic: about two CTAs per SM, every split keeps at least 8 chunks (512 rows of the reduction)
    s = static_cast<int>(2 * kNumSms / tiles);
    s = min(s, chunks / 8);
    s = min(s, 16);
  }
  s = max(1, min(s, chunks));
  *cps = (chunks + s - 1) / s;
  *splits = (chunks + *cps - 1) / *cps;  // no empty splits
}

static bool out_ok(const void* p, long long ld, int dtype) {
  return (reinterpret_cast<uintptr_t>(p) & 15) == 0 && ld % 8 == 0 && (dtype == MDB_DTYPE_F16 || dtype == MDB_DTYPE_F32);
}

// igemm: the conv at any latent size (mdb_conv3x3_igemm_bwd_f16): dB and stride-1 dA through im2col loads, one or
// two sources; fn names the entry point in messages
static int plan_bwd(const mdb_gemm_bwd_desc* g, GbPlan* pl, bool igemm, const char* fn) {
  MDB_REQUIRE(g != nullptr, "%s: null descriptor", fn);
  const mdb_gemm_desc* f = &g->fwd;
  memset(pl, 0, sizeof(*pl));
  MDB_REQUIRE(f->epilogue == MDB_EPI_NONE,
              "%s: the GEGLU epilogue has no backward here (differentiate the plain GEMM and the "
              "activation separately)", fn);
  MDB_REQUIRE(f->ln_u == nullptr, "%s: the folded LayerNorm (ln_u) has no backward here", fn);
  MDB_REQUIRE(f->m > 0 && f->n > 0 && f->k > 0 && f->k % 64 == 0, "%s: bad shape m=%d n=%d k=%d", fn,
              f->m, f->n, f->k);
  MDB_REQUIRE(g->dd != nullptr && g->lddd % 8 == 0 && g->lddd >= f->n && (reinterpret_cast<uintptr_t>(g->dd) & 15) == 0,
              "%s: dd must be 16B aligned with lddd %% 8 == 0 and lddd >= n (lddd=%lld)", fn,
              (long long)g->lddd);
  MDB_REQUIRE(g->splits >= 0 && f->splits >= 0, "%s: negative split count", fn);
  pl->da = g->da != nullptr || g->da2 != nullptr;
  pl->db = g->db != nullptr;
  pl->dbias = g->dbias != nullptr;
  if (g->da) MDB_REQUIRE(out_ok(g->da, g->ldda, g->da_dtype), "%s: da must be 16B aligned, ldda %% 8 == 0, dtype 0|1", fn);
  if (g->da2) MDB_REQUIRE(out_ok(g->da2, g->ldda2, g->da2_dtype), "%s: da2 must be 16B aligned, ldda2 %% 8 == 0, dtype 0|1", fn);
  if (g->db) MDB_REQUIRE(out_ok(g->db, g->lddb, g->db_dtype), "%s: db must be 16B aligned, lddb %% 8 == 0, dtype 0|1", fn);
  if (pl->da) MDB_REQUIRE(f->b != nullptr && f->ldb % 8 == 0, "%s: dA needs the forward's b (ldb %% 8 == 0)", fn);
  if (pl->db) MDB_REQUIRE(f->a != nullptr, "%s: dB needs the forward's a", fn);
  if (f->bias_batch_stride != 0)
    MDB_REQUIRE(f->rows_per_batch > 0 && f->bias_batch_stride >= f->n,
                "%s: a per-batch bias needs rows_per_batch > 0 and bias_batch_stride >= n", fn);
  pl->m = f->m;
  if (igemm) MDB_REQUIRE(f->conv != 0, "%s: conv must be the stride, 1 or 2 (got 0)", fn);
  if (f->conv) {
    MDB_REQUIRE(f->conv == 1 || f->conv == 2, "%s: conv must be 1 or 2 (stride), got %d", fn, f->conv);
    MDB_REQUIRE(igemm || f->a2 == nullptr, "%s: conv mode takes a single source", fn);
    MDB_REQUIRE(f->c % 64 == 0 && f->k == 9 * f->c && f->nb > 0 && f->h > 0 && f->w > 0,
                "%s: conv needs c %% 64 == 0 and k == 9c (c=%d k=%d)", fn, f->c, f->k);
    pl->cs = f->conv;
    pl->ho = (f->h - 1) / pl->cs + 1;
    pl->wo = (f->w - 1) / pl->cs + 1;
    MDB_REQUIRE(f->m == f->nb * pl->ho * pl->wo, "%s: conv m != nb*ho*wo", fn);
    if (igemm) {
      // two sources: channels [0, k1) of every pixel from a (and dA to da), [k1, c) from a2 (dA to da2)
      const int c1 = f->a2 ? f->k1 : f->c;
      MDB_REQUIRE(c1 > 0 && c1 % 64 == 0 && (f->a2 ? c1 < f->c : c1 == f->c),
                  "%s: with a2, k1 (the channels taken from a) must be a multiple of 64 below c (k1=%d c=%d)", fn, c1,
                  f->c);
      const long long lda = f->lda > 0 ? f->lda : c1, lda2 = f->lda2 > 0 ? f->lda2 : f->c - c1;
      if (pl->db)
        MDB_REQUIRE(lda >= c1 && lda % 8 == 0 && (!f->a2 || (lda2 >= f->c - c1 && lda2 % 8 == 0)),
                    "%s: the pixel strides lda / lda2 must cover their channels and be multiples of 8", fn);
      MDB_REQUIRE(g->da2 == nullptr || f->a2 != nullptr, "%s: da2 without a second source", fn);
      MDB_REQUIRE(!(pl->da && f->a2 && pl->cs == 2), "%s: stride-2 dA of a two-source conv is not supported", fn);
    } else if (pl->da) {
      MDB_REQUIRE(g->da != nullptr && g->da2 == nullptr, "%s: conv dA goes to da only", fn);
    }
    // pixels that do not form TMA boxes take the column path (igemm: only stride-2 dA, im2col loads otherwise)
    uint32_t box[4];
    pl->da_col = pl->cs == 2 || (!igemm && pixel_box(f->h, f->w, 1, kGbM, false, box) != kBoxOk);
    pl->db_col = !igemm && pixel_box(pl->ho, pl->wo, pl->cs, 64, false, box) != kBoxOk;
  } else {
    const int k1 = f->a2 ? f->k1 : f->k;
    MDB_REQUIRE(k1 % 64 == 0 && k1 > 0 && k1 <= f->k, "%s: k1=%d must be a multiple of 64 within K", fn, k1);
    if (pl->db) MDB_REQUIRE(f->lda % 8 == 0 && (!f->a2 || f->lda2 % 8 == 0), "%s: lda %% 8 == 0", fn);
    MDB_REQUIRE(g->da2 == nullptr || f->a2 != nullptr, "%s: da2 without a second source", fn);
  }
  long long ws = 0;
  const long long k_tiles = (f->k + kGbN - 1) / kGbN;
  if (pl->da) {
    // implicit conv: [nb*h*w][c] over 9 taps of N; otherwise [M][K] over N (the column path's dCol is [M_out][9c])
    const bool implicit = f->conv && !pl->da_col;
    const int chunks = implicit ? 9 * ((f->n + 63) / 64) : (f->n + 63) / 64;
    const long long dst_rows = implicit ? static_cast<long long>(f->nb) * f->h * f->w : f->m;
    const long long dst_cols = implicit ? f->c : f->k;
    pick_splits(f->splits, (dst_rows + kGbM - 1) / kGbM * ((dst_cols + kGbN - 1) / kGbN), chunks, &pl->da_splits,
                &pl->da_cps);
    pl->da_col_floats = pl->da_col ? static_cast<long long>(f->m) * f->k : 0;
    const long long slabs = pl->da_splits > 1 ? pl->da_splits * dst_rows * dst_cols : 0;
    ws = max(ws, pl->da_col_floats + slabs);
  }
  if (pl->db) {
    const int chunks = (f->m + 63) / 64;
    pick_splits(g->splits, (long long)(f->n + kGbM - 1) / kGbM * k_tiles, chunks, &pl->db_splits, &pl->db_cps);
    pl->db_col_floats = pl->db_col ? (static_cast<long long>(f->m) * f->k / 2 + 3) / 4 * 4 : 0;  // fp16 im2col
    const long long slabs = pl->db_splits > 1 ? static_cast<long long>(pl->db_splits) * f->n * f->k : 0;
    ws = max(ws, pl->db_col_floats + slabs);
  }
  if (pl->dbias) {
    pl->bias_rpb = f->bias_batch_stride != 0 ? f->rows_per_batch : f->m;
    pl->bias_segs = (f->m + pl->bias_rpb - 1) / pl->bias_rpb;
    pl->bias_parts = (pl->bias_rpb + kBiasRows - 1) / kBiasRows;
    ws = max(ws, static_cast<long long>(pl->bias_segs) * pl->bias_parts * f->n);
  }
  pl->ws_floats = ws;
  return MDB_OK;
}

template <auto kern>
static int launch_bwd_kernel(const GemmBwdKParams& kp, dim3 grid, cudaStream_t st) {
  if (int rc = set_max_dyn_smem<kern>(kGbSmem)) return rc;
  MDB_CHECK_CUDA(launch_pdl(kern, grid, dim3(kWsThreads), kGbSmem, st, kp));
  return MDB_OK;
}

static int launch_bwd_gemm(int ta, GemmBwdKParams& kp, int tiles_x, int splits, int cps, cudaStream_t st,
                           bool igemm = false) {
  kp.splits = splits;
  kp.chunks_per_split = cps;
  const dim3 grid(tiles_x, (kp.cols + kGbN - 1) / kGbN, splits);
  const int rc = igemm ? (ta == 0 ? launch_bwd_kernel<gemm_bwd_igemm_kernel<0>>(kp, grid, st)
                                  : launch_bwd_kernel<gemm_bwd_igemm_kernel<1>>(kp, grid, st))
                       : (ta == 0 ? launch_bwd_kernel<gemm_bwd_kernel<0>>(kp, grid, st)
                                  : launch_bwd_kernel<gemm_bwd_kernel<1>>(kp, grid, st));
  if (rc) return rc;
  count_launch();
  if (splits > 1) {
    const long long pairs = static_cast<long long>(kp.rows) * kp.cols / 2;
    const int blocks = static_cast<int>(min((pairs + 255) / 256, static_cast<long long>(kNumSms) * 8));
    MDB_CHECK_CUDA(launch_pdl(gemm_bwd_finalize_kernel, dim3(blocks), dim3(256), 0, st, kp));
    count_launch();
  }
  return MDB_OK;
}

static int run_da(const mdb_gemm_bwd_desc* g, const GbPlan& pl, cudaStream_t st, bool igemm = false) {
  const mdb_gemm_desc* f = &g->fwd;
  GemmBwdKParams kp;
  memset(&kp, 0, sizeof(kp));
  int rc;
  // the forward's B [N][K]: 64 columns x 64 rows (the reduction) per box, read MN-major
  if ((rc = tmap_rows(&kp.tmB, f->b, f->k, f->n, f->ldb, 64, 64))) return rc;
  kp.cols = f->k;
  int tiles_x;
  if (f->conv && !pl.da_col) {  // stride 1, implicit: the row tiles are input pixels
    if (igemm) {
      if ((rc = tmap_nhwc_im2col(&kp.tmD, g->dd, f->n, f->w, f->h, f->nb, g->lddd, kGbM, 1))) return rc;
    } else {
      uint32_t box[4];
      pixel_box(f->h, f->w, 1, kGbM, false, box);
      if ((rc = tmap_nhwc(&kp.tmD, g->dd, f->n, f->w, f->h, f->nb, g->lddd, box, 1))) return rc;
    }
    kp.conv = 1;
    kp.chunks_per_tap = (f->n + 63) / 64;
    kp.chunks = 9 * kp.chunks_per_tap;
    kp.c = f->c;
    kp.w = f->w;
    kp.hw = f->h * f->w;
    kp.cs = 1;
    kp.rows = f->nb * f->h * f->w;
    kp.cols = f->c;
    kp.out[0] = gb_out(g->da, g->ldda, g->da_dtype, g->da_accumulate);
    kp.split_col = f->c;
    if (igemm && f->a2) {  // channels [k1, c) of every input pixel are the second source's
      kp.out[1] = gb_out(g->da2, g->ldda2, g->da2_dtype, g->da2_accumulate);
      kp.split_col = f->k1;
    }
  } else {
    if ((rc = tmap_rows(&kp.tmD, g->dd, f->n, f->m, g->lddd, 64, kGbM))) return rc;
    kp.chunks = (f->n + 63) / 64;
    kp.rows = f->m;
    if (pl.da_col) {
      kp.out[0] = gb_out(g->ws, f->k, MDB_DTYPE_F32, 0);
      kp.split_col = f->k;
    } else {
      kp.out[0] = gb_out(g->da, g->ldda, g->da_dtype, g->da_accumulate);
      kp.out[1] = gb_out(g->da2, g->ldda2, g->da2_dtype, g->da2_accumulate);
      kp.split_col = f->a2 ? f->k1 : f->k;
    }
  }
  tiles_x = (kp.rows + kGbM - 1) / kGbM;
  kp.ws = g->ws + pl.da_col_floats;
  if ((rc = launch_bwd_gemm(0, kp, tiles_x, pl.da_splits, pl.da_cps, st, igemm && kp.conv))) return rc;
  if (pl.da_col) {
    const long long total = static_cast<long long>(f->nb) * f->h * f->w * (f->c / 2);
    const int blocks = static_cast<int>(min((total + 255) / 256, static_cast<long long>(kNumSms) * 16));
    MDB_CHECK_CUDA(launch_pdl(col2im_gather_kernel, dim3(blocks), dim3(256), 0, st, static_cast<const float*>(g->ws),
                              gb_out(g->da, g->ldda, g->da_dtype, g->da_accumulate), f->nb, f->h, f->w, f->c, pl.cs,
                              pl.ho, pl.wo));
    count_launch();
  }
  return MDB_OK;
}

static int run_db(const mdb_gemm_bwd_desc* g, const GbPlan& pl, cudaStream_t st, bool igemm = false) {
  const mdb_gemm_desc* f = &g->fwd;
  GemmBwdKParams kp;
  memset(&kp, 0, sizeof(kp));
  int rc;
  // dD^T: 64 of N x 64 of M per box, read MN-major
  if ((rc = tmap_rows(&kp.tmD, g->dd, f->n, f->m, g->lddd, 64, 64))) return rc;
  if (igemm) {  // 64 output pixels x 64 channels of one tap per im2col load, from a or a2
    const int c1 = f->a2 ? f->k1 : f->c;
    if ((rc = tmap_nhwc_im2col(&kp.tmB, f->a, c1, f->w, f->h, f->nb, f->lda > 0 ? f->lda : c1, 64, pl.cs))) return rc;
    if (f->a2 && (rc = tmap_nhwc_im2col(&kp.tmB2, f->a2, f->c - c1, f->w, f->h, f->nb,
                                        f->lda2 > 0 ? f->lda2 : f->c - c1, 64, pl.cs)))
      return rc;
    kp.conv = 1;
    kp.c = f->c;
    kp.k1 = c1;
    kp.w = pl.wo;
    kp.hw = pl.ho * pl.wo;
    kp.cs = pl.cs;
  } else if (f->conv && !pl.db_col) {  // the forward's shifted pixel boxes, 64 output pixels x 64 channels of one tap
    uint32_t box[4];
    pixel_box(pl.ho, pl.wo, pl.cs, 64, false, box);
    if ((rc = tmap_nhwc(&kp.tmB, f->a, f->c, f->w, f->h, f->nb, f->c, box, pl.cs))) return rc;
    kp.conv = 1;
    kp.c = f->c;
    kp.w = pl.wo;
    kp.hw = pl.ho * pl.wo;
    kp.cs = pl.cs;
  } else if (f->conv) {  // latents that do not tile: im2col into the workspace, then the plain path
    if ((rc = mdb_im2col3x3_f16(f->a, g->ws, f->nb, f->h, f->w, f->c, pl.cs, st))) return rc;
    if ((rc = tmap_rows(&kp.tmB, g->ws, f->k, f->m, f->k, 64, 64))) return rc;
    kp.k1 = f->k;
  } else {
    const int k1 = f->a2 ? f->k1 : f->k;
    if ((rc = tmap_rows(&kp.tmB, f->a, k1, f->m, f->lda, 64, 64))) return rc;
    if (f->a2 && (rc = tmap_rows(&kp.tmB2, f->a2, f->k - k1, f->m, f->lda2, 64, 64))) return rc;
    kp.k1 = k1;
  }
  kp.rows = f->n;
  kp.cols = f->k;
  kp.chunks = (f->m + 63) / 64;
  kp.out[0] = gb_out(g->db, g->lddb, g->db_dtype, g->db_accumulate);
  kp.split_col = f->k;
  kp.ws = g->ws + pl.db_col_floats;
  return launch_bwd_gemm(1, kp, (f->n + kGbM - 1) / kGbM, pl.db_splits, pl.db_cps, st, igemm);
}

static int run_dbias(const mdb_gemm_bwd_desc* g, const GbPlan& pl, cudaStream_t st) {
  const mdb_gemm_desc* f = &g->fwd;
  const dim3 grid((f->n + 31) / 32, pl.bias_segs * pl.bias_parts);
  MDB_CHECK_CUDA(launch_pdl(colsum_partial_kernel, grid, dim3(32, 8), 0, st, static_cast<const __half*>(g->dd),
                            (long long)g->lddd, f->m, f->n, pl.bias_rpb, pl.bias_parts, g->ws));
  count_launch();
  return launch_colsum_finalize(g->ws, f->n, pl.bias_segs, pl.bias_parts, g->dbias,
                                f->bias_batch_stride != 0 ? f->bias_batch_stride : 0, g->dbias_accumulate, st);
}

int launch_colsum_finalize(const float* ws, int n, int segs, int parts, float* out, long long stride, int acc,
                           cudaStream_t st) {
  const long long total = static_cast<long long>(segs) * n;
  MDB_CHECK_CUDA(launch_pdl(colsum_finalize_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, st,
                            ws, n, segs, parts, out, stride, acc));
  count_launch();
  return MDB_OK;
}

}  // namespace mdb

using namespace mdb;

static int run_bwd(const mdb_gemm_bwd_desc* g, mdb_stream_t stream, bool igemm, const char* fn, const char* ws_fn) {
  GbPlan pl;
  int rc = plan_bwd(g, &pl, igemm, fn);
  if (rc) return rc;
  MDB_REQUIRE(pl.ws_floats == 0 || (g->ws != nullptr && (reinterpret_cast<uintptr_t>(g->ws) & 15) == 0),
              "%s: needs a 16B-aligned workspace of %s() = %lld floats", fn, ws_fn, (long long)pl.ws_floats);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // the phases run one after the other on the stream and share the workspace
  if (pl.da && (rc = run_da(g, pl, st, igemm))) return rc;
  if (pl.db && (rc = run_db(g, pl, st, igemm))) return rc;
  if (pl.dbias && (rc = run_dbias(g, pl, st))) return rc;
  return MDB_OK;
}

extern "C" int64_t mdb_gemm_bwd_ws_floats(const mdb_gemm_bwd_desc* g) {
  GbPlan pl;
  const int rc = plan_bwd(g, &pl, false, "mdb_gemm_bwd_f16");
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_gemm_bwd_f16(const mdb_gemm_bwd_desc* g, mdb_stream_t stream) {
  return run_bwd(g, stream, false, "mdb_gemm_bwd_f16", "mdb_gemm_bwd_ws_floats");
}

extern "C" int64_t mdb_conv3x3_igemm_bwd_ws_floats(const mdb_gemm_bwd_desc* g) {
  GbPlan pl;
  const int rc = plan_bwd(g, &pl, true, "mdb_conv3x3_igemm_bwd_f16");
  return rc ? rc : pl.ws_floats;
}

extern "C" int mdb_conv3x3_igemm_bwd_f16(const mdb_gemm_bwd_desc* g, mdb_stream_t stream) {
  return run_bwd(g, stream, true, "mdb_conv3x3_igemm_bwd_f16", "mdb_conv3x3_igemm_bwd_ws_floats");
}
