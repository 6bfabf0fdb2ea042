// Pieces the GroupNorm / LayerNorm forward (norm.cu) and backward (norm_bwd.cu) share: source addressing of the
// fused channel concat, the group pivot, the LayerNorm row statistics and the GroupNorm statistics launch.
#pragma once

#include "common.cuh"

namespace mdb {

constexpr int kGnMaxBatch = 1024;  // batch elements of the two-kernel path (size of the ticket region)

#ifdef __CUDACC__
__device__ __forceinline__ const uint4* gn_src(const __half* x1, int c1, const __half* x2, int c2, long long row,
                                                int ch) {
  // channel ch (multiple of 8) of concatenated row -> address of its 16-byte vector
  return (ch < c1) ? reinterpret_cast<const uint4*>(x1 + row * c1 + ch)
                   : reinterpret_cast<const uint4*>(x2 + row * c2 + (ch - c1));
}

// pivot of group g of batch element b: the group's first channel at pixel 0
__device__ __forceinline__ float gn_pivot(const __half* x1, int c1, const __half* x2, int c2, int b, int hw, int ch) {
  return (ch < c1) ? __half2float(x1[static_cast<long long>(b) * hw * c1 + ch])
                   : __half2float(x2[static_cast<long long>(b) * hw * c2 + (ch - c1)]);
}

// LayerNorm row statistics, one warp per row: lane holds the half2 pairs lane, lane + 32, ... of the row in v; the
// backward recomputes them with this same code, so its mean / rstd are bit-identical to the forward's
template <int VPL>  // half2 pairs per lane
__device__ __forceinline__ void ln_row_stats(const __half2* xr, int lane, int c, float eps, float2 (&v)[VPL],
                                             float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    v[i] = __half22float2(xr[lane + i * 32]);
    s += v[i].x + v[i].y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  mean = s / c;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean;
    q += dx * dx + dy * dy;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  rstd = rsqrtf(q / c + eps);
}
#endif  // __CUDACC__

// rows per stats CTA / stats grid of gn_stats_kernel (norm.cu)
void gn_stats_geometry(int c, int batch, int hw, int* threads_out, int* rows_per_cta_out, int* nblk_out);
// launches gn_stats_kernel: (mean, var) of every (batch element, group) at ws + kGnMaxBatch, [batch][32][2]; ws as
// mdb_groupnorm_ws_floats sizes it, ZERO when first used.  Counts no launch.
int launch_gn_stats(const __half* x1, int c1, const __half* x2, int c2, float* ws, int batch, int hw,
                    cudaStream_t st);

}  // namespace mdb
