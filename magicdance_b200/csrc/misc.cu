// HBM-bound helper kernels of the denoising step: direct 3x3 conv for non-GEMM-shaped layers,
// im2col (stride-2 downsample), nearest x2 upsample, residual add, timestep embedding, skinny
// Linear for the timestep MLPs, NCHW fp32 <-> NHWC fp16 boundary converts, fused CFG + DDIM update.
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include "common.cuh"

namespace mdb {

// ---------------------------------------------------------------------------------------------
// plumbing
// ---------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
bool pdl_enabled() { return true; }  // every launch carries the programmatic-stream-serialization attribute

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

// fp16 tiled map with 128B swizzle; dims[0] is the contiguous dimension; strides_bytes[i] is the byte stride of
// dims[i+1]; elem_strides: TMA element strides (nullptr = 1 along every dimension)
static int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides = nullptr) {
  if (g_encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
      return MDB_ERR_CUDA;
    }
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("TMA base address %p is not 16-byte aligned", base);
    return MDB_ERR_INVALID;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("TMA stride %d (%llu bytes) is not a multiple of 16", i, (unsigned long long)gstr[i]);
      return MDB_ERR_INVALID;
    }
  }
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstr, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu,%llu box %u,%u)", (int)r, rank,
              (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0), bx[0], rank > 1 ? bx[1] : 0);
    return MDB_ERR_CUDA;
  }
  return MDB_OK;
}

int tmap_rows(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, long long ld, uint32_t box_inner,
              uint32_t box_rows) {
  const uint64_t dims[2] = {inner, rows};
  const uint64_t str[1] = {(uint64_t)ld * 2};
  const uint32_t box[2] = {box_inner, box_rows};
  return make_tmap_f16(out, base, 2, dims, str, box);
}

int tmap_heads(CUtensorMap* out, const void* base, int d, int heads, uint64_t tokens, long long ld,
               uint32_t box_tokens) {
  const uint64_t dims[3] = {(uint64_t)d, (uint64_t)heads, tokens};
  const uint64_t str[2] = {(uint64_t)d * 2, (uint64_t)ld * 2};
  const uint32_t box[3] = {64, 1, box_tokens};
  return make_tmap_f16(out, base, 3, dims, str, box);
}

int tmap_heads_per_sample(CUtensorMap* out, const void* base, int d, int heads, int n, int nb, long long ld,
                          uint32_t box_tokens) {
  const uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)n, (uint64_t)nb};
  const uint64_t str[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)ld * n * 2};
  const uint32_t box[4] = {64, 1, box_tokens, 1};
  return make_tmap_f16(out, base, 4, dims, str, box);
}

int tmap_vt(CUtensorMap* out, const void* base, int n, int nb, long long ldvb, int rows, long long ldvt,
            uint32_t box_rows) {
  const uint64_t dims[3] = {(uint64_t)n, (uint64_t)nb, (uint64_t)rows};
  const uint64_t str[2] = {(uint64_t)ldvb * 2, (uint64_t)ldvt * 2};
  const uint32_t box[3] = {64, 1, box_rows};
  return make_tmap_f16(out, base, 3, dims, str, box);
}

int tmap_nhwc(CUtensorMap* out, const void* base, int c, int w, int h, int nb, long long ld, const uint32_t box[4],
              int cs) {
  const uint64_t dims[4] = {(uint64_t)c, (uint64_t)w, (uint64_t)h, (uint64_t)nb};
  const uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * w * 2, (uint64_t)ld * h * w * 2};
  const uint32_t estr[4] = {1u, (uint32_t)cs, (uint32_t)cs, 1u};
  return make_tmap_f16(out, base, 4, dims, str, box, cs == 2 ? estr : nullptr);
}

static PFN_cuTensorMapEncodeIm2col_v12000 g_encode_im2col = nullptr;

int tmap_nhwc_im2col(CUtensorMap* out, const void* base, int c, int w, int h, int nb, long long ld, int pixels,
                     int cs) {
  if (g_encode_im2col == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeIm2col not available from the driver (%s)", cudaGetErrorString(e));
      return MDB_ERR_CUDA;
    }
    g_encode_im2col = reinterpret_cast<PFN_cuTensorMapEncodeIm2col_v12000>(fn);
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || ld % 8 != 0) {
    set_error("TMA im2col map: base %p must be 16-byte aligned and the pixel stride (%lld) a multiple of 8", base, ld);
    return MDB_ERR_INVALID;
  }
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)nb};
  const cuuint64_t str[3] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * w * 2, (cuuint64_t)ld * h * w * 2};
  // The bounding box of window corners, per image, runs along w from lower[0] to w - 1 + upper[0] (and likewise along
  // h) in steps of cs: corners -1 .. w - 2 are the (w - 1) / cs + 1 output columns of a pad-1 3x3 conv, and a
  // corner plus its tap offset (0..2) is the input pixel read, -1 .. w (the halo, zero-filled)
  const int lower[2] = {-1, -1};
  const int upper[2] = {-1, -1};
  const cuuint32_t estr[4] = {1u, (cuuint32_t)cs, (cuuint32_t)cs, 1u};
  CUresult r = g_encode_im2col(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, str, lower, upper,
                               64, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeIm2col failed with CUresult %d (c %d, w %d, h %d, nb %d, %d pixels, stride %d)", (int)r,
              c, w, h, nb, pixels, cs);
    return MDB_ERR_CUDA;
  }
  return MDB_OK;
}

// ---------------------------------------------------------------------------------------------
// direct 3x3 conv, pad 1, stride 1|2, NHWC fp16, fp32 accumulate.
// CTA: 8x8 output pixels x 32 output channels; input patch (with halo) and the weight slab for a
// 16-channel slice of cin are staged in shared memory; each thread owns 1 pixel x 8 couts.
// ---------------------------------------------------------------------------------------------
constexpr int kDcTile = 8;
constexpr int kDcCout = 32;
constexpr int kDcCin = 16;

template <int STRIDE>
__global__ void __launch_bounds__(256) direct_conv3x3_kernel(const __half* __restrict__ x, const __half* __restrict__ wt,
                                                             const float* __restrict__ bias,
                                                             const __half* __restrict__ residual, __half* __restrict__ y,
                                                             int h, int w, int cin, int cout, int ho, int wo, int silu) {
  constexpr int PH = (kDcTile - 1) * STRIDE + 3;  // patch height/width
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_in[PH * PH * kDcCin];
  __shared__ float s_w[kDcCout * 9 * kDcCin];
  const int tiles_x = (wo + kDcTile - 1) / kDcTile;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int co0 = blockIdx.y * kDcCout;
  const int b = blockIdx.z;
  const int px = threadIdx.x % 64;            // pixel within tile
  const int cgp = threadIdx.x / 64;           // cout group of 8 (4 groups)
  const int oy = ty * kDcTile + px / kDcTile, ox = tx * kDcTile + px % kDcTile;
  const int iy0 = ty * kDcTile * STRIDE - 1, ix0 = tx * kDcTile * STRIDE - 1;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  for (int c0 = 0; c0 < cin; c0 += kDcCin) {
    const int cs = min(kDcCin, cin - c0);
    for (int i = threadIdx.x; i < PH * PH * kDcCin; i += blockDim.x) {
      const int ci = i % kDcCin, pp = i / kDcCin;
      const int yy = iy0 + pp / PH, xx = ix0 + pp % PH;
      float v = 0.f;
      if (ci < cs && yy >= 0 && yy < h && xx >= 0 && xx < w)
        v = __half2float(x[((static_cast<long long>(b) * h + yy) * w + xx) * cin + c0 + ci]);
      s_in[i] = v;
    }
    for (int i = threadIdx.x; i < kDcCout * 9 * kDcCin; i += blockDim.x) {
      const int ci = i % kDcCin, t = (i / kDcCin) % 9, co = i / (kDcCin * 9);
      float v = 0.f;
      if (ci < cs && co0 + co < cout) v = __half2float(wt[(static_cast<long long>(co0 + co) * 9 + t) * cin + c0 + ci]);
      s_w[i] = v;
    }
    __syncthreads();
    const int py = (px / kDcTile) * STRIDE, pxx = (px % kDcTile) * STRIDE;
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float* ip = &s_in[((py + t / 3) * PH + pxx + t % 3) * kDcCin];
#pragma unroll
      for (int ci = 0; ci < kDcCin; ++ci) {
        const float xv = ip[ci];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += xv * s_w[((cgp * 8 + j) * 9 + t) * kDcCin + ci];
      }
    }
    __syncthreads();
  }
  if (oy < ho && ox < wo) {
    const long long o = ((static_cast<long long>(b) * ho + oy) * wo + ox) * cout;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int co = co0 + cgp * 8 + j;
      if (co < cout) {
        float v = acc[j] + (bias ? bias[co] : 0.f);
        if (silu) v = silu_f(v);
        if (residual) v += __half2float(residual[o + co]);
        y[o + co] = __float2half_rn(v);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// 3x3 stride-1 conv with a tiny input-channel count (the 4->320 input conv): K = 9*CIN.
// CTA = 8 pixel slots x (cout/8) channel groups, each thread walks 4 pixels; the weights sit in shared
// memory as fp32 laid out [k][j][group] so that a warp's reads are conflict-free; they are constants,
// so they are staged BEFORE the PDL wait and overlap the previous kernel's tail.
// ---------------------------------------------------------------------------------------------
constexpr int kCiSlots = 8;
constexpr int kCiPixPerThread = 4;
constexpr int kCiMaxThreads = 512;
// Blocks of kCiSlots * (cout / 8) <= kCiMaxThreads threads: the register budget must admit the largest.
template <int CIN>
__global__ void __launch_bounds__(kCiMaxThreads) conv3x3_smallcin_kernel(const __half* __restrict__ x, const __half* __restrict__ wt,
                                                                const float* __restrict__ bias, const __half* __restrict__ residual,
                                                                __half* __restrict__ y, int batch, int h, int w, int cout,
                                                                int silu) {
  extern __shared__ float s_wt[];  // [9*CIN][8][groups]
  constexpr int KK = 9 * CIN;
  const int groups = cout / 8;
  pdl_launch_dependents();
  for (int i = threadIdx.x; i < cout * KK; i += blockDim.x) {
    const int co = i / KK, k = i - co * KK;
    s_wt[(k * 8 + (co & 7)) * groups + (co >> 3)] = __half2float(wt[i]);
  }
  __syncthreads();
  pdl_wait();
  const int g = threadIdx.x % groups;
  const int slot = threadIdx.x / groups;
  if (slot >= kCiSlots) return;
  const long long npix = static_cast<long long>(batch) * h * w;
  float bj[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bj[j] = bias ? bias[g * 8 + j] : 0.f;
  for (int pp = 0; pp < kCiPixPerThread; ++pp) {
    const long long pix = (static_cast<long long>(blockIdx.x) * kCiPixPerThread + pp) * kCiSlots + slot;
    if (pix >= npix) break;
    const int xx = static_cast<int>(pix % w), yy = static_cast<int>((pix / w) % h);
    const long long b = pix / (static_cast<long long>(w) * h);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = bj[j];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int iy = yy + t / 3 - 1, ix = xx + t % 3 - 1;
      if (iy < 0 || iy >= h || ix < 0 || ix >= w) continue;
      const __half* xp = x + ((b * h + iy) * w + ix) * CIN;
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        const float xv = __half2float(xp[ci]);
        const float* wr = &s_wt[((t * CIN + ci) * 8) * groups + g];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += xv * wr[j * groups];
      }
    }
    if (silu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = silu_f(acc[j]);
    }
    const long long o = pix * cout + g * 8;
    if (residual) {
      uint4 r4 = *reinterpret_cast<const uint4*>(residual + o);
      const __half2* h2 = reinterpret_cast<const __half2*>(&r4);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float2 f = __half22float2(h2[e]);
        acc[2 * e] += f.x; acc[2 * e + 1] += f.y;
      }
    }
    uint4 o4;
    o4.x = pack_half2(acc[0], acc[1]); o4.y = pack_half2(acc[2], acc[3]);
    o4.z = pack_half2(acc[4], acc[5]); o4.w = pack_half2(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(y + o) = o4;
  }
}

// 3x3 stride-1 conv with a tiny output-channel count (the 320->4 output conv): one warp per pixel,
// lanes split the K = 9*cin reduction in 16-byte vectors, weights in shared memory.
template <int COUT>
__global__ void conv3x3_smallcout_kernel(const __half* __restrict__ x, const __half* __restrict__ wt,
                                         const float* __restrict__ bias, __half* __restrict__ y, int batch, int h,
                                         int w, int cin, int silu) {
  extern __shared__ __half s_wh[];  // [COUT][9*cin]
  const int kk = 9 * cin;
  pdl_launch_dependents();
  for (int i = threadIdx.x * 8; i < COUT * kk; i += blockDim.x * 8)
    *reinterpret_cast<uint4*>(&s_wh[i]) = *reinterpret_cast<const uint4*>(&wt[i]);
  __syncthreads();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  const long long npix = static_cast<long long>(batch) * h * w;
  const int vecs = cin / 8;
  for (long long pix = static_cast<long long>(blockIdx.x) * warps + (threadIdx.x >> 5); pix < npix;
       pix += static_cast<long long>(gridDim.x) * warps) {
    const int xx = static_cast<int>(pix % w), yy = static_cast<int>((pix / w) % h);
    const long long b = pix / (static_cast<long long>(w) * h);
    float acc[COUT];
#pragma unroll
    for (int j = 0; j < COUT; ++j) acc[j] = 0.f;
    for (int t = 0; t < 9; ++t) {
      const int iy = yy + t / 3 - 1, ix = xx + t % 3 - 1;
      if (iy < 0 || iy >= h || ix < 0 || ix >= w) continue;  // warp-uniform
      const __half* xp = x + ((b * h + iy) * w + ix) * cin;
      for (int v = lane; v < vecs; v += 32) {
        uint4 u = *reinterpret_cast<const uint4*>(xp + v * 8);
        const __half2* xh = reinterpret_cast<const __half2*>(&u);
        float xf[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f2 = __half22float2(xh[e]);
          xf[2 * e] = f2.x; xf[2 * e + 1] = f2.y;
        }
#pragma unroll
        for (int j = 0; j < COUT; ++j) {
          uint4 wu = *reinterpret_cast<const uint4*>(&s_wh[j * kk + t * cin + v * 8]);
          const __half2* wh = reinterpret_cast<const __half2*>(&wu);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float2 f2 = __half22float2(wh[e]);
            acc[j] += xf[2 * e] * f2.x + xf[2 * e + 1] * f2.y;
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < COUT; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    }
    if (lane < COUT) {
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < COUT; ++j)
        if (j == lane) v = acc[j];
      v += bias ? bias[lane] : 0.f;
      if (silu) v = silu_f(v);
      y[pix * COUT + lane] = __float2half_rn(v);
    }
  }
}

// ---------------------------------------------------------------------------------------------
__global__ void im2col3x3_kernel(const __half* __restrict__ x, __half* __restrict__ col, int batch, int h, int w,
                                 int c, int stride, int ho, int wo) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = c / 8;
  const long long total = static_cast<long long>(batch) * ho * wo * 9 * vecs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int t = static_cast<int>(r % 9);
    r /= 9;  // output pixel index
    const int ox = static_cast<int>(r % wo);
    const int oy = static_cast<int>((r / wo) % ho);
    const int b = static_cast<int>(r / (static_cast<long long>(wo) * ho));
    const int yy = oy * stride - 1 + t / 3, xx = ox * stride - 1 + t % 3;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (yy >= 0 && yy < h && xx >= 0 && xx < w)
      val = *reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * h + yy) * w + xx) * c + v * 8);
    *reinterpret_cast<uint4*>(col + (r * 9 + t) * c + v * 8) = val;
  }
}

// Same gather with the window anchored at the output pixel (no top/left halo) and zero fill past the bottom /
// right edge: the first-stage VAE encoder's Downsample pads (0,1,0,1) and convolves with stride 2, padding 0
// (ldm/modules/diffusionmodules/model.py:82-84).  Used by the VAE encoder (tests/test_vae_gpu.py).
__global__ void im2col3x3_br_kernel(const __half* __restrict__ x, __half* __restrict__ col, int batch, int h, int w,
                                    int c, int stride, int ho, int wo) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = c / 8;
  const long long total = static_cast<long long>(batch) * ho * wo * 9 * vecs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int t = static_cast<int>(r % 9);
    r /= 9;  // output pixel index
    const int ox = static_cast<int>(r % wo);
    const int oy = static_cast<int>((r / wo) % ho);
    const int b = static_cast<int>(r / (static_cast<long long>(wo) * ho));
    const int yy = oy * stride + t / 3, xx = ox * stride + t % 3;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (yy < h && xx < w)
      val = *reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * h + yy) * w + xx) * c + v * 8);
    *reinterpret_cast<uint4*>(col + (r * 9 + t) * c + v * 8) = val;
  }
}

__global__ void upsample2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, int batch, int h, int w, int c) {
  pdl_launch_dependents();
  pdl_wait();
  const int vecs = c / 8;
  const long long total = static_cast<long long>(batch) * (2 * h) * (2 * w) * vecs;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % vecs);
    long long r = i / vecs;
    const int ox = static_cast<int>(r % (2 * w));
    const int oy = static_cast<int>((r / (2 * w)) % (2 * h));
    const int b = static_cast<int>(r / (static_cast<long long>(4) * w * h));
    const uint4 val = *reinterpret_cast<const uint4*>(x + ((static_cast<long long>(b) * h + oy / 2) * w + ox / 2) * c + v * 8);
    *reinterpret_cast<uint4*>(y + r * c + v * 8) = val;
  }
}

__global__ void add_kernel(const __half* __restrict__ a, const __half* __restrict__ b, __half* __restrict__ y,
                           long long n_per_batch, int batch, int b_batches) {
  pdl_launch_dependents();
  pdl_wait();
  const long long vec_per = n_per_batch / 8;
  const long long total = vec_per * batch;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bi = (b_batches == 1) ? (i % vec_per) : i;
    uint4 ua = reinterpret_cast<const uint4*>(a)[i];
    uint4 ub = reinterpret_cast<const uint4*>(b)[bi];
    __half2* ha = reinterpret_cast<__half2*>(&ua);
    const __half2* hb = reinterpret_cast<const __half2*>(&ub);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 fa = __half22float2(ha[e]), fb = __half22float2(hb[e]);
      ha[e] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
    }
    reinterpret_cast<uint4*>(y)[i] = ua;
  }
}

__global__ void timestep_embedding_kernel(const int64_t* __restrict__ t, float* __restrict__ out, int batch, int dim,
                                          int t_count) {
  pdl_launch_dependents();
  pdl_wait();
  const int half = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * half) return;
  const int b = i / half, k = i % half;
  const float freq = expf(-logf(10000.0f) * static_cast<float>(k) / static_cast<float>(half));
  const float arg = static_cast<float>(t[b % t_count]) * freq;  // t_count < batch: the timesteps repeat (cond | uncond)
  out[b * dim + k] = cosf(arg);
  out[b * dim + half + k] = sinf(arg);
}

// out[r][n] = sum_k f(x[r][k]) * W[n][k] + bias[n]; one warp per output column n, all rows at once
template <int ROWS>
__global__ void skinny_linear_kernel(const float* __restrict__ x, const __half* __restrict__ w,
                                     const float* __restrict__ bias, float* __restrict__ out, int rows, int n, int k,
                                     int silu_in, int silu_out) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n) return;
  float acc[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) acc[r] = 0.f;
  const __half* wr = w + static_cast<long long>(warp) * k;
  for (int kk = lane * 8; kk < k; kk += 32 * 8) {
    uint4 u = *reinterpret_cast<const uint4*>(wr + kk);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
    float wf[8];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = __half22float2(h2[e]);
      wf[2 * e] = f.x; wf[2 * e + 1] = f.y;
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      if (r < rows) {
        const float* xr = x + static_cast<long long>(r) * k + kk;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float xv = xr[e];
          if (silu_in) xv = silu_f(xv);
          acc[r] += xv * wf[e];
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
  }
  if (lane == 0) {
    for (int r = 0; r < rows && r < ROWS; ++r) {
      float v = acc[r] + (bias ? bias[warp] : 0.f);
      if (silu_out) v = silu_f(v);
      out[static_cast<long long>(r) * n + warp] = v;
    }
  }
}

// copies > 1: the output holds the batch `copies` times over (the paired cond | uncond batch of p_sample_ddim)
__global__ void nchw_f32_to_nhwc_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, int batch, int c, int h,
                                            int w, int copies) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(batch) * copies * c * h * w;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // i indexes the NHWC output
    const int ch = static_cast<int>(i % c);
    long long r = i / c;
    const int xx = static_cast<int>(r % w);
    const int yy = static_cast<int>((r / w) % h);
    const int b = static_cast<int>(r / (static_cast<long long>(w) * h)) % batch;
    y[i] = __float2half_rn(x[((static_cast<long long>(b) * c + ch) * h + yy) * w + xx]);
  }
}

__global__ void nhwc_f16_to_nchw_f32_kernel(const __half* __restrict__ x, float* __restrict__ y, int batch, int c, int h,
                                            int w) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = static_cast<long long>(batch) * c * h * w;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // i indexes the NCHW output
    const int xx = static_cast<int>(i % w);
    long long r = i / w;
    const int yy = static_cast<int>(r % h);
    r /= h;
    const int ch = static_cast<int>(r % c);
    const int b = static_cast<int>(r / c);
    y[i] = __half2float(x[((static_cast<long long>(b) * h + yy) * w + xx) * c + ch]);
  }
}

__global__ void cfg_ddim_update_kernel(float* x, const float* __restrict__ ec, const float* __restrict__ eu,
                                       const float* __restrict__ noise, float* __restrict__ x_prev,
                                       float* __restrict__ pred_x0, long long n, const float* __restrict__ coef,
                                       int update_x) {
  pdl_launch_dependents();
  pdl_wait();
  // coef (device, so one captured CUDA graph serves all 50 steps):
  //   {cfg scale, sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev - sigma^2), sigma, sqrt(1 - a_t)}
  const float scale = coef[0], sqrt_at = coef[1], sqrt_aprev = coef[2], dir_coef = coef[3], sigma = coef[4],
              s1m = coef[5];
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float u = eu[i];
    const float e = u + scale * (ec[i] - u);
    const float p0 = (x[i] - s1m * e) / sqrt_at;
    float xp = sqrt_aprev * p0 + dir_coef * e;
    if (noise != nullptr) xp += sigma * noise[i];
    x_prev[i] = xp;
    pred_x0[i] = p0;
    if (update_x) x[i] = xp;  // the chain's state advances in place: the next step reads x
  }
}


static inline int grid_for(long long total, int threads = 256, int cap = kNumSms * 16) {
  long long b = (total + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace mdb

using namespace mdb;

extern "C" int mdb_abi_version(void) { return MDB_ABI_VERSION; }

extern "C" int64_t mdb_abi_struct_bytes(int32_t which) {
  switch (which) {
    case 0:
      return (int64_t)sizeof(mdb_gemm_desc);
    case 1:
      return (int64_t)sizeof(mdb_attn_desc);
    case 2:
      return (int64_t)sizeof(mdb_attn_bwd_desc);
    case 3:
      return (int64_t)sizeof(mdb_gemm_bwd_desc);
    case 4:
      return (int64_t)sizeof(mdb_groupnorm_bwd_desc);
    case 5:
      return (int64_t)sizeof(mdb_layernorm_bwd_desc);
    case 6:
      return (int64_t)sizeof(mdb_conv3x3_bwd_desc);
    case 7:
      return (int64_t)sizeof(mdb_skinny_linear_bwd_desc);
    default:
      return -1;
  }
}

extern "C" int mdb_set_tuning(int32_t key, int32_t value) {
  switch (key) {
    case MDB_TUNE_GEMM_PAIR_MIN_TILES:
    case MDB_TUNE_GEMM_BN80_BELOW:
    case MDB_TUNE_GEMM_SKINNY_CTAS:
    case MDB_TUNE_GEMM_SPLIT_MIN_CHUNKS:
      mdb::set_gemm_tuning(key, value);
      return MDB_OK;
    case MDB_TUNE_ATTN40_2Q_MIN_CTAS:
      mdb::set_attn_tuning(value);
      return MDB_OK;
    default:
      mdb::set_error("mdb_set_tuning: unknown key %d", key);
      return MDB_ERR_INVALID;
  }
}

extern "C" int32_t mdb_get_tuning(int32_t key) {
  if (key == MDB_TUNE_ATTN40_2Q_MIN_CTAS) return mdb::get_attn_tuning();
  return mdb::get_gemm_tuning(key);
}
extern "C" const char* mdb_last_error(void) { return mdb::g_err; }
extern "C" int64_t mdb_launch_count(void) { return mdb::g_launches.load(); }

extern "C" int mdb_device_check(void) {
  int dev = 0;
  MDB_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  MDB_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major, prop.minor);
    return MDB_ERR_UNSUPPORTED;
  }
  return MDB_OK;
}

namespace {
// one CTA per row; three passes over the row (max, sum of exp2, normalise) — rows of a few KB stay in L1/L2
__global__ void __launch_bounds__(256) softmax_rows_kernel(__half* __restrict__ x, long long ld, int cols, float scale_log2) {
  mdb::pdl_launch_dependents();
  mdb::pdl_wait();
  __shared__ float red[8];
  __shared__ float bcast;
  __half* row = x + static_cast<long long>(blockIdx.x) * ld;
  const int vecs = cols >> 3;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + v * 8);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      m = fmaxf(m, fmaxf(f.x, f.y));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int w = 1; w < 8; ++w) t = fmaxf(t, red[w]);
    bcast = t;
  }
  __syncthreads();
  m = bcast * scale_log2;  // scale > 0: the maximum of the scaled row
  float sum = 0.f;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + v * 8);
    const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      sum += exp2f(fmaf(f.x, scale_log2, -m)) + exp2f(fmaf(f.y, scale_log2, -m));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  __syncthreads();  // red[] / bcast of the first reduction have been consumed
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    bcast = 1.0f / t;
  }
  __syncthreads();
  const float inv = bcast;
  for (int v = threadIdx.x; v < vecs; v += blockDim.x) {
    uint4 u = *reinterpret_cast<const uint4*>(row + v * 8);
    __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      h2[e] = __floats2half2_rn(exp2f(fmaf(f.x, scale_log2, -m)) * inv, exp2f(fmaf(f.y, scale_log2, -m)) * inv);
    }
    *reinterpret_cast<uint4*>(row + v * 8) = u;
  }
}
}  // namespace

extern "C" int mdb_softmax_rows_f16(void* x, int64_t ld, int32_t rows, int32_t cols, float scale, mdb_stream_t stream) {
  MDB_REQUIRE(x != nullptr && rows > 0 && cols > 0, "mdb_softmax_rows_f16: bad arguments");
  MDB_REQUIRE(cols % 8 == 0 && ld % 8 == 0 && ld >= cols && (reinterpret_cast<uintptr_t>(x) & 15) == 0,
              "mdb_softmax_rows_f16: cols and ld must be multiples of 8, ld >= cols, x 16-byte aligned (cols=%d)", cols);
  MDB_REQUIRE(scale > 0.f, "mdb_softmax_rows_f16: scale must be positive");
  MDB_CHECK_CUDA(mdb::launch_pdl(softmax_rows_kernel, dim3(static_cast<unsigned>(rows)), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), static_cast<__half*>(x), static_cast<long long>(ld),
                                 cols, scale * 1.4426950408889634f));
  mdb::count_launch();
  return MDB_OK;
}

extern "C" int mdb_conv3x3_direct_f16(const void* x, const void* wt, const float* bias, const void* residual, void* y,
                                      int32_t batch, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t stride,
                                      int32_t silu, mdb_stream_t stream) {
  MDB_REQUIRE(x && wt && y, "mdb_conv3x3_direct_f16: null pointer");
  MDB_REQUIRE(stride == 1 || stride == 2, "mdb_conv3x3_direct_f16: stride must be 1 or 2");
  const int ho = (h + 2 - 3) / stride + 1, wo = (w + 2 - 3) / stride + 1;
  dim3 grid(((wo + kDcTile - 1) / kDcTile) * ((ho + kDcTile - 1) / kDcTile), (cout + kDcCout - 1) / kDcCout, batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long npix = static_cast<long long>(batch) * h * w;
  if (stride == 1 && cin == 4 && cout % 8 == 0 && cout * 36 * 4 <= 96 * 1024 && kCiSlots * (cout / 8) <= kCiMaxThreads) {
    // tiny-cin path (input conv)
    const int smem = cout * 36 * 4;
    if (int rc = set_max_dyn_smem<conv3x3_smallcin_kernel<4>>(96 * 1024)) return rc;
    const int threads = ((kCiSlots * (cout / 8) + 31) / 32) * 32;
    const int per_block = kCiSlots * kCiPixPerThread;
    MDB_CHECK_CUDA(launch_pdl(conv3x3_smallcin_kernel<4>, dim3(static_cast<unsigned>((npix + per_block - 1) / per_block)),
                              dim3(threads), smem, st, static_cast<const __half*>(x), static_cast<const __half*>(wt),
                              bias, static_cast<const __half*>(residual), static_cast<__half*>(y), batch, h, w, cout,
                              silu));
    count_launch();
    return MDB_OK;
  }
  if (stride == 1 && cout == 4 && cin % 8 == 0 && residual == nullptr && cout * 9 * cin * 2 <= 96 * 1024) {
    // tiny-cout path (output conv)
    const int smem = cout * 9 * cin * 2;
    if (int rc = set_max_dyn_smem<conv3x3_smallcout_kernel<4>>(96 * 1024)) return rc;
    int blocks = static_cast<int>((npix + 7) / 8);
    if (blocks > kNumSms * 4) blocks = kNumSms * 4;
    MDB_CHECK_CUDA(launch_pdl(conv3x3_smallcout_kernel<4>, dim3(blocks), dim3(256), smem, st,
                              static_cast<const __half*>(x), static_cast<const __half*>(wt), bias,
                              static_cast<__half*>(y), batch, h, w, cin, silu));
    count_launch();
    return MDB_OK;
  }
  if (stride == 1)
    MDB_CHECK_CUDA(launch_pdl(direct_conv3x3_kernel<1>, grid, dim3(256), 0, st, static_cast<const __half*>(x),
                              static_cast<const __half*>(wt), bias, static_cast<const __half*>(residual),
                              static_cast<__half*>(y), h, w, cin, cout, ho, wo, silu));
  else
    MDB_CHECK_CUDA(launch_pdl(direct_conv3x3_kernel<2>, grid, dim3(256), 0, st, static_cast<const __half*>(x),
                              static_cast<const __half*>(wt), bias, static_cast<const __half*>(residual),
                              static_cast<__half*>(y), h, w, cin, cout, ho, wo, silu));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_im2col3x3_f16(const void* x, void* col, int32_t batch, int32_t h, int32_t w, int32_t c,
                                 int32_t stride, mdb_stream_t stream) {
  MDB_REQUIRE(x && col, "mdb_im2col3x3_f16: null pointer");
  MDB_REQUIRE(c % 8 == 0 && (stride == 1 || stride == 2), "mdb_im2col3x3_f16: need c %% 8 == 0 and stride 1 or 2");
  const int ho = (h - 1) / stride + 1, wo = (w - 1) / stride + 1;
  const long long total = static_cast<long long>(batch) * ho * wo * 9 * (c / 8);
  MDB_CHECK_CUDA(launch_pdl(im2col3x3_kernel, dim3(grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                            static_cast<const __half*>(x), static_cast<__half*>(col), batch, h, w, c, stride, ho, wo));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_im2col3x3_br_f16(const void* x, void* col, int32_t batch, int32_t h, int32_t w, int32_t c,
                                    int32_t stride, mdb_stream_t stream) {
  MDB_REQUIRE(x && col, "mdb_im2col3x3_br_f16: null pointer");
  MDB_REQUIRE(c % 8 == 0 && (stride == 1 || stride == 2), "mdb_im2col3x3_br_f16: need c %% 8 == 0 and stride 1 or 2");
  MDB_REQUIRE(h >= 2 && w >= 2, "mdb_im2col3x3_br_f16: image too small");
  // input padded by one row / column at the bottom / right, 3x3 window, no other padding
  const int ho = (h + 1 - 3) / stride + 1, wo = (w + 1 - 3) / stride + 1;
  const long long total = static_cast<long long>(batch) * ho * wo * 9 * (c / 8);
  MDB_CHECK_CUDA(launch_pdl(im2col3x3_br_kernel, dim3(grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                            static_cast<const __half*>(x), static_cast<__half*>(col), batch, h, w, c, stride, ho, wo));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_upsample2x_f16(const void* x, void* y, int32_t batch, int32_t h, int32_t w, int32_t c,
                                  mdb_stream_t stream) {
  MDB_REQUIRE(x && y && c % 8 == 0, "mdb_upsample2x_f16: bad arguments");
  const long long total = static_cast<long long>(batch) * 4 * h * w * (c / 8);
  MDB_CHECK_CUDA(launch_pdl(upsample2x_kernel, dim3(grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                            static_cast<const __half*>(x), static_cast<__half*>(y), batch, h, w, c));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_add_f16(const void* a, const void* b, void* y, int64_t n_per_batch, int32_t batch, int32_t b_batches,
                           mdb_stream_t stream) {
  MDB_REQUIRE(a && b && y && n_per_batch % 8 == 0, "mdb_add_f16: bad arguments");
  MDB_REQUIRE(b_batches == 1 || b_batches == batch, "mdb_add_f16: b_batches must be 1 or batch");
  MDB_CHECK_CUDA(launch_pdl(add_kernel, dim3(grid_for(n_per_batch / 8 * batch)), dim3(256), 0,
                            static_cast<cudaStream_t>(stream), static_cast<const __half*>(a),
                            static_cast<const __half*>(b), static_cast<__half*>(y), static_cast<long long>(n_per_batch),
                            batch, b_batches));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_timestep_embedding_f32(const int64_t* t, int32_t t_count, float* out, int32_t batch, int32_t dim,
                                          mdb_stream_t stream) {
  MDB_REQUIRE(t && out && dim % 2 == 0 && t_count >= 1 && batch % t_count == 0, "mdb_timestep_embedding_f32: bad arguments");
  const int total = batch * dim / 2;
  MDB_CHECK_CUDA(launch_pdl(timestep_embedding_kernel, dim3((total + 127) / 128), dim3(128), 0,
                            static_cast<cudaStream_t>(stream), t, out, batch, dim, t_count));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_skinny_linear_f32(const float* x, const void* w, const float* bias, float* out, int32_t rows,
                                     int32_t n, int32_t k, int32_t silu_in, int32_t silu_out, mdb_stream_t stream) {
  MDB_REQUIRE(x && w && out, "mdb_skinny_linear_f32: null pointer");
  MDB_REQUIRE(rows >= 1 && rows <= 16 && k % 8 == 0, "mdb_skinny_linear_f32: rows must be 1..16 and k %% 8 == 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = 256;
  const int blocks = (n * 32 + threads - 1) / threads;
  const __half* wp = static_cast<const __half*>(w);
  if (rows <= 2)
    MDB_CHECK_CUDA(launch_pdl(skinny_linear_kernel<2>, dim3(blocks), dim3(threads), 0, st, x, wp, bias, out, rows, n, k,
                              silu_in, silu_out));
  else if (rows <= 8)
    MDB_CHECK_CUDA(launch_pdl(skinny_linear_kernel<8>, dim3(blocks), dim3(threads), 0, st, x, wp, bias, out, rows, n, k,
                              silu_in, silu_out));
  else
    MDB_CHECK_CUDA(launch_pdl(skinny_linear_kernel<16>, dim3(blocks), dim3(threads), 0, st, x, wp, bias, out, rows, n, k,
                              silu_in, silu_out));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_nchw_f32_to_nhwc_f16(const float* x, void* y, int32_t batch, int32_t c, int32_t h, int32_t w,
                                        int32_t copies, mdb_stream_t stream) {
  MDB_REQUIRE(x && y && copies >= 1, "mdb_nchw_f32_to_nhwc_f16: bad arguments");
  const long long total = static_cast<long long>(batch) * copies * c * h * w;
  MDB_CHECK_CUDA(launch_pdl(nchw_f32_to_nhwc_f16_kernel, dim3(grid_for(total)), dim3(256), 0,
                            static_cast<cudaStream_t>(stream), x, static_cast<__half*>(y), batch, c, h, w, copies));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_nhwc_f16_to_nchw_f32(const void* x, float* y, int32_t batch, int32_t c, int32_t h, int32_t w,
                                        mdb_stream_t stream) {
  MDB_REQUIRE(x && y, "mdb_nhwc_f16_to_nchw_f32: null pointer");
  const long long total = static_cast<long long>(batch) * c * h * w;
  MDB_CHECK_CUDA(launch_pdl(nhwc_f16_to_nchw_f32_kernel, dim3(grid_for(total)), dim3(256), 0,
                            static_cast<cudaStream_t>(stream), static_cast<const __half*>(x), y, batch, c, h, w));
  count_launch();
  return MDB_OK;
}

extern "C" int mdb_cfg_ddim_update_f32(float* x, const float* eps_c, const float* eps_u, const float* noise,
                                       float* x_prev, float* pred_x0, int64_t n, const float* coef, int32_t update_x,
                                       mdb_stream_t stream) {
  MDB_REQUIRE(x && eps_c && eps_u && x_prev && pred_x0 && coef && n > 0, "mdb_cfg_ddim_update_f32: bad arguments");
  MDB_CHECK_CUDA(launch_pdl(cfg_ddim_update_kernel, dim3(grid_for(n)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                            x, eps_c, eps_u, noise, x_prev, pred_x0, static_cast<long long>(n), coef, update_x));
  count_launch();
  return MDB_OK;
}
