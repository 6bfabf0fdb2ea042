// Shared device/host helpers for the sm_90a kernels: mbarrier, TMA, cluster and wgmma PTX wrappers,
// the operand ring of the warp-specialised kernels, wgmma descriptors, TMA tensor-map construction
// and error plumbing for the C ABI.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/magicdance_b200.h"
#include "wgmma.cuh"

namespace mdb {

// ----------------------------------------------------------------------------------------------
// error plumbing: every extern "C" entry returns 0 or a negative code; text via mdb_last_error()
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);

#define MDB_CHECK_CUDA(expr)                                                                     \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      mdb::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return MDB_ERR_CUDA;                                                                       \
    }                                                                                            \
  } while (0)

#define MDB_REQUIRE(cond, ...)      \
  do {                              \
    if (!(cond)) {                  \
      mdb::set_error(__VA_ARGS__);  \
      return MDB_ERR_INVALID;       \
    }                               \
  } while (0)

// launch counter behind mdb_launch_count(); launch heuristics behind mdb_set_tuning() / mdb_get_tuning()
void count_launch(int n = 1);
int get_gemm_tuning(int key);
void set_gemm_tuning(int key, int value);
int get_attn_tuning();
void set_attn_tuning(int v);

constexpr int kNumSms = 132;  // H100 SXM: the SM count that the grid-size heuristics plan for

// ----------------------------------------------------------------------------------------------
// TMA tensor maps (host): fp16 tiled maps with 128-byte swizzle.  Each returns 0 or an MDB_ERR_* code.
// ----------------------------------------------------------------------------------------------
// [rows][inner] row-major, `ld` elements between rows; boxes of box_rows x box_inner
int tmap_rows(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, long long ld, uint32_t box_inner,
              uint32_t box_rows);
// the head slices of [tokens][heads * d] activations (row stride ld) as (d, heads, tokens); boxes of 64 channels x
// 1 head x box_tokens tokens, zero-filled beyond d
int tmap_heads(CUtensorMap* out, const void* base, int d, int heads, uint64_t tokens, long long ld,
               uint32_t box_tokens);
// The same head slices of nb samples of n tokens each as (d, heads, token, sample); boxes of 64 channels x 1 head x
// box_tokens tokens x 1 sample.  Tokens >= n are zero-filled, so a sample's last ragged box never reaches into the
// next sample's rows.
int tmap_heads_per_sample(CUtensorMap* out, const void* base, int d, int heads, int n, int nb, long long ld,
                          uint32_t box_tokens);
// V^T of attention: `rows` channel rows (row stride ldvt) of nb samples' column blocks of ldvb columns, the first n
// of each used, as (key, sample, row); boxes of 64 keys x 1 sample x box_rows rows.  Keys >= n are zero-filled, so
// the padding columns n..ldvb and the next sample's keys never reach shared memory.
int tmap_vt(CUtensorMap* out, const void* base, int n, int nb, long long ldvb, int rows, long long ldvt,
            uint32_t box_rows);
// NHWC images [nb][h][w] of pixels `ld` elements apart, c channels used, as (c, w, h, nb); cs = 2 reads every second
// pixel along w and h (TMA element strides)
int tmap_nhwc(CUtensorMap* out, const void* base, int c, int w, int h, int nb, long long ld, const uint32_t box[4],
              int cs);
// The same NHWC images as an im2col-mode map for a 3x3 pad-1 window: one load walks `pixels` consecutive window
// positions (output pixels) across row and image boundaries, 64 channels each, into the [pixels][64] 128B-swizzled
// tile a tiled box of `pixels` rows gives.  The load's coordinates are the window's top-left input pixel
// (cs * x - 1, cs * y - 1) of the first output pixel; its im2col offsets (0..2 along w and h) pick the tap; pixels
// outside the image are zero-filled.  cs = 2 steps the window by two input pixels (TMA element strides).
int tmap_nhwc_im2col(CUtensorMap* out, const void* base, int c, int w, int h, int nb, long long ld, int pixels,
                     int cs);

// The 4-D TMA box {64 channels, x, y, images} that covers `rows` consecutive output pixels of a 3x3 conv with ho x wo
// output pixels per image, reading every cs-th input pixel.  `fwd` selects the forward kernel's rule for rows at
// least as wide as the box: only rows strictly wider are cut into single-row boxes, and only at stride 1.  Returns
// kBoxOk, or the condition that fails (such runs of pixels are then not boxes).
enum { kBoxOk, kBoxWideRows, kBoxRowsPerTile, kBoxImagesPerTile, kBoxTooLarge };
int pixel_box(int ho, int wo, int cs, int rows, bool fwd, uint32_t box[4]);

// ----------------------------------------------------------------------------------------------
// device-side PTX wrappers
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__

// launch helper: cudaLaunchKernelEx with the programmatic-stream-serialization attribute (PDL);
// MDB_PDL=0 in the environment turns the attribute off (then griddepcontrol.* are no-ops).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster2(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                       cudaStream_t stream, unsigned cluster_x, unsigned cluster_z, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_z > 1 || cluster_x > 1) {
    // thread-block cluster: along z = split-K partners (GEMM) or the CTAs of one GroupNorm group, which
    // reduce through distributed shared memory
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = cluster_z;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                      cudaStream_t stream, unsigned cluster_z, Args&&... args) {
  return launch_pdl_cluster2(kernel, grid, block, smem, stream, 1u, cluster_z, static_cast<Args&&>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  return launch_pdl_cluster2(kernel, grid, block, smem, stream, 1u, 1u, static_cast<Args&&>(args)...);
}
// raises the dynamic shared-memory limit of Kernel to `bytes`, once.  The flag belongs to the kernel itself: kernels
// of the same type (gemm_bwd_kernel<0> and <1>) each get their own.
template <auto Kernel>
inline int set_max_dyn_smem(int bytes) {
  static bool done = false;
  if (!done) {
    MDB_CHECK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done = true;
  }
  return MDB_OK;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------
// Every kernel of this library starts with pdl_launch_dependents() (the NEXT kernel in the stream may
// begin its prologue: barrier init, descriptor prefetch, index math) and calls pdl_wait()
// before it touches global memory (waits until the PREVIOUS kernel has completed and flushed).  With
// ~650 small kernels per denoise step this was meant to hide launch-to-launch latency (measured: neutral).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- mbarrier --------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = smem_u32(bar);
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t}"
      ::"r"(addr), "r"(parity)
      : "memory");
}

// ---- warp-specialised TMA -> wgmma kernels ------------------------------------------------------
// Warp roles: warps 0-7 are two MMA warpgroups (the consumers), warp 8 is the TMA producer.
constexpr int kConsumers = 256;
constexpr int kProducerWarp = kConsumers / 32;
constexpr int kWsThreads = kConsumers + 32;

// 128-byte-swizzled TMA tiles and wgmma descriptors need 1024-byte-aligned shared memory
__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~uintptr_t(1023));
}

// The S-stage operand ring: step `it` uses stage it % S.  The producer fills a stage once its `empty` barrier shows
// that the consumers released the previous round; the consumers read it once its `full` barrier completes.
template <int S>
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, uint32_t full_count) {
  for (int s = 0; s < S; ++s) {
    mbar_init(&full[s], full_count);
    mbar_init(&empty[s], kConsumers);  // every consumer thread arrives when it is done with the stage
  }
}
// producer: wait until the stage of step `it` is free and return it (the caller then arms `full` with expect_tx)
template <int S>
__device__ __forceinline__ int ring_acquire(uint64_t* empty, int it) {
  const int s = it % S;
  mbar_wait(&empty[s], ((it / S) & 1) ^ 1);
  return s;
}
// consumer: wait until the stage of step `it` is loaded and return it
template <int S>
__device__ __forceinline__ int ring_wait_full(uint64_t* full, int it) {
  const int s = it % S;
  mbar_wait(&full[s], (it / S) & 1);
  return s;
}

// ---- TMA loads (global -> shared, completion on an mbarrier) -----------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col-mode load of a tmap_nhwc_im2col map: coordinates (channel, w, h, image) of the first window's corner, offsets
// (ow, oh) of the tap inside the window
__device__ __forceinline__ void tma_load_im2col_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                   int c2, int c3, int ow, int oh) {
  const uint16_t w16 = static_cast<uint16_t>(ow), h16 = static_cast<uint16_t>(oh);
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
        "h"(w16), "h"(h16)
      : "memory");
}

// ---- thread-block clusters / distributed shared memory ---------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// all threads of all CTAs of the cluster
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// address of `local_smem_addr` (a shared::cta address of THIS CTA) in the shared memory of cluster CTA `rank`
__device__ __forceinline__ uint32_t dsmem_map(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local_smem_addr), "r"(rank));
  return a;
}
__device__ __forceinline__ float4 dsmem_ld_f4(uint32_t cluster_addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"(cluster_addr));
  return v;
}

// ---- proxies / fences ---------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads of smem)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- warpgroup MMA (sm_90a) -------------------------------------------------------------------------
// K-major operand tile stored as [rows][64 halves] (128-byte rows, TMA SWIZZLE_128B, 1024B-aligned):
// 8-row groups are 1024 B apart (SBO), LBO is unused for swizzled K-major layouts (set to 1),
// layout type 1 = SWIZZLE_128B.  A K step of 16 halves (32 B) inside the swizzle row is +2 on the descriptor.
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);   // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                      // LBO (unused)   [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // SBO = 1024 B   [32,46)
  d |= static_cast<uint64_t>(1) << 62;                      // SWIZZLE_128B   [62,64)
  return d;
}
// MN-major operand tile (wgmma trans = 1) stored as [K rows][64 M-or-N halves] per 64-wide chunk, the same 128-byte
// swizzled rows TMA writes: one swizzle atom is 64 M/N elements x 8 K rows (1024 B).  SBO = 1024 B steps 8 K rows,
// LBO = `chunk_bytes` steps to the next 64 M/N elements.  A K step of 16 rows is +2048 B on the start address.
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(uint32_t smem_addr, uint32_t chunk_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);   // start address  [0,14)
  d |= static_cast<uint64_t>((chunk_bytes >> 4) & 0x3FFF) << 16;  // LBO      [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // SBO = 1024 B   [32,46)
  d |= static_cast<uint64_t>(1) << 62;                      // SWIZZLE_128B   [62,64)
  return d;
}
// before the first wgmma of a batch: orders earlier register / shared-memory accesses of the warpgroup
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N committed groups of this warpgroup may still be in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma_wait
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over `threads` threads (a multiple of 32) of this CTA; id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// single-instruction MUFU.EX2 (inputs here are <= 8 in magnitude on the positive side; flush-to-zero is fine)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// derivatives: silu'(x) = s (1 + x (1 - s)) with s = sigmoid(x); gelu'(x) = Phi(x) + x phi(x)
__device__ __forceinline__ float dsilu(float x) {
  const float s = 1.0f / (1.0f + __expf(-x));
  return s * (1.0f + x * (1.0f - s));
}
__device__ __forceinline__ float dgelu_erf(float x) {
  return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * __expf(-0.5f * x * x);
}

// ---- gradient destinations of the backward kernels -------------------------------------------------
struct GbOut {  // fp16 or fp32 rows, overwritten or accumulated into; p == nullptr: dropped
  void* p;
  long long ld;
  int f32, acc;
};

__device__ __forceinline__ void gb_store2(const GbOut& o, long long row, int col, float v0, float v1) {
  if (o.p == nullptr) return;
  if (o.f32) {
    float2* d = reinterpret_cast<float2*>(static_cast<float*>(o.p) + row * o.ld + col);
    if (o.acc) {
      const float2 x = *d;
      v0 += x.x;
      v1 += x.y;
    }
    *d = make_float2(v0, v1);
  } else {
    __half2* d = reinterpret_cast<__half2*>(static_cast<__half*>(o.p) + row * o.ld + col);
    if (o.acc) {
      const float2 x = __half22float2(*d);
      v0 += x.x;
      v1 += x.y;
    }
    *d = __floats2half2_rn(v0, v1);
  }
}
#endif  // __CUDACC__

inline GbOut gb_out(void* p, long long ld, int dtype, int acc) {
  GbOut o;
  o.p = p;
  o.ld = ld;
  o.f32 = dtype == MDB_DTYPE_F32;
  o.acc = acc != 0;
  return o;
}

// second pass of a fixed-order column sum (gemm_bwd.cu): out[seg * stride + col] (+)= sum over q < parts, in order, of
// ws[(seg * parts + q) * n + col], for seg < segs and col < n.  Counts its launch.
int launch_colsum_finalize(const float* ws, int n, int segs, int parts, float* out, long long stride, int acc,
                           cudaStream_t st);

}  // namespace mdb
