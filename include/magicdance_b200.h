/*
 * magicdance_b200 — C ABI of the H100 (sm_90a) kernels behind MagicPose's DDIM denoising hot path.
 *
 * The reference (Boese0601/MagicDance) has no FFI: its "plugin API" is Python classes looked up by
 * YAML `target:` strings (model_lib/ControlNet/ldm/util.py:72-87).  The drop-in Python classes in
 * this repo (model_lib/ControlNet/cldm/cldm.py, .../ldm/...) keep those names and signatures and
 * call THIS library for every per-step tensor op.  Each entry point below names the reference
 * interface (file:line, relative to /root/reference/model_lib/ControlNet/) it replaces.
 *
 * Conventions
 *   - all data pointers are DEVICE pointers (cudaMalloc'ed / torch CUDA storage) unless noted;
 *   - activations are fp16, channels-last: an NCHW tensor (B,C,H,W) is stored as [B][H][W][C],
 *     which is also the token-major (B, H*W, C) matrix the transformer blocks use;
 *   - weights are fp16, "K-major": Linear (out,in) as is; Conv2d OIHW repacked to [O][kh][kw][I];
 *   - `stream` is a cudaStream_t (0 = legacy default stream); every call is asynchronous;
 *   - return value: 0 on success, negative MDB_ERR_* otherwise; mdb_last_error() gives the text.
 *   - there is NO CPU fallback: without an sm_90 device every compute entry returns an error.
 */
#ifndef MAGICDANCE_B200_H_
#define MAGICDANCE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDB_OK 0
#define MDB_ERR_INVALID (-1)
#define MDB_ERR_CUDA (-2)
#define MDB_ERR_UNSUPPORTED (-3)

#define MDB_ABI_VERSION 2

typedef void* mdb_stream_t;

/* library plumbing */
int mdb_abi_version(void);
const char* mdb_last_error(void);
/* 0 if the current CUDA device is compute capability 10.x, MDB_ERR_UNSUPPORTED otherwise */
int mdb_device_check(void);
/* number of kernels launched by this library since load (bench.py's gpu_launches) */
int64_t mdb_launch_count(void);
/* sizeof(mdb_gemm_desc) (which = 0) / sizeof(mdb_attn_desc) (which = 1) / sizeof(mdb_attn_bwd_desc) (which = 2) /
 * sizeof(mdb_gemm_bwd_desc) (which = 3) / sizeof(mdb_groupnorm_bwd_desc) (which = 4) /
 * sizeof(mdb_layernorm_bwd_desc) (which = 5) / sizeof(mdb_conv3x3_bwd_desc) (which = 6) /
 * sizeof(mdb_skinny_linear_bwd_desc) (which = 7): a binding checks its struct mirrors */
int64_t mdb_abi_struct_bytes(int32_t which);

/* Launch heuristics, process-wide (defaults in parentheses); tests use the setter to force a kernel variant onto small
 * problems. */
#define MDB_TUNE_GEMM_PAIR_MIN_TILES 1 /* grids of >= this many tiles use the one-CTA-per-SM large-grid tiles (128) */
#define MDB_TUNE_ATTN40_2Q_MIN_CTAS 3  /* d=40 attention grids of >= this many CTAs run two CTAs per SM (512) */
#define MDB_TUNE_GEMM_BN80_BELOW 4     /* N %% 160 == 0 layers with fewer 160-wide CTAs than this take 80-wide tiles (100) */
enum {
  MDB_TUNE_GEMM_SKINNY_CTAS = 5,     /* automatic plan of long-K grids (K >= 4096) of at most half this many tiles:
                                      * 80-wide tiles, K split up to this many CTAs (96); 0 = the compute-bound plan
                                      * (powers of two, >= 16 K chunks per split) */
  MDB_TUNE_GEMM_SPLIT_MIN_CHUNKS = 6 /* ... with at least this many 64-wide K chunks per split (8) */
};
int mdb_set_tuning(int32_t key, int32_t value);
int32_t mdb_get_tuning(int32_t key);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core GEMM / implicit-GEMM convolution (wgmma + TMA).
 *   D[M,N] = epilogue( A[M,K] * B[N,K]^T )     fp16 in, fp32 accumulate, fp16 out
 * Replaces: nn.Linear in CrossAttention.to_q/to_k/to_v/to_out (ldm/modules/attention.py:154-161),
 * GEGLU.proj / FeedForward.net[2] (attention.py:53-56,68-72), the 1x1 convs proj_in/proj_out
 * (attention.py:342-361), ResBlock.skip_connection and the ControlNet zero convs
 * (openaimodel.py:254-261, cldm.py:733-734), and — in conv mode — every 3x3 stride-1 pad-1
 * conv_nd of ResBlock / Upsample / Downsample-after-im2col (openaimodel.py:225,249-252,127,175).
 * ---------------------------------------------------------------------------------------------- */
#define MDB_EPI_NONE 0
#define MDB_EPI_GEGLU 1 /* B/bias rows interleaved [32 value | 32 gate]; D is [M][N/2] = v*gelu_erf(g) */

typedef struct mdb_gemm_desc {
  const void* a;   /* plain: fp16 [M][k1], row stride lda.  conv: NHWC fp16 [nb][h][w][c]        */
  int64_t lda;
  const void* a2;  /* optional 2nd source for K columns [k1, K) (fused torch.cat along channels) */
  int64_t lda2;
  int32_t k1;      /* columns taken from a; == k when a2 == NULL                                  */
  int32_t conv;    /* 0 plain; 1 | 2 = 3x3 pad-1 implicit GEMM with stride 1 | 2 over the NHWC input
                      (K = 9*c, M = nb*ho*wo, ho = (h-1)/stride+1): no im2col buffer (TMA element strides) */
  int32_t nb, h, w, c;
  const void* b;   /* fp16 [N][K], row stride ldb                                                 */
  int64_t ldb;
  void* d;         /* fp16 [M][N] (GEGLU: [M][N/2]), row stride ldd                               */
  int64_t ldd;
  const float* bias;          /* fp32, may be NULL; bias[(row / rows_per_batch) * bias_batch_stride + col] */
  int64_t bias_batch_stride;  /* 0 => one bias row for all batches                                */
  int32_t rows_per_batch;     /* rows of D per batch element (ignored when bias_batch_stride == 0) */
  int32_t epilogue;           /* MDB_EPI_*                                                        */
  const void* residual;       /* fp16 [M][N] added after bias, may be NULL                        */
  int64_t ldr;
  int32_t m, n, k;
  int32_t splits;             /* 0: automatic (1 ... 8, in-cluster reduction); 1: none; >1: as given */
  float* splitk_ws;           /* fp32 [splits][M][N] scratch, only for explicit split counts above 8 */
  /* LayerNorm over A's rows folded into the GEMM (norm2 -> attn2.to_q of BasicTransformerBlock,
   * attention.py:271,312-314): with B = W diag(gamma) and bias = W beta (+ the layer's own bias) supplied by the
   * caller, ln_u[n] = sum_k B[n][k] makes D = rstd_r (A B^T - mean_r ln_u) + bias equal to LayerNorm(A) W^T + b; K must
   * be the normalised width.  Small grids only: every N tile recomputes the statistics of its rows (no split-K, no
   * GEGLU epilogue, single-CTA tiles).  NULL = off. */
  const float* ln_u;
  float ln_eps;
} mdb_gemm_desc;

int mdb_gemm_f16(const mdb_gemm_desc* desc, mdb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of mdb_gemm_f16 (EPI_NONE, no ln_u): with D = A B^T (+ bias + residual) and dD its gradient,
 *   dA    = dD B       reduces over N: the input gradient of nn.Linear / 1x1 conv (attention.py:154-161,342-361),
 *                      and in conv mode of the 3x3 conv_nd (openaimodel.py:225,249-252,175) — col2im by gather;
 *   dB    = dD^T A     reduces over M (tokens / pixels): the weight gradient of the same layers;
 *   dbias = column sums of dD (per segment of rows_per_batch rows when bias_batch_stride != 0: the gradient of the
 *           per-sample timestep bias of ResBlock.emb_layers, openaimodel.py:238-244,262-263).
 * The residual's gradient is dD itself.  Deterministic: no atomics; split reductions go through fp32 slabs summed in
 * a fixed order, so two calls give bit-equal results.  Nothing is transposed in memory: B (dA) and both operands
 * (dB) are read MN-major by wgmma from the TMA tiles.
 *   fwd     : the forward's descriptor; its a / a2 / b / geometry / bias geometry are used, d / residual / bias
 *             pointers ignored; fwd.splits is the split count of the dA reduction (0 automatic, 1 none)
 *   dd      : fp16 [M][N], row stride lddd (a multiple of 8, 16-byte aligned base)
 *   da      : [M][k1] (conv: NHWC like fwd.a), da2: [M][K - k1] (the a2 columns); db: [N][K] (conv: [O][kh][kw][I])
 *   dbias   : fp32, dbias[(row / rows_per_batch) * bias_batch_stride + col] like the forward's bias
 *   NULL    = that gradient is not wanted; *_dtype MDB_DTYPE_F16 | MDB_DTYPE_F32; *_accumulate != 0 adds the
 *             gradient to the destination's contents instead of overwriting them
 *   splits  : split count of the dB reduction over M (0 automatic, 1 none)
 *   ws      : fp32 workspace of mdb_gemm_bwd_ws_floats(desc) floats (no initial value needed)
 * Stride-2 convs and latents whose rows do not tile into the TMA boxes (e.g. 12x8) take dA through an fp32 column
 * buffer and a gather kernel; non-tiling latents take dB through mdb_im2col3x3_f16.
 * ---------------------------------------------------------------------------------------------- */
#define MDB_DTYPE_F16 0
#define MDB_DTYPE_F32 1

typedef struct mdb_gemm_bwd_desc {
  mdb_gemm_desc fwd;
  const void* dd; int64_t lddd;
  void* da; int64_t ldda; int32_t da_dtype; int32_t da_accumulate;
  void* da2; int64_t ldda2; int32_t da2_dtype; int32_t da2_accumulate;
  void* db; int64_t lddb; int32_t db_dtype; int32_t db_accumulate;
  float* dbias; int32_t dbias_accumulate;
  int32_t splits;
  float* ws;
} mdb_gemm_bwd_desc;

int mdb_gemm_bwd_f16(const mdb_gemm_bwd_desc* desc, mdb_stream_t stream);
/* workspace floats mdb_gemm_bwd_f16 needs for this descriptor; negative MDB_ERR_* for a descriptor it rejects */
int64_t mdb_gemm_bwd_ws_floats(const mdb_gemm_bwd_desc* desc);

/* ------------------------------------------------------------------------------------------------
 * 3x3 pad-1 convolution (conv_nd of ResBlock / Upsample / Downsample, openaimodel.py:127,175,225,249-252) at ANY
 * latent size, forward and backward, on the same wgmma kernels: the activation tiles come from TMA im2col-mode loads,
 * which walk 128 consecutive output pixels across row and image boundaries and zero-fill the halo, instead of the 4-D
 * boxes of mdb_gemm_f16's conv mode (which need the pixels of a tile to form a box, e.g. 16x16 ... 128x128 latents).
 * At sizes both take, the two give bit-equal results.  Same descriptors as mdb_gemm_f16 / mdb_gemm_bwd_f16 with:
 *   conv     1 | 2: the stride (required);  nb, h, w, c: the input, c % 64 == 0;  k = 9c;  m = nb * ho * wo
 *   a, lda   NHWC fp16 input, lda = the pixel stride in elements (0: the channel count)
 *   a2, lda2 optional second source (a fused torch.cat along channels): channels [0, k1) of every pixel come from a,
 *            [k1, c) from a2; k1 a multiple of 64.  Ignored (k1 = c) when a2 == NULL
 *   epilogue MDB_EPI_NONE, ln_u NULL; bias / per-batch bias / residual / splits / splitk_ws as in mdb_gemm_f16
 * The backward's gradients are those of mdb_gemm_bwd_f16 (da: [nb*h*w][k1], da2: [nb*h*w][c - k1]); dA at stride 2
 * goes through the fp32 column buffer and gather kernel (single source only), everything else through im2col loads.
 * ---------------------------------------------------------------------------------------------- */
int mdb_conv3x3_igemm_f16(const mdb_gemm_desc* desc, mdb_stream_t stream);
int mdb_conv3x3_igemm_bwd_f16(const mdb_gemm_bwd_desc* desc, mdb_stream_t stream);
/* workspace floats mdb_conv3x3_igemm_bwd_f16 needs; negative MDB_ERR_* for a descriptor it rejects */
int64_t mdb_conv3x3_igemm_bwd_ws_floats(const mdb_gemm_bwd_desc* desc);

/* ------------------------------------------------------------------------------------------------
 * Fused attention, FlashAttention-style tile loop on wgmma, with TWO key/value sources whose
 * keys are concatenated in-kernel:  out = softmax([Q K0^T | Q K1^T] * scale) [V0 ; V1].
 * Replaces CrossAttention._forward (attention.py:168-199) / MemoryEfficientCrossAttention
 * (attention.py:225-250) AND the torch.cat([x_norm1] + bank) of BasicTransformerBlock 'read'
 * mode (attention.py:303-307): source 0 = the layer's own tokens, source 1 = the appearance bank.
 *   q   : fp16 [B*Nq][heads*d]                    (row stride ldq)
 *   k0  : fp16 [kv0_batches*N0][heads*d]          (row stride ldk0); kv0_batches is B or 1 (shared)
 *   vt0 : fp16 [heads*d][kv0_batches*ldv0_batch]  V TRANSPOSED: row = channel, col = key; each
 *         batch occupies ldv0_batch columns (>= N0, multiple of 8), row stride ldvt0
 *   k1/vt1 : same for source 1 (NULL / N1 = 0 when absent); only batches b < bank_batches use it
 *   out : fp16 [B*Nq][heads*d] (row stride ldo)
 * d in {40, 80, 160}.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mdb_attn_desc {
  const void* q; int64_t ldq;
  const void* k0; int64_t ldk0; const void* vt0; int64_t ldvt0; int32_t n0; int32_t kv0_batches; int32_t ldv0_batch;
  const void* k1; int64_t ldk1; const void* vt1; int64_t ldvt1; int32_t n1; int32_t kv1_batches; int32_t ldv1_batch;
  void* out; int64_t ldo;
  int32_t batch, heads, d, nq;
  int32_t bank_batches;
  float scale; /* d^-0.5 (attention.py:152) */
} mdb_attn_desc;

int mdb_attention_f16(const mdb_attn_desc* desc, mdb_stream_t stream);

/* The same forward, which also stores the softmax statistics the backward needs:
 *   lse : fp32 [batch][heads][nq], lse = log(sum_j exp(scale * q k_j^T)) over the row's keys of both sources
 *         (natural log of the SCALED scores).
 * `out` is bit-equal to mdb_attention_f16's for the same descriptor. */
int mdb_attention_lse_f16(const mdb_attn_desc* desc, float* lse, mdb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of mdb_attention_f16: the gradients of  out = softmax([Q K0^T | Q K1^T] * scale) [V0 ; V1]
 * with respect to q, k0, v0, k1, v1 — the differentiation of CrossAttention._forward (attention.py:168-199) and of
 * the torch.cat([x_norm1] + bank) of BasicTransformerBlock 'read' mode (attention.py:303-307), which carries the
 * gradient of a frozen UNet into the appearance bank.  FlashAttention-2 recompute from the stored log-sum-exp.
 * Deterministic: no atomics, two runs give bit-equal gradients.
 *   fwd          : the forward's descriptor; fwd.out is the forward's output O
 *   dout         : fp16 [B*Nq][heads*d], the gradient of out (row stride lddout, a multiple of 8)
 *   lse          : from mdb_attention_lse_f16
 *   dq           : fp16, laid out like q  [B*Nq][heads*d]          (row stride lddq)
 *   dk0 / dk1    : fp16, laid out like k* [B*N][heads*d]           (row stride lddk*)
 *   dvt0 / dvt1  : fp16, laid out like vt* [heads*d][B*ldv_batch]  (row stride lddvt*, the forward's ldv*_batch):
 *                  only valid key columns are written; padding columns, and the bank rows / columns of batch
 *                  elements b >= bank_batches, are left as they are; those bank rows of k1 and columns of vt1 are
 *                  never read, so they may hold anything, NaN and Inf included
 *   ws           : fp32 workspace of mdb_attention_bwd_ws_floats(batch, heads, nq) floats (no initial value needed)
 * Shared sources (kv*_batches == 1 with batch > 1) are rejected: their gradient needs a reduction across batch
 * elements.  Training has one bank and one prompt per sample.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mdb_attn_bwd_desc {
  mdb_attn_desc fwd;
  const void* dout; int64_t lddout;
  const float* lse;
  void* dq; int64_t lddq;
  void* dk0; int64_t lddk0; void* dvt0; int64_t lddvt0;
  void* dk1; int64_t lddk1; void* dvt1; int64_t lddvt1;
  float* ws;
} mdb_attn_bwd_desc;

int mdb_attention_bwd_f16(const mdb_attn_bwd_desc* desc, mdb_stream_t stream);
int64_t mdb_attention_bwd_ws_floats(int32_t batch, int32_t heads, int32_t nq);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm(32 groups, affine) [+ SiLU], fp32 statistics, over channels-last fp16; optionally the
 * input is the channel-concatenation of two tensors (fuses torch.cat([h, hs.pop()], 1),
 * cldm.py:104).  Replaces GroupNorm32 (ldm/modules/diffusionmodules/util.py:252-254) + nn.SiLU in
 * ResBlock.in_layers/out_layers and UNet.out (openaimodel.py:222-226,246-248,744-748), and
 * Normalize (attention.py:89-90, eps 1e-6) in SpatialTransformer.
 *   x1 [B][hw][c1], x2 [B][hw][c2] (x2 NULL => c2 = 0), y [B][hw][c1+c2].
 * Deterministic (fixed-order reductions, no atomics on data) and pivot-shifted (sums of x - x[b,0,first channel of
 * the group]), so large-mean activations do not cancel.  Two paths, chosen by batch size (mode 0), or forced
 * (mode 1 = two kernels, mode 2 = cluster):
 *   - ONE launch: a thread-block cluster per (batch element, group) exchanges its partial sums through
 *     distributed shared memory (channels per group even, i.e. c a multiple of 64); ws may be NULL;
 *   - stats (+ last-CTA fold) -> apply: needs ws of mdb_groupnorm_ws_floats(c, batch, hw) floats that were ZERO
 *     when first used (self-resetting tickets; calls of any shape on one stream may share one workspace).
 * ---------------------------------------------------------------------------------------------- */
int mdb_groupnorm_f16(const void* x1, int32_t c1, const void* x2, int32_t c2, const float* gamma, const float* beta,
                      void* y, float* ws, int32_t batch, int32_t hw, float eps, int32_t silu, int32_t mode,
                      mdb_stream_t stream);
int64_t mdb_groupnorm_ws_floats(int32_t c, int32_t batch, int32_t hw);

/* LayerNorm over the last dim (eps 1e-5), fp16 [rows][c] -> fp16; replaces nn.LayerNorm norm1/2/3 of
 * BasicTransformerBlock (attention.py:270-272). */
int mdb_layernorm_f16(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int32_t c,
                      float eps, mdb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of mdb_groupnorm_f16: the differentiation of GroupNorm32 (+ SiLU) (util.py:252-254, openaimodel.py:222-226,
 * 246-248) and Normalize (attention.py:89-90).  Per (batch element b, group g) with n = (c/32) hw, xhat = (x-mean) rstd,
 * z = gamma xhat + beta, dz = dy silu'(z) (dy without SiLU), A_bc = sum_pix dz, B_bc = sum_pix dz xhat:
 *   dx = rstd (gamma_c dz - (sum_{c in g} gamma_c A_bc + xhat sum_{c in g} gamma_c B_bc) / n),
 *   dbeta_c = sum_b A_bc, dgamma_c = sum_b B_bc (batch order).
 * The statistics are recomputed by the forward's statistics kernel.  Deterministic: fixed-order reductions through
 * fp32 partial slabs, no atomics on data.  c = c1 + c2 with c1, c2 multiples of 8, c % 32 == 0, 320 <= c <= 2560
 * (groups of 10 channels or more; the first-stage VAE's 4-channel groups are rejected), batch <= 1024.
 *   x1, x2, gamma, beta, batch, hw, eps, silu : the forward's arguments (x2 NULL => c2 = 0)
 *   dy           : fp16 [B][hw][c1+c2], the gradient of the forward's y
 *   dx1 / dx2    : [B][hw][c1] / [B][hw][c2], MDB_DTYPE_F16 | MDB_DTYPE_F32; NULL = not wanted
 *   dgamma/dbeta : fp32 [c]; NULL = not wanted (the frozen UNet needs dx only)
 *   *_accumulate : != 0 adds the gradient to the destination's contents instead of overwriting them
 *   ws           : fp32 workspace of mdb_groupnorm_bwd_ws_floats(desc) floats, ZERO when first used (the statistics
 *                  kernel's self-resetting tickets); calls of any shape on one stream may share it
 * Every pointer but gamma / beta / dgamma / dbeta is 16-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mdb_groupnorm_bwd_desc {
  const void* x1; const void* x2; int32_t c1; int32_t c2;
  const float* gamma; const float* beta;
  const void* dy;
  int32_t batch; int32_t hw; float eps; int32_t silu;
  void* dx1; int32_t dx1_dtype; int32_t dx1_accumulate;
  void* dx2; int32_t dx2_dtype; int32_t dx2_accumulate;
  float* dgamma; float* dbeta; int32_t dgamma_accumulate; int32_t dbeta_accumulate;
  float* ws;
} mdb_groupnorm_bwd_desc;

int mdb_groupnorm_bwd_f16(const mdb_groupnorm_bwd_desc* desc, mdb_stream_t stream);
/* workspace floats mdb_groupnorm_bwd_f16 needs for this descriptor; negative MDB_ERR_* for a descriptor it rejects */
int64_t mdb_groupnorm_bwd_ws_floats(const mdb_groupnorm_bwd_desc* desc);

/* Backward of mdb_layernorm_f16 (nn.LayerNorm norm1/2/3 of BasicTransformerBlock, attention.py:270-272; c = 320, 640,
 * 1280): with xhat = (x - mean) rstd and dxhat = dy gamma,
 *   dx = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)),  dgamma = sum_rows dy xhat,  dbeta = sum_rows dy.
 * One warp per row; mean and rstd are recomputed by the forward's own code (bit-identical statistics).  dgamma / dbeta
 * are deterministic column sums (per-CTA partials summed in a fixed order).
 *   x, gamma, rows, c, eps : the forward's arguments; dy fp16 [rows][c]
 *   dx     : [rows][c], dx_dtype MDB_DTYPE_F16 | MDB_DTYPE_F32; NULL = not wanted
 *   dgamma / dbeta : fp32 [c]; NULL = not wanted; *_accumulate as above
 *   ws     : fp32 workspace of mdb_layernorm_bwd_ws_floats(desc) floats (no initial value needed)
 * ---------------------------------------------------------------------------------------------- */
typedef struct mdb_layernorm_bwd_desc {
  const void* x; const float* gamma; const void* dy;
  int64_t rows; int32_t c; float eps;
  void* dx; int32_t dx_dtype; int32_t dx_accumulate;
  float* dgamma; float* dbeta; int32_t dgamma_accumulate; int32_t dbeta_accumulate;
  float* ws;
} mdb_layernorm_bwd_desc;

int mdb_layernorm_bwd_f16(const mdb_layernorm_bwd_desc* desc, mdb_stream_t stream);
int64_t mdb_layernorm_bwd_ws_floats(const mdb_layernorm_bwd_desc* desc);

/* GEGLU activation in the projection's own row order (attention.py:53-56): h = proj(x) is fp16 [m][2n] (row stride
 * ldh), values in columns [0, n), gates in [n, 2n) — a plain mdb_gemm_f16 with proj.weight / proj.bias as they are.
 *   forward : out[m][n] = v * gelu_erf(g)                                  (row stride ldo)
 *   backward: dh[m][2n] = [dout * gelu_erf(g) | dout * v * gelu_erf'(g)]    (row strides lddout, lddh)
 * n % 8 == 0, row strides multiples of 8, 16-byte aligned pointers.  The interleaved MDB_EPI_GEGLU epilogue is the
 * inference path; training differentiates this pair and the plain GEMM. */
int mdb_geglu_f16(const void* h, int64_t ldh, void* out, int64_t ldo, int64_t m, int32_t n, mdb_stream_t stream);
int mdb_geglu_bwd_f16(const void* h, int64_t ldh, const void* dout, int64_t lddout, void* dh, int64_t lddh, int64_t m,
                      int32_t n, mdb_stream_t stream);

/* Generic direct 3x3 conv (pad 1, stride 1|2) for shapes the tensor-core path does not take
 * (cin or cout not a multiple of 64): the ControlNet hint encoder (cldm.py:599-615), the 4->320
 * input conv (openaimodel.py:554-558) and the 320->4 output conv (openaimodel.py:744-748).
 *   x NHWC fp16 [B][h][w][cin]; wt fp16 [cout][3][3][cin]; y NHWC fp16 [B][ho][wo][cout];
 *   y = act(conv(x) + bias) + residual, act = SiLU when silu != 0, residual (same shape as y) optional
 *   (the ControlNet's `h += guided_hint`, cldm.py:745-749). */
int mdb_conv3x3_direct_f16(const void* x, const void* wt, const float* bias, const void* residual, void* y,
                           int32_t batch, int32_t h, int32_t w, int32_t cin, int32_t cout, int32_t stride,
                           int32_t silu, mdb_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of mdb_conv3x3_direct_f16: the differentiation of the ControlNet hint encoder (cldm.py:599-615), the 4->320
 * input conv (openaimodel.py:554-558) and the 320->4 output conv (openaimodel.py:744-748).  With z = conv(x) + bias,
 * y = act(z) + residual and dz = dy silu'(z) (dy without SiLU):
 *   dx = the transposed conv of dz, dW[o][i][kh][kw] = sum_pix dz_o x_i(shifted), dbias = sum_pix dz.
 * z is recomputed by the forward kernel (silu = 0) into the workspace; the forward's own output is never changed.
 * Stride 1: dx is the forward kernel applied to dz with wt_t, the flipped and transposed weight
 * wt_t[i][kh][kw][o] = wt[o][2-kh][2-kw][i] (at most a few hundred KB; the caller relayouts it).  Stride 2: dx by a
 * gather over the 1, 2 or 4 taps each input pixel's parity admits (any h, w).  dW / dbias: per-CTA fp32 slabs summed
 * in a fixed order, no atomics: two calls give bit-equal results.  The residual's gradient is dy itself.
 *   x, wt, bias, batch, h, w, cin, cout, stride, silu : the forward's arguments (bias may be NULL)
 *   dy     : fp16 NHWC [B][ho][wo][cout], ho = (h-1)/stride+1
 *   dx     : fp16 NHWC [B][h][w][cin], overwritten; NULL = not wanted (the first hint conv's input is the pose map)
 *   dw     : fp32 [cout][cin][3][3] (the Conv2d parameter's own OIHW layout); dbias: fp32 [cout]; NULL = not wanted;
 *            *_accumulate != 0 adds into the destination instead of overwriting it
 *   ws     : fp32 workspace of mdb_conv3x3_direct_bwd_ws_floats(desc) floats (no initial value needed)
 * x, wt, wt_t, dy, dx and ws are 16-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
typedef struct mdb_conv3x3_bwd_desc {
  const void* x; const void* wt; const void* wt_t; const float* bias; const void* dy;
  int32_t batch; int32_t h; int32_t w; int32_t cin; int32_t cout; int32_t stride; int32_t silu;
  void* dx;
  float* dw; int32_t dw_accumulate;
  float* dbias; int32_t dbias_accumulate;
  float* ws;
} mdb_conv3x3_bwd_desc;

int mdb_conv3x3_direct_bwd_f16(const mdb_conv3x3_bwd_desc* desc, mdb_stream_t stream);
/* workspace floats mdb_conv3x3_direct_bwd_f16 needs for this descriptor; negative MDB_ERR_* for one it rejects */
int64_t mdb_conv3x3_direct_bwd_ws_floats(const mdb_conv3x3_bwd_desc* desc);

/* im2col for 3x3 pad-1 convolutions, stride 1 or 2: x NHWC [B][h][w][c] -> col [B*ho*wo][9*c] with K order
 * (kh, kw, c), ho = (h-1)/stride+1, consumed by mdb_gemm_f16.  Used for Downsample.op (stride 2,
 * openaimodel.py:154-180) and as the general path for latent sizes whose rows do not tile into the
 * 128-pixel TMA boxes of the implicit-GEMM conv (any image size the reference accepts works). */
int mdb_im2col3x3_f16(const void* x, void* col, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t stride,
                      mdb_stream_t stream);

/* The same gather for a window anchored at the output pixel with ONE padding row / column at the bottom / right
 * only: ho = (h + 1 - 3)/stride + 1.  Replaces F.pad(x, (0,1,0,1)) + Conv2d(k=3, stride=2, padding=0) of the
 * first-stage VAE encoder's Downsample (ldm/modules/diffusionmodules/model.py:71-90) together with mdb_gemm_f16. */
int mdb_im2col3x3_br_f16(const void* x, void* col, int32_t batch, int32_t h, int32_t w, int32_t c, int32_t stride,
                         mdb_stream_t stream);

/* nearest x2 upsample (Upsample.forward, openaimodel.py:129-139): NHWC [B][h][w][c] -> [B][2h][2w][c] */
int mdb_upsample2x_f16(const void* x, void* y, int32_t batch, int32_t h, int32_t w, int32_t c, mdb_stream_t stream);
/* its backward: dx[B][h][w][c] (+)= the sum of each 2x2 block of dy [B][2h][2w][c] (fp16), in a fixed order;
 * dx_dtype MDB_DTYPE_F16 | MDB_DTYPE_F32, accumulate != 0 adds into dx.  c % 8 == 0, 16-byte aligned pointers. */
int mdb_upsample2x_bwd_f16(const void* dy, void* dx, int32_t dx_dtype, int32_t accumulate, int32_t batch, int32_t h,
                           int32_t w, int32_t c, mdb_stream_t stream);

/* y = a + b (b broadcast over the batch when b_batches == 1); the ControlNet residual adds
 * `h += pose_control.pop()` / `hs.pop() + pose_control.pop()` (cldm.py:93-104). n = elements per batch */
int mdb_add_f16(const void* a, const void* b, void* y, int64_t n_per_batch, int32_t batch, int32_t b_batches,
                mdb_stream_t stream);

/* timestep_embedding (util.py:189-209): t int64 [t_count] -> fp32 [batch][dim], [cos | sin], max_period 1e4; row b
 * uses t[b % t_count] (t_count = batch: one timestep per sample; fewer: the timesteps repeat, e.g. cond | uncond) */
int mdb_timestep_embedding_f32(const int64_t* t, int32_t t_count, float* out, int32_t batch, int32_t dim,
                               mdb_stream_t stream);

/* Skinny Linear for the timestep path (rows <= 16): out[r][n] = sum_k f(x[r][k]) W[n][k] + bias[n],
 * f = SiLU when silu_in, fp32 in/out, fp16 weights.  Replaces time_embed (openaimodel.py:547-551)
 * and every ResBlock.emb_layers (openaimodel.py:238-244) — all 22 of a network in one launch by
 * stacking their weights along n.  silu_out applies SiLU to the result (time_embed's middle SiLU). */
int mdb_skinny_linear_f32(const float* x, const void* w, const float* bias, float* out, int32_t rows, int32_t n,
                          int32_t k, int32_t silu_in, int32_t silu_out, mdb_stream_t stream);

/* Backward of mdb_skinny_linear_f32 without silu_out (training runs time_embed.0 with silu_out = 0 and time_embed.2
 * with silu_in = 1, which is bit-identical to the fused forward and keeps the pre-activation):
 *   dx[r][k]  = sum_n dy[r][n] W[n][k]  (* silu'(x[r][k]) when silu_in),
 *   dw[n][k]  = sum_r dy[r][n] f(x[r][k]),  dbias[n] = sum_r dy[r][n]   (f = SiLU when silu_in), all fp32.
 * Deterministic: dx sums per-chunk fp32 slabs over n in chunk order; dw / dbias sum the rows in row order.  Inputs
 * taller than 16 rows go through in row chunks: dx per chunk, dw / dbias of later chunks with *_accumulate = 1.
 *   x, w, rows, n, k, silu_in : the forward's arguments (rows 1..16, k % 8 == 0); dy fp32 [rows][n]
 *   dx fp32 [rows][k], dw fp32 [n][k], dbias fp32 [n]: NULL = not wanted; *_accumulate as above
 *   ws     : fp32 workspace of mdb_skinny_linear_bwd_ws_floats(desc) floats (no initial value needed)
 * x, w, dy, dx, dw and ws are 16-byte aligned. */
typedef struct mdb_skinny_linear_bwd_desc {
  const float* x; const void* w; const float* dy;
  int32_t rows; int32_t n; int32_t k; int32_t silu_in;
  float* dx; int32_t dx_accumulate;
  float* dw; int32_t dw_accumulate;
  float* dbias; int32_t dbias_accumulate;
  float* ws;
} mdb_skinny_linear_bwd_desc;

int mdb_skinny_linear_bwd_f32(const mdb_skinny_linear_bwd_desc* desc, mdb_stream_t stream);
int64_t mdb_skinny_linear_bwd_ws_floats(const mdb_skinny_linear_bwd_desc* desc);


/* Row softmax in place over fp16 logits x[rows][cols] (row pitch ld elements), fp32 arithmetic:
 * x <- softmax(scale * x) along the columns.  The single-head, 512-channel attention of the first-stage VAE's
 * middle block (ldm/modules/diffusionmodules/model.py:186-193: torch.bmm -> * c^-0.5 -> softmax) is run as
 * GEMM -> this -> GEMM, its head dimension being outside the fused attention kernel's range (<= 160). */
int mdb_softmax_rows_f16(void* x, int64_t ld, int32_t rows, int32_t cols, float scale, mdb_stream_t stream);

/* layout/precision boundary: the reference passes NCHW fp32 tensors (cldm.py:1099) */
/* y holds the batch `copies` times over ([copies*batch][h][w][c]): the paired cond | uncond batch of p_sample_ddim */
int mdb_nchw_f32_to_nhwc_f16(const float* x, void* y, int32_t batch, int32_t c, int32_t h, int32_t w, int32_t copies,
                             mdb_stream_t stream);
int mdb_nhwc_f16_to_nchw_f32(const void* x, float* y, int32_t batch, int32_t c, int32_t h, int32_t w, mdb_stream_t stream);

/* CFG combine + DDIM update in one pass (ddim.py:605,617-645; eps-parameterisation):
 *   e = e_u + scale (e_c - e_u); pred_x0 = (x - sqrt(1-a_t) e)/sqrt(a_t);
 *   x_prev = sqrt(a_prev) pred_x0 + sqrt(1 - a_prev - sigma^2) e + sigma * noise   (noise may be NULL when sigma == 0)
 * all tensors fp32, n elements.  coef is a DEVICE array of 6 floats
 *   {scale, sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev - sigma^2), sigma, sqrt(1 - a_t)}
 * so that one captured CUDA graph serves every DDIM step.  update_x != 0: x is overwritten with x_prev as well
 * (the chain's state advances in place). */
int mdb_cfg_ddim_update_f32(float* x, const float* eps_c, const float* eps_u, const float* noise, float* x_prev,
                            float* pred_x0, int64_t n, const float* coef, int32_t update_x, mdb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MAGICDANCE_B200_H_ */
