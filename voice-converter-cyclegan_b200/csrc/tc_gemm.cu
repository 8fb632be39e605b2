// Tensor-core gather-GEMM kernels of libcgvc.so (sm_90a): the dense contractions of the CycleGAN-VC hot path
// (module.py:22-64 convolutions, forward / data-gradient / weight-gradient) on the Hopper tensor cores (wgmma).
//
// Arithmetic: every fp32 operand x is kept in HBM as two bf16 planes (hi = bf16(x), lo = bf16(x - hi)); a product
// is evaluated as hi*hi + hi*lo + lo*hi by three wgmma (bf16 inputs) accumulating in fp32 registers ("bf16x3", ~2^-16
// relative error per product); CGVC_PREC_BF16 issues the first MMA only.  CGVC_PREC_F16F8 keeps fp16 + two scaled e4m3 planes
// instead and spends 2 MMA units per product: the two cross terms first (e4m3 wgmma), then the accumulator is rescaled by 2^-15
// and the fp16 hi*hi wgmma follow.
//
// Kernel anatomy (both kernels are persistent, one CTA per SM, 384 threads, tiles / work items walked with stride gridDim.x):
//   warps 0-3   producers: gather the activation rows (im2col rows, zero-filled at the TF-SAME borders) with 16-byte cp.async
//               into SWIZZLE_128B shared memory; one thread TMA-loads the weight (NT) / gradient (TN) tile; both complete on
//               the stage's "full" mbarrier.  Forward / data-gradient tiles that are boxes of the source planes (nt_tma_maps) take
//               the TMA form instead: one thread loads both operand tiles by TMA, the padding zero-filled by the hardware.  So do
//               weight-gradient stages of whole output rows (tn_tma_maps): the lanes of warp 0 issue the gradient atoms and one
//               activation box per output row (or per stage) and channel atom.
//   warps 4-11  two consumer warpgroups, 64 accumulator rows each: wgmma from the shared-memory stages into registers, stages
//               released through the "empty" mbarriers.  NT: the plain epilogue (bias / accumulate) stores the accumulator
//               fragments from registers; for the fused instance-norm (+GLU / +residual) forward epilogues and the opt-in fused
//               backward epilogues the finished tile is passed through shared memory, and their global stores are transposed
//               through a per-warp patch so that 8 lanes write one row.
//               TN: red.global.add of the accumulator fragments into the weight gradient.
#include "tc_gemm.cuh"
#include "geom.h"
#include "kernels.cuh"
#include "wgmma.cuh"

#include <cuda.h>      // CUtensorMap (types only: the encoder is fetched with cudaGetDriverEntryPoint, no libcuda link)
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace {

// ------------------------------------------------------------------------------------------------ TMA descriptors (host)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encoder() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
// bf16 tensor [d2][d1][d0] (d0 contiguous), box [1][b1][64], SWIZZLE_128B: lands as b1 rows of 128 bytes
bool make_tmap3(CUtensorMap* m, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b1) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return false;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * 2, d0 * d1 * 2};
  cuuint32_t box[3] = {64, b1, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// same for any element type: tensor [d2][d1][d0] (d0 contiguous, esize bytes), box [1][b1][b0], rows of b0 * esize bytes (128 or 64,
// the swizzle span: SWIZZLE_128B or SWIZZLE_64B)
bool make_tmap3_t(CUtensorMap* m, const void* base, CUtensorMapDataType dt, int esize, uint64_t d0, uint64_t d1, uint64_t d2, uint32_t b0, uint32_t b1) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return false;
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {d0 * (uint64_t)esize, d0 * d1 * (uint64_t)esize};
  cuuint32_t box[3] = {b0, b1, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(m, dt, 3, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             b0 * esize == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// An activation plane [B][Hs][Ws][ld] (esize-byte elements) as the 4-D tensor (channel, x, y, sample), box [nb][1][bx][64 channels]
// with traversal stride sx along x: a box at (c0, x * sx + ox, y * sy + oy, b) is the gathered operand of bx / sx output positions
// x, x + 1, ... of nb samples b, b + 1, ..., one 64 * esize-byte row each (SWIZZLE_128B for 128-byte rows, else SWIZZLE_64B).
// TF-SAME padding, negative coordinates included, and samples past the batch read as zeros (OOB fill NONE fills zeros).
bool make_tmap_act(CUtensorMap* m, const void* base, int esize, uint64_t ld, const GatherGeom& g, uint32_t bx, uint32_t nb) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return false;
  cuuint64_t dims[4] = {ld, (cuuint64_t)g.Ws, (cuuint64_t)g.Hs, (cuuint64_t)g.B};
  cuuint64_t strides[3] = {ld * esize, ld * esize * g.Ws, ld * esize * g.Ws * g.Hs};
  cuuint32_t box[4] = {64, bx, 1, nb};
  cuuint32_t es[4] = {1, (cuuint32_t)g.sx, 1, 1};
  return enc(m, esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, esize == 1 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier receives one arrival from this thread once all of its prior cp.async have completed
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA tile load (rank 3) into swizzled shared memory; completes `bytes` on the mbarrier
__device__ __forceinline__ void tma_load3(uint32_t dst_smem, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst_smem), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
// rank 4 (the activation maps of make_tmap_act); out-of-bounds coordinates, negative ones included, land as zeros
__device__ __forceinline__ void tma_load4(uint32_t dst_smem, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
               ::"r"(dst_smem), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Shared-memory matrix descriptor of wgmma, SWIZZLE_128B (layout type 1 in bits 62-63):
//   K-major : 8-row groups of 128-byte rows, SBO = 1024 B between groups, LBO unused
//   MN-major: atoms of (64 MN-elements x 8 K-rows) = 1024 B; LBO = stride between atoms along MN, SBO = along K
// make_desc64: SWIZZLE_64B (layout type 2), K-major: 8-row groups of 64-byte rows, SBO = 512 B
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout = 1) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (layout << 62);
}
__device__ __forceinline__ uint64_t make_desc64(uint32_t smem_addr) { return make_desc(smem_addr, 16, 512, 2); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous wgmma
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// the 256 consumer threads (two warpgroups) of a CTA; ids 1 and 2 are the epilogue groups' barriers
__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 3, 256;" ::: "memory"); }
__device__ __forceinline__ void st_shared16(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// 8 e4m3 values -> 8 fp16 values (exact: every e4m3 number is an fp16 number)
__device__ __forceinline__ uint4 e4m3x8_to_f16x8(uint2 v) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t src = (i < 2 ? v.x : v.y) >> (16 * (i & 1));
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(src & 0xFFFFu), __NV_E4M3);
    w[i] = (uint32_t)h.x | ((uint32_t)h.y << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// exact unsigned division by a runtime constant (n < 2^31): q = (umulhi(n, mul) + n) >> shr, Granlund-Montgomery round-up form
struct FastDiv { uint32_t mul, shr, d; };
__host__ inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f; f.d = d;
  uint32_t l = 0; while ((1ull << l) < d) ++l;
  f.mul = (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1);
  f.shr = l;
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, const FastDiv& f) { return (uint32_t)(((uint64_t)__umulhi(n, f.mul) + n) >> f.shr); }

// byte offset of (row r, 16-byte chunk c) inside a [rows x 128 B] SWIZZLE_128B tile (tile base 1024-aligned)
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4)); }

// ------------------------------------------------------------------------------------------------ parameters
struct TcNTParams {                 // forward / data-gradient form: D[m,n] = sum_t sum_c A[src(m,t), c] * B[t][n][c]
  GatherGeom g;
  const __nv_bfloat16 *a_hi, *a_lo; int a_ld; int C;     // gathered operand planes, row stride (elements), contraction channels
  const __nv_bfloat16 *b_hi, *b_lo; int Nw;              // weights [slab][Nw][C]
  int N;                                                 // real output columns (stores are guarded; tiles cover Nw)
  int n_tiles;                                           // column tiles to compute (host: covers the real columns only)
  int debug;                                             // diagnostic knobs (option "tc_debug", TcWeights::debug): 1 = epilogue skips its global stores, 2 = also skips
                                                         // the accumulator reads (the plain epilogue reads registers only: 2 acts as 1 there),
                                                         // 4 = producers skip the A gather (the weight gradient's too: TcTNParams::debug).
                                                         // Results are garbage; timing only.
  float* dst; int d_ld; const float* bias; int accumulate;
  int perm; int Cc;                                      // gated layers: weight rows / bias are stored tile-interleaved: tile j =
                                                         // [a-channels j*128..+127 | g-channels j*128..+127]; Cc = channels per branch
  // fused forward epilogue (EPI 1: instance norm + GLU, EPI 2: instance norm + residual); rows = whole samples of R positions
  int R;                                                 // positions per sample (32, 64 or 128)
  const float *gamma_a, *beta_a, *gamma_g, *beta_g;
  float* stats;                                          // [B,4,C]: mean_a, rstd_a, mean_g, rstd_g
  const float* resid;                                    // [M,C] (EPI 2)
  float* y; __nv_bfloat16 *y_hi, *y_lo;                  // [M,C] outputs (y may be null)
  int C_out;                                             // channels of y (Cc for gated, N for EPI 2); channels per branch (EPI 3, 4)
  // fused backward epilogue of the data-gradient form (EPI 3: GLU + instance-norm backward of the gated layer whose output this
  // gradient is; EPI 4: instance-norm backward of a residual block's second convolution).  dY = accumulator (+ dst when accumulate).
  const float* bp; int bp_ld;                            // that layer's saved pre-norm conv outputs [M, bp_ld] (a columns, then gate columns)
  __nv_bfloat16 *dp_hi, *dp_lo; int dp_ld;               // its dP planes, written here [M, dp_ld]
  float *dbeta_a, *dgamma_a, *dbeta_g, *dgamma_g;        // instance-norm parameter gradients (atomically accumulated; may be null)
  CUtensorMap tm_b_hi, tm_b_lo;                          // TMA maps of the weight planes, box [1][BN][64]
  // F16F8 mode (NPL == 3, forward only): a_hi / tm_b_hi are the fp16 planes; the e4m3 planes of both operands:
  const uint8_t *a8_hi, *a8_lo;                          // [rows, a_ld] bytes
  CUtensorMap tm_b8_hi, tm_b8_lo;                        // box [1][BN][64 bytes], SWIZZLE_64B
  uint8_t* y8;                                           // fused epilogues: q8hi plane of y [M, C_out] bytes, q8lo follows at + M * C_out (y_hi = q16)
  // packed variable-length utterances (the PK kernels, plain epilogue only): g is the 1-D geometry of all rows, pk.div the source
  // level's divisor; the output level's is pk.div * g.sx
  PackGeom pk;
  FastDiv div_bw, div_w;                                 // B * Wx and Wx: row m -> (y, b, x), see nt_row
  // the TMA form of the dense kernel (TA, see nt_tma_maps): the activation planes as make_tmap_act maps, one box per plane and stage.
  // NPL 1 / 2: the bf16 planes; NPL 3: tm_a_hi = the fp16 plane, tm_a8_hi / tm_a8_lo = the e4m3 planes (SWIZZLE_64B tiles)
  CUtensorMap tm_a_hi, tm_a_lo, tm_a8_hi, tm_a8_lo;
};
static_assert(sizeof(TcNTParams) <= 4096, "kernel parameters are limited to 4 KB");

// Rows of the NT kernel are walked output row y outermost: m = (y * B + b) * Wx + x, so that a 128-row tile spans few output rows and
// skips the taps that read only the padding for all of them (gather_tap_mask).  With Hy == 1 this is the sample order m = b * Wx + x.
struct RowPos { int b, y, x; };
__device__ __forceinline__ RowPos nt_row(const TcNTParams& p, long long m) {
  RowPos r;
  r.y = (int)fdiv((uint32_t)m, p.div_bw);
  const uint32_t rem = (uint32_t)m - (uint32_t)r.y * p.div_bw.d;
  r.b = (int)fdiv(rem, p.div_w);
  r.x = (int)(rem - (uint32_t)r.b * p.div_w.d);
  return r;
}
// the taps the tile of rows m0 .. m0 + 127 contracts over: the same list for its producers and its consumers.  PK 2 (packed 2-D
// grids): a tile inside one utterance drops the taps as the dense form does, a tile that spans utterances walks every tap
template <int PK = 0>
__device__ __forceinline__ uint32_t nt_tile_taps(const TcNTParams& p, long long m0, long long M) {
  const long long m1 = m0 + 127 < M ? m0 + 127 : M - 1;
  if constexpr (PK == 2) {
    const int dout = p.pk.div * p.g.sx;
    const Pack2Pos a = pack2_pos(p.pk, p.g.Hy, dout, m0), b = pack2_pos(p.pk, p.g.Hy, dout, m1);
    return a.u == b.u ? gather_tap_mask(p.g, a.y, b.y) : (1u << p.g.ntaps) - 1u;
  }
  return gather_tap_mask(p.g, nt_row(p, m0).y, nt_row(p, m1).y);
}

struct TcTNParams {                 // weight-gradient form: D_t[c,n] = sum_m X[src(m,t), c] * G[m, n]
  GatherGeom g;
  const __nv_bfloat16 *x_hi, *x_lo; int x_ld; int C;     // gathered operand planes [.., x_ld] (x_ld = C rounded up to 64); C = real channels (GEMM M)
  const __nv_bfloat16 *g_hi, *g_lo; int g_ld; int N;     // dense gradient planes [M, g_ld] (g_ld = N rounded up to 64); N = real columns
  float* dw_a; float* dw_g; int n_split;                 // columns [0,n_split) -> dw_a[t][c][n], rest -> dw_g[t][c][n-n_split]
  int ksplit;
  FastDiv div_hw, div_w;                                 // m -> (b, y, x) without integer division
  CUtensorMap tm_g_hi, tm_g_lo;                          // TMA maps of the gradient planes [M][g_ld], box [64 rows][64 cols]
  // F16F8 (NPL 3): x_hi / tm_g_hi are the fp16 planes; the e4m3 planes of both operands (widened to fp16 by the producers)
  const uint8_t *x8_hi, *x8_lo;                          // [rows_in, x_ld] bytes
  const uint8_t *g8_hi, *g8_lo;                          // [M, g_ld] bytes
  int w16;                                               // 1: fp16 planes only (one MMA unit per product; weight gradients are leaves of the graph)
  int fold_n;                                            // != 0: tap-folded layer (TcLayer::fold): column = t * fold_n + n of a [taps][C][fold_n] TF kernel
  // deterministic form (DET): split k stores its partial tile to part + k * part_k, laid out like [dw_a | dw_g] (dw_g at numel_a)
  float* part; long long part_k, numel_a;
  // packed variable-length utterances (the PK kernels): g is the 1-D forward geometry of all rows, pk.div the source level's divisor
  PackGeom pk;
  int debug;                                             // TcNTParams::debug; the TN kernel reads bit 4 only (producers skip the X loads)
  // the TMA form of the dense kernel (TA, see tn_tma_maps): the activation planes as make_tmap_act maps, one box per output row (or
  // per stage when Hy == 1) and channel atom.  NPL 1 / 2: the bf16 planes; NPL 3 with W16: tm_x_hi = the fp16 plane
  CUtensorMap tm_x_hi, tm_x_lo;
};
static_assert(sizeof(TcTNParams) <= 4096, "kernel parameters are limited to 4 KB");

// address of weight-gradient element (tap slab, channel c, column col) in the TF-layout kernel [taps][C][ncols]; with fold_n the layer's
// real taps live in the column dimension (col = t * fold_n + n) and the kernel in memory is [taps][C][fold_n]
__device__ __forceinline__ float* tn_dst(float* base, int slab, int C, int c, int ncols, int col, int fold_n) {
  if (fold_n) { const int t = col / fold_n; return base + ((long long)t * C + c) * fold_n + (col - t * fold_n); }
  return base + ((long long)slab * C + c) * ncols + col;
}

constexpr int kProducerThreads = 128;


// Stages of 64 contraction channels.  F16F8 (NPL = 3) stages hold one 128-byte-row tile per operand, like NPL 1: an fp16 stage the
// fp16 tiles; a cross-term stage the A rows as [64 a8_hi bytes | 64 a8_lo bytes] (SWIZZLE_128B; the TMA form: two SWIZZLE_64B tiles
// of 64-byte rows, a8_hi then a8_lo) and the weight tile as two SWIZZLE_64B tiles, b8_hi then b8_lo (TMA boxes of 64 bytes).
template <int BN, int NPL>
struct NTCfg {
  static constexpr int A_PLANE = 128 * 128;            // bytes: 128 rows x 128 B
  static constexpr int B_PLANE = BN * 128;
  static constexpr int PLANES = NPL == 2 ? 2 : 1;
  static constexpr int STAGE = PLANES * (A_PLANE + B_PLANE);
  static constexpr int STAGES = (192 * 1024) / STAGE;   // BN = 256 / 128 / 32: 2 / 3 / 4 (x3), 4 / 6 / 9 (x1, f16f8)
  static constexpr int SMEM = STAGES * STAGE + 1024;
  static_assert(STAGES * STAGE >= 128 * BN * 4, "the finished fp32 tile is staged over the pipeline stages");
};

// The finished 128 x BN fp32 tile in shared memory: row r, column n at r * BN + (n & ~31) + (((n >> 2) & 7) ^ (r & 7)) * 4 + (n & 3)
// (16-byte chunks of every 32-column block XOR-swizzled by the row: the row-per-lane reads of acc_ld32 are conflict-free)
template <int BN>
__device__ __forceinline__ int acc_off(int r, int n) { return r * BN + (n & ~31) + ((((n >> 2) & 7) ^ (r & 7)) << 2) + (n & 3); }
// columns [col, col + 32) of tile row r (col a multiple of 32)
template <int BN>
__device__ __forceinline__ void acc_ld32(const float* acc, int r, int col, uint32_t (&v)[32]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const float4 x = *reinterpret_cast<const float4*>(acc + r * BN + col + ((c ^ (r & 7)) << 2));
    v[4 * c] = __float_as_uint(x.x); v[4 * c + 1] = __float_as_uint(x.y); v[4 * c + 2] = __float_as_uint(x.z); v[4 * c + 3] = __float_as_uint(x.w);
  }
}

// ---- fused instance-norm epilogue helpers -----------------------------------------------------------------------
// Column sums over the 32 rows of a warp (row = lane): butterfly transpose-reduce, 31 shuffles for 32 columns.
// On return lane j holds the sum of column j (in t[0]).  t is destroyed.
__device__ __forceinline__ float warp_colsum32(float (&t)[32], int lane) {
#pragma unroll
  for (int o = 16, n = 32; o >= 1; o >>= 1, n >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      float send = up ? t[i] : t[i + n / 2];
      float keep = up ? t[i + n / 2] : t[i];
      t[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return t[0];
}
__device__ __forceinline__ void epi_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }      // the 4 epilogue warps of a group (barrier 1 + group)

// combine a per-warp column statistic over the warps that share a sample (spw = R/32 warps) through shared memory
__device__ __forceinline__ float sample_sum(float v, float (*xch)[32], int q, int lane, int spw, int barid) {
  if (spw == 1) return v;
  epi_bar(barid);
  xch[q][lane] = v;
  epi_bar(barid);
  const int q0 = (q / spw) * spw;
  float r = 0.f;
  for (int w = 0; w < spw; ++w) r += xch[q0 + w][lane];
  return r;
}
__device__ __forceinline__ void bc4(const float* p, float (&v)[4]) { const float4 x = *reinterpret_cast<const float4*>(p); v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; }
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
// Instance-norm statistics of one 32-column chunk held as v[32] per row-thread; writes per-column scale/offset
// (norm(x) = x*sc + of) for the 32 columns into bc[0..31] / bc[32..63] of this warp's broadcast area and returns the
// column's (mean, rstd) in lane == column.
__device__ __forceinline__ void chunk_norm_coeffs(const float (&v)[32], const float* __restrict__ gamma, const float* __restrict__ beta,
                                                  int ch, int R, float (*xch)[32], float* bc, int q, int lane, int spw, int barid, float& mean, float& rstd) {
  float t[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) t[k] = v[k];
  float s = warp_colsum32(t, lane);
  s = sample_sum(s, xch, q, lane, spw, barid);
  mean = s / (float)R;
  __syncwarp();
  bc[lane] = mean;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 32; k += 4) {
    float4 m4 = *reinterpret_cast<const float4*>(bc + k);
    float d0 = v[k] - m4.x, d1 = v[k + 1] - m4.y, d2 = v[k + 2] - m4.z, d3 = v[k + 3] - m4.w;
    t[k] = d0 * d0; t[k + 1] = d1 * d1; t[k + 2] = d2 * d2; t[k + 3] = d3 * d3;
  }
  float ss = warp_colsum32(t, lane);
  ss = sample_sum(ss, xch, q, lane, spw, barid);
  rstd = 1.f / sqrtf(ss / (float)R + 1e-6f);                       // module.py:11 epsilon
  const float sc = rstd * gamma[ch + lane];
  const float of = beta[ch + lane] - mean * sc;
  __syncwarp();
  bc[lane] = sc; bc[32 + lane] = of;
  __syncwarp();
}

// The same for a pixel-shuffled layer (module.py:135-146): post-shuffle channel c holds the conv channels c (v0) and c + C/2 (v1) of
// every conv row, so its statistics run over 2R values.
__device__ __forceinline__ void pair_norm_coeffs(const float (&v0)[32], const float (&v1)[32], const float* __restrict__ gamma, const float* __restrict__ beta,
                                                 int ch, int R, float (*xch)[32], float* bc, int q, int lane, int spw, int barid, float& mean, float& rstd) {
  float t[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) t[k] = v0[k] + v1[k];
  float s = warp_colsum32(t, lane);
  s = sample_sum(s, xch, q, lane, spw, barid);
  const float inv = 1.f / (float)(2 * R);
  mean = s * inv;
  __syncwarp();
  bc[lane] = mean;
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 32; k += 4) {
    float4 m4 = *reinterpret_cast<const float4*>(bc + k);
    const float m[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float d0 = v0[k + j] - m[j], d1 = v1[k + j] - m[j]; t[k + j] = fmaf(d0, d0, d1 * d1); }
  }
  float ss = warp_colsum32(t, lane);
  ss = sample_sum(ss, xch, q, lane, spw, barid);
  rstd = 1.f / sqrtf(ss * inv + 1e-6f);                              // module.py:11 epsilon
  const float sc = rstd * gamma[ch + lane];
  const float of = beta[ch + lane] - mean * sc;
  __syncwarp();
  bc[lane] = sc; bc[32 + lane] = of;
  __syncwarp();
}

// ---- warp-cooperative coalesced row stores -----------------------------------------------------------------------
// Every lane of an epilogue warp owns one tile row.  If each lane stored its own 32 columns, one warp-wide 16-byte store would
// touch 32 different rows (32 half-used sectors); instead the warp transposes its rows through a shared-memory patch and writes
// them back with several lanes per row.
// ---- half-width transposition patch (NT epilogues) -------------------------------------------------------------------------
// The forward / data-gradient epilogues run on 8 warps per CTA, and shared memory is full with the
// pipeline stages, so their per-warp patch is 32 rows x 16 words = 2 KB: a 32-word row passes through it in two halves.  16-byte
// chunk c (0..3) of row r lives at word r*16 + ((c ^ ((r >> 1) & 3)) << 2): conflict-free for the row-wise writes (lane = row) and
// for the write-back role (chunk lane & 3 of rows (lane >> 2) + 8 i), which covers 8 rows x 64 bytes per warp instruction.
__device__ __forceinline__ uint32_t hp_off(int r, int c) { return (uint32_t)(r * 16 + ((c ^ ((r >> 1) & 3)) << 2)); }
// this lane's 32 words (its tile row) -> f(rr, w0, val): val = words [w0, w0 + 4) of tile row rr; 8 calls per lane
template <class F>
__device__ __forceinline__ void rows_out(float* stg, const float (&o)[32], int lane, F f) {
  const int hc = lane & 3, hr = lane >> 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __syncwarp();                                          // earlier readers of the patch are done
#pragma unroll
    for (int c = 0; c < 4; ++c)
      *reinterpret_cast<float4*>(stg + hp_off(lane, c)) = make_float4(o[16 * h + 4 * c], o[16 * h + 4 * c + 1], o[16 * h + 4 * c + 2], o[16 * h + 4 * c + 3]);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = hr + 8 * i;
      f(rr, 16 * h + 4 * hc, *reinterpret_cast<const float4*>(stg + hp_off(rr, hc)));
    }
  }
}
// the inverse: pre[4 h + i] = words [16 h + 4 (lane & 3), + 4) of tile row (lane >> 2) + 8 i (fetched by the caller, 8 rows x 64 bytes
// per warp instruction) -> v = this lane's row
__device__ __forceinline__ void rows_in(float* stg, float (&v)[32], int lane, const float4 (&pre)[8]) {
  const int hc = lane & 3, hr = lane >> 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i) *reinterpret_cast<float4*>(stg + hp_off(hr + 8 * i, hc)) = pre[4 * h + i];
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float4 x = *reinterpret_cast<const float4*>(stg + hp_off(lane, c));
      v[16 * h + 4 * c] = x.x; v[16 * h + 4 * c + 1] = x.y; v[16 * h + 4 * c + 2] = x.z; v[16 * h + 4 * c + 3] = x.w;
    }
  }
}
// fetch for rows_in: 32 columns [col, col + 32) of the dense rows mq .. mq + 31 of a [M, ld] fp32 matrix (rows >= M read as zero)
__device__ __forceinline__ void rows_fetch(float4 (&pre)[8], const float* base, long long ld, long long mq, long long M, int col, int lane) {
  const int hc = lane & 3, hr = lane >> 2;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int rr = hr + 8 * i;
      pre[4 * h + i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (mq + rr < M) pre[4 * h + i] = *reinterpret_cast<const float4*>(base + (mq + rr) * ld + col + 16 * h + 4 * hc);
    }
}
__device__ __forceinline__ void hload_rows(float* stg, float (&v)[32], const float* base, long long ld, long long mq, long long M, int col, int lane) {
  float4 pre[8];
  rows_fetch(pre, base, ld, mq, M, col, lane);
  rows_in(stg, v, lane, pre);
}
// the staged block to 32 arbitrary destination rows (null = row outside the tensor), columns [col0, col0 + 32)
__device__ __forceinline__ void hwrite_rows_f32(float* stg, const float (&o)[32], float* const* rowp, int col0, int lane) {
  rows_out(stg, o, lane, [&](int rr, int w0, float4 val) {
    float* rp = rowp[rr];
    if (rp != nullptr) *reinterpret_cast<float4*>(rp + col0 + w0) = val;
  });
}
// y[32] of this lane's row -> optional fp32 copy and the bf16 hi/lo planes of the dense [M, C] activation (rows mq .. mq + 31)
// rs / ro: destination row of tile row r is r * rs + ro (pixel shuffle: the two halves of a conv row are output rows 2r and 2r + 1)
__device__ __forceinline__ void hwrite_y(float* stg, const float (&y)[32], float* yf, __nv_bfloat16* yhi, __nv_bfloat16* ylo,
                                         long long mq, long long M, int C, int ch, int lane, int rs = 1, int ro = 0) {
  if (yf)
    rows_out(stg, y, lane, [&](int rr, int w0, float4 val) {
      if (mq + rr < M) *reinterpret_cast<float4*>(yf + ((mq + rr) * rs + ro) * C + ch + w0) = val;
    });
  // planes: the row's 32 words are [16 words of hi bf16 pairs | 16 words of lo bf16 pairs]; word w of a half = columns 2w, 2w + 1
  float hl[32];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    __nv_bfloat162 hh = __floats2bfloat162_rn(y[2 * k], y[2 * k + 1]);
    float2 f = __bfloat1622float2(hh);
    __nv_bfloat162 ll = __floats2bfloat162_rn(y[2 * k] - f.x, y[2 * k + 1] - f.y);
    hl[k] = __uint_as_float(*reinterpret_cast<uint32_t*>(&hh)); hl[16 + k] = __uint_as_float(*reinterpret_cast<uint32_t*>(&ll));
  }
  rows_out(stg, hl, lane, [&](int rr, int w0, float4 val) {
    __nv_bfloat16* plane = (w0 < 16) ? yhi : ylo;
    if (mq + rr < M) *reinterpret_cast<float4*>(plane + ((mq + rr) * rs + ro) * C + ch + 2 * (w0 & 15)) = val;
  });
}
// F16F8 variant: the row's 32 words are [16 words of fp16 pairs | 8 words of e4m3 hi quads | 8 words of e4m3 lo quads]
__device__ __forceinline__ void hwrite_yq(float* stg, const float (&y)[32], float* yf, __nv_bfloat16* q16, uint8_t* q8,
                                          long long mq, long long M, int C, int ch, int lane, int rs = 1, int ro = 0) {
  if (yf)
    rows_out(stg, y, lane, [&](int rr, int w0, float4 val) {
      if (mq + rr < M) *reinterpret_cast<float4*>(yf + ((mq + rr) * rs + ro) * C + ch + w0) = val;
    });
  float w[32];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float v[4] = {y[4 * k], y[4 * k + 1], y[4 * k + 2], y[4 * k + 3]};
    uint2 h; uint32_t b_hi, b_lo;
    cgvc_quant4(v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO, h, b_hi, b_lo);
    w[2 * k] = __uint_as_float(h.x); w[2 * k + 1] = __uint_as_float(h.y);
    w[16 + k] = __uint_as_float(b_hi); w[24 + k] = __uint_as_float(b_lo);
  }
  rows_out(stg, w, lane, [&](int rr, int w0, float4 val) {
    if (mq + rr >= M) return;
    const long long r = (mq + rr) * rs + ro;
    uint8_t* dst;
    if (w0 < 16) dst = reinterpret_cast<uint8_t*>(q16) + (r * C + ch + 2 * w0) * 2;                  // 8 fp16 columns
    else if (w0 < 24) dst = q8 + r * C + ch + 4 * (w0 - 16);                                           // 16 e4m3 columns
    else dst = q8 + M * rs * C + r * C + ch + 4 * (w0 - 24);
    *reinterpret_cast<float4*>(dst) = val;
  });
}

// ---- epilogue of one 128-row x BN-column accumulator tile ------------------------------------------------------------------
// Called by the 8 consumer warps of a CTA once the finished tile is in shared memory (acc, layout acc_off): 4 warps (one per 32-row
// quarter q) form a group; group grp of ngrp takes the 32-column chunks grp, grp + ngrp, ... of the tile.  m0 = first row of the
// tile, n0 = its first column.  stg / rowp / bc: this warp's 2 KB transposition patch, destination-row table and coefficient
// broadcast area; epi_xch: the group's cross-warp exchange area (statistics of samples that span several warps; barrier 1 + grp).
template <int BN, int NPL, int EPI>
__device__ __forceinline__ void nt_tile_epilogue(const TcNTParams& p, const long long M, const long long m0, const int n0,
                                                 const int q, const int lane, float* stg, float** rowp, float* bc, float (*epi_xch)[32],
                                                 const float* acc, const int grp = 0, const int ngrp = 1) {
  const GatherGeom& g = p.g;
  const int barid = 1 + grp;
  const int arow = q * 32 + lane;                        // this lane's tile row
  const long long mq = m0 + q * 32;                      // first row of this warp
  const long long m = mq + lane;
  float* drow = nullptr;
  if (m < M && p.dst) {                                  // dst may be null for the fused forward epilogues (inference: nothing kept for backward)
    const RowPos o = nt_row(p, m);
    long long dr = ((long long)(o.b * g.Hd + o.y * g.dsy + g.doy) * g.Wd + o.x * g.dsx + g.dox);
    drow = p.dst + dr * p.d_ld;
  }
  __syncwarp();
  rowp[lane] = drow;                                     // destination row of every tile row, for the write-back lanes
  __syncwarp();
  {
    // ---- fused forward epilogue: the 128 rows of the tile are whole samples of R positions (R = 32, 64, 128) ----
    const int spw = p.R >> 5;                              // warps per sample
    const long long sample = mq / p.R;
    const bool stat_writer = (q % spw) == 0 && mq < M && p.stats != nullptr;
    if (EPI == 1) {
      // gated: tile = [128 a-channels | the same 128 g-channels]; y = IN(a) * sigmoid(IN(g))   (module.py:3-20,85-98)
      const int ch0 = n0 >> 1;
#pragma unroll 1
      for (int cb = grp; cb < 4; cb += ngrp) {
        const int ch = ch0 + cb * 32;
        float va[32], vg[32];
        { uint32_t u[32]; acc_ld32<BN>(acc, arow, (cb * 32), u);
#pragma unroll
          for (int k = 0; k < 32; k += 4) { float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + cb * 32 + k);
            va[k] = __uint_as_float(u[k]) + bb.x; va[k + 1] = __uint_as_float(u[k + 1]) + bb.y; va[k + 2] = __uint_as_float(u[k + 2]) + bb.z; va[k + 3] = __uint_as_float(u[k + 3]) + bb.w; } }
        { uint32_t u[32]; acc_ld32<BN>(acc, arow, (128 + cb * 32), u);
#pragma unroll
          for (int k = 0; k < 32; k += 4) { float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + 128 + cb * 32 + k);
            vg[k] = __uint_as_float(u[k]) + bb.x; vg[k + 1] = __uint_as_float(u[k + 1]) + bb.y; vg[k + 2] = __uint_as_float(u[k + 2]) + bb.z; vg[k + 3] = __uint_as_float(u[k + 3]) + bb.w; } }
        // pre-norm outputs are kept for the backward pass
        if (p.dst) {
          hwrite_rows_f32(stg, va, rowp, ch, lane);
          hwrite_rows_f32(stg, vg, rowp, p.Cc + ch, lane);
        }
        float mean_a, rstd_a, mean_g, rstd_g;
        chunk_norm_coeffs(va, p.gamma_a, p.beta_a, ch, p.R, epi_xch, bc, q, lane, spw, barid, mean_a, rstd_a);
        chunk_norm_coeffs(vg, p.gamma_g, p.beta_g, ch, p.R, epi_xch, bc + 64, q, lane, spw, barid, mean_g, rstd_g);
        if (stat_writer) {
          float* st = p.stats + sample * 4 * p.C_out + ch + lane;
          st[0] = mean_a; st[p.C_out] = rstd_a; st[2 * p.C_out] = mean_g; st[3 * p.C_out] = rstd_g;
        }
#pragma unroll
        for (int k = 0; k < 32; k += 4) {                  // y overwrites va
          float4 sa = *reinterpret_cast<const float4*>(bc + k), oa = *reinterpret_cast<const float4*>(bc + 32 + k);
          float4 sg = *reinterpret_cast<const float4*>(bc + 64 + k), og = *reinterpret_cast<const float4*>(bc + 96 + k);
          va[k]     = fmaf(va[k],     sa.x, oa.x) * fast_sigmoid(fmaf(vg[k],     sg.x, og.x));
          va[k + 1] = fmaf(va[k + 1], sa.y, oa.y) * fast_sigmoid(fmaf(vg[k + 1], sg.y, og.y));
          va[k + 2] = fmaf(va[k + 2], sa.z, oa.z) * fast_sigmoid(fmaf(vg[k + 2], sg.z, og.z));
          va[k + 3] = fmaf(va[k + 3], sa.w, oa.w) * fast_sigmoid(fmaf(vg[k + 3], sg.w, og.w));
        }
        if (NPL == 3) hwrite_yq(stg, va, p.y, p.y_hi, p.y8, mq, M, p.C_out, ch, lane);
        else hwrite_y(stg, va, p.y, p.y_hi, p.y_lo, mq, M, p.C_out, ch, lane);
      }
    } else if (EPI == 5) {
      // gated + pixel shuffle (upsample1d_block, module.py:115-146): the tile holds, for 64 post-shuffle channels c, the conv columns
      // [a(c) | a(c + Ch) | g(c) | g(c + Ch)], 64 each (Ch = Cc / 2 post-shuffle channels).  Conv row r of a sample becomes output rows
      // 2r (columns c) and 2r + 1 (columns c + Ch); the statistics of channel c run over both: 2R positions.
      const int Ch = p.C_out;
      const int ch0 = n0 >> 2;
#pragma unroll 1
      for (int cb = grp; cb < 2; cb += ngrp) {
        const int ch = ch0 + cb * 32;
        auto load = [&](float (&v)[32], int tcol) {
          uint32_t u[32]; acc_ld32<BN>(acc, arow, tcol, u);
#pragma unroll
          for (int k = 0; k < 32; k += 4) { float4 bb = *reinterpret_cast<const float4*>(p.bias + n0 + tcol + k);
            v[k] = __uint_as_float(u[k]) + bb.x; v[k + 1] = __uint_as_float(u[k + 1]) + bb.y; v[k + 2] = __uint_as_float(u[k + 2]) + bb.z; v[k + 3] = __uint_as_float(u[k + 3]) + bb.w; }
        };
        float mean_a, rstd_a, mean_g, rstd_g;
        {                                                  // gate branch first: statistics only, the values are re-read from the tile below
          float g0[32], g1[32];
          load(g0, 128 + cb * 32); load(g1, 192 + cb * 32);
          if (p.dst) { hwrite_rows_f32(stg, g0, rowp, p.Cc + ch, lane); hwrite_rows_f32(stg, g1, rowp, p.Cc + Ch + ch, lane); }
          pair_norm_coeffs(g0, g1, p.gamma_g, p.beta_g, ch, p.R, epi_xch, bc + 64, q, lane, spw, barid, mean_g, rstd_g);
        }
        float a0[32], a1[32];
        load(a0, cb * 32); load(a1, 64 + cb * 32);
        if (p.dst) { hwrite_rows_f32(stg, a0, rowp, ch, lane); hwrite_rows_f32(stg, a1, rowp, Ch + ch, lane); }
        pair_norm_coeffs(a0, a1, p.gamma_a, p.beta_a, ch, p.R, epi_xch, bc, q, lane, spw, barid, mean_a, rstd_a);
        if (stat_writer) {
          float* st = p.stats + sample * 4 * Ch + ch + lane;
          st[0] = mean_a; st[Ch] = rstd_a; st[2 * Ch] = mean_g; st[3 * Ch] = rstd_g;
        }
        auto emit = [&](const float (&a)[32], const int s) {
          float gg[32];
          load(gg, 128 + s * 64 + cb * 32);
#pragma unroll
          for (int k = 0; k < 32; k += 4) {
            float4 sa = *reinterpret_cast<const float4*>(bc + k), oa = *reinterpret_cast<const float4*>(bc + 32 + k);
            float4 sg = *reinterpret_cast<const float4*>(bc + 64 + k), og = *reinterpret_cast<const float4*>(bc + 96 + k);
            gg[k]     = fmaf(a[k],     sa.x, oa.x) * fast_sigmoid(fmaf(gg[k],     sg.x, og.x));
            gg[k + 1] = fmaf(a[k + 1], sa.y, oa.y) * fast_sigmoid(fmaf(gg[k + 1], sg.y, og.y));
            gg[k + 2] = fmaf(a[k + 2], sa.z, oa.z) * fast_sigmoid(fmaf(gg[k + 2], sg.z, og.z));
            gg[k + 3] = fmaf(a[k + 3], sa.w, oa.w) * fast_sigmoid(fmaf(gg[k + 3], sg.w, og.w));
          }
          if (NPL == 3) hwrite_yq(stg, gg, p.y, p.y_hi, p.y8, mq, M, Ch, ch, lane, 2, s);
          else hwrite_y(stg, gg, p.y, p.y_hi, p.y_lo, mq, M, Ch, ch, lane, 2, s);
        };
        emit(a1, 1);
        emit(a0, 0);
      }
    } else if (EPI == 2) {
      // EPI 2: y = resid + IN(conv)   (residual1d_block second half, module.py:79-83); 256 independent channels per tile
#pragma unroll 1
      for (int cb = grp; cb < BN / 32; cb += ngrp) {
        const int ch = n0 + cb * 32;
        if (ch >= p.N) break;
        // the residual input (read 4 lanes per row, 8 rows per instruction) is fetched first: its global-memory latency hides behind the
        // accumulator load and the statistics of this chunk
        float4 rpre[8];
        rows_fetch(rpre, p.resid, p.C_out, mq, M, ch, lane);
        float va[32];
        { uint32_t u[32]; acc_ld32<BN>(acc, arow, (cb * 32), u);
#pragma unroll
          for (int k = 0; k < 32; k += 4) { float4 bb = *reinterpret_cast<const float4*>(p.bias + ch + k);
            va[k] = __uint_as_float(u[k]) + bb.x; va[k + 1] = __uint_as_float(u[k + 1]) + bb.y; va[k + 2] = __uint_as_float(u[k + 2]) + bb.z; va[k + 3] = __uint_as_float(u[k + 3]) + bb.w; } }
        if (p.dst) hwrite_rows_f32(stg, va, rowp, ch, lane);
        float mean_a, rstd_a;
        chunk_norm_coeffs(va, p.gamma_a, p.beta_a, ch, p.R, epi_xch, bc, q, lane, spw, barid, mean_a, rstd_a);
        if (stat_writer) {
          float* st = p.stats + sample * 4 * p.C_out + ch + lane;
          st[0] = mean_a; st[p.C_out] = rstd_a; st[2 * p.C_out] = 0.f; st[3 * p.C_out] = 1.f;
        }
        // transpose the residual through the patch: every lane then holds its own row
        float res[32];
        rows_in(stg, res, lane, rpre);
#pragma unroll
        for (int k = 0; k < 32; k += 4) {
          float4 scl = *reinterpret_cast<const float4*>(bc + k), of = *reinterpret_cast<const float4*>(bc + 32 + k);
          va[k] = fmaf(va[k], scl.x, of.x) + res[k]; va[k + 1] = fmaf(va[k + 1], scl.y, of.y) + res[k + 1];
          va[k + 2] = fmaf(va[k + 2], scl.z, of.z) + res[k + 2]; va[k + 3] = fmaf(va[k + 3], scl.w, of.w) + res[k + 3];
        }
        if (NPL == 3) hwrite_yq(stg, va, p.y, p.y_hi, p.y8, mq, M, p.C_out, ch, lane);
        else hwrite_y(stg, va, p.y, p.y_hi, p.y_lo, mq, M, p.C_out, ch, lane);
      }
    } else {
      // ---- EPI 3 / 4: fused backward (SURVEY.md Appendix A.7).  The tile holds dY for 256 output channels of whole samples.
      //   EPI 3 (gated layer):  y = na * sigmoid(ng), na = IN(a), ng = IN(g):  dna = dY * s, dng = dna * na * (1 - s)
      //   EPI 4 (residual h2):  y = resid + IN(a):                             dna = dY (also written back: it is the skip gradient)
      //   IN backward per (sample, channel):  dx = sc * (dn - mean_R(dn) - xhat * mean_R(dn * xhat)),  sc = gamma * rstd
      const int C = p.C_out;
      const float invR = 1.f / (float)p.R;
      const bool live = mq < M;
#pragma unroll 1
      for (int cb = grp; cb < BN / 32; cb += ngrp) {
        const int ch = n0 + cb * 32;
        if (ch >= p.N) break;
        float dy[32], xa[32];
        { uint32_t u[32]; acc_ld32<BN>(acc, arow, (cb * 32), u);
#pragma unroll
          for (int k = 0; k < 32; ++k) dy[k] = __uint_as_float(u[k]); }
        if (p.accumulate) {
          hload_rows(stg, xa, p.dst, p.d_ld, mq, M, ch, lane);
#pragma unroll
          for (int k = 0; k < 32; ++k) dy[k] += xa[k];
        }
        if (EPI == 4) {                                    // gradient w.r.t. the block output: the next block's skip gradient
          rows_out(stg, dy, lane, [&](int rr, int w0, float4 val) {
            if (mq + rr < M) *reinterpret_cast<float4*>(p.dst + (mq + rr) * p.d_ld + ch + w0) = val;
          });
        }
        // per-column coefficients of this warp's sample (lane == column): xhat = x * r + h ; norm = x * sc + of
        {
          const float* st = p.stats + sample * 4 * C + ch + lane;
          const float mean = live ? st[0] : 0.f, rstd = live ? st[C] : 1.f;
          const float scl = rstd * p.gamma_a[ch + lane];
          __syncwarp();
          bc[lane] = rstd; bc[32 + lane] = -mean * rstd; bc[64 + lane] = scl;
          if (EPI == 3) {
            bc[96 + lane] = p.beta_a[ch + lane] - mean * scl;
            const float mg = live ? st[2 * C] : 0.f, rg = live ? st[3 * C] : 1.f;
            const float sg = rg * p.gamma_g[ch + lane];
            bc[128 + lane] = rg; bc[160 + lane] = -mg * rg; bc[192 + lane] = sg; bc[224 + lane] = p.beta_g[ch + lane] - mg * sg;
          }
          __syncwarp();
        }
        hload_rows(stg, xa, p.bp, p.bp_ld, mq, M, ch, lane);
        float dg[32], xg[32];
        if (EPI == 3) {
          hload_rows(stg, xg, p.bp, p.bp_ld, mq, M, C + ch, lane);
#pragma unroll
          for (int k = 0; k < 32; k += 4) {
            float ra[4], ha[4], sa[4], oa[4], rg[4], hg[4], sg[4], og[4];
            bc4(bc + k, ra); bc4(bc + 32 + k, ha); bc4(bc + 64 + k, sa); bc4(bc + 96 + k, oa);
            bc4(bc + 128 + k, rg); bc4(bc + 160 + k, hg); bc4(bc + 192 + k, sg); bc4(bc + 224 + k, og);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float na = fmaf(xa[k + j], sa[j], oa[j]), ng = fmaf(xg[k + j], sg[j], og[j]);
              const float sgm = fast_sigmoid(ng);
              const float dna = dy[k + j] * sgm;
              dy[k + j] = dna; dg[k + j] = dna * na * (1.f - sgm);
              xa[k + j] = fmaf(xa[k + j], ra[j], ha[j]);      // xhat_a
              xg[k + j] = fmaf(xg[k + j], rg[j], hg[j]);      // xhat_g
            }
          }
        } else {
#pragma unroll
          for (int k = 0; k < 32; k += 4) {
            float ra[4], ha[4];
            bc4(bc + k, ra); bc4(bc + 32 + k, ha);
#pragma unroll
            for (int j = 0; j < 4; ++j) xa[k + j] = fmaf(xa[k + j], ra[j], ha[j]);
          }
        }
        // column sums over this warp's 32 rows (lane == column), parameter gradients, then over the whole sample
        float t[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) t[k] = dy[k];
        float s1a = warp_colsum32(t, lane);
#pragma unroll
        for (int k = 0; k < 32; ++k) t[k] = dy[k] * xa[k];
        float s2a = warp_colsum32(t, lane);
        float s1g = 0.f, s2g = 0.f;
        if (EPI == 3) {
#pragma unroll
          for (int k = 0; k < 32; ++k) t[k] = dg[k];
          s1g = warp_colsum32(t, lane);
#pragma unroll
          for (int k = 0; k < 32; ++k) t[k] = dg[k] * xg[k];
          s2g = warp_colsum32(t, lane);
        }
        if (p.dbeta_a && live) {
          atomicAdd(p.dbeta_a + ch + lane, s1a); atomicAdd(p.dgamma_a + ch + lane, s2a);
          if (EPI == 3) { atomicAdd(p.dbeta_g + ch + lane, s1g); atomicAdd(p.dgamma_g + ch + lane, s2g); }
        }
        s1a = sample_sum(s1a, epi_xch, q, lane, spw, barid); s2a = sample_sum(s2a, epi_xch, q, lane, spw, barid);
        if (EPI == 3) { s1g = sample_sum(s1g, epi_xch, q, lane, spw, barid); s2g = sample_sum(s2g, epi_xch, q, lane, spw, barid); }
        {
          const float sca = bc[64 + lane], scg = EPI == 3 ? bc[192 + lane] : 0.f;
          __syncwarp();
          bc[256 + lane] = sca * s1a * invR; bc[288 + lane] = sca * s2a * invR;
          if (EPI == 3) { bc[320 + lane] = scg * s1g * invR; bc[352 + lane] = scg * s2g * invR; }
          __syncwarp();
        }
#pragma unroll
        for (int k = 0; k < 32; k += 4) {
          float c1[4], c2[4], c3[4];
          bc4(bc + 64 + k, c1); bc4(bc + 256 + k, c2); bc4(bc + 288 + k, c3);
#pragma unroll
          for (int j = 0; j < 4; ++j) dy[k + j] = fmaf(c1[j], dy[k + j], -fmaf(xa[k + j], c3[j], c2[j]));
        }
        hwrite_y(stg, dy, nullptr, p.dp_hi, p.dp_lo, mq, M, p.dp_ld, ch, lane);
        if (EPI == 3) {
#pragma unroll
          for (int k = 0; k < 32; k += 4) {
            float c1[4], c2[4], c3[4];
            bc4(bc + 192 + k, c1); bc4(bc + 320 + k, c2); bc4(bc + 352 + k, c3);
#pragma unroll
            for (int j = 0; j < 4; ++j) dg[k + j] = fmaf(c1[j], dg[k + j], -fmaf(xg[k + j], c3[j], c2[j]));
          }
          hwrite_y(stg, dg, nullptr, p.dp_hi, p.dp_lo, mq, M, p.dp_ld, C + ch, lane);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ consumer K loop
// MMAs of one pipeline stage.  The kind is a template argument, so that no wgmma sits under a runtime branch (which makes ptxas
// serialise the asynchronous MMAs): F16F8 walks its two passes as two calls.
// MMA_E4M3_CROSS64: the same products from A rows held as two SWIZZLE_64B tiles (a8_hi, then a8_lo), as the TMA form loads them
enum { MMA_BF16 = 0, MMA_BF16X3 = 1, MMA_E4M3_CROSS = 2, MMA_F16 = 3, MMA_F16_CROSS = 4, MMA_E4M3_CROSS64 = 5 };

// One consumer warpgroup walks nkb pipeline stages: wait for the stage, issue its MMAs, release the previous stage once those have
// completed.  TN = 0: both operands K-major, 128-byte rows (forward / data gradient); TN = 1: both MN-major, 64-element atoms at
// 8192 B (weight gradient).  The warpgroup's A rows (NT) / channels (TN) start at wg * 8192 (MMA_E4M3_CROSS64: 64-byte rows, wg * 4096).
template <int BN, int KIND, int TN, class Cfg>
__device__ __forceinline__ void consume_stages(float (&d)[BN / 2], int nkb, int& stage, uint32_t& phase, int& prev,
                                               uint64_t* full_bar, uint64_t* empty_bar, uint32_t smem_base, int wg, int lane) {
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    fence_proxy_async();                                     // producers' generic-proxy writes (cp.async, st.shared) -> wgmma reads
    const uint32_t sA = smem_base + stage * Cfg::STAGE + wg * (KIND == MMA_E4M3_CROSS64 ? 4096 : 8192);
    const uint32_t sB = smem_base + stage * Cfg::STAGE + Cfg::PLANES * Cfg::A_PLANE;
    fence_acc(d);
    wgmma_fence();
    if constexpr (TN == 0) {
      if constexpr (KIND == MMA_E4M3_CROSS) {                // K = 32 e4m3 per instruction: a8_hi x b8_lo + a8_lo x b8_hi
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_e4m3<BN>(d, make_desc(sA + k * 32, 16, 1024), make_desc64(sB + Cfg::B_PLANE / 2 + k * 32), 1);
          wgmma_e4m3<BN>(d, make_desc(sA + 64 + k * 32, 16, 1024), make_desc64(sB + k * 32), 1);
        }
      } else if constexpr (KIND == MMA_E4M3_CROSS64) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_e4m3<BN>(d, make_desc64(sA + k * 32), make_desc64(sB + Cfg::B_PLANE / 2 + k * 32), 1);
          wgmma_e4m3<BN>(d, make_desc64(sA + Cfg::A_PLANE / 2 + k * 32), make_desc64(sB + k * 32), 1);
        }
      } else if constexpr (KIND == MMA_F16) {                // fp16 hi x hi, one 64-channel tile of K = 16 steps
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_f16<BN, 0, 0>(d, make_desc(sA + k * 32, 16, 1024), make_desc(sB + k * 32, 16, 1024), 1);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {                        // K = 16 bf16 = 32 bytes along the swizzled row
          const uint64_t a_hi = make_desc(sA + k * 32, 16, 1024), b_hi = make_desc(sB + k * 32, 16, 1024);
          wgmma_bf16<BN, 0, 0>(d, a_hi, b_hi, 1);
          if constexpr (KIND == MMA_BF16X3) {
            const uint64_t a_lo = make_desc(sA + Cfg::A_PLANE + k * 32, 16, 1024), b_lo = make_desc(sB + Cfg::B_PLANE + k * 32, 16, 1024);
            wgmma_bf16<BN, 0, 0>(d, a_hi, b_lo, 1);
            wgmma_bf16<BN, 0, 0>(d, a_lo, b_hi, 1);
          }
        }
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {                          // K = 16 K-rows = two 8-row groups = 2048 bytes
        const uint64_t a0 = make_desc(sA + k * 2048, 8192, 1024), b0 = make_desc(sB + k * 2048, 8192, 1024);
        const uint64_t a1 = make_desc(sA + Cfg::A_PLANE + k * 2048, 8192, 1024), b1 = make_desc(sB + Cfg::B_PLANE + k * 2048, 8192, 1024);
        if constexpr (KIND == MMA_F16_CROSS) {               // the widened e4m3 planes: x8hi x g8lo + x8lo x g8hi
          wgmma_f16<BN, 1, 1>(d, a0, b1, 1);
          wgmma_f16<BN, 1, 1>(d, a1, b0, 1);
        } else if constexpr (KIND == MMA_F16) {
          wgmma_f16<BN, 1, 1>(d, a0, b0, 1);
        } else {
          wgmma_bf16<BN, 1, 1>(d, a0, b0, 1);
          if constexpr (KIND == MMA_BF16X3) {
            wgmma_bf16<BN, 1, 1>(d, a0, b1, 1);
            wgmma_bf16<BN, 1, 1>(d, a1, b0, 1);
          }
        }
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                                         // the previous stage's MMAs have completed: release it
    fence_acc(d);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
  }
}
// all MMAs issued so far complete, then D *= scale (folds the common power of two of the F16F8 cross products out of D)
template <int N>
__device__ __forceinline__ void rescale_acc(float (&d)[N], float scale) {
  wgmma_wait<0>();
  fence_acc(d);
#pragma unroll
  for (int i = 0; i < N; ++i) d[i] *= scale;
}

// ---- plain epilogue (EPI 0) straight from the accumulator fragments ----------------------------------------------------------
// This thread's fragments are tile rows r and r + 8, columns 8 j + c + {0, 1} of every 8-column block j (c = 2 (t % 4)).  y = D (+ bias),
// stored or (accumulate) added.  One float2 store of a warp covers 8 rows x 32 contiguous bytes: whole sectors.  Nothing passes through
// the pipeline stages, so the producers fill them with the next tile's operands meanwhile.
// PK 2: row m of the packed output grid goes to its own utterance's rows of the packed destination grid
template <int BN, int PK = 0>
__device__ __forceinline__ void nt_store_fragments(const TcNTParams& p, const float (&d)[BN / 2], const long long M,
                                                   const long long m0, const int n0, const int r, const int c) {
  const GatherGeom& g = p.g;
  float* rowp[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long long m = m0 + r + 8 * h;
    rowp[h] = nullptr;
    if (m < M && p.dst) {
      if constexpr (PK == 2) {
        const int dout = p.pk.div * g.sx;
        const Pack2Pos o = pack2_pos(p.pk, g.Hy, dout, m);
        const long long r = pack2_row(o.o0, o.o1, g.Hd, dout / g.dsx, o.y * g.dsy + g.doy, o.x * g.dsx + g.dox);
        if (r >= 0) rowp[h] = p.dst + r * p.d_ld;            // (a data-gradient class row always lies inside its utterance)
      } else {
        const RowPos o = nt_row(p, m);
        rowp[h] = p.dst + ((long long)(o.b * g.Hd + o.y * g.dsy + g.doy) * g.Wd + o.x * g.dsx + g.dox) * p.d_ld;
      }
    }
  }
  const bool vec = (p.d_ld & 1) == 0;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int cb = j >> 2;                                   // 32-column block of the tile
    // gated layers store their weight rows tile-interleaved ([128 a | 128 g] per 256-wide tile): map back
    // (shuffled gated layers: [64 a s0 | 64 a s1 | 64 g s0 | 64 g s1] for 64 post-shuffle channels, see EPI 5)
    const int n = (p.perm == 2 ? (cb >> 2) * p.Cc + ((cb >> 1) & 1) * (p.Cc >> 1) + (n0 >> 2) + (cb & 1) * 32
                   : p.perm    ? ((cb < 4) ? (n0 >> 1) + cb * 32 : p.Cc + (n0 >> 1) + (cb - 4) * 32) : n0 + cb * 32) + ((8 * j) & 31) + c;
    if (n >= p.N) continue;                                  // padded columns are never stored
    float2 bb = make_float2(0.f, 0.f);
    if (p.bias) bb = *reinterpret_cast<const float2*>(p.bias + n0 + 8 * j + c);   // bias in weight-row order
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float* rp = rowp[h];
      if (rp == nullptr) continue;
      float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      if (p.bias) { v0 += bb.x; v1 += bb.y; }
      if (vec && n + 2 <= p.N) {
        if (p.accumulate)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(rp + n), "f"(v0), "f"(v1) : "memory");
        else
          *reinterpret_cast<float2*>(rp + n) = make_float2(v0, v1);
      } else {                                               // a data gradient with an odd cin (the discriminator's one-channel input)
        if (p.accumulate) atomicAdd(rp + n, v0); else rp[n] = v0;
        if (n + 1 < p.N) { if (p.accumulate) atomicAdd(rp + n + 1, v1); else rp[n + 1] = v1; }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ NT kernel
// Persistent: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ... (m or n fastest, see n_fast).
// 384 threads:
//   warps 0-3   producers (A rows by cp.async, weight tile by TMA), running ahead across K-blocks
//   warps 4-11  two consumer warpgroups: wgmma of tile rows 64 wg .. + 63 into registers (BN / 2 per thread).  The plain epilogue
//               (EPI 0) stores the fragments from registers (nt_store_fragments) while the producers already load the next tile.
//               The fused epilogues write the whole tile to shared memory over the pipeline stages -- they hold nothing at that
//               point, because the producers wait for the epilogue of a tile before they load the next one -- and the 8 warps run
//               the epilogue in two groups of 4.  (The accumulator of a 256-wide tile does not fit next to the stages: 128 KB.)
constexpr int kNTThreads = 384;

// PK 1: the packed form (cgvc_generator_forward_packed).  Row m's source rows are those of its own utterance: the producers keep
// (first source row of the utterance, its length at the source level, local position * stride) where the dense form keeps (b, y, x).
// PK 2: the packed 2-D form (cgvc_discriminator_forward_packed, kernels.cuh PackGeom2): the producers keep (first source row of the
// utterance, y * sy, x * sx) and the utterance's source width
// TA: the dense form whose tiles are boxes of the activation planes (nt_tma_maps): one producer thread issues, per stage, one TMA of
// each A plane beside the weight tile, and the full barriers expect that one arrival plus the bytes.  The stages' contents are those
// of the gather, so every MMA sees the same operands in the same order.
template <int BN, int NPL, int EPI, int PK = 0, int TA = 0>
__global__ void __launch_bounds__(kNTThreads, 1)
tc_gg_nt_kernel(const __grid_constant__ TcNTParams p) {
  static_assert(!PK || EPI == 0, "packed rows never take the fused epilogues (they need whole equal-length samples per tile)");
  static_assert(!PK || !TA, "the TMA form is dense");
  using Cfg = NTCfg<BN, NPL>;
  __shared__ float epi_xch[2][4][32];                        // cross-warp exchange of the fused epilogue, per group
  __shared__ __align__(16) float epi_bc[8][(EPI == 3 || EPI == 4) ? 384 : 128];   // per-warp broadcast of per-column coefficients (32 floats per quantity)
  __shared__ __align__(16) float epi_stage[8][32 * 16];      // per-warp half-width transposition patch of the coalesced row stores
  __shared__ float* epi_rowp[8][32];                         // destination row of every tile row
  constexpr int S = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[S], empty_bar[S], acc_free_bar;

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GatherGeom& g = p.g;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  // K blocks ("stages"): 64 channels each; F16F8 walks the contraction twice -- first the two fp8 cross products (planes
  // a8_hi x b8_lo and a8_lo x b8_hi), then the fp16 hi x hi product after the rescale of D.  A tile walks only its taps
  // (nt_tile_taps): cchunks stages per tap and pass
  const int cchunks = p.C >> 6;
  const int m_tiles = (int)((M + 127) / 128);
  const int n_tiles = p.n_tiles;
  const int num_tiles = m_tiles * n_tiles;
  // Tile order.  1-D layers walk m fastest: the CTAs that run at once share the weight tile in L2.  2-D layers (rows output row y
  // outermost, see nt_row) walk n fastest: the CTAs that run at once share the activation rows of a few m tiles, which all kernel
  // rows re-read, while the m tiles of different output rows read overlapping source rows at different times
  const bool n_fast = g.Hy > 1;

  if (threadIdx.x == 0) {
    // full: 128 cp.async arrivals (A rows) + 1 arrive.expect_tx whose bytes the weight-tile TMA completes (TA: that one arrival,
    // whose bytes both operand TMAs complete); empty / acc_free: one arrival per consumer warp
    for (int s = 0; s < S; ++s) { mbar_init(&full_bar[s], TA ? 1 : kProducerThreads + 1); mbar_init(&empty_bar[s], 8); }
    mbar_init(&acc_free_bar, 8);
    fence_barrier_init();
    tma_prefetch_desc(&p.tm_b_hi);
    if (NPL == 2) tma_prefetch_desc(&p.tm_b_lo);
    if (NPL == 3) { tma_prefetch_desc(&p.tm_b8_hi); tma_prefetch_desc(&p.tm_b8_lo); }
    if (TA) {
      tma_prefetch_desc(&p.tm_a_hi);
      if (NPL == 2) tma_prefetch_desc(&p.tm_a_lo);
      if (NPL == 3) { tma_prefetch_desc(&p.tm_a8_hi); tma_prefetch_desc(&p.tm_a8_lo); }
    }
  }
  __syncthreads();

  if (TA && warp < 4) {
    // ===================== producer (TMA form): thread 0 issues both operand tiles of every stage =====================
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const long long m0 = (long long)(n_fast ? tile / n_tiles : tile % m_tiles) * 128;
        const int n0 = (n_fast ? tile % n_tiles : tile / m_tiles) * BN;
        if (EPI != 0 && it > 0) mbar_wait(&acc_free_bar, (uint32_t)(it - 1) & 1u);
        const uint32_t taps = nt_tile_taps<PK>(p, m0, M);
        const RowPos o = nt_row(p, m0);                        // the tile: positions o.x .. of samples o.b .. at output row o.y
        const uint32_t a_bytes = (p.debug & 4) ? 0u : (uint32_t)Cfg::PLANES * Cfg::A_PLANE;
        for (int pass = 0; pass < (NPL == 3 ? 2 : 1); ++pass)
        for (int tap = 0; tap < g.ntaps; ++tap) {
          if (!((taps >> tap) & 1u)) continue;
          const int xs = o.x * g.sx + g.ox[tap], ys = o.y * g.sy + g.oy[tap];
          for (int cc = 0; cc < cchunks; ++cc) {
            const int c0 = cc << 6;
            mbar_wait(&empty_bar[stage], phase ^ 1);
            const uint32_t sA = smem_base + stage * Cfg::STAGE;
            const uint32_t sB = sA + Cfg::PLANES * Cfg::A_PLANE;
            mbar_expect_tx(&full_bar[stage], a_bytes + Cfg::PLANES * Cfg::B_PLANE);
            if (NPL == 3 && pass == 0) {
              tma_load3(sB, &p.tm_b8_hi, c0, n0, g.widx[tap], &full_bar[stage]);
              tma_load3(sB + Cfg::B_PLANE / 2, &p.tm_b8_lo, c0, n0, g.widx[tap], &full_bar[stage]);
              if (a_bytes) {
                tma_load4(sA, &p.tm_a8_hi, c0, xs, ys, o.b, &full_bar[stage]);
                tma_load4(sA + Cfg::A_PLANE / 2, &p.tm_a8_lo, c0, xs, ys, o.b, &full_bar[stage]);
              }
            } else {
              tma_load3(sB, &p.tm_b_hi, c0, n0, g.widx[tap], &full_bar[stage]);
              if (NPL == 2) tma_load3(sB + Cfg::B_PLANE, &p.tm_b_lo, c0, n0, g.widx[tap], &full_bar[stage]);
              if (a_bytes) {
                tma_load4(sA, &p.tm_a_hi, c0, xs, ys, o.b, &full_bar[stage]);
                if (NPL == 2) tma_load4(sA + Cfg::A_PLANE, &p.tm_a_lo, c0, xs, ys, o.b, &full_bar[stage]);
              }
            }
            if (++stage == S) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp < 4) {
    // ===================== producers =====================
    const int t = threadIdx.x;
    const int chunk = t & 7, rsub = t >> 3;                 // 8 threads cover one 128-byte row; 16 rows per pass
    int stage = 0; uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const long long m0 = (long long)(n_fast ? tile / n_tiles : tile % m_tiles) * 128;
      const int n0 = (n_fast ? tile % n_tiles : tile / m_tiles) * BN;
      if (EPI != 0 && it > 0) mbar_wait(&acc_free_bar, (uint32_t)(it - 1) & 1u);   // the previous tile's epilogue has left the stages
      const uint32_t taps = nt_tile_taps<PK>(p, m0, M);
      int rb[8], ry[8], rx[8];                              // decoded output coordinates of this thread's 8 A rows
      int rw[PK == 2 ? 8 : 1];                              // PK 2: the source width of the row's utterance
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        long long m = m0 + rsub + 16 * i;
        if (m < M) {
          if constexpr (PK == 2) {
            const Pack2Pos o = pack2_pos(p.pk, g.Hy, p.pk.div * g.sx, m);
            rb[i] = (int)(g.Hs * o.o0 / p.pk.div); rw[i] = (int)((o.o1 - o.o0) / p.pk.div); ry[i] = o.y * g.sy; rx[i] = o.x * g.sx;
          } else if constexpr (PK) {                         // rb = first source row, ry = source length, rx = local position * stride
            const int dout = p.pk.div * g.sx;
            const int u = pack_find(p.pk.off, p.pk.n, m * dout);
            const long long o0 = __ldg(p.pk.off + u), o1 = __ldg(p.pk.off + u + 1);
            rb[i] = (int)(o0 / p.pk.div); ry[i] = (int)((o1 - o0) / p.pk.div); rx[i] = (int)(m - o0 / dout) * g.sx;
          } else {
            const RowPos o = nt_row(p, m);
            rb[i] = o.b; ry[i] = o.y * g.sy; rx[i] = o.x * g.sx;
          }
        } else { rb[i] = -1; ry[i] = 0; rx[i] = 0; }
      }
      for (int pass = 0; pass < (NPL == 3 ? 2 : 1); ++pass)
      for (int tap = 0; tap < g.ntaps; ++tap) {
        if (!((taps >> tap) & 1u)) continue;                 // its A tile would be all zeros
        long long aoff[8];                                   // element offset of the source row, or -1
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int cofs = NPL == 3 && pass == 0 ? (chunk & 3) * 16 : chunk * 8;
          if constexpr (PK == 2) {
            const int yy = ry[i] + g.oy[tap], xx = rx[i] + g.ox[tap];
            aoff[i] = rb[i] >= 0 && yy >= 0 && yy < g.Hs && xx >= 0 && xx < rw[i] ? ((long long)rb[i] + yy * rw[i] + xx) * p.a_ld + cofs : -1;
          } else if constexpr (PK) {
            const int xx = rx[i] + g.ox[tap];
            aoff[i] = rb[i] >= 0 && xx >= 0 && xx < ry[i] ? (long long)(rb[i] + xx) * p.a_ld + cofs : -1;
          } else {
            int yy = ry[i] + g.oy[tap], xx = rx[i] + g.ox[tap];
            bool ok = rb[i] >= 0 && yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws;
            aoff[i] = ok ? ((long long)(rb[i] * g.Hs + yy) * g.Ws + xx) * p.a_ld + cofs : -1;
          }
        }
        for (int cc = 0; cc < cchunks; ++cc) {
          const int c0 = cc << 6;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const uint32_t sA = smem_base + stage * Cfg::STAGE;
          const uint32_t sB = sA + Cfg::PLANES * Cfg::A_PLANE;
          if (t == 0) {                                      // weight tile [BN rows n][128 bytes of c] by TMA (hardware swizzle)
            mbar_expect_tx(&full_bar[stage], Cfg::PLANES * Cfg::B_PLANE);
            if (NPL == 3) {
              if (pass == 0) {                               // e4m3: two tiles of 64-byte rows
                tma_load3(sB, &p.tm_b8_hi, c0, n0, g.widx[tap], &full_bar[stage]);
                tma_load3(sB + Cfg::B_PLANE / 2, &p.tm_b8_lo, c0, n0, g.widx[tap], &full_bar[stage]);
              } else {
                tma_load3(sB, &p.tm_b_hi, c0, n0, g.widx[tap], &full_bar[stage]);
              }
            } else {
              tma_load3(sB, &p.tm_b_hi, c0, n0, g.widx[tap], &full_bar[stage]);
              if (NPL == 2) tma_load3(sB + Cfg::B_PLANE, &p.tm_b_lo, c0, n0, g.widx[tap], &full_bar[stage]);
            }
          }
          if (!(p.debug & 4)) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int r = rsub + 16 * i;
              const uint32_t so = sw128(r, chunk);
              const bool ok = aoff[i] >= 0;
              const long long off = ok ? aoff[i] + c0 : 0;
              if (NPL == 3) {
                if (pass == 0)                               // row = [64 a8_hi bytes | 64 a8_lo bytes]
                  cp_async16(sA + so, (chunk < 4 ? p.a8_hi : p.a8_lo) + off, ok ? 16u : 0u);
                else                                         // 64 fp16
                  cp_async16(sA + so, p.a_hi + off, ok ? 16u : 0u);
              } else {
                cp_async16(sA + so, p.a_hi + off, ok ? 16u : 0u);
                if (NPL == 2) cp_async16(sA + Cfg::A_PLANE + so, p.a_lo + off, ok ? 16u : 0u);
              }
            }
          }
          cp_async_arrive_noinc(&full_bar[stage]);
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: MMA, then epilogue =====================
    const int cw = warp - 4;                                 // consumer warp 0..7
    const int wg = cw >> 2;                                  // warpgroup: tile rows 64 wg .. + 63
    const int tw = threadIdx.x - 128 * (wg + 1);             // thread within the warpgroup
    float* acc_s = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)));
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long m0 = (long long)(n_fast ? tile / n_tiles : tile % m_tiles) * 128;
      const int n0 = (n_fast ? tile % n_tiles : tile / m_tiles) * BN;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int prev = -1;                                         // stage whose MMAs may still be in flight
      const int kb_pass = __popc(nt_tile_taps<PK>(p, m0, M)) * cchunks;   // (> 0 for TF-SAME geometries; 0 is safe)
      if constexpr (NPL == 3) {                             // e4m3 cross products, then the fp16 hi x hi products after the rescale of D
        consume_stages<BN, TA ? MMA_E4M3_CROSS64 : MMA_E4M3_CROSS, 0, Cfg>(d, kb_pass, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
        rescale_acc(d, 1.f / (float)(1 << CGVC_Q_ACC_SHIFT));
        consume_stages<BN, MMA_F16, 0, Cfg>(d, kb_pass, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
      } else {
        consume_stages<BN, NPL == 2 ? MMA_BF16X3 : MMA_BF16, 0, Cfg>(d, kb_pass, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
      }
      wgmma_wait<0>();
      fence_acc(d);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      const int r0 = wg * 64 + (tw >> 5) * 16 + ((tw & 31) >> 2), c0 = 2 * (tw & 3);   // this thread's fragment rows r0, r0 + 8
      if constexpr (EPI == 0) {
        if (!(p.debug & 3)) nt_store_fragments<BN, PK>(p, d, M, m0, n0, r0, c0);
      } else {
        // the tile into shared memory once both warpgroups are done reading the stages
        consumer_bar();
        if (!(p.debug & 2)) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(acc_s + acc_off<BN>(r0, 8 * j + c0)) = make_float2(d[4 * j], d[4 * j + 1]);
            *reinterpret_cast<float2*>(acc_s + acc_off<BN>(r0 + 8, 8 * j + c0)) = make_float2(d[4 * j + 2], d[4 * j + 3]);
          }
        }
        consumer_bar();
        nt_tile_epilogue<BN, NPL, EPI>(p, M, m0, n0, cw & 3, lane, epi_stage[cw], epi_rowp[cw], epi_bc[cw], epi_xch[wg], acc_s, wg, 2);
        fence_proxy_async();                                 // generic accesses of the stages before the next tile's TMA writes
        __syncwarp();
        if (lane == 0) mbar_arrive(&acc_free_bar);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ TN kernel (wgrad)
// Tile: 128 channels (GEMM M, operand A = X, MN-major) x 256 gradient columns (GEMM N, operand B = G, MN-major);
// the contraction runs over rows m of the forward output grid, 64 rows per stage.  NPL 1 / 2: the bf16 planes (hi | hi + lo).
// NPL 3 (CGVC_PREC_F16F8): X and G are kept as fp16 + two scaled e4m3 planes, both with the activation-role scales (1, 2^12), so
// both cross products x8hi * g8lo and x8lo * g8hi carry 2^12.  Unless p.w16 is set, the row range of a work item is walked twice:
// first the cross products -- e4m3 wgmma reads K-major operands only, and both operands are MN-major here, so the producers widen
// the e4m3 tiles to fp16 (exactly) on their way into shared memory and the products run as fp16 MMAs --, then the accumulator is
// rescaled by 2^-12 and the fp16 hi x hi products follow.  W16 (selected by p.w16) is the fp16-only form: its stages hold one plane
// per operand, so twice as many fit.
#define CGVC_Q_WGRAD_SHIFT 12
template <int NPL, int W16>
struct TNCfg {
  static constexpr int A_PLANE = 64 * 256;              // 64 K-rows x 128 channels x 2 B  (2 MN-atoms side by side: LBO = 8192)
  static constexpr int B_PLANE = 64 * 512;              // 64 K-rows x 256 columns x 2 B  (4 MN-atoms: LBO = 8192)
  static constexpr int PLANES = (NPL == 1 || W16) ? 1 : 2;
  static constexpr int STAGE = PLANES * (A_PLANE + B_PLANE);
  static constexpr int STAGES = (192 * 1024) / STAGE;   // 2 (x3, f16f8), 4 (x1, f16f8 with W16)
  static constexpr int SMEM = STAGES * STAGE + 1024;
};

// Persistent like the NT kernel: work items (n-tile, c-tile, tap, K-split) are walked with stride gridDim.x (n fastest, so
// concurrently running CTAs share the same rows of X and dP in L2).  Each consumer warpgroup owns 64 of the 128 channels.
// DET (deterministic mode, ksplit > 1): the fragments are stored to the K-split's partial slab instead of added into dW; launch_tn then
// adds the partials in K-split order (launch_reduce_parts)
// PK: the packed form (packed generator tapes).  K-row m (an output row of all packed rows) gathers its source row from its own
// utterance u = pack_find(m * dout): local position (m - off[u] / dout) * stride + tap offset, a zero row outside [0, len_u / div)
// PK 2: packed 2-D grids (kernels.cuh PackGeom2): K-row m finds (u, y, x) in the output grid and reads its own utterance's source row,
// a zero row outside it
// TA: the dense form whose stages are boxes of the activation planes (tn_tma_maps): the lanes of producer warp 0 issue, per stage, the
// gradient atoms and one TMA per box of whole output rows and channel atom; lane 0 arms the full barrier with every box's bytes first.
// The stages' contents are those of the gather (the boxes zero-fill padding, samples past the batch and channels past x_ld), so
// every MMA sees the same operands in the same order.
template <int NPL, int W16, int DET, int PK = 0, int TA = 0>
__global__ void __launch_bounds__(kNTThreads, 1)
tc_gg_tn_kernel(const __grid_constant__ TcTNParams p) {
  static_assert(W16 == 0 || NPL == 3, "the fp16-only weight gradient is a form of CGVC_PREC_F16F8");
  static_assert(!TA || (!PK && (NPL != 3 || W16)), "the TMA form is dense and loads the planes as they are (no e4m3 widening)");
  using Cfg = TNCfg<NPL, W16>;
  constexpr int S = Cfg::STAGES;
  constexpr int BN = 256;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[S], empty_bar[S];

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const GatherGeom& g = p.g;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  const int HW = g.Hy * g.Wx;
  const int n_tiles = (p.g_ld + BN - 1) / BN, c_tiles = (p.x_ld + 127) / 128;
  const int num_items = n_tiles * c_tiles * g.ntaps * p.ksplit;
  constexpr int pass0 = (NPL == 3 && !W16) ? 0 : 1;       // pass 0: the F16F8 cross products; pass 1: the main products
  long long chunk_rows = (M + p.ksplit - 1) / p.ksplit;
  chunk_rows = (chunk_rows + 63) / 64 * 64;

  struct Item { int n0, c0, tap, ks; long long mbeg, mend; int num_kb; };
  auto decode = [&](int item) -> Item {
    Item w;
    int n_t = item % n_tiles; int t1 = item / n_tiles;
    int c_t = t1 % c_tiles; int t2 = t1 / c_tiles;
    w.tap = t2 % g.ntaps; const int ks = t2 / g.ntaps; w.ks = ks;
    w.n0 = n_t * BN; w.c0 = c_t * 128;
    w.mbeg = (long long)ks * chunk_rows;
    w.mend = (w.mbeg + chunk_rows < M) ? w.mbeg + chunk_rows : M;
    w.num_kb = w.mend > w.mbeg ? (int)((w.mend - w.mbeg + 63) / 64) : 0;
    return w;
  };

  if (threadIdx.x == 0) {
    // full: 128 cp.async arrivals (X rows) + 1 arrive.expect_tx whose bytes the gradient-tile TMA completes (TA: that one arrival,
    // whose bytes both operands' TMAs complete); empty: one arrival per consumer warp
    for (int s = 0; s < S; ++s) { mbar_init(&full_bar[s], TA ? 1 : kProducerThreads + 1); mbar_init(&empty_bar[s], 8); }
    fence_barrier_init();
    tma_prefetch_desc(&p.tm_g_hi);
    if (NPL == 2) tma_prefetch_desc(&p.tm_g_lo);
    if (TA) { tma_prefetch_desc(&p.tm_x_hi); if (NPL == 2) tma_prefetch_desc(&p.tm_x_lo); }
  }
  __syncthreads();

  if (TA && warp < 4) {
    // ---- producer (TMA form): lanes 0-3 load the gradient atoms, lanes 4 .. 4 + 2 * nbox - 1 one X box each (box j, atom a).  A box
    // is box_rows K-rows: 64 / Wx whole samples at y = 0 (Hy == 1), one output row (b, y) of a 2-D grid, or 64 positions of one row;
    // box j lands at row j * box_rows of both MN atoms, a 1024-byte boundary (Wx >= 8), so the 128B swizzle is the one sw128 writes
    if (warp == 0) {
      const int box_rows = (g.Hy == 1 || g.Wx >= 64) ? 64 : g.Wx;
      const int nbox = 64 / box_rows;
      const uint32_t x_bytes = (p.debug & 4) ? 0u : (uint32_t)Cfg::PLANES * Cfg::A_PLANE;   // both atoms, OOB-filled ones included
      int stage = 0; uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const Item w = decode(item);
        for (int kb = 0; kb < w.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const uint32_t sA = smem_base + stage * Cfg::STAGE;
          const uint32_t sB = sA + Cfg::PLANES * Cfg::A_PLANE;
          const int row0 = (int)(w.mbeg + (long long)kb * 64);
          if (lane == 0) {
            int natoms = 0;
#pragma unroll
            for (int a = 0; a < 4; ++a) natoms += (w.n0 + a * 64) < p.g_ld ? 1 : 0;
            mbar_expect_tx(&full_bar[stage], Cfg::PLANES * natoms * 8192 + x_bytes);
          }
          __syncwarp();                                        // the barrier expects the bytes before any of them can land
          if (lane < 4) {
            if ((w.n0 + lane * 64) < p.g_ld) {
              tma_load3(sB + lane * 8192, &p.tm_g_hi, w.n0 + lane * 64, row0, 0, &full_bar[stage]);
              if (NPL == 2) tma_load3(sB + Cfg::B_PLANE + lane * 8192, &p.tm_g_lo, w.n0 + lane * 64, row0, 0, &full_bar[stage]);
            }
          } else if (x_bytes && lane < 4 + 2 * nbox) {
            const int j = (lane - 4) >> 1, a = (lane - 4) & 1;
            const uint32_t mu = (uint32_t)(row0 + j * box_rows);     // rows past M are samples past the batch: zeros
            const int b = (int)fdiv(mu, p.div_hw); const int rem = (int)(mu - (uint32_t)b * (uint32_t)HW);
            const int y = (int)fdiv((uint32_t)rem, p.div_w); const int x = rem - y * g.Wx;
            const int c0 = w.c0 + a * 64, xs = x * g.sx + g.ox[w.tap], ys = y * g.sy + g.oy[w.tap];
            const uint32_t dst = sA + a * 8192 + j * box_rows * 128;
            tma_load4(dst, &p.tm_x_hi, c0, xs, ys, b, &full_bar[stage]);
            if (NPL == 2) tma_load4(dst + Cfg::A_PLANE, &p.tm_x_lo, c0, xs, ys, b, &full_bar[stage]);
          }
          if (++stage == S) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < 4) {
    // ---- producers: every K-row (one output position m) is a contiguous run of channels / columns in global memory
    const int t = threadIdx.x;
    const int chunk = t & 7, rsub = t >> 3;                 // 8 threads x 16 B = one 128-byte atom row; 16 rows per pass
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const Item w = decode(item);
      for (int pass = pass0; pass < 2; ++pass)
      for (int kb = 0; kb < w.num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        const uint32_t sA = smem_base + stage * Cfg::STAGE;
        const uint32_t sB = sA + Cfg::PLANES * Cfg::A_PLANE;
        long long xoff[4];                                   // source row of each of this thread's 4 K-rows (-1: zero row)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const long long m = w.mbeg + (long long)kb * 64 + rsub + 16 * i;
          xoff[i] = -1;
          if (m < w.mend) {
            if constexpr (PK == 2) {
              const Pack2Pos o = pack2_pos(p.pk, g.Hy, p.pk.div * g.sx, m);
              const long long r = pack2_row(o.o0, o.o1, g.Hs, p.pk.div, o.y * g.sy + g.oy[w.tap], o.x * g.sx + g.ox[w.tap]);
              if (r >= 0) xoff[i] = r * p.x_ld + w.c0 + chunk * 8;
            } else if constexpr (PK) {
              const int dout = p.pk.div * g.sx;
              const int u = pack_find(p.pk.off, p.pk.n, m * dout);
              const long long o0 = __ldg(p.pk.off + u), o1 = __ldg(p.pk.off + u + 1);
              const int xx = (int)(m - o0 / dout) * g.sx + g.ox[w.tap];
              if (xx >= 0 && xx < (int)((o1 - o0) / p.pk.div)) xoff[i] = (o0 / p.pk.div + xx) * p.x_ld + w.c0 + chunk * 8;
            } else {
              const uint32_t mu = (uint32_t)m;
              int b = (int)fdiv(mu, p.div_hw); int rem = (int)(mu - (uint32_t)b * (uint32_t)HW);
              int y = (int)fdiv((uint32_t)rem, p.div_w); int x = rem - y * g.Wx;
              int yy = y * g.sy + g.oy[w.tap], xx = x * g.sx + g.ox[w.tap];
              if (yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws)
                xoff[i] = ((long long)(b * g.Hs + yy) * g.Ws + xx) * p.x_ld + w.c0 + chunk * 8;
            }
          }
        }
        if (NPL == 3 && pass == 0) {
          // e4m3 planes, widened to fp16 here: plane 0 = hi, plane 1 = lo, for both operands
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int kr = rsub + 16 * i;
            const uint32_t so = sw128(kr, chunk);
#pragma unroll
            for (int a = 0; a < 2; ++a) {                     // 2 channel atoms of 64
              if (p.debug & 4) break;                           // (tc_debug 4: the X rows are not loaded)
              const bool ok = xoff[i] >= 0 && (w.c0 + a * 64) < p.x_ld;
              uint2 vh = make_uint2(0u, 0u), vl = make_uint2(0u, 0u);
              if (ok) { vh = __ldg(reinterpret_cast<const uint2*>(p.x8_hi + xoff[i] + a * 64)); vl = __ldg(reinterpret_cast<const uint2*>(p.x8_lo + xoff[i] + a * 64)); }
              st_shared16(sA + a * 8192 + so, e4m3x8_to_f16x8(vh));
              st_shared16(sA + Cfg::A_PLANE + a * 8192 + so, e4m3x8_to_f16x8(vl));
            }
            const long long m = w.mbeg + (long long)kb * 64 + kr;
#pragma unroll
            for (int a = 0; a < 4; ++a) {                     // 4 gradient-column atoms of 64
              const int col = w.n0 + a * 64 + chunk * 8;
              const bool ok = m < w.mend && col < p.g_ld;
              uint2 vh = make_uint2(0u, 0u), vl = make_uint2(0u, 0u);
              if (ok) { vh = __ldg(reinterpret_cast<const uint2*>(p.g8_hi + m * p.g_ld + col)); vl = __ldg(reinterpret_cast<const uint2*>(p.g8_lo + m * p.g_ld + col)); }
              st_shared16(sB + a * 8192 + so, e4m3x8_to_f16x8(vh));
              st_shared16(sB + Cfg::B_PLANE + a * 8192 + so, e4m3x8_to_f16x8(vl));
            }
          }
          fence_proxy_async();                               // generic stores -> visible to the tensor cores' reads
          if (t == 0) mbar_expect_tx(&full_bar[stage], 0);   // (the arrival the TMA thread makes in the other pass)
          mbar_arrive(&full_bar[stage]);
        } else {
          if (t == 0) {
            // gradient tile: 64 K-rows x 256 columns = 4 MN-atoms of [64 rows][64 cols]; rows >= M are zero-filled by TMA
            // (a stage never straddles two K-splits: split boundaries are multiples of 64 rows)
            const int row0 = (int)(w.mbeg + (long long)kb * 64);
            int natoms = 0;
#pragma unroll
            for (int a = 0; a < 4; ++a) natoms += (w.n0 + a * 64) < p.g_ld ? 1 : 0;
            mbar_expect_tx(&full_bar[stage], (NPL == 2 ? 2 : 1) * natoms * 8192);
#pragma unroll
            for (int a = 0; a < 4; ++a) {
              if ((w.n0 + a * 64) < p.g_ld) {
                tma_load3(sB + a * 8192, &p.tm_g_hi, w.n0 + a * 64, row0, 0, &full_bar[stage]);
                if (NPL == 2) tma_load3(sB + Cfg::B_PLANE + a * 8192, &p.tm_g_lo, w.n0 + a * 64, row0, 0, &full_bar[stage]);
              }
            }
          }
          if (!(p.debug & 4))                                  // (tc_debug 4: the X rows are not loaded)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint32_t so = sw128(rsub + 16 * i, chunk);   // (kr/8)*1024 + (kr%8)*128 + swizzled chunk
#pragma unroll
            for (int a = 0; a < 2; ++a) {                     // 2 channel atoms of 64
              const bool ok = xoff[i] >= 0 && (w.c0 + a * 64) < p.x_ld;
              const long long off = ok ? xoff[i] + a * 64 : 0;
              cp_async16(sA + a * 8192 + so, p.x_hi + off, ok ? 16u : 0u);
              if (NPL == 2) cp_async16(sA + Cfg::A_PLANE + a * 8192 + so, p.x_lo + off, ok ? 16u : 0u);
            }
          }
          cp_async_arrive_noinc(&full_bar[stage]);
        }
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ---- consumers: MMA, then red.global.add of the fragments into dW (TF layout [t][c][n]); split-K partials meet there
    const int cw = warp - 4;
    const int wg = cw >> 2;                                  // warpgroup: channels c0 + 64 wg .. + 63 (MN atom wg of the X tile)
    const int tw = threadIdx.x - 128 * (wg + 1);
    int stage = 0; uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const Item w = decode(item);
      if (w.num_kb == 0) continue;
      float d[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      int prev = -1;
      if constexpr (NPL == 3 && !W16) {
        consume_stages<BN, MMA_F16_CROSS, 1, Cfg>(d, w.num_kb, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
        rescale_acc(d, 1.f / (float)(1 << CGVC_Q_WGRAD_SHIFT));
        consume_stages<BN, MMA_F16, 1, Cfg>(d, w.num_kb, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
      } else if constexpr (NPL == 3) {
        consume_stages<BN, MMA_F16, 1, Cfg>(d, w.num_kb, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
      } else {
        consume_stages<BN, NPL == 2 ? MMA_BF16X3 : MMA_BF16, 1, Cfg>(d, w.num_kb, stage, phase, prev, full_bar, empty_bar, smem_base, wg, lane);
      }
      wgmma_wait<0>();
      fence_acc(d);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      const int c = w.c0 + wg * 64 + (tw >> 5) * 16 + ((tw & 31) >> 2);   // fragment rows c and c + 8
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = w.n0 + 8 * j + 2 * (tw & 3);
        if (n >= p.N) continue;
        float* base; int nn; int ncols;                      // (n even and n_split even: a column pair never straddles the split)
        if (n < p.n_split) { base = DET ? p.part + w.ks * p.part_k : p.dw_a; nn = n; ncols = p.n_split; }
        else { base = DET ? p.part + w.ks * p.part_k + p.numel_a : p.dw_g; nn = n - p.n_split; ncols = p.N - p.n_split; }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (c + 8 * h >= p.C) continue;
          float* dst = tn_dst(base, g.widx[w.tap], p.C, c + 8 * h, ncols, nn, p.fold_n);
          if constexpr (DET) asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1]) : "memory");
          else asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(d[4 * j + 2 * h]), "f"(d[4 * j + 2 * h + 1]) : "memory");
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ weight planes
// Row of the forward weight / bias planes that holds output channel co of a branch (noff = 0: a, != 0: gate) of a layer with cout channels
// per branch.  perm 0: branches one after the other.  perm 1 (gated): 256-row tiles [128 a | 128 g].  perm 2 (gated + pixel shuffle,
// Ch = cout / 2 post-shuffle channels): 256-row tiles [64 a(c) | 64 a(c + Ch) | 64 g(c) | 64 g(c + Ch)] for 64 post-shuffle channels c.
__host__ __device__ __forceinline__ int perm_row(int perm, int co, int cout, int noff) {
  if (perm == 1) return (co >> 7) * 256 + (noff ? 128 : 0) + (co & 127);
  if (perm == 2) { const int Ch = cout >> 1; const int s = co >= Ch ? 1 : 0; const int c = co - s * Ch; return (c >> 6) * 256 + (noff ? 128 : 0) + s * 64 + (c & 63); }
  return noff + co;
}
// element (tap, ci, co) of a TF kernel [taps][cin][cout].  fold_n != 0 (TcLayer::fold): the layer is registered as a 1 x 1 layer whose
// `cout` columns are (t, n) pairs, co = t * fold_n + n, of a kernel that lies in memory as [cout / fold_n taps][cin][fold_n]
__host__ __device__ __forceinline__ long long w_src(int tap, int ci, int co, int cin, int cout, int fold_n) {
  if (fold_n) { const int t = co / fold_n; return ((long long)t * cin + ci) * fold_n + (co - t * fold_n); }
  return ((long long)tap * cin + ci) * cout + co;
}
// TF kernel [taps][cin][cout] (fp32) -> wd[taps][cin][Ntot] (+ column offset) and wf[taps][Ntot][cin], bf16 hi/lo
__global__ void __launch_bounds__(256)
prep_weights_kernel(const float* __restrict__ w, int taps, int cin, int cout, int nt_n, int cin_k, int cin_n, int nt_k, int noff, int perm, int fold_n,
                    __nv_bfloat16* __restrict__ wf_hi, __nv_bfloat16* __restrict__ wf_lo,
                    __nv_bfloat16* __restrict__ wd_hi, __nv_bfloat16* __restrict__ wd_lo) {
  // 32x32 transposing tiles over (cin, cout) for each tap
  __shared__ float tile[32][33];
  const int tap = blockIdx.z;
  const int ci0 = blockIdx.y * 32, co0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 8 rows per pass
  for (int r = ty; r < 32; r += 8) {
    int ci = ci0 + r, co = co0 + tx;
    float v = 0.f;
    if (ci < cin && co < cout) {
      v = w[w_src(tap, ci, co, cin, cout, fold_n)];
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
      long long o = ((long long)tap * cin_n + ci) * nt_k + noff + co;
      wd_hi[o] = h; wd_lo[o] = l;
    }
    tile[r][tx] = v;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    int co = co0 + r, ci = ci0 + tx;
    if (ci < cin && co < cout) {
      float v = tile[tx][r];
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
      // forward rows of gated layers are tile-interleaved: row = (co/128)*256 + branch*128 + co%128 (branch = noff/cout)
      const int nrow = perm_row(perm, co, cout, noff);
      long long o = ((long long)tap * nt_n + nrow) * cin_k + ci;
      wf_hi[o] = h; wf_lo[o] = l;
    }
  }
}

__global__ void copy_bias_kernel(const float* __restrict__ b, float* __restrict__ dst, int n, int noff, int perm) {
  int i = blockIdx.x * 256 + threadIdx.x;
  if (i < n) dst[perm_row(perm, i, n, noff)] = b[i];
}

// TF kernel [taps][cin][cout] (fp32) -> F16F8 forward planes wq[taps][nt_n][cin_q] (weight scales); 4 input channels per thread
__global__ void __launch_bounds__(256)
prep_weights_q_kernel(const float* __restrict__ w, int taps, int cin, int cout, int nt_n, int cin_q, int noff, int perm, int fold_n,
                      __half* __restrict__ q16, uint8_t* __restrict__ q8hi, uint8_t* __restrict__ q8lo) {
  const int cq = cin / 4;
  const long long total = (long long)taps * cout * cq;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c4 = (int)(i % cq); long long r = i / cq;
    const int co = (int)(r % cout); const int tap = (int)(r / cout);
    const int ci = c4 * 4;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = w[w_src(tap, ci + k, co, cin, cout, fold_n)];
    const int nrow = perm_row(perm, co, cout, noff);
    const long long o = ((long long)tap * nt_n + nrow) * cin_q + ci;
    uint2 hh; uint32_t b_hi, b_lo;
    cgvc_quant4(v, CGVC_Q_W_SHI, CGVC_Q_W_SLO, hh, b_hi, b_lo);
    *reinterpret_cast<uint2*>(q16 + o) = hh;
    *reinterpret_cast<uint32_t*>(q8hi + o) = b_hi;
    *reinterpret_cast<uint32_t*>(q8lo + o) = b_lo;
  }
}

// TF kernel [taps][cin][cout] (fp32) -> F16F8 data-gradient planes wdq[taps][cin_n][nt_q] (K = output columns contiguous, weight
// scales); 4 output columns per thread.  Column of (branch, co) = noff + co, like the bf16 wd planes.
__global__ void __launch_bounds__(256)
prep_weights_qd_kernel(const float* __restrict__ w, int taps, int cin, int cout, int cin_n, int nt_q, int noff, int fold_n,
                       __half* __restrict__ q16, uint8_t* __restrict__ q8hi, uint8_t* __restrict__ q8lo) {
  const int cq = cout / 4;
  const long long total = (long long)taps * cin * cq;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int c4 = (int)(i % cq); long long r = i / cq;
    const int ci = (int)(r % cin); const int tap = (int)(r / cin);
    const float4 v4 = *reinterpret_cast<const float4*>(w + w_src(tap, ci, c4 * 4, cin, cout, fold_n));      // (fold_n % 4 == 0: a quad never straddles two taps)
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
    const long long o = ((long long)tap * cin_n + ci) * nt_q + noff + c4 * 4;
    uint2 hh; uint32_t b_hi, b_lo;
    cgvc_quant4(v, CGVC_Q_W_SHI, CGVC_Q_W_SLO, hh, b_hi, b_lo);
    *reinterpret_cast<uint2*>(q16 + o) = hh;
    *reinterpret_cast<uint32_t*>(q8hi + o) = b_hi;
    *reinterpret_cast<uint32_t*>(q8lo + o) = b_lo;
  }
}

// ---- F16F8 planes of every layer in ONE launch (per refresh, or per network range) --------------------------------------------------
// The per-layer kernels above cost ~210 launches per train step (forward planes, data-gradient planes and bias of 70 layer branches) and
// prep_weights_q_kernel reads its source with a stride of `cout` floats between neighbouring threads.  This kernel walks a job table --
// one job per layer branch -- in 32-channel x 64-column tiles: the tile is read once, coalesced along the output columns, written to the
// data-gradient planes in that orientation, transposed through shared memory and written to the forward planes as whole 32-byte sectors
// (8 consecutive input channels per thread); the first tile of a job also copies the bias.  Same arithmetic (cgvc_quant4, weight scales),
// bit-identical planes (tests/test_gpu_model.py::test_batched_weight_planes_match_per_layer_kernels).
struct PrepJob {                               // one branch (a or g) of one layer
  long long w_off, b_off;                      // offsets of its TF kernel / bias in the PARAM arena (b_off < 0: no bias, tap-folded layers)
  int taps, cin, cout, nt_n, cin_q, cin_n, nt_q, noff, perm, fold_n;
  __half* q16; uint8_t *q8hi, *q8lo;           // forward planes [taps][nt_n][cin_q]
  __half* dq16; uint8_t *dq8hi, *dq8lo;        // data-gradient planes [taps][cin_n][nt_q] (null: forward-only engine)
  float* bias;                                 // [nt_n], weight-row order
  int tiles_ci, tiles_co;                      // tiles per tap
  int first_block;                             // blocks of the jobs before this one
};

__global__ void __launch_bounds__(256)
prep_weights_q_all_kernel(const float* __restrict__ params, const PrepJob* __restrict__ jobs, int j0, int j1, int block0) {
  __shared__ float tile[32][65];
  const int blk = (int)blockIdx.x + block0;
  int lo = j0, hi = j1 - 1;                     // last job whose first block is <= blk (block-uniform)
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (jobs[mid].first_block <= blk) lo = mid; else hi = mid - 1; }
  const PrepJob& J = jobs[lo];
  int r = blk - J.first_block;
  const int tco = r % J.tiles_co; r /= J.tiles_co;
  const int tci = r % J.tiles_ci; const int tap = r / J.tiles_ci;
  const int ci0 = tci * 32, co0 = tco * 64;
  const float* __restrict__ w = params + J.w_off;
  const int t = threadIdx.x;
  {
    const int c4 = (t & 15) * 4;
    for (int rr = t >> 4; rr < 32; rr += 16) {
      const int ci = ci0 + rr, co = co0 + c4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (ci < J.cin && co < J.cout) {           // cout % 4 == 0 (layer_ok): whole quads
        const float4 q = *reinterpret_cast<const float4*>(w + w_src(tap, ci, co, J.cin, J.cout, J.fold_n));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        if (J.dq16) {
          const long long o = ((long long)tap * J.cin_n + ci) * J.nt_q + J.noff + co;
          uint2 hh; uint32_t b_hi, b_lo;
          cgvc_quant4(v, CGVC_Q_W_SHI, CGVC_Q_W_SLO, hh, b_hi, b_lo);
          *reinterpret_cast<uint2*>(J.dq16 + o) = hh;
          *reinterpret_cast<uint32_t*>(J.dq8hi + o) = b_hi;
          *reinterpret_cast<uint32_t*>(J.dq8lo + o) = b_lo;
        }
      }
      tile[rr][c4] = v[0]; tile[rr][c4 + 1] = v[1]; tile[rr][c4 + 2] = v[2]; tile[rr][c4 + 3] = v[3];
    }
  }
  __syncthreads();
  {
    const int lane = t & 31, warp = t >> 5;
    const int cig = (lane & 3) * 8;               // 8 consecutive input channels: 16 bytes of q16, 8 of each e4m3 plane
    const int col = warp * 8 + (lane >> 2);
    const int co = co0 + col;
    if (co < J.cout && ci0 + cig < J.cin_q) {     // channels in [cin, cin_q) are written as zeros (they are zero in the tile)
      float va[4], vb[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) { va[k] = tile[cig + k][col]; vb[k] = tile[cig + 4 + k][col]; }
      const int nrow = perm_row(J.perm, co, J.cout, J.noff);
      const long long o = ((long long)tap * J.nt_n + nrow) * J.cin_q + ci0 + cig;
      uint2 ha, hb; uint32_t a_hi, a_lo, b_hi, b_lo;
      cgvc_quant4(va, CGVC_Q_W_SHI, CGVC_Q_W_SLO, ha, a_hi, a_lo);
      cgvc_quant4(vb, CGVC_Q_W_SHI, CGVC_Q_W_SLO, hb, b_hi, b_lo);
      *reinterpret_cast<uint4*>(J.q16 + o) = make_uint4(ha.x, ha.y, hb.x, hb.y);
      *reinterpret_cast<uint2*>(J.q8hi + o) = make_uint2(a_hi, b_hi);
      *reinterpret_cast<uint2*>(J.q8lo + o) = make_uint2(a_lo, b_lo);
    }
  }
  if (tap == 0 && tci == 0 && tco == 0 && J.b_off >= 0)
    for (int i = t; i < J.cout; i += 256) J.bias[perm_row(J.perm, i, J.cout, J.noff)] = params[J.b_off + i];
}

// opt-in to > 48 KB dynamic shared memory, once per kernel (never inside a stream capture: see tc_init_kernels)
template <class K>
cudaError_t set_smem(K kernel, int bytes) {
  static std::vector<const void*> done;
  const void* key = (const void*)kernel;
  for (const void* d : done) if (d == key) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done.push_back(key);
  return e;
}

// ---- optional per-launch event timing (bench.py roofline): class 0 = NT (fwd/dgrad, plain epilogue), 1 = TN (wgrad),
//      2 = NT with the fused instance-norm epilogue
struct ProfRec { cudaEvent_t a, b; double flops; int cls; long long M; int N, K; };
bool g_prof_on = false;
std::vector<ProfRec> g_prof;
void prof_begin(cudaStream_t st, double flops, int cls, long long M = 0, int N = 0, int K = 0) {
  if (!g_prof_on) return;
  ProfRec r; r.flops = flops; r.cls = cls; r.M = M; r.N = N; r.K = K;
  cudaEventCreate(&r.a); cudaEventCreate(&r.b);
  cudaEventRecord(r.a, st);
  g_prof.push_back(r);
}
void prof_end(cudaStream_t st) { if (g_prof_on && !g_prof.empty()) cudaEventRecord(g_prof.back().b, st); }

// output-column tile width: 256 where the padded width allows, 32 for the 24-column edge layers (G.o1 forward, G.h1 data
// gradient: a 128-wide tile would spend 5x the MMAs on zero padding), else 128
inline int tile_rows(int n_real, int n_padded) { return (n_padded % 256 == 0) ? 256 : (n_real <= 32 ? 32 : 128); }

int num_sms() {
  static int n = 0;
  if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); }
  return n;
}

// The TMA form of the dense kernel takes the geometries whose 128-row tiles are boxes of the source planes: a tile is 128 / Wx whole
// samples (Wx divides 128) or 128 positions of one sample (128 divides Wx), all at one output row (rows are y-major, see nt_row: true
// when Hy == 1 or 128 divides B * Wx).  Rows past M in the last tile are samples past the batch, which the box reads as zeros, as the
// gather does.  Encodes p's activation maps and returns true; false leaves the geometry (or a plane the encoder refuses) to the gather.
static bool nt_tma_maps(TcNTParams& p, int npl) {
  const GatherGeom& g = p.g;
  const int wx = g.Wx < 128 ? g.Wx : 128;
  if (128 % wx || g.Wx % wx || (g.Hy > 1 && ((long long)g.B * g.Wx) % 128) || wx * g.sx > 256 || g.sx > 8) return false;
  const uint32_t bx = (uint32_t)(wx * g.sx), nb = (uint32_t)(128 / wx);
  if (npl == 3)
    return make_tmap_act(&p.tm_a_hi, p.a_hi, 2, p.a_ld, g, bx, nb) && make_tmap_act(&p.tm_a8_hi, p.a8_hi, 1, p.a_ld, g, bx, nb) &&
           make_tmap_act(&p.tm_a8_lo, p.a8_lo, 1, p.a_ld, g, bx, nb);
  return make_tmap_act(&p.tm_a_hi, p.a_hi, 2, p.a_ld, g, bx, nb) && (npl != 2 || make_tmap_act(&p.tm_a_lo, p.a_lo, 2, p.a_ld, g, bx, nb));
}

cudaError_t launch_nt(TcNTParams p, int precision, cudaStream_t st, int epi) {
  const long long M = (long long)p.g.B * p.g.Hy * p.g.Wx;
  if (M == 0) return cudaSuccess;
  if (M >= (1ll << 31)) return cudaErrorInvalidValue;    // (nt_row divides 32-bit row indices)
  const bool x3 = precision == 1;
  if (p.g.ntaps == 0) return cudaErrorInvalidValue;      // empty contractions are the caller's business
  p.div_bw = make_fastdiv((uint32_t)(p.g.B * p.g.Wx)); p.div_w = make_fastdiv((uint32_t)p.g.Wx);
  const int bn = tile_rows(p.N, p.Nw);
  p.n_tiles = bn == 32 ? 1 : p.Nw / bn;                  // the 32-wide tile only ever covers the (<= 32) real columns
  const long long tiles = ((M + 127) / 128) * p.n_tiles;
  dim3 grid((unsigned)(tiles < num_sms() ? tiles : num_sms()));
  cudaError_t e;
  ++g_cgvc_launches;
  prof_begin(st, 2.0 * (double)M * p.N * p.g.ntaps * p.C, (epi == 1 || epi == 2 || epi == 5) ? 2 : 0, M, p.N, p.g.ntaps * p.C);
#define LAUNCH_NT(BN_, NPL_, EPI_, ...)                                                                        \
  do {                                                                                                         \
    e = set_smem(tc_gg_nt_kernel<BN_, NPL_, EPI_, ##__VA_ARGS__>, NTCfg<BN_, NPL_>::SMEM);                     \
    if (e != cudaSuccess) return e;                                                                            \
    tc_gg_nt_kernel<BN_, NPL_, EPI_, ##__VA_ARGS__><<<grid, kNTThreads, NTCfg<BN_, NPL_>::SMEM, st>>>(p);      \
  } while (0)
  if (epi != 0 && bn != 256) return cudaErrorInvalidValue;
  if (p.pk.off && (p.g.Hy > 1 || p.g.Hs > 1 || p.g.Hd > 1)) {   // packed 2-D grids (the discriminator's layers)
    if (epi != 0 || p.g.B != 1 || p.g.ntaps > 31) return cudaErrorInvalidValue;
    const int npl = precision == 3 ? 3 : x3 ? 2 : 1;
    if (bn == 256)      { if (npl == 3) LAUNCH_NT(256, 3, 0, 2); else if (npl == 2) LAUNCH_NT(256, 2, 0, 2); else LAUNCH_NT(256, 1, 0, 2); }
    else if (bn == 128) { if (npl == 3) LAUNCH_NT(128, 3, 0, 2); else if (npl == 2) LAUNCH_NT(128, 2, 0, 2); else LAUNCH_NT(128, 1, 0, 2); }
    else                { if (npl == 3) LAUNCH_NT(32, 3, 0, 2);  else if (npl == 2) LAUNCH_NT(32, 2, 0, 2);  else LAUNCH_NT(32, 1, 0, 2); }
  }
  else if (p.pk.off) {                                      // packed utterances: plain epilogue only
    if (epi != 0 || p.g.B != 1 || p.g.Hy != 1) return cudaErrorInvalidValue;
    const int npl = precision == 3 ? 3 : x3 ? 2 : 1;
    if (bn == 256)      { if (npl == 3) LAUNCH_NT(256, 3, 0, 1); else if (npl == 2) LAUNCH_NT(256, 2, 0, 1); else LAUNCH_NT(256, 1, 0, 1); }
    else if (bn == 128) { if (npl == 3) LAUNCH_NT(128, 3, 0, 1); else if (npl == 2) LAUNCH_NT(128, 2, 0, 1); else LAUNCH_NT(128, 1, 0, 1); }
    else                { if (npl == 3) LAUNCH_NT(32, 3, 0, 1);  else if (npl == 2) LAUNCH_NT(32, 2, 0, 1);  else LAUNCH_NT(32, 1, 0, 1); }
  }
  else {
    // dense rows: the TMA form where the tiles are boxes of the activation planes, else the gather
    const bool ta = nt_tma_maps(p, precision == 3 ? 3 : x3 ? 2 : 1);
#define LAUNCH_NT_D(BN_, NPL_, EPI_) do { if (ta) LAUNCH_NT(BN_, NPL_, EPI_, 0, 1); else LAUNCH_NT(BN_, NPL_, EPI_); } while (0)
    if (precision == 3) {                                // F16F8 (no fused backward epilogues in this precision)
      if (epi == 1)       LAUNCH_NT_D(256, 3, 1);
      else if (epi == 2)  LAUNCH_NT_D(256, 3, 2);
      else if (epi == 5)  LAUNCH_NT_D(256, 3, 5);
      else if (epi != 0)  return cudaErrorInvalidValue;
      else if (bn == 256) LAUNCH_NT_D(256, 3, 0);
      else if (bn == 128) LAUNCH_NT_D(128, 3, 0);
      else                LAUNCH_NT_D(32, 3, 0);
    }
    else if (epi == 1)  { if (x3) LAUNCH_NT_D(256, 2, 1); else LAUNCH_NT_D(256, 1, 1); }
    else if (epi == 2)  { if (x3) LAUNCH_NT_D(256, 2, 2); else LAUNCH_NT_D(256, 1, 2); }
    else if (epi == 3)  { if (x3) LAUNCH_NT_D(256, 2, 3); else LAUNCH_NT_D(256, 1, 3); }
    else if (epi == 4)  { if (x3) LAUNCH_NT_D(256, 2, 4); else LAUNCH_NT_D(256, 1, 4); }
    else if (epi == 5)  { if (x3) LAUNCH_NT_D(256, 2, 5); else LAUNCH_NT_D(256, 1, 5); }
    else if (bn == 256) { if (x3) LAUNCH_NT_D(256, 2, 0); else LAUNCH_NT_D(256, 1, 0); }
    else if (bn == 128) { if (x3) LAUNCH_NT_D(128, 2, 0); else LAUNCH_NT_D(128, 1, 0); }
    else                { if (x3) LAUNCH_NT_D(32, 2, 0);  else LAUNCH_NT_D(32, 1, 0); }
#undef LAUNCH_NT_D
  }
#undef LAUNCH_NT
  prof_end(st);
  return cudaGetLastError();
}

// The TMA form of the weight-gradient kernel takes the dense geometries whose 64-row stages are boxes of the source planes: a stage is
// 64 / Wx whole output rows (Wx divides 64) or 64 positions of one output row (64 divides Wx).  K-rows are sample-major, so a box of
// whole rows may start in one sample and the next box in the next; with Hy == 1 the 64 / Wx samples of a stage share one box.  Wx >= 8
// keeps every box on a 1024-byte boundary of the stage.  Rows past M in the last stage are samples past the batch, zeros in the box as
// in the gather.  Encodes p's activation maps and returns true; false leaves the geometry (or a plane the encoder refuses) to the gather.
static bool tn_tma_maps(TcTNParams& p, int npl) {
  const GatherGeom& g = p.g;
  const int wx = g.Wx < 64 ? g.Wx : 64;
  if (g.Wx < 8 || 64 % wx || g.Wx % wx || wx * g.sx > 256 || g.sx > 8) return false;
  const uint32_t bx = (uint32_t)(wx * g.sx), nb = g.Hy == 1 ? (uint32_t)(64 / wx) : 1u;
  return make_tmap_act(&p.tm_x_hi, p.x_hi, 2, p.x_ld, g, bx, nb) && (npl != 2 || make_tmap_act(&p.tm_x_lo, p.x_lo, 2, p.x_ld, g, bx, nb));
}

cudaError_t launch_tn(TcTNParams p, int precision, cudaStream_t st, const DetSlab* det) {
  const long long M = (long long)p.g.B * p.g.Hy * p.g.Wx;
  if (M == 0) return cudaSuccess;
  if (M >= (1ll << 31)) return cudaErrorInvalidValue;
  const int tiles = ((p.g_ld + 255) / 256) * ((p.x_ld + 127) / 128) * p.g.ntaps;
  const int nsm = num_sms();
  // split the row (contraction) range so that the work items fill whole rounds of the persistent grid; every item keeps
  // >= 16 stages so that the wait of its epilogue stays small next to its MMAs
  long long maxsplit = M / 1024; if (maxsplit < 1) maxsplit = 1; if (maxsplit > 32) maxsplit = 32;
  int ksplit = 1; double best = 0.0;
  for (int ks = 1; ks <= (int)maxsplit; ++ks) {
    long long items = (long long)tiles * ks;
    double eff = (double)items / (double)(((items + nsm - 1) / nsm) * nsm);
    if (items < nsm) eff *= 0.5;                           // a single partial round: prefer more, smaller items
    if (eff > best + 0.02) { best = eff; ksplit = ks; }
  }
  // deterministic mode: every element of every split's partial tile is stored (so no split may have an empty row range), and the
  // ksplit partial copies of dW must fit the slab; a layer too large for two copies runs unsplit, whose adds are one per element
  const long long numel = (long long)p.g.ntaps * p.C * p.N;
  auto chunk_of = [&](int ks) { return ((M + ks - 1) / ks + 63) / 64 * 64; };
  if (det && det->p)
    while (ksplit > 1 && ((long long)ksplit * numel > det->cap || (long long)(ksplit - 1) * chunk_of(ksplit) >= M)) --ksplit;
  const bool det_split = det && det->p && ksplit > 1;
  if (det_split) { p.part = det->p; p.part_k = numel; p.numel_a = (long long)p.g.ntaps * p.C * p.n_split; }
  p.ksplit = ksplit;
  p.div_hw = make_fastdiv((uint32_t)(p.g.Hy * p.g.Wx)); p.div_w = make_fastdiv((uint32_t)p.g.Wx);
  const long long items = (long long)tiles * ksplit;
  dim3 grid((unsigned)(items < nsm ? items : nsm));
  cudaError_t e;
  ++g_cgvc_launches;
  prof_begin(st, 2.0 * (double)M * p.N * p.g.ntaps * p.C, 1, M, p.N, p.g.ntaps * p.C);
#define LAUNCH_TN(NPL_, W16_, DET_, ...)                                                                      \
  do {                                                                                                        \
    e = set_smem(tc_gg_tn_kernel<NPL_, W16_, DET_, ##__VA_ARGS__>, TNCfg<NPL_, W16_>::SMEM);                  \
    if (e != cudaSuccess) return e;                                                                           \
    tc_gg_tn_kernel<NPL_, W16_, DET_, ##__VA_ARGS__><<<grid, kNTThreads, TNCfg<NPL_, W16_>::SMEM, st>>>(p);   \
  } while (0)
  if (p.pk.off && (p.g.Hy > 1 || p.g.Hs > 1)) {             // packed 2-D grids
    if (p.g.B != 1) return cudaErrorInvalidValue;
    if (det_split) {
      if (precision == 3) { if (p.w16) LAUNCH_TN(3, 1, 1, 2); else LAUNCH_TN(3, 0, 1, 2); }
      else if (precision == 1) LAUNCH_TN(2, 0, 1, 2);
      else                     LAUNCH_TN(1, 0, 1, 2);
    } else {
      if (precision == 3) { if (p.w16) LAUNCH_TN(3, 1, 0, 2); else LAUNCH_TN(3, 0, 0, 2); }
      else if (precision == 1) LAUNCH_TN(2, 0, 0, 2);
      else                     LAUNCH_TN(1, 0, 0, 2);
    }
  } else if (p.pk.off) {                                    // packed utterances
    if (p.g.B != 1 || p.g.Hy != 1) return cudaErrorInvalidValue;
    if (det_split) {
      if (precision == 3) { if (p.w16) LAUNCH_TN(3, 1, 1, 1); else LAUNCH_TN(3, 0, 1, 1); }
      else if (precision == 1) LAUNCH_TN(2, 0, 1, 1);
      else                     LAUNCH_TN(1, 0, 1, 1);
    } else {
      if (precision == 3) { if (p.w16) LAUNCH_TN(3, 1, 0, 1); else LAUNCH_TN(3, 0, 0, 1); }
      else if (precision == 1) LAUNCH_TN(2, 0, 0, 1);
      else                     LAUNCH_TN(1, 0, 0, 1);
    }
  } else {
    // dense rows: the TMA form where the stages are boxes of the activation planes (not F16F8's cross pass, whose producers widen
    // the e4m3 planes), else the gather
    const bool ta = (precision != 3 || p.w16) && tn_tma_maps(p, precision == 1 ? 2 : 1);
#define LAUNCH_TN_D(NPL_, W16_, DET_) do { if (ta) LAUNCH_TN(NPL_, W16_, DET_, 0, 1); else LAUNCH_TN(NPL_, W16_, DET_); } while (0)
    if (det_split) {
      if (precision == 3) { if (p.w16) LAUNCH_TN_D(3, 1, 1); else LAUNCH_TN(3, 0, 1); }
      else if (precision == 1) LAUNCH_TN_D(2, 0, 1);
      else                     LAUNCH_TN_D(1, 0, 1);
    } else {
      if (precision == 3) { if (p.w16) LAUNCH_TN_D(3, 1, 0); else LAUNCH_TN(3, 0, 0); }
      else if (precision == 1) LAUNCH_TN_D(2, 0, 0);
      else                     LAUNCH_TN_D(1, 0, 0);
    }
#undef LAUNCH_TN_D
  }
#undef LAUNCH_TN
  prof_end(st);
  if (!det_split) return cudaGetLastError();
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_reduce_parts(p.part, ksplit, numel, DetSegs{{p.dw_a, p.dw_g}, {0, p.numel_a}, {p.numel_a, p.dw_g ? numel - p.numel_a : 0}}, st);
}

inline int ru(int v, int m) { return (v + m - 1) / m * m; }
inline int Ntot(const TcLayer& L) { return L.cout * (L.gated ? 2 : 1); }
// padded extents: *_k = as a contraction dimension (multiple of 64), *_n = as an output-tile dimension (multiple of 128)
inline int cin_k(const TcLayer& L) { return ru(L.cin, 64); }
inline int cin_n(const TcLayer& L) { return ru(L.cin, 128); }
inline int nt_k(const TcLayer& L) { return ru(Ntot(L), 64); }
inline int nt_n(const TcLayer& L) { return ru(Ntot(L), 128); }
inline int cin_q(const TcLayer& L) { return ru(L.cin, 128); }
inline int nt_q(const TcLayer& L) { return ru(Ntot(L), 128); }      // output columns as an F16F8 contraction dimension (128-byte e4m3 lines)
inline size_t wq_elems(const TcLayer& L) { return (size_t)L.kh * L.kw * nt_n(L) * cin_q(L); }
inline size_t wdq_elems(const TcLayer& L) { return (size_t)L.kh * L.kw * cin_n(L) * nt_q(L); }
inline size_t wf_elems(const TcLayer& L) { return (size_t)L.kh * L.kw * nt_n(L) * cin_k(L); }
inline size_t wd_elems(const TcLayer& L) { return (size_t)L.kh * L.kw * cin_n(L) * nt_k(L); }
// gated layers whose branch width is a multiple of 128 keep their forward weight rows tile-interleaved (see TcNTParams::perm)
inline int layer_perm(const TcLayer& L) {
  if (L.gated && L.shuffle == 2 && L.cout % 128 == 0) return 2;      // see perm_row
  return (L.gated && L.cout % 128 == 0) ? 1 : 0;
}
inline bool layer_ok(const TcLayer& L) {
  if (L.fold && (L.gated || L.kh * L.kw != 1 || L.cout % L.fold || (L.cout / L.fold) % 4)) return false;      // see TcLayer::fold
  return L.kh * L.kw <= CGVC_MAX_TAPS && Ntot(L) % 4 == 0;
}
// the F16F8 planes pack quads of input channels (cgvc_quant4)
inline bool layer_ok_q(const TcLayer& L) { return layer_ok(L) && L.cin % 4 == 0; }


// TMA descriptors of a layer's weight planes (call after wf_/wd_ pointers are set)
bool make_layer_maps(TcLayer& L) {
  const int taps = L.kh * L.kw;
  const int bf = tile_rows(Ntot(L), nt_n(L)), bd = tile_rows(L.cin, cin_n(L));   // must match launch_nt's choice of BN
  return make_tmap3(&L.tm_f_hi, L.wf_hi, cin_k(L), nt_n(L), taps, bf) &&
         make_tmap3(&L.tm_f_lo, L.wf_lo, cin_k(L), nt_n(L), taps, bf) &&
         make_tmap3(&L.tm_d_hi, L.wd_hi, nt_k(L), cin_n(L), taps, bd) &&
         make_tmap3(&L.tm_d_lo, L.wd_lo, nt_k(L), cin_n(L), taps, bd);
}

bool make_layer_maps_q(TcLayer& L) {
  const int taps = L.kh * L.kw;
  const int bf = tile_rows(Ntot(L), nt_n(L)), bd = tile_rows(L.cin, cin_n(L));
  const CUtensorMapDataType F16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16, U8 = CU_TENSOR_MAP_DATA_TYPE_UINT8;
  bool ok = make_tmap3_t(&L.tm_q16, L.wq16, F16, 2, cin_q(L), nt_n(L), taps, 64, bf) &&
            make_tmap3_t(&L.tm_q8hi, L.wq8hi, U8, 1, cin_q(L), nt_n(L), taps, 64, bf) &&
            make_tmap3_t(&L.tm_q8lo, L.wq8lo, U8, 1, cin_q(L), nt_n(L), taps, 64, bf);
  if (ok && L.wdq16)
    ok = make_tmap3_t(&L.tm_dq16, L.wdq16, F16, 2, nt_q(L), cin_n(L), taps, 64, bd) &&
         make_tmap3_t(&L.tm_dq8hi, L.wdq8hi, U8, 1, nt_q(L), cin_n(L), taps, 64, bd) &&
         make_tmap3_t(&L.tm_dq8lo, L.wdq8lo, U8, 1, nt_q(L), cin_n(L), taps, 64, bd);
  return ok;
}

}  // namespace

// ------------------------------------------------------------------------------------------------ public API
int tc_refresh_layer(TcLayer& L, const float* ka, const float* kg, const float* ba, const float* bg, cudaStream_t st) {
  const int taps = L.kh * L.kw;
  dim3 grid((L.cout + 31) / 32, (L.cin + 31) / 32, taps);
  g_cgvc_launches += L.gated ? 4 : 2;
  const int perm = layer_perm(L);
  const int fn = L.fold ? L.cout / L.fold : 0;          // tap-folded layer: columns are (t, n) pairs of a [fold][cin][fn] kernel; no bias of its own
  // (an engine in the F16F8 precision never reads the bf16 planes: only the quantised planes below are refreshed)
  if (!L.wq16) prep_weights_kernel<<<grid, 256, 0, st>>>(ka, taps, L.cin, L.cout, nt_n(L), cin_k(L), cin_n(L), nt_k(L), 0, perm, fn, L.wf_hi, L.wf_lo, L.wd_hi, L.wd_lo);
  if (!L.fold) copy_bias_kernel<<<(L.cout + 255) / 256, 256, 0, st>>>(ba, L.bias, L.cout, 0, perm);
  if (L.gated) {
    if (!L.wq16) prep_weights_kernel<<<grid, 256, 0, st>>>(kg, taps, L.cin, L.cout, nt_n(L), cin_k(L), cin_n(L), nt_k(L), L.cout, perm, fn, L.wf_hi, L.wf_lo, L.wd_hi, L.wd_lo);
    copy_bias_kernel<<<(L.cout + 255) / 256, 256, 0, st>>>(bg, L.bias, L.cout, L.cout, perm);
  }
  if (L.wq16) {
    long long tot = (long long)taps * L.cout * (L.cin / 4); long long nb = (tot + 255) / 256; if (nb > num_sms() * 32) nb = num_sms() * 32;
    g_cgvc_launches += L.gated ? 2 : 1;
    prep_weights_q_kernel<<<(unsigned)nb, 256, 0, st>>>(ka, taps, L.cin, L.cout, nt_n(L), cin_q(L), 0, perm, fn, (__half*)L.wq16, L.wq8hi, L.wq8lo);
    if (L.gated) prep_weights_q_kernel<<<(unsigned)nb, 256, 0, st>>>(kg, taps, L.cin, L.cout, nt_n(L), cin_q(L), L.cout, perm, fn, (__half*)L.wq16, L.wq8hi, L.wq8lo);
    if (L.wdq16) {
      g_cgvc_launches += L.gated ? 2 : 1;
      prep_weights_qd_kernel<<<(unsigned)nb, 256, 0, st>>>(ka, taps, L.cin, L.cout, cin_n(L), nt_q(L), 0, fn, (__half*)L.wdq16, L.wdq8hi, L.wdq8lo);
      if (L.gated) prep_weights_qd_kernel<<<(unsigned)nb, 256, 0, st>>>(kg, taps, L.cin, L.cout, cin_n(L), nt_q(L), L.cout, fn, (__half*)L.wdq16, L.wdq8hi, L.wdq8lo);
    }
  }
  return (int)cudaGetLastError();
}

// x planes: [n,H,W,cin_k] (channels beyond cin are zero)
int tc_conv_fwd(const TcLayer& L, int precision, int debug, const __nv_bfloat16* xhi, const __nv_bfloat16* xlo, int n, int H, int W, int sh, int sw,
                float* P, cudaStream_t st, const TcFuse* fuse, bool* fused_out, const PackGeom* pk) {
  if (!layer_ok(L) || (precision == 3 && !layer_ok_q(L))) return TC_UNSUPPORTED;
  if (pk && (n != 1 || (H == 1 && L.kh != 1) || fuse)) return (int)cudaErrorInvalidValue;     // H > 1: packed 2-D grids
  TcNTParams p; memset(&p, 0, sizeof p);
  p.g = fwd_geom(n, H, W, L.kh, L.kw, sh, sw);
  if (pk) p.pk = *pk;
  p.a_hi = xhi; p.a_lo = xlo; p.a_ld = cin_k(L); p.C = cin_k(L);
  p.b_hi = L.wf_hi; p.b_lo = L.wf_lo; p.Nw = nt_n(L); p.N = Ntot(L);
  p.dst = P; p.d_ld = Ntot(L); p.bias = L.bias; p.accumulate = 0;
  p.perm = layer_perm(L); p.Cc = L.cout;
  p.tm_b_hi = L.tm_f_hi; p.tm_b_lo = L.tm_f_lo; p.debug = debug;
  if (precision == 3) {
    // F16F8: x planes are [rows, cin_q] -- xhi = q16, xlo = q8hi followed by q8lo (kernels.cuh)
    if (!L.wq16) return TC_UNSUPPORTED;
    p.a_ld = cin_q(L); p.C = cin_q(L); p.a_lo = nullptr;
    p.a8_hi = reinterpret_cast<const uint8_t*>(xlo); p.a8_lo = p.a8_hi + (size_t)n * H * W * cin_q(L);
    p.tm_b_hi = L.tm_q16; p.tm_b8_hi = L.tm_q8hi; p.tm_b8_lo = L.tm_q8lo;
  }
  int epi = 0;
  if (fuse && fuse->R > 0) {
    // fused instance-norm epilogue: 1-D layer, whole samples per 128-row tile, 256-wide tiles
    const bool shape_ok = H == 1 && (fuse->R == 32 || fuse->R == 64 || fuse->R == 128) && p.g.Wx == fuse->R && nt_n(L) % 256 == 0 && Ntot(L) == nt_n(L);
    if (shape_ok && L.gated && p.perm == 1) epi = 1; else if (shape_ok && L.gated && p.perm == 2) epi = 5; else if (shape_ok && !L.gated) epi = 2;
    if (epi) {
      p.R = fuse->R; p.gamma_a = fuse->gamma_a; p.beta_a = fuse->beta_a; p.gamma_g = fuse->gamma_g; p.beta_g = fuse->beta_g;
      p.stats = fuse->stats; p.resid = fuse->resid; p.y = fuse->y; p.y_hi = fuse->y_hi; p.y_lo = fuse->y_lo;
      p.y8 = reinterpret_cast<uint8_t*>(fuse->y_lo);
      p.C_out = epi == 5 ? L.cout / 2 : (L.gated ? L.cout : Ntot(L));
      if (!p.y_hi || (epi == 2 && !p.resid)) epi = 0;
    }
  }
  if (fused_out) *fused_out = epi != 0;
  if (!epi && !P) return (int)cudaErrorInvalidValue;          // only the fused epilogues can do without the pre-norm output
  return (int)launch_nt(p, precision, st, epi);
}

// dP planes: [rows_out, nt_k]
int tc_conv_dgrad(const TcLayer& L, int precision, int debug, const __nv_bfloat16* dPhi, const __nv_bfloat16* dPlo, int n, int H, int W, int sh, int sw,
                  float* dx, int accumulate, cudaStream_t st, const TcBwdFuse* fuse, bool* fused_out, const PackGeom* pk) {
  if (fused_out) *fused_out = false;
  if (!layer_ok(L) || (precision == 3 && (!layer_ok_q(L) || !L.wdq16))) return TC_UNSUPPORTED;     // F16F8 needs the data-gradient planes (training engines)
  if (pk && (n != 1 || (H == 1 && L.kh != 1))) return (int)cudaErrorInvalidValue;     // H > 1: packed 2-D grids
  if (pk) fuse = nullptr;
  std::vector<GatherGeom> gs = dgrad_geoms(n, H, W, L.kh, L.kw, sh, sw);
  for (const GatherGeom& g : gs) if (g.ntaps == 0) return TC_UNSUPPORTED;     // (never the case for this model's layers)
  // fused backward epilogue: stride-1 1-D layer (one geometry, dense rows), whole samples per 128-row tile, 256-wide tiles
  int epi = 0;
  if (fuse && fuse->R > 0 && gs.size() == 1 && H == 1 && sh == 1 && sw == 1 && (fuse->R == 32 || fuse->R == 64 || fuse->R == 128) &&
      gs[0].Wx == fuse->R && cin_n(L) % 256 == 0 && L.cin == cin_n(L) && fuse->bp && fuse->stats && fuse->dp_hi && fuse->dp_lo && fuse->gamma_a &&
      (fuse->gated ? (fuse->gamma_g && fuse->beta_a && fuse->beta_g) : (dx != nullptr)) && precision != 3)
    epi = fuse->gated ? 3 : 4;
  for (const GatherGeom& g : gs) {
    TcNTParams p; memset(&p, 0, sizeof p);
    p.g = g;
    if (pk) {
      // packed: every class reads dP at the output level, of divisor pk->div * sw (see DESIGN.md section 12 for the parity classes)
      p.pk = *pk; p.pk.div = pk->div * sw;
    }
    p.a_hi = dPhi; p.a_lo = dPlo; p.a_ld = nt_k(L); p.C = nt_k(L);
    p.b_hi = L.wd_hi; p.b_lo = L.wd_lo; p.Nw = cin_n(L); p.N = L.cin;
    p.dst = dx; p.d_ld = L.cin; p.bias = nullptr; p.accumulate = accumulate;
    p.tm_b_hi = L.tm_d_hi; p.tm_b_lo = L.tm_d_lo; p.debug = debug;
    if (precision == 3) {
      // F16F8: dP planes are [rows, nt_q] -- dPhi = q16, dPlo = q8hi followed by q8lo (activation-role scales); weights from the wdq planes
      p.a_ld = nt_q(L); p.C = nt_q(L); p.a_lo = nullptr;
      p.a8_hi = reinterpret_cast<const uint8_t*>(dPlo); p.a8_lo = p.a8_hi + (size_t)g.B * g.Hs * g.Ws * nt_q(L);
      p.tm_b_hi = L.tm_dq16; p.tm_b8_hi = L.tm_dq8hi; p.tm_b8_lo = L.tm_dq8lo;
    }
    if (epi) {
      p.R = fuse->R; p.C_out = L.cin; p.stats = const_cast<float*>(fuse->stats);
      p.gamma_a = fuse->gamma_a; p.beta_a = fuse->beta_a; p.gamma_g = fuse->gamma_g; p.beta_g = fuse->beta_g;
      p.bp = fuse->bp; p.bp_ld = fuse->bp_ld; p.dp_hi = fuse->dp_hi; p.dp_lo = fuse->dp_lo; p.dp_ld = fuse->dp_ld;
      p.dbeta_a = fuse->dbeta_a; p.dgamma_a = fuse->dgamma_a; p.dbeta_g = fuse->dbeta_g; p.dgamma_g = fuse->dgamma_g;
    }
    cudaError_t e = launch_nt(p, precision, st, epi);
    if (e != cudaSuccess) return (int)e;
  }
  if (fused_out) *fused_out = epi != 0;
  return 0;
}

int tc_conv_wgrad(const TcLayer& L, int precision, int debug, int w16, const __nv_bfloat16* xhi, const __nv_bfloat16* xlo,
                  const __nv_bfloat16* dPhi, const __nv_bfloat16* dPlo, int n, int H, int W, int sh, int sw,
                  float* dwa, float* dwg, cudaStream_t st, const DetSlab* det, const PackGeom* pk) {
  if (!layer_ok(L) || (precision == 3 && !layer_ok_q(L))) return TC_UNSUPPORTED;
  if (pk && (n != 1 || (H == 1 && L.kh != 1))) return (int)cudaErrorInvalidValue;     // H > 1: packed 2-D grids
  TcTNParams p; memset(&p, 0, sizeof p);
  if (pk) p.pk = *pk;
  p.w16 = (precision == 3 && w16) ? 1 : 0; p.debug = debug;
  p.fold_n = L.fold ? L.cout / L.fold : 0;
  p.g = fwd_geom(n, H, W, L.kh, L.kw, sh, sw);
  p.x_hi = xhi; p.x_lo = xlo; p.x_ld = cin_k(L); p.C = L.cin;
  p.g_hi = dPhi; p.g_lo = dPlo; p.g_ld = nt_k(L); p.N = Ntot(L);
  p.dw_a = dwa; p.dw_g = dwg; p.n_split = L.cout;
  const long long M = (long long)p.g.B * p.g.Hy * p.g.Wx;
  if (precision == 3) {
    // F16F8: x planes [rows_in, cin_q] and dP planes [M, nt_q], each q16 (xhi / dPhi) + q8hi followed by q8lo (xlo / dPlo)
    const long long rows_in = (long long)n * H * W;
    p.x_ld = cin_q(L); p.g_ld = nt_q(L); p.x_lo = p.g_lo = nullptr;
    p.x8_hi = reinterpret_cast<const uint8_t*>(xlo); p.x8_lo = p.x8_hi + rows_in * p.x_ld;
    p.g8_hi = reinterpret_cast<const uint8_t*>(dPlo); p.g8_lo = p.g8_hi + M * p.g_ld;
    if (!make_tmap3_t(&p.tm_g_hi, dPhi, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (uint64_t)p.g_ld, (uint64_t)M, 1, 64, 64))
      return (int)cudaErrorInvalidValue;
  } else if (!make_tmap3(&p.tm_g_hi, dPhi, (uint64_t)nt_k(L), (uint64_t)M, 1, 64) || !make_tmap3(&p.tm_g_lo, dPlo, (uint64_t)nt_k(L), (uint64_t)M, 1, 64)) {
    return (int)cudaErrorInvalidValue;
  }
  return (int)launch_tn(p, precision, st, det);
}

int tc_register(TcWeights& w, size_t ka, size_t kg, size_t ba, size_t bg, int kh, int kw, int cin, int cout, int gated, int shuffle, int fold) {
  TcLayer L{}; L.ka = ka; L.kg = kg; L.ba = ba; L.bg = bg; L.kh = kh; L.kw = kw; L.cin = cin; L.cout = cout; L.gated = gated; L.shuffle = shuffle; L.fold = fold;
  w.layers.push_back(L);
  return (int)w.layers.size() - 1;
}

static cudaError_t tc_init_kernels();

int tc_alloc(TcWeights& w, int precision, bool train) {
  { cudaError_t ie = tc_init_kernels(); if (ie != cudaSuccess) return (int)ie; }
  w.quant = precision == 3;
  w.quant_bwd = w.quant && train;
  w.wgrad16 = w.quant;                              // option "wgrad_f16"
  size_t total = 0;
  auto rnd = [](size_t b) { return (b + 255) & ~(size_t)255; };
  for (TcLayer& L : w.layers) {
    total += 2 * rnd(wf_elems(L) * sizeof(__nv_bfloat16)) + 2 * rnd(wd_elems(L) * sizeof(__nv_bfloat16)) + rnd((size_t)nt_n(L) * sizeof(float));
    if (w.quant && layer_ok_q(L)) total += rnd(wq_elems(L) * 2) + 2 * rnd(wq_elems(L));
    if (w.quant && w.quant_bwd && layer_ok_q(L)) total += rnd(wdq_elems(L) * 2) + 2 * rnd(wdq_elems(L));
  }
  cudaError_t err = cudaMalloc(&w.pool, total);
  if (err != cudaSuccess) return (int)err;
  err = cudaMemset(w.pool, 0, total);               // padded rows / channels / bias entries stay zero forever
  if (err != cudaSuccess) return (int)err;
  w.pool_bytes = total;
  char* p = (char*)w.pool;
  for (TcLayer& L : w.layers) {
    size_t ef = rnd(wf_elems(L) * sizeof(__nv_bfloat16)), ed = rnd(wd_elems(L) * sizeof(__nv_bfloat16));
    L.wf_hi = (__nv_bfloat16*)p; p += ef; L.wf_lo = (__nv_bfloat16*)p; p += ef;
    L.wd_hi = (__nv_bfloat16*)p; p += ed; L.wd_lo = (__nv_bfloat16*)p; p += ed;
    L.bias = (float*)p; p += rnd((size_t)nt_n(L) * sizeof(float));
    if (!make_layer_maps(L)) return (int)cudaErrorInvalidValue;
    L.wq16 = nullptr; L.wq8hi = L.wq8lo = nullptr; L.wdq16 = nullptr; L.wdq8hi = L.wdq8lo = nullptr;
    if (w.quant && layer_ok_q(L)) {
      L.wq16 = p; p += rnd(wq_elems(L) * 2);
      L.wq8hi = (uint8_t*)p; p += rnd(wq_elems(L)); L.wq8lo = (uint8_t*)p; p += rnd(wq_elems(L));
      if (w.quant_bwd) {
        L.wdq16 = p; p += rnd(wdq_elems(L) * 2);
        L.wdq8hi = (uint8_t*)p; p += rnd(wdq_elems(L)); L.wdq8lo = (uint8_t*)p; p += rnd(wdq_elems(L));
      }
      if (!make_layer_maps_q(L)) return (int)cudaErrorInvalidValue;
    }
  }
  // job table of prep_weights_q_all_kernel: one job per branch of every layer that has F16F8 planes, in layer order
  w.job_first.clear(); w.job_ka.clear();
  if (w.quant) {
    std::vector<PrepJob> jobs;
    int blocks = 0;
    for (TcLayer& L : w.layers) {
      if (!L.wq16) continue;
      for (int br = 0; br < (L.gated ? 2 : 1); ++br) {
        PrepJob J; memset(&J, 0, sizeof J);
        J.w_off = (long long)(br ? L.kg : L.ka); J.b_off = L.fold ? -1 : (long long)(br ? L.bg : L.ba);
        J.taps = L.kh * L.kw; J.cin = L.cin; J.cout = L.cout; J.nt_n = nt_n(L); J.cin_q = cin_q(L); J.cin_n = cin_n(L); J.nt_q = nt_q(L);
        J.noff = br ? L.cout : 0; J.perm = layer_perm(L); J.fold_n = L.fold ? L.cout / L.fold : 0;
        J.q16 = (__half*)L.wq16; J.q8hi = L.wq8hi; J.q8lo = L.wq8lo;
        J.dq16 = (__half*)L.wdq16; J.dq8hi = L.wdq8hi; J.dq8lo = L.wdq8lo;
        J.bias = L.bias;
        J.tiles_ci = (L.cin + 31) / 32; J.tiles_co = (L.cout + 63) / 64;
        J.first_block = blocks;
        blocks += J.taps * J.tiles_ci * J.tiles_co;
        jobs.push_back(J); w.job_first.push_back(J.first_block); w.job_ka.push_back(L.ka);
      }
    }
    w.job_first.push_back(blocks);
    if (!jobs.empty()) {
      err = cudaMalloc(&w.prep_jobs, jobs.size() * sizeof(PrepJob));
      if (err != cudaSuccess) return (int)err;
      err = cudaMemcpy(w.prep_jobs, jobs.data(), jobs.size() * sizeof(PrepJob), cudaMemcpyHostToDevice);
      if (err != cudaSuccess) return (int)err;
    }
  }
  w.ready = false;
  return 0;
}

// configure every tensor-core kernel instantiation up front (so that no attribute call happens during graph capture)
static cudaError_t tc_init_kernels() {
  cudaError_t e;
#define INIT_NT(BN_, NPL_, EPI_) if ((e = set_smem(tc_gg_nt_kernel<BN_, NPL_, EPI_>, NTCfg<BN_, NPL_>::SMEM)) != cudaSuccess) return e;
  INIT_NT(256, 2, 0) INIT_NT(256, 1, 0) INIT_NT(128, 2, 0) INIT_NT(128, 1, 0) INIT_NT(32, 2, 0) INIT_NT(32, 1, 0)
  INIT_NT(256, 2, 1) INIT_NT(256, 1, 1) INIT_NT(256, 2, 2) INIT_NT(256, 1, 2)
  INIT_NT(256, 2, 3) INIT_NT(256, 1, 3) INIT_NT(256, 2, 4) INIT_NT(256, 1, 4) INIT_NT(256, 2, 5) INIT_NT(256, 1, 5)
  INIT_NT(256, 3, 0) INIT_NT(128, 3, 0) INIT_NT(32, 3, 0) INIT_NT(256, 3, 1) INIT_NT(256, 3, 2) INIT_NT(256, 3, 5)
#undef INIT_NT
#define INIT_NT(BN_, NPL_, EPI_) if ((e = set_smem(tc_gg_nt_kernel<BN_, NPL_, EPI_, 0, 1>, NTCfg<BN_, NPL_>::SMEM)) != cudaSuccess) return e;
  INIT_NT(256, 2, 0) INIT_NT(256, 1, 0) INIT_NT(128, 2, 0) INIT_NT(128, 1, 0) INIT_NT(32, 2, 0) INIT_NT(32, 1, 0)
  INIT_NT(256, 2, 1) INIT_NT(256, 1, 1) INIT_NT(256, 2, 2) INIT_NT(256, 1, 2)
  INIT_NT(256, 2, 3) INIT_NT(256, 1, 3) INIT_NT(256, 2, 4) INIT_NT(256, 1, 4) INIT_NT(256, 2, 5) INIT_NT(256, 1, 5)
  INIT_NT(256, 3, 0) INIT_NT(128, 3, 0) INIT_NT(32, 3, 0) INIT_NT(256, 3, 1) INIT_NT(256, 3, 2) INIT_NT(256, 3, 5)
#undef INIT_NT
#define INIT_NT_PK(BN_, NPL_, PK_) if ((e = set_smem(tc_gg_nt_kernel<BN_, NPL_, 0, PK_>, NTCfg<BN_, NPL_>::SMEM)) != cudaSuccess) return e;
  INIT_NT_PK(256, 1, 1) INIT_NT_PK(256, 2, 1) INIT_NT_PK(256, 3, 1) INIT_NT_PK(128, 1, 1) INIT_NT_PK(128, 2, 1) INIT_NT_PK(128, 3, 1)
  INIT_NT_PK(32, 1, 1) INIT_NT_PK(32, 2, 1) INIT_NT_PK(32, 3, 1)
  INIT_NT_PK(256, 1, 2) INIT_NT_PK(256, 2, 2) INIT_NT_PK(256, 3, 2) INIT_NT_PK(128, 1, 2) INIT_NT_PK(128, 2, 2) INIT_NT_PK(128, 3, 2)
  INIT_NT_PK(32, 1, 2) INIT_NT_PK(32, 2, 2) INIT_NT_PK(32, 3, 2)
#undef INIT_NT_PK
#define INIT_TN(NPL_, W16_, DET_) if ((e = set_smem(tc_gg_tn_kernel<NPL_, W16_, DET_>, TNCfg<NPL_, W16_>::SMEM)) != cudaSuccess) return e;
  INIT_TN(3, 1, 0) INIT_TN(3, 0, 0) INIT_TN(2, 0, 0) INIT_TN(1, 0, 0)
  INIT_TN(3, 1, 1) INIT_TN(3, 0, 1) INIT_TN(2, 0, 1) INIT_TN(1, 0, 1)
#define INIT_TN_TA(NPL_, W16_, DET_) if ((e = set_smem(tc_gg_tn_kernel<NPL_, W16_, DET_, 0, 1>, TNCfg<NPL_, W16_>::SMEM)) != cudaSuccess) return e;
  INIT_TN_TA(3, 1, 0) INIT_TN_TA(2, 0, 0) INIT_TN_TA(1, 0, 0)
  INIT_TN_TA(3, 1, 1) INIT_TN_TA(2, 0, 1) INIT_TN_TA(1, 0, 1)
#undef INIT_TN_TA
#define INIT_TN_PK(NPL_, W16_, DET_, PK_) if ((e = set_smem(tc_gg_tn_kernel<NPL_, W16_, DET_, PK_>, TNCfg<NPL_, W16_>::SMEM)) != cudaSuccess) return e;
  INIT_TN_PK(3, 1, 0, 1) INIT_TN_PK(3, 0, 0, 1) INIT_TN_PK(2, 0, 0, 1) INIT_TN_PK(1, 0, 0, 1)
  INIT_TN_PK(3, 1, 1, 1) INIT_TN_PK(3, 0, 1, 1) INIT_TN_PK(2, 0, 1, 1) INIT_TN_PK(1, 0, 1, 1)
  INIT_TN_PK(3, 1, 0, 2) INIT_TN_PK(3, 0, 0, 2) INIT_TN_PK(2, 0, 0, 2) INIT_TN_PK(1, 0, 0, 2)
  INIT_TN_PK(3, 1, 1, 2) INIT_TN_PK(3, 0, 1, 2) INIT_TN_PK(2, 0, 1, 2) INIT_TN_PK(1, 0, 1, 2)
#undef INIT_TN_PK
#undef INIT_TN
  return cudaSuccess;
}

void tc_free(TcWeights& w) {
  if (w.pool) cudaFree(w.pool);
  if (w.prep_jobs) cudaFree(w.prep_jobs);
  w.pool = nullptr; w.prep_jobs = nullptr; w.ready = false;
}

// the jobs [j0, j1) of the batched F16F8 plane kernel (contiguous: the layers of a network are registered together)
static int refresh_jobs(TcWeights& w, const float* params, int j0, int j1, cudaStream_t st) {
  if (j1 <= j0) return 0;
  const int b0 = w.job_first[j0], nb = w.job_first[j1] - b0;
  ++g_cgvc_launches;
  prep_weights_q_all_kernel<<<(unsigned)nb, 256, 0, st>>>(params, (const PrepJob*)w.prep_jobs, j0, j1, b0);
  return (int)cudaGetLastError();
}

int tc_refresh_weights(TcWeights& w, const float* params, cudaStream_t st) {
  if (!w.pool) return 0;
  const bool batched = w.prep_batched && w.prep_jobs;
  for (TcLayer& L : w.layers) {
    if (batched && L.wq16) continue;
    int r = tc_refresh_layer(L, params + L.ka, params + L.kg, params + L.ba, params + L.bg, st);
    if (r != 0) return r;
  }
  if (batched) { int r = refresh_jobs(w, params, 0, (int)w.job_ka.size(), st); if (r != 0) return r; }
  w.ready = true;
  return 0;
}

// the layers whose kernels live in [begin, end) of the parameter arena (one network)
int tc_refresh_weights_range(TcWeights& w, const float* params, size_t begin, size_t end, cudaStream_t st) {
  if (!w.pool) return 0;
  const bool batched = w.prep_batched && w.prep_jobs;
  for (TcLayer& L : w.layers) {
    if (L.ka < begin || L.ka >= end) continue;
    if (batched && L.wq16) continue;
    int r = tc_refresh_layer(L, params + L.ka, params + L.kg, params + L.ba, params + L.bg, st);
    if (r != 0) return r;
  }
  if (batched) {
    const int nj = (int)w.job_ka.size();
    int j = 0;
    while (j < nj) {                             // maximal runs of jobs inside the range (one run per network in practice)
      if (w.job_ka[j] < begin || w.job_ka[j] >= end) { ++j; continue; }
      int k = j; while (k < nj && w.job_ka[k] >= begin && w.job_ka[k] < end) ++k;
      int r = refresh_jobs(w, params, j, k, st); if (r != 0) return r;
      j = k;
    }
  }
  return 0;
}

void tc_layer_dims(const TcWeights& w, int slot, int dims[7]) {
  const TcLayer& L = w.layers[slot];
  const int d[7] = {nt_n(L), cin_k(L), cin_n(L), nt_k(L), cin_q(L), nt_q(L), layer_ok_q(L) ? 1 : 0};
  for (int i = 0; i < 7; ++i) dims[i] = d[i];
}

int tc_layer_plane(const TcWeights& w, int slot, const char* name, const void** p, size_t* bytes) {
  const TcLayer& L = w.layers[slot];
  const bool bf = w.pool && !L.wq16;                 // tc_refresh_layer writes the bf16 planes only for layers without F16F8 planes
  struct Plane { const char* name; const void* p; size_t bytes; };
  const Plane planes[] = {
    {"wf_hi", bf ? L.wf_hi : nullptr, wf_elems(L) * 2}, {"wf_lo", bf ? L.wf_lo : nullptr, wf_elems(L) * 2},
    {"wd_hi", bf ? L.wd_hi : nullptr, wd_elems(L) * 2}, {"wd_lo", bf ? L.wd_lo : nullptr, wd_elems(L) * 2},
    {"wq16", L.wq16, wq_elems(L) * 2}, {"wq8hi", L.wq8hi, wq_elems(L)}, {"wq8lo", L.wq8lo, wq_elems(L)},
    {"wdq16", L.wdq16, wdq_elems(L) * 2}, {"wdq8hi", L.wdq8hi, wdq_elems(L)}, {"wdq8lo", L.wdq8lo, wdq_elems(L)},
    {"bias", w.pool ? L.bias : nullptr, (size_t)nt_n(L) * sizeof(float)},
  };
  for (const Plane& q : planes)
    if (!strcmp(q.name, name)) { *p = q.p; *bytes = q.p ? q.bytes : 0; return 0; }
  return -1;
}

cudaError_t tc_split_planes(int precision, const float* x, long long rows, int C, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st,
                            unsigned long long* sat, unsigned long long* ufl) {
  return precision == 3 ? launch_pad_split_q(x, rows, C, C, ru(C, 128), hi, lo, st, sat, ufl) : launch_pad_split(x, rows, C, C, ru(C, 64), hi, lo, st);
}

bool tc_profile_is_on() { return g_prof_on; }

void tc_profile_enable(int on) {
  for (ProfRec& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  g_prof.clear();
  g_prof_on = on != 0;
}

// sums per class over everything recorded since tc_profile_enable(1); synchronises the device
int tc_profile_collect(double ms[3], double flops[3], long long launches[3]) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  for (int c = 0; c < 3; ++c) { ms[c] = 0; flops[c] = 0; launches[c] = 0; }
  for (ProfRec& r : g_prof) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) continue;
    ms[r.cls] += t; flops[r.cls] += r.flops; launches[r.cls] += 1;
  }
  return 0;
}

// every recorded launch in order: ms / flops per launch, meta = (class, M rows, N columns, K = taps * channels) x 4 ints
int tc_profile_launches(double* ms, double* flops, long long* meta4, int capacity, int* n_out) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return (int)e;
  int n = 0;
  for (ProfRec& r : g_prof) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) continue;
    if (n < capacity) { ms[n] = t; flops[n] = r.flops; meta4[4 * n] = r.cls; meta4[4 * n + 1] = r.M; meta4[4 * n + 2] = r.N; meta4[4 * n + 3] = r.K; }
    ++n;
  }
  if (n_out) *n_out = n;
  return 0;
}
