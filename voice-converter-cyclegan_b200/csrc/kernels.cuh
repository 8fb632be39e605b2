// Internal kernel-launcher declarations for libcgvc.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <stdint.h>
#ifdef __CUDACC__
#include <cooperative_groups.h>
#include <cooperative_groups/reduce.h>
#endif

// ---- "F16F8" operand planes (CGVC_PREC_F16F8; forward, data gradient and weight gradient since round 2): an fp32 tensor x is kept as
//        q16  = fp16(x)                                   2 bytes / element   (hi * hi product: one kind::f16 MMA)
//        q8hi = e4m3(sat(float(q16) * S_hi))              1 byte              } the two cross products hi * lo, lo * hi as
//        q8lo = e4m3(sat((x - float(q16)) * S_lo))        1 byte              } kind::f8f6f4 MMAs at twice the rate
//      with static power-of-two scales chosen so that BOTH cross products carry 2^15, which the first kind::f16 MMA of a
//      tile removes again (scale-input-d = 15):  activations S_hi = 1, S_lo = 2^12;  weights S_hi = 2^3, S_lo = 2^15.
//      Emulated end to end in tests/precision_study.py (scheme fp16_f8_static): 4.7e-5 on the generator output.
#define CGVC_Q_ACT_SHI 1.0f
#define CGVC_Q_ACT_SLO 4096.0f
#define CGVC_Q_W_SHI 8.0f
#define CGVC_Q_W_SLO 32768.0f
#define CGVC_Q_ACC_SHIFT 15
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t cgvc_e4m3x4(float a, float b, float c, float d) {      // 4 floats -> 4 saturating e4m3 bytes
  const uint32_t lo = (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
// 4 consecutive values -> 8 bytes of q16, 4 bytes of q8hi, 4 bytes of q8lo
__device__ __forceinline__ void cgvc_quant4(const float (&v)[4], float s_hi, float s_lo, uint2& q16, uint32_t& q8hi, uint32_t& q8lo) {
  const __half2 h01 = __floats2half2_rn(v[0], v[1]), h23 = __floats2half2_rn(v[2], v[3]);
  const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  q16.x = *reinterpret_cast<const uint32_t*>(&h01); q16.y = *reinterpret_cast<const uint32_t*>(&h23);
  q8hi = cgvc_e4m3x4(f01.x * s_hi, f01.y * s_hi, f23.x * s_hi, f23.y * s_hi);
  q8lo = cgvc_e4m3x4((v[0] - f01.x) * s_lo, (v[1] - f01.y) * s_lo, (v[2] - f23.x) * s_lo, (v[3] - f23.y) * s_lo);
}
// Whether cgvc_quant4's planes of 4 values are wrong: true if an e4m3 conversion clamped (|scaled value| > 448, the largest e4m3 number, in
// the hi or the lo plane) or fp16(x) is not finite.  With the activation-role scales the hi plane clamps once |fp16(x)| > 448 and the lo
// plane, whose rounding residual reaches |x| * 2^-11, from |x| >= 256; fp16(x) itself overflows at 65504.
#define CGVC_E4M3_MAX 448.f
__device__ __forceinline__ bool cgvc_sat4(const float (&v)[4], float s_hi, float s_lo) {
  bool bad = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float f = __half2float(__float2half_rn(v[k]));
    bad |= !(fabsf(f * s_hi) <= CGVC_E4M3_MAX) || !(fabsf((v[k] - f) * s_lo) <= CGVC_E4M3_MAX);     // NaN / inf compare false
  }
  return bad;
}
// *ctr += hits, aggregated over the lanes of the warp that reach this call together: one reduction and, only if the sum is non-zero,
// one atomic per such group.  The writers call this inside divergent loops, so the group is discovered (coalesced_threads), not
// assumed to be the full warp
__device__ __forceinline__ void cgvc_count_hits(unsigned long long* ctr, unsigned hits) {
  namespace cg = cooperative_groups;
  const cg::coalesced_group g = cg::coalesced_threads();
  const unsigned n = cg::reduce(g, hits, cg::plus<unsigned>());
  if (n && g.thread_rank() == 0) atomicAdd(ctr, (unsigned long long)n);
}
// Whether cgvc_quant4's fp16 plane of 4 values lies below its lower edge: one of them is finite and non-zero while |fp16(x)| < 2^-14, i.e.
// fp16(x) is subnormal or flushed to zero.  Below that edge an F16F8 product loses a bit per octave (DESIGN.md section 10)
__device__ __forceinline__ bool cgvc_ufl4(const float (&v)[4]) {
  bool low = false;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    low |= isfinite(v[k]) && v[k] != 0.f && fabsf(__half2float(__float2half_rn(v[k]))) < 0x1p-14f;
  return low;
}
// The counters of a plane writer for one 4-value group (each null: not counted): sat += cgvc_sat4, ufl[0] += cgvc_ufl4, ufl[1] += 1
// (the groups counted, so that ufl[0] reads as a fraction).  Activation-role scales
__device__ __forceinline__ void cgvc_count_planes(unsigned long long* sat, unsigned long long* ufl, const float (&v)[4]) {
  if (sat) cgvc_count_hits(sat, cgvc_sat4(v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO));
  if (ufl) { cgvc_count_hits(ufl, cgvc_ufl4(v)); cgvc_count_hits(ufl + 1, 1u); }
}
#endif

// ---- dynamic loss scaling (engine option "loss_scale"; DESIGN.md section 10).  One per engine, in device memory.  The first fields
// are cgvc_loss_scale_info of include/cgvc.h, in its layout (cgvc_loss_scale_state copies them out); the counters and the non-finite
// flag are zeroed at the start of every train step and filled by the plane writers and the GRAD check
struct LossScaler {
  float scale;                    // loss scale the next step's gradients are formed with
  int good_steps;                 // consecutive steps that were not skipped
  long long skipped;              // steps skipped so far
  int last_skipped;               // the last step was skipped
  unsigned nonfinite;             // the last step's GRAD held a non-finite value: bit 0 generators, bit 1 discriminators
  unsigned long long sat_grad;    // the last step's saturated 4-value groups in gradient planes
  unsigned long long sat_act;     // ... in activation planes (diagnostic)
  // engine-internal
  long long t;                    // Adam step count (dynamic mode)
  float scale_used;               // the scale the last step's gradients were formed with
  // option "loss_scale_per_network": [0] the generators, [1] the discriminators.  Net has the layout of the head's first two fields;
  // cnt[k] = {sat, ufl, groups} of network k's gradient planes in the last step (the writers' targets: sat = cnt[k], ufl = cnt[k] + 1,
  // see cgvc_count_planes), one contiguous block so that one all-reduce sums both networks' counts over ranks
  struct Net {
    float scale;                  // the scale this network's passes form their gradients with
    int good_steps;               // consecutive steps in which this network's planes and GRAD range did not overflow (dynamic)
  } net[2];
  unsigned long long cnt[2][3];
};
// the Adam hyper-parameters of both optimizers after a step: hyper = d_scalars + 2 = [lr_G, 1/nranks, lr_D, 1/nranks] as the host wrote
// them on entry, overwritten with [lr_t G, grad_scale, lr_t D, grad_scale] unless the step is skipped (see simt_kernels.cu)
// nets = 1: a scale per network (F16F8): the step is skipped when either network overflowed, only an overflowing network's scale halves,
// each grows after growth_interval of its own good steps, and grad_scale divides by that network's scale.  nets = 2 (monitor mode) only
// sums the counters: sat_grad = cnt[0][0] + cnt[1][0]
cudaError_t launch_loss_scale_update(LossScaler* s, float* hyper, int adapt, int growth_interval, float beta1, float beta2, cudaStream_t st,
                                     int nets = 0);
// nonfinite |= (bit 0 if a non-finite value lies in g[0, cut), bit 1 if in g[cut, n))
cudaError_t launch_check_finite(const float* g, long long n, long long cut, unsigned* nonfinite, cudaStream_t st);

extern unsigned long long g_cgvc_launches;   // incremented by every kernel launch of the library

// grid caps of the streaming kernels: multiples of the SM count of an H100 SXM
#define CGVC_NUM_SMS 132

#define CGVC_MAX_TAPS 18   // largest filter on the path: discriminator d3, 6x3 (module.py:208)

// ---- deterministic mode (engine option "deterministic"; DESIGN.md section 11).  A writer that would add into GRAD or a loss slot from
// many CTAs at once instead stores each CTA's contribution as one row of a partials slab with plain stores; launch_reduce_parts then
// sums the rows in index order and makes one add per element.  The slab is carved from the WORK arena, CGVC_DET_SLAB_FLOATS floats
// per lane; every launcher checks on the host that its rows fit and returns an error, never launches, when they do not.
#define CGVC_DET_SLAB_FLOATS (8ll << 20)
struct DetSlab { float* p; long long cap; };          // cap: floats; p == null: the default atomic accumulation
// up to four destinations of one partial row: dst[i][j] += sum_k part[k * row + off[i] + j], j < len[i] (null dst: skipped)
struct DetSegs { float* dst[4]; long long off[4]; long long len[4]; };
cudaError_t launch_reduce_parts(const float* part, long long nparts, long long row, const DetSegs& s, cudaStream_t st);

// Geometry of a "gather-GEMM":  D[m, n] = sum_t sum_c  S[src(m,t), c] * Wt[t][c][n]
//   m enumerates a logical output grid (b, y, x); src(m,t) = (b, y*sy + oy[t], x*sx + ox[t]) in the source
//   tensor [B,Hs,Ws,*] (zero outside), and row m is written to (b, y*dsy + doy, x*dsx + dox) of the
//   destination tensor [B,Hd,Wd,*].  This one primitive expresses
//     - forward conv (TF SAME, any stride):  oy = i - pad_top, sy = stride
//     - data gradient, stride 1:             oy = pad_top - i (flipped taps), source = dY
//     - data gradient, stride 2:             one launch per output-parity class p with the taps of matching
//                                            parity, oy = (p + pad - i)/2, dsy = 2, doy = p
//   (SURVEY.md Appendix A.1/A.2; module.py:22-64 of the reference).
struct GatherGeom {
  int B, Hy, Wx;
  int Hs, Ws;
  int sy, sx;
  int ntaps;
  int Hd, Wd, dsy, dsx, doy, dox;
  short oy[CGVC_MAX_TAPS], ox[CGVC_MAX_TAPS], widx[CGVC_MAX_TAPS];
};
#ifdef __CUDACC__
// The taps that rows of output rows y_lo .. y_hi can read (bit t): those with some y in the range and 0 <= y*sy + oy[t] < Hs.  Every
// other tap reads only the zero padding for all of these rows.  Along x nothing is dropped.
__host__ __device__ __forceinline__ uint32_t gather_tap_mask(const GatherGeom& g, int y_lo, int y_hi) {
  uint32_t mask = 0;
  for (int t = 0; t < g.ntaps; ++t) {
    const int oy = g.oy[t];
    int y = y_lo;                                            // the first y >= y_lo whose source row is not above the tensor
    if (oy < 0 && (-oy + g.sy - 1) / g.sy > y) y = (-oy + g.sy - 1) / g.sy;
    if (y <= y_hi && y * g.sy + oy < g.Hs) mask |= 1u << t;
  }
  return mask;
}
#endif

// Packed variable-length 1-D geometry (cgvc_generator_forward_packed): n utterances concatenated along time.  off = n + 1 device
// frame prefix sums at full resolution, every length a multiple of 4, so at a level of divisor div (1, 2 or 4: the T, T/2, T/4
// resolutions of the generator) utterance u owns the rows [off[u] / div, off[u+1] / div) exactly.  max_len: the longest utterance at
// full resolution (launch sizing on the host).
struct PackGeom { const long long* off; int n; int div; int max_len; };
#ifdef __CUDACC__
// the utterance holding full-resolution frame f: off[u] <= f < off[u+1] (binary search; off is small and stays in L1 / L2)
__device__ __forceinline__ int pack_find(const long long* __restrict__ off, int n, long long f) {
  int lo = 0, hi = n;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (__ldg(off + mid) <= f) lo = mid; else hi = mid; }
  return lo;
}
#endif

// Packed variable-length 2-D grids (cgvc_discriminator_forward_packed): every length a multiple of 16, and a grid of H rows at divisor
// div (<= 16) holds utterance u as [H][len_u / div] at rows H * off[u] / div ... H * off[u+1] / div, so that the levels of the
// discriminator lie utterance after utterance.  A gather over such grids takes its GatherGeom from fwd_geom / dgrad_geoms(1, H, total
// frames / div, ...) and its PackGeom as for the 1-D form: pk.div the source grid's divisor, pk.div * g.sx the output grid's and
// pk.div * g.sx / g.dsx the destination grid's.  PackGeom2 is that PackGeom as the trailing argument of the 2-D kernel instantiations.
struct PackGeom2 { PackGeom pk; };
#ifdef __CUDACC__
// row m of a grid of H rows at divisor div: its utterance u (frames o0 .. o1) and its (y, x) there
struct Pack2Pos { int u; long long o0, o1; int y, x; };
__device__ __forceinline__ Pack2Pos pack2_pos(const PackGeom& pk, int H, int div, long long m) {
  Pack2Pos r;
  r.u = pack_find(pk.off, pk.n, m * div / H);               // H off[u] / div <= m  <=>  off[u] <= floor(m div / H)
  r.o0 = __ldg(pk.off + r.u); r.o1 = __ldg(pk.off + r.u + 1);
  const int w = (int)((r.o1 - r.o0) / div);
  const long long l = m - H * r.o0 / div;
  r.y = (int)(l / w); r.x = (int)(l - (long long)r.y * w);
  return r;
}
// the row of (y, x) of utterance o0 .. o1 in a grid of H rows at divisor div, or -1 outside its [0, H) x [0, len / div)
__device__ __forceinline__ long long pack2_row(long long o0, long long o1, int H, int div, int y, int x) {
  const int w = (int)((o1 - o0) / div);
  return y >= 0 && y < H && x >= 0 && x < w ? H * o0 / div + (long long)y * w + x : -1;
}
#endif

struct GemmOperands {
  const float* src; int s_ld; int s_coff; int C;      // gathered operand: row stride, column offset, #channels contracted
  const float* w; long long w_ts; int w_cs; int w_ns; // weight element (tap slab, c, n) = w[widx*w_ts + c*w_cs + n*w_ns]
  int N;
  float* dst; int d_ld; int d_coff;
  const float* bias;                                  // [N] or null
  int accumulate;                                     // dst += result
};

// ---- fp32 SIMT path (reference arithmetic on the GPU; also the permanent path for the tiny-K layers)
cudaError_t launch_gg_simt(const GatherGeom& g, const GemmOperands& op, cudaStream_t st);
// the same over a packed geometry: g = fwd_geom(1, 1, rows at the source level, 1, kw, 1, sw) of a 1-D layer, pk.div = the source
// level's divisor; taps read only their own utterance's rows (TF-SAME zero padding at every utterance edge).  A geometry with more
// than one row along y is a 2-D packed one (PackGeom2)
cudaError_t launch_gg_simt_packed(const GatherGeom& g, const GemmOperands& op, const PackGeom& pk, cudaStream_t st);
// weight gradient in forward geometry: dW[widx[t]][c][n] += sum_m S[src(m,t), c] * G[m, n]   (atomic accumulate)
// pk: packed utterances, g and pk as launch_gg_simt_packed takes them; a tap outside its row's utterance contributes a zero row
cudaError_t launch_wgrad_simt(const GatherGeom& g, const float* src, int s_ld, int s_coff, int C,
                              const float* grad, int g_ld, int g_coff, int N,
                              float* dw, long long w_ts, int w_cs, int w_ns, cudaStream_t st, int det = 0, const PackGeom* pk = nullptr);
// db[n] += sum_m G[m, g_coff + n]
cudaError_t launch_colsum(const float* grad, long long rows, int g_ld, int g_coff, int N, float* db, cudaStream_t st,
                          const DetSlab* det = nullptr);

// ---- instance-norm / GLU / residual "post" kernels (module.py:3-20, 66-146)
struct PostParams {
  const float* p; int ldp; int Cc;      // conv output rows [B*(R/sh), ldp]; 'a' cols [0,Cc), gate cols [Cc,2Cc); Cc = C*sh
  int B, R, C, sh;                      // after the pixel-shuffle view: R positions x C channels per sample
  const float *beta_a, *gamma_a, *beta_g, *gamma_g;
  int has_in, has_gate;
  const float* resid;                   // [B,R,C] added to the result (residual1d_block), or null
  float* y;                             // [B,R,C] (may be null when only the planes are wanted)
  float* stats;                         // [B,4,C]: mean_a, rstd_a, mean_g, rstd_g (written if has_in)
  __nv_bfloat16 *y_hi, *y_lo;           // optional bf16 split planes of y for the tensor-core path
  float* scratch;                       // [B,4,C] fp32 workspace for the instance-norm sums (required when has_in)
  int qmode;                            // 1: the planes are F16F8 planes instead: y_hi = q16 [B*R*C halves], y_lo = q8hi [B*R*C bytes] followed by q8lo
  // packed variable-length samples (seg.off != null): sample b = view rows [seg.off[b] / seg.div, seg.off[b+1] / seg.div) of seg_rows
  // rows in all (the planes' extent is seg_rows * C); R = the longest sample (grid size).  launch_post_fwd only
  PackGeom seg; long long seg_rows;
  unsigned long long* sat;              // qmode: count of saturated 4-value groups of the planes (cgvc_quant4_sat), or null
  unsigned long long* ufl;              // qmode: [ufl, groups] of the planes (cgvc_count_planes), or null
};
// Which forms of the kernels a launch may take (the engine's options "post_onepass" and "post_stream", include/cgvc.h).
// onepass: samples of <= 64 positions take the one-pass backward kernel, else always sums + apply.  stream: the layer shapes that
// have one take the streaming (cp.async double-buffered) form, the backward's only with onepass
struct PostForms { int onepass, stream; };
cudaError_t launch_post_fwd(const PostParams& pp, PostForms forms, cudaStream_t st);

struct PostBwdParams {
  const float* dy1; const float* dy2;   // upstream gradient(s) [B,R,C]; dy2 may be null (summed if present)
  const float* p; int ldp; int Cc;
  int B, R, C, sh;
  const float *beta_a, *gamma_a, *beta_g, *gamma_g;
  int has_in, has_gate;
  const float* stats;
  float* dp;                            // same layout as p (fp32), may be null if only planes wanted
  __nv_bfloat16 *dp_hi, *dp_lo;         // optional bf16 split planes, same layout as p
  float *dbeta_a, *dgamma_a, *dbeta_g, *dgamma_g;   // accumulated atomically (may be null when has_in == 0)
  float *dbias_a, *dbias_g;             // conv-bias gradients [Cc] = column sums of dp (accumulated atomically; may be null)
  int qmode;                            // 1: dp_hi / dp_lo are F16F8 planes (q16; q8hi followed by q8lo) with the activation-role scales
  float* scratch;                       // [B,4,C] fp32 workspace (required when has_in)
  unsigned long long* sat;              // qmode: count of saturated 4-value groups of the planes (cgvc_quant4_sat), or null
  unsigned long long* ufl;              // qmode: [ufl, groups] of the planes (cgvc_count_planes), or null
  DetSlab det;                          // deterministic mode (det.p != null): the sums + apply form, parameter and bias gradients reduced in order
};
// Packed variable-length samples of launch_post_bwd (instance-normed layers; the sums + apply form only): sample b = view rows
// [seg.off[b] / seg.div, seg.off[b+1] / seg.div) of `rows` view rows in all, with its own statistics; PostBwdParams::B = seg.n and R =
// the longest sample (grid size).  A kernel argument of the packed instantiations only: PostBwdParams, the parameter block of the
// equal-length kernels, stays as it is
struct PostBwdSeg { PackGeom seg; long long rows; };
cudaError_t launch_post_bwd(const PostBwdParams& pp, PostForms forms, cudaStream_t st, const PostBwdSeg* seg = nullptr);
cudaError_t post_init_kernels();   // shared-memory opt-in of the streaming kernels (call once, outside any stream capture)

// ---- discriminator head: dense(1024->1) + sigmoid (module.py:211) and LSGAN loss (model.py:68-69,81-86)
cudaError_t launch_head_fwd(const float* y, long long rows, int C, const float* w, const float* b, float* prob, cudaStream_t st);
// loss_slot += coef * mean((p - target)^2) over `rows`; dz = coef * 2 (p-target)/rows * p (1-p);
// dy[row,:] = dz * w (if dy);  dw += sum dz*y[row,:], db += sum dz (if dw)
// dprob (may be null): an upstream gradient d prob [rows] instead of the loss: dz = grad_mult * dprob[row] * p (1-p), target and coef
// unused, loss_slot must be null
cudaError_t launch_head_loss_bwd(const float* prob, const float* y, long long rows, int C, const float* w,
                                 float target, float coef, float* loss_slot,
                                 float* dy, float* dw, float* db, cudaStream_t st, const float* grad_mult_dev = nullptr,
                                 const DetSlab* det = nullptr, const float* dprob = nullptr);

// ---- L1 loss + gradient (utils.py:6-8): loss_slot += mean|yhat - y|; d[i] = gscale * sign(yhat - y)/n  (accumulate optional)
cudaError_t launch_l1_loss_grad(const float* yhat, const float* y, long long n, float* loss_slot,
                                const float* gscale_dev, float* d, int accumulate, cudaStream_t st, const float* grad_mult_dev = nullptr,
                                const DetSlab* det = nullptr);
// grad_mult_dev (both loss kernels, null: 1): the gradients -- not the loss values -- are multiplied by *grad_mult_dev, the loss scale of the
// F16F8 gradient planes; a device pointer, so that a captured step follows the dynamic scale
// x *= a, or with div_dev x *= a / *div_dev
cudaError_t launch_scale(float* x, long long n, float a, cudaStream_t st, const float* div_dev = nullptr);
// x *= a * *mul_dev (a tape backward's upstream gradient times the scaler's current loss scale)
cudaError_t launch_scale_by(float* x, long long n, float a, const float* mul_dev, cudaStream_t st);
// [B,F,T] <-> [B,T,F]
cudaError_t launch_transpose_ft(const float* in, float* out, int B, int F, int T, cudaStream_t st);
// packed [F][len_u] blocks (block u at element F * off[u]) <-> channels-last rows [off[n], F]; to_rows = 1: blocks -> rows
cudaError_t launch_transpose_packed(const float* in, float* out, const long long* off, int n, long long rows, int F, int to_rows, cudaStream_t st);
// y = a + b
cudaError_t launch_add(const float* a, const float* b, float* y, long long n, cudaStream_t st);

// ---- TF-style Adam over a flat range (tf.train.AdamOptimizer; SURVEY.md Appendix A.6)
// hyper_dev: [0] = lr_t (already bias-corrected step size), [1] = grad_scale.  skip_dev (may be null): when *skip_dev != 0, p, m, v stay untouched
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, long long n,
                        const float* hyper_dev, float beta1, float beta2, float eps, cudaStream_t st, const int* skip_dev = nullptr);
// final loss algebra (model.py:72,83,88,90) on the 8-slot buffer
cudaError_t launch_finalize_losses(float* losses8, const float* lambdas_dev, cudaStream_t st);

// fp32 -> bf16 hi/lo split planes (x ~= hi + lo, |x - hi - lo| <= 2^-17 |x|)
cudaError_t launch_split_bf16(const float* x, __nv_bfloat16* hi, __nv_bfloat16* lo, long long n, cudaStream_t st);

// ---- single-input-channel specials (discriminator h1, K = 9, HBM-bound)
// dW[t][0][n] += sum_m x[src(m,t)] * G[m,n]; columns [0,n_split) -> dw_a, the rest -> dw_g; db = column sums (optional)
cudaError_t launch_wgrad_c1(const GatherGeom& g, const float* src, const float* grad, int g_ld, int N,
                            float* dw_a, float* dw_g, int n_split, float* db_a, float* db_g, cudaStream_t st, const DetSlab* det = nullptr,
                            const PackGeom* pk = nullptr);
// dx[B,H,W] = conv-transpose of G [rows, C] with w = [wa | wg] ([taps][c_split], [taps][C - c_split]); Z is scratch [rows, taps]
cudaError_t launch_dgrad_c1(const float* G, int C, const float* wa, const float* wg, int c_split, float* Z, float* dx,
                            int B, int H, int W, int kh, int kw, int sh, int sw, cudaStream_t st, const PackGeom* pk = nullptr);
// fp32 [M, C] (row stride ld) -> zero-padded bf16 hi/lo planes [M, Cpad]
cudaError_t launch_pad_split(const float* x, long long M, int C, int ld, int Cpad, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st);
// same into F16F8 planes: q16 [M, Cpad] halves, q8 = [M*Cpad bytes of q8hi | M*Cpad bytes of q8lo] (activation scales)
// sat (may be null): count of saturated 4-value groups (cgvc_quant4_sat); ufl (may be null): [ufl, groups] (cgvc_count_planes)
cudaError_t launch_pad_split_q(const float* x, long long M, int C, int ld, int Cpad, void* q16, void* q8, cudaStream_t st,
                               unsigned long long* sat = nullptr, unsigned long long* ufl = nullptr);
// tap lowering of the generator's 15-tap edge layers (simt_kernels.cu): im2col of a narrow channels-last tensor over the taps of a
// stride-1 1-D TF-SAME convolution into operand planes [M, Cpad] (qmode 1: F16F8 planes q16 / q8hi|q8lo, else bf16 hi / lo), dir = +1:
// out[m, t*C + c] = x[m + t - pl, c], dir = -1: x[m - t + pl, c] (zero outside the sample, pl = (kw - 1) / 2), and the matching sum
// y[m, c] = bias[c] + sum_t z[m + dir*(t - pl), t*C + c]
// With off (n + 1 device frame prefix sums, packed utterances) the samples are [off[u], off[u+1]) instead of T-row blocks (T ignored).
// sat (qmode, may be null): count of saturated 4-value groups (cgvc_quant4_sat); ufl (qmode, may be null): [ufl, groups]
cudaError_t launch_im2col_taps(const float* x, long long M, int T, int C, int kw, int dir, int Cpad, int qmode, void* hi, void* lo, cudaStream_t st,
                               const long long* off = nullptr, int n_off = 0, unsigned long long* sat = nullptr,
                               unsigned long long* ufl = nullptr);
cudaError_t launch_col2im_taps(const float* z, int ldz, long long M, int T, int C, int kw, int dir, const float* bias, float* y, cudaStream_t st,
                               const long long* off = nullptr, int n_off = 0);
// P[m, 0:2*cout] = [bias_a | bias_g] + sum_t x[src(m,t)] * [wa | wg][t]   (single input channel, TF kernels [taps][1][cout])
// pk (both c1 forwards, may be null): x and P are packed 2-D grids (PackGeom2), g = fwd_geom(1, H, total frames, ...)
cudaError_t launch_conv_c1_fwd(const GatherGeom& g, const float* x, const float* wa, const float* wg, const float* ba, const float* bg,
                               int cout, float* P, cudaStream_t st, const PackGeom* pk = nullptr);

// ... and with the layer's GLU in the same pass (gate without instance norm): also y = a * sigmoid(g) as fp32 [M, cout] (optional) and as
// operand planes (bf16 hi / lo, or with qmode the F16F8 planes q16; q8hi followed by q8lo); <= 9 taps
cudaError_t launch_conv_c1_glu_fwd(const GatherGeom& g, const float* x, const float* wa, const float* wg, const float* ba, const float* bg,
                                   int cout, float* P, float* y, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, int qmode, cudaStream_t st,
                                   unsigned long long* sat = nullptr, unsigned long long* ufl = nullptr, const PackGeom* pk = nullptr);

// s[off .. off+n) = v6_host[0..n)  (n <= 6), passed by value in the kernel arguments (no host-memory copy node)
cudaError_t launch_set_scalars(float* s, int off, int n, const float* v6_host, cudaStream_t st);

// ---- device-resident training data: epoch plan (pairing + crops from a counter-based generator) and minibatch gather
// (train.py:90-107, preprocess.py:207-238; contract in simt_kernels.cu).  off_X: n_X + 1 frame prefix sums; plan: [4][min(n_A, n_B)] ints;
// err: one int, set to (utterance index + 1, bit 30 = side B) if an utterance is shorter than the crop
cudaError_t launch_sample_plan(const long long* off_A, int n_A, const long long* off_B, int n_B, unsigned long long seed, long long epoch,
                               int crop, int* plan, int* err, cudaStream_t st);
cudaError_t launch_gather_minibatch(const float* cA, const long long* off_A, const float* cB, const long long* off_B, const int* plan,
                                    int num_pairs, int first_pair, int batch, int F, int crop, float* out_A, float* out_B, cudaStream_t st);

// ---- discriminator input layer backward, fused (no instance norm, one input channel): dP = GLU backward of (dY, P = [a | g]) is
// formed in registers and consumed in place -- weight + bias gradients, or the data gradient (Z scratch [rows, taps]) -- instead of
// being written to HBM and read back.  C = channels per branch (128).
cudaError_t launch_glu_bwd_wgrad_c1(const GatherGeom& g, const float* src, const float* dy, const float* P, int C,
                                    float* dw_a, float* dw_g, float* db_a, float* db_g, cudaStream_t st, const DetSlab* det = nullptr,
                                    const PackGeom* pk = nullptr);
cudaError_t launch_glu_bwd_dgrad_c1(const float* dy, const float* P, int C, const float* wa, const float* wg, float* Z, float* dx,
                                    int B, int H, int W, int kh, int kw, int sh, int sw, cudaStream_t st, const PackGeom* pk = nullptr);
// pk (the six c1 kernels, may be null): x / dx, P and dy are packed 2-D grids (PackGeom2: B = 1, W = all frames, pk.div = 1)
