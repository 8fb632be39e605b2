// wgmma (Hopper tensor core) gather-GEMM path of libcgvc.so: bf16 hi/lo split operands, fp32 register accumulators.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stddef.h>
#include <vector>
#include "kernels.cuh"

#define TC_UNSUPPORTED (-12345)

// One convolution (or gated pair of convolutions sharing an input) whose weights are kept as bf16 hi/lo planes in
// the operand layouts the tensor-core kernels consume.
struct TcLayer {
  size_t ka, kg, ba, bg;          // offsets (elements) of kernel_a / kernel_g / bias_a / bias_g in the PARAM arena
  int kh, kw, cin, cout, gated;   // TF shapes [kh,kw,cin,cout]; Ntot = cout * (gated ? 2 : 1)
  int shuffle;                    // 2: the layer's output goes through the pixel shuffler (module.py:135-146); forward weight rows are then
                                  // stored so that one 256-column tile holds both conv channels of 64 post-shuffle channels (tc_gemm.cu perm_row)
  int fold;                       // > 0: a 1 x 1 layer whose `cout` output columns are (t, n) pairs, column = t * (cout / fold) + n, of a TF kernel
                                  // [1, fold, cin, cout / fold] at ka (a stride-1 multi-tap layer with few output channels, computed as one dense GEMM
                                  // whose per-tap results the caller sums with the tap shifts: engine.cu `edge_lower`); not gated, no bias
  // padded extents: x_k = rounded up to 64 (contraction), x_n = rounded up to 128 (output tile); pads are zero
  __nv_bfloat16 *wf_hi, *wf_lo;   // forward B operand  [taps][Ntot_n][cin_k]   (K = cin contiguous)
  __nv_bfloat16 *wd_hi, *wd_lo;   // dgrad   B operand  [taps][cin_n][Ntot_k]   (K = Ntot contiguous)
  float* bias;                    // [Ntot_n]
  CUtensorMap tm_f_hi, tm_f_lo;   // TMA descriptors of wf (box [1][BN][64]) and wd, built once the planes are allocated
  CUtensorMap tm_d_hi, tm_d_lo;
  // CGVC_PREC_F16F8 (allocated when TcWeights::quant): forward operand [taps][Ntot_n][cin_q], cin_q = cin rounded up
  // to 128, as fp16 + two e4m3 planes with the weight scales of kernels.cuh
  void* wq16; uint8_t *wq8hi, *wq8lo;
  CUtensorMap tm_q16, tm_q8hi, tm_q8lo;
  // F16F8 training (TcWeights::quant_bwd): data-gradient operand [taps][cin_n][nt_q], nt_q = Ntot rounded up to 128
  void* wdq16; uint8_t *wdq8hi, *wdq8lo;
  CUtensorMap tm_dq16, tm_dq8hi, tm_dq8lo;
};

struct TcWeights {
  std::vector<TcLayer> layers;
  void* pool = nullptr;
  size_t pool_bytes = 0;
  bool ready = false;
  bool quant = false;             // also keep the F16F8 forward planes (precision F16F8)
  bool quant_bwd = false;         // ... and the F16F8 data-gradient planes (training in that precision)
  void* prep_jobs = nullptr;      // device job table of the batched F16F8 plane kernel (tc_gemm.cu PrepJob), one job per layer branch
  std::vector<int> job_first;     // first block of every job + total (size jobs + 1)
  std::vector<size_t> job_ka;     // PARAM offset of the job's layer (range filter of tc_refresh_weights_range)
  // options of the engine that only this module reads (include/cgvc.h cgvc_set_option)
  int wgrad16 = 0;                // "wgrad_f16" (F16F8 only; tc_alloc sets it there): weight gradients from the fp16 planes alone
                                  // (one MMA unit per product instead of two)
  int prep_batched = 1;           // "prep_batched": F16F8 weight planes of all layers in one launch; 0: per-layer kernels
  int debug = 0;                  // "tc_debug": diagnostic knobs of the gather-GEMMs (timing experiments only; see TcNTParams::debug)
};

// what the fused forward epilogue needs besides the convolution itself (see tc_conv_fwd)
struct TcFuse {
  int R;                                            // positions per sample of the layer output
  const float *gamma_a, *beta_a, *gamma_g, *beta_g; // instance-norm affine parameters (g: gate branch, null when not gated)
  float* stats;                                     // [n,4,C] saved (mean, rstd) pairs for the backward pass
  const float* resid;                               // residual input [rows, C] (non-gated residual layer) or null
  float* y; __nv_bfloat16 *y_hi, *y_lo;             // outputs [rows, C] (fp32 optional)
};

// what the fused backward epilogue of a data-gradient launch needs (see tc_conv_dgrad): the gradient this launch computes
// is d loss / d (output of an upstream layer); that layer's instance-norm (+ GLU) backward runs in the epilogue
struct TcBwdFuse {
  int R;                                            // positions per sample
  int gated;                                        // 1: y = IN(a) * sigmoid(IN(g)) (EPI 3); 0: y = resid + IN(a) (EPI 4, dx also receives dY)
  const float* bp; int bp_ld;                       // the upstream layer's saved pre-norm conv outputs [rows, bp_ld]
  const float* stats;                               // its saved (mean_a, rstd_a, mean_g, rstd_g) [n,4,C]
  const float *gamma_a, *beta_a, *gamma_g, *beta_g;
  __nv_bfloat16 *dp_hi, *dp_lo; int dp_ld;          // its dP planes (output) [rows, dp_ld]
  float *dbeta_a, *dgamma_a, *dbeta_g, *dgamma_g;   // parameter gradients (accumulated; null: data gradient only)
};

int tc_register(TcWeights& w, size_t ka, size_t kg, size_t ba, size_t bg, int kh, int kw, int cin, int cout, int gated, int shuffle = 1, int fold = 0);
// precision: CGVC_PREC_*; train: an F16F8 engine also keeps the data-gradient planes.  cudaError_t as int
int tc_alloc(TcWeights& w, int precision, bool train);
void tc_free(TcWeights& w);
int tc_refresh_weights(TcWeights& w, const float* params, cudaStream_t st);
// the planes and bias of one layer from its TF kernels ka / kg and biases ba / bg (the per-layer step of tc_refresh_weights)
int tc_refresh_layer(TcLayer& L, const float* ka, const float* kg, const float* ba, const float* bg, cudaStream_t st);
int tc_refresh_weights_range(TcWeights& w, const float* params, size_t begin, size_t end, cudaStream_t st);
// Read-only view of registered layer `slot` (include/cgvc.h cgvc_weight_planes).  dims = {nt_n, cin_k, cin_n, nt_k, cin_q, nt_q, layer_ok_q}.
// tc_layer_plane: the device address and size in bytes (padding included) of a named plane; *p = null when the store keeps no such plane
// current (not allocated, or the bf16 planes of a layer that an F16F8 store serves from its F16F8 planes).  Returns -1 for an unknown name.
void tc_layer_dims(const TcWeights& w, int slot, int dims[7]);
int tc_layer_plane(const TcWeights& w, int slot, const char* name, const void** p, size_t* bytes);

// x [rows, C] fp32 -> the operand planes of `precision` with C zero-padded to the contraction width: bf16 hi / lo [rows, ru64(C)],
// F16F8: q16 (hi) and q8hi followed by q8lo (lo) [rows, ru128(C)].  cudaError_t
// sat (F16F8, may be null): count of saturated 4-value groups of the planes (kernels.cuh cgvc_quant4_sat); ufl: [ufl, groups] likewise
cudaError_t tc_split_planes(int precision, const float* x, long long rows, int C, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st,
                            unsigned long long* sat = nullptr, unsigned long long* ufl = nullptr);

// The convolutions of layer L below read and write the planes of `precision` (tc_split_planes), with their channel count rounded up
// (zero-filled): x [n,H,W,cin], dP [rows, Ntot].  debug and w16: the store's TcWeights::debug and TcWeights::wgrad16.  They return
// 0, TC_UNSUPPORTED (no launch: the shape has no tensor-core form) or a cudaError_t.
// P[rows, Ntot] = conv(x) + bias.
//   fuse: instance norm (+ GLU | + residual) fused into the epilogue when the shape allows (1-D layer, whole samples per 128-row
//         tile: R in {32,64,128}); *fused tells the caller whether it happened (if not, P is written and the caller runs the
//         separate instance-norm kernels).
//   pk:   a 1-D layer over packed variable-length utterances (kernels.cuh PackGeom): n = H = 1, x planes [W, .] at the source level
//         of divisor pk->div; every tap reads only its own utterance's rows.  Plain epilogue only.
int tc_conv_fwd(const TcLayer& L, int precision, int debug, const __nv_bfloat16* xhi, const __nv_bfloat16* xlo, int n, int H, int W,
                int sh, int sw, float* P, cudaStream_t st, const TcFuse* fuse = nullptr, bool* fused = nullptr, const PackGeom* pk = nullptr);
// dx[n,H,W,cin] (+)= dgrad(dP)            (dP planes [rows_out, Ntot]; H, W are the INPUT dims)
//   fuse: the upstream layer's instance-norm (+ GLU) backward fused into the epilogue when the shape allows (stride-1 1-D layer,
//         whole samples per 128-row tile): the launch then writes that layer's dP planes (and, for gated = 0, dx = dY) instead
//         of / besides dx; *fused tells whether it happened (if not, dx holds the plain data gradient).
//   pk:   packed utterances as in tc_conv_fwd, pk->div the divisor of the INPUT level; plain epilogue only (fuse is ignored)
int tc_conv_dgrad(const TcLayer& L, int precision, int debug, const __nv_bfloat16* dPhi, const __nv_bfloat16* dPlo, int n, int H, int W,
                  int sh, int sw, float* dx, int accumulate, cudaStream_t st, const TcBwdFuse* fuse = nullptr, bool* fused = nullptr,
                  const PackGeom* pk = nullptr);
// dW_a/dW_g (TF layout) += x^T dP  (the bias gradients are column sums of dP: the instance-norm backward kernels or launch_colsum)
//   pk:   packed utterances as in tc_conv_fwd (x planes at the source level of divisor pk->div): a tap outside its row's utterance
//         contributes a zero row
int tc_conv_wgrad(const TcLayer& L, int precision, int debug, int w16, const __nv_bfloat16* xhi, const __nv_bfloat16* xlo,
                  const __nv_bfloat16* dPhi, const __nv_bfloat16* dPlo, int n, int H, int W, int sh, int sw,
                  float* dwa, float* dwg, cudaStream_t st, const DetSlab* det = nullptr,   // det: deterministic mode (kernels.cuh DetSlab)
                  const PackGeom* pk = nullptr);

// per-launch CUDA-event timing of the tensor-core kernels (class 0 = forward/dgrad kernel with the plain epilogue,
// 1 = wgrad kernel, 2 = forward kernel with the fused instance-norm epilogue)
void tc_profile_enable(int on);
bool tc_profile_is_on();
int tc_profile_collect(double ms[3], double flops[3], long long launches[3]);
int tc_profile_launches(double* ms, double* flops, long long* meta4, int capacity, int* n_out);
