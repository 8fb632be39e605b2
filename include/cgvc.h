/*
 * cgvc.h -- C ABI of libcgvc.so, the H100-native CycleGAN-VC training/inference engine.
 *
 * The reference (leimao/Voice-Converter-CycleGAN) has no FFI of its own: its seam is the Python
 * class `CycleGAN` (model.py:7-169) driving a TensorFlow-1 session.  Each entry point below names
 * the reference interface it replaces (file:line into /root/reference).  The Python mirror of the
 * reference class lives in voice-converter-cyclegan_b200/model.py and binds these symbols with ctypes;
 * INTEGRATION.md shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every call returns int: 0 = ok, <0 = error (message via cgvc_last_error); nothing throws across the ABI
 *   - pointers are DEVICE pointers unless the parameter name ends in _host
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); calls enqueue work and do
 *     not synchronise unless documented
 *   - one handle per device, not thread-safe per handle
 *   - storage (all arenas) is owned by the caller (torch tensors on the Python side); the engine never frees it
 *   - activations/IO are fp32; MCEP frames are [batch, 24, frames] row-major exactly like the reference's
 *     placeholders (model.py:35-42)
 */
#ifndef CGVC_H
#define CGVC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CGVC_ABI_VERSION 1
#define CGVC_NUM_LOSSES 8   /* model.py:153-169, in that order: cycle, identity, G_A2B, G_B2A, generator, D_A, D_B, discriminator */

typedef struct cgvc_engine* cgvc_handle;

typedef struct cgvc_config {
  int num_features;   /* 24: model.py:9 num_features (only 24 is supported; the discriminator head needs H=24) */
  int max_batch;      /* largest per-GPU minibatch a train step / forward will be called with */
  int max_frames;     /* largest frame count T (multiple of 4, module.py:166-179); training uses 128 (train.py:24) */
  int precision;      /* CGVC_PREC_*: arithmetic of the tensor-core contractions */
  int device;         /* CUDA device ordinal */
  int train;          /* 1: size arenas for training (model.py mode='train'); 0: forward only */
} cgvc_config;

enum {
  CGVC_PREC_FP32_SIMT = 0,  /* every contraction in fp32 FFMA (reference arithmetic; slow, used as on-GPU cross-check) */
  CGVC_PREC_BF16X3 = 1,     /* wgmma bf16 hi/lo split, 3 MMAs per product, fp32 accumulate (~2^-16 rel error; parity mode) */
  CGVC_PREC_BF16 = 2,       /* wgmma single bf16 MMA (fast, NOT parity-grade) */
  CGVC_PREC_F16F8 = 3       /* fp16 hi*hi MMA + the two cross terms as e4m3 kind::f8f6f4 MMAs at twice the rate, their common power of
                             * two folded out by scale-input-d: 2 MMA units per product instead of 3, parity-grade (4.7e-5 on the
                             * generator output).  Forward and data gradient; the weight gradient -- a leaf of the graph, its rounding
                             * error is not propagated into any other tensor -- reads the fp16 planes alone (1 unit; option "wgrad_f16" = 0
                             * restores the 2-unit form).  Training applies a power-of-two loss scale to the gradient planes and
                             * removes it in Adam (DESIGN.md section 10) */
};

enum cgvc_arena {
  CGVC_ARENA_PARAM = 0,     /* fp32 trainable variables, TF layouts, order [G_A2B | G_B2A | D_A | D_B] (model.py:93-95) */
  CGVC_ARENA_GRAD = 1,      /* fp32 gradients, same layout (what `minimize` computes, model.py:107-108) */
  CGVC_ARENA_ADAM_M = 2,    /* Adam first moment  (<var>/Adam   slots of tf.train.AdamOptimizer) */
  CGVC_ARENA_ADAM_V = 3,    /* Adam second moment (<var>/Adam_1 slots) */
  CGVC_ARENA_WORK = 4,      /* activations saved for backward, gradient scratch, bf16 operand planes */
  CGVC_ARENA_COUNT = 5
};

/* -- lifecycle: replaces CycleGAN.__init__ / build_model / optimizer_initializer (model.py:9-30,32-108) -- */
int cgvc_abi_version(void);
int cgvc_create(const cgvc_config* cfg, cgvc_handle* out);
int cgvc_destroy(cgvc_handle h);
const char* cgvc_last_error(cgvc_handle h);    /* h may be NULL: last error of a failed cgvc_create */

/* Bytes the caller must provide for an arena (WORK depends on cfg.max_batch/max_frames/train). */
int cgvc_arena_bytes(cgvc_handle h, int arena, size_t* bytes);
int cgvc_bind_arena(cgvc_handle h, int arena, void* dev_ptr, size_t bytes);

/* Variable table: TF variable names -> arena offsets (elements) and shapes, for checkpoints and weight
 * injection; replaces tf.trainable_variables() / tf.train.Saver (model.py:21,93,140-150). */
int cgvc_param_count(cgvc_handle h, int* n_tensors, size_t* n_elements);
int cgvc_param_info(cgvc_handle h, int index, const char** name, size_t* offset, int* ndim, int shape_out[4]);

/* Must be called after the caller (re)writes the PARAM arena (init, checkpoint load): refreshes the engine's
 * derived bf16 operand copies.  Replaces sess.run(global_variables_initializer) / Saver.restore side effects. */
int cgvc_params_updated(cgvc_handle h, void* stream);
/* Reset Adam step count t (beta-power accumulators of both optimizers, model.py:107-108).  With option "loss_scale" = 2 the count
 * lives on the device (a skipped step does not advance it): both calls then synchronise the device. */
int cgvc_set_adam_step(cgvc_handle h, long long t);
int cgvc_get_adam_step(cgvc_handle h, long long* t);

/* -- loss scaling of the F16F8 gradient planes (option "loss_scale", DESIGN.md section 10) ---------------------------------------
 * The planes of a gradient tensor x are fp16(x) and two e4m3 cross terms (S_hi = 1, S_lo = 2^12).  They are exact only in a window:
 * the hi plane clamps once |fp16(x)| > 448, the lo plane from |x| >= 256, fp16(x) overflows to inf at 65504 -- and a clamped cross term
 * is a wrong product, not a NaN.  Training multiplies every loss gradient by a power-of-two scale and Adam divides it out again.
 *   "loss_scale" = 0 (default): static, 2^(9 + floor(log2 batch)) in F16F8, 1 otherwise.  No extra work per step.
 *                = 1: monitor.  The static scale and the kernels of 0 (same arithmetic), but every train step counts its saturated plane
 *                     groups and checks GRAD for non-finite values (read with cgvc_loss_scale_state).
 *                = 2: dynamic.  A step whose gradient planes saturated (summed over ranks) or whose all-reduced GRAD holds a
 *                     non-finite value is skipped -- PARAM, ADAM_M, ADAM_V and the Adam step count stay as they were -- and the
 *                     scale halves (floor 1); after "loss_scale_growth_interval" (default 2000) good steps in a row it doubles
 *                     (cap 2^24).  It starts from the static scale of the first step's batch unless set with
 *                     cgvc_set_loss_scale_state.  In bf16x3, bf16 and fp32 the scale stays 1 and only non-finite steps are skipped.
 * Counted: the planes the instance-norm / GLU kernels (forward and backward), the input and output-gradient splits of the generator
 * and the discriminator's input layer write in a train step.  Not counted: the fused instance-norm epilogues of the forward GEMMs
 * (activation planes: with "fuse_in" = 1, the default, the generator layers whose instance norm is fused into the GEMM) and the weight
 * planes; with loss_scale != 0 the opt-in fused backward epilogues ("fuse_bwd") are not used, so with "fuse_bwd" = 1 modes 1 and 2 run
 * the unfused backward kernels and are not bit-identical to mode 0 (the unfused path is the default one).
 * Changing either option invalidates the captured step graphs.  With a communicator and "pipelined_comm", mode 2 makes every
 * network's Adam wait for the whole all-reduce and the scaler.
 * The window, measured on one H100 80GB HBM3 (700 W power limit; DESIGN.md section 10, tests/test_gpu_planes.py): an F16F8 GEMM stays
 * within 4e-4 of float64 while an activation / gradient operand's RMS lies in 2^-14 .. 2^12 (full precision for 2^-6 .. 2^6 with no
 * element above 256), a weight operand's from about 2^-13 up.  The batch-2 train step's gradients are within 1e-3 of float64 at every
 * scale from 2^4 up whose planes did not saturate (2^2: 1.2e-3, 2^0: 1.9e-3; the first saturation at 2^14), so the static scale
 * (2^10 at batch 2) lies 2^6 above the lower edge.  With one scale, at batch 1 with lambda_cycle = 1e4 it settles on 2, where the worst
 * gradient is 1.2e-3 from float64 -- not parity-grade: the generators' L1 gradients force the scale down and the discriminators' LSGAN
 * gradients, which do not grow with the lambdas, fall below the fp16 lower edge.  With "loss_scale_per_network" the same case settles
 * on s_G = 2, s_D = 512 and the worst of the 280 gradients is 3.6e-4.  Below the edge the underflow count rises: at batch 2 the
 * discriminators' ufl_grad / groups is 1.3e-2 at s_D = 2^10 and 1.6e-1 at 2^6, where their first update moves 1.2e-3.
 * "loss_scale_per_network" = 1 (F16F8, modes 1 and 2; default 0, and 0 changes nothing): two scales.  s_D multiplies the discriminators'
 *     D-loss heads and so everything that pass back-propagates, their weight gradients included; s_G the cycle and identity L1 gradients
 *     and the adversarial head, and so the adversarial data gradient through the discriminator and both generator backward passes.  Adam
 *     divides each GRAD range by its own network's scale.  The gradient-plane writers count per pass: sat_grad (saturated groups),
 *     ufl_grad (groups with a finite non-zero value whose fp16 plane is subnormal or flushed, |fp16(x)| < 2^-14: the edge below which an
 *     F16F8 product loses a bit per octave) and groups (all groups counted).  Dynamic mode skips a step when either network overflowed
 *     (saturation in its block, or a non-finite value in its GRAD range), halves only the scale of a network that did, and doubles each
 *     scale after "loss_scale_growth_interval" steps in which that network did not overflow.  ufl_grad is reported, not acted on.
 *     Monitor mode uses the static scale for both.  cgvc_loss_scale_info keeps its meaning, with scale = s_G, sat_grad = both networks'
 *     saturated groups and good_steps = consecutive steps not skipped. */
typedef struct cgvc_loss_scale_info {
  float scale;                    /* the scale the next step's gradients are formed with (static: that of the last step's batch) */
  int good_steps;                 /* consecutive steps not skipped (dynamic) */
  long long skipped;              /* steps skipped so far (dynamic) */
  int last_skipped;               /* the last step was skipped (dynamic) */
  unsigned nonfinite;             /* the last step's GRAD held a non-finite value: bit 0 generators, bit 1 discriminators */
  unsigned long long sat_grad;    /* the last step's saturated 4-value groups in gradient planes (dynamic: summed over ranks) */
  unsigned long long sat_act;     /* ... in activation planes: a diagnostic, the loss scale cannot fix a forward activation */
} cgvc_loss_scale_info;
/* asynchronous: copies the state into out_dev (device memory) on the stream */
int cgvc_loss_scale_state(cgvc_handle h, cgvc_loss_scale_info* out_dev, void* stream);
/* resume a dynamic scale: scale in [1, 2^24]; last_skipped, nonfinite, sat_grad and sat_act are cleared.  Synchronises the stream.
 * Sets both networks' scales and good-step counts too (a single-scale state resumed with "loss_scale_per_network"). */
int cgvc_set_loss_scale_state(cgvc_handle h, float scale, int good_steps, long long skipped, void* stream);
/* one network's share of the state with "loss_scale_per_network" (index 0 the generators, 1 the discriminators) */
typedef struct cgvc_loss_scale_net_info {
  float scale;                    /* s_G / s_D: the scale the next step's gradients of this network's passes are formed with */
  int good_steps;                 /* consecutive steps in which this network did not overflow (dynamic) */
  unsigned long long sat_grad;    /* the last step's saturated 4-value groups in this network's gradient planes (dynamic: summed over ranks) */
  unsigned long long ufl_grad;    /* ... groups below the fp16 lower edge (see above; dynamic: summed over ranks) */
  unsigned long long groups;      /* ... groups counted (dynamic: summed over ranks) */
} cgvc_loss_scale_net_info;
/* asynchronous: copies both networks' states into info_dev[2] (device memory) on the stream */
int cgvc_loss_scale_net_state(cgvc_handle h, cgvc_loss_scale_net_info* info_dev, void* stream);
/* resume one network's dynamic scale: net 0 or 1, scale in [1, 2^24] (net 0 also sets cgvc_loss_scale_info.scale).  Before any scale was
 * set it calls cgvc_set_loss_scale_state(scale, good_steps, 0) first, so the other network starts from the same scale.  Synchronises the
 * stream. */
int cgvc_set_loss_scale_net_state(cgvc_handle h, int net, float scale, int good_steps, void* stream);

/* -- the hot path: replaces CycleGAN.train (model.py:110-125) ------------------------------------------
 * One G step + one D step from the same pre-update weights, then both Adam updates.
 *   A_dev, B_dev       [batch, 24, frames] fp32 real samples of domain A / B
 *   gen_A_dev/gen_B_dev optional outputs [batch, 24, frames]: generation_A / generation_B (model.py:112)
 *   losses_dev         8 fp32 scalars (CGVC_NUM_LOSSES order), pre-update values, local-batch means
 * With a communicator attached (cgvc_comm_init) gradients are sum-all-reduced over ranks and averaged
 * before Adam; losses stay local. */
int cgvc_train_step(cgvc_handle h, const float* A_dev, const float* B_dev, int batch, int frames,
                    float lambda_cycle, float lambda_identity, float lr_generator, float lr_discriminator,
                    float* gen_A_dev, float* gen_B_dev, float* losses_dev, void* stream);

/* Same graph, but stops after the backward pass (GRAD arena holds d generator_loss/d G-vars and
 * d discriminator_loss/d D-vars); no all-reduce, no Adam.  For parity tests against the oracle. */
int cgvc_compute_gradients(cgvc_handle h, const float* A_dev, const float* B_dev, int batch, int frames,
                           float lambda_cycle, float lambda_identity,
                           float* gen_A_dev, float* gen_B_dev, float* losses_dev, void* stream);

/* TF-style Adam on the bound arenas (model.py:107-108; tf.train.AdamOptimizer beta1=0.5): advances t by one.
 * grad_scale multiplies every gradient first (1/nranks after a sum-all-reduce).  The same in every "loss_scale" mode (no skip: the
 * GRAD arena is the caller's); with "loss_scale" = 2, where t lives on the device, the call synchronises the device twice.
 * Loss scale of the tape backward calls (cgvc_*_backward_tape): in CGVC_PREC_F16F8 they leave their GRAD contributions multiplied by
 * the static loss scale of their tape's batch, s = 2^(9 + floor(log2 batch)) (1 in the other precisions; see cgvc_loss_scale_state);
 * Adam over such gradients takes grad_scale = 1 / s (times 1/nranks after an all-reduce).  Gradients of tapes of batches with different
 * scales do not share one GRAD: zero it in between.  No all-reduce: with a communicator, call cgvc_allreduce_grads first. */
int cgvc_adam_step(cgvc_handle h, float lr_generator, float lr_discriminator, float grad_scale, void* stream);

/* The optimizer tail of cgvc_train_step over the gradients that tape backward calls accumulated in GRAD (option "tape_loss_scale" = 1,
 * which needs "loss_scale" = 2).  With a communicator: the per-network all-reduce of GRAD and of the counters (pipelined with each
 * network's Adam when "pipelined_comm" is on).  Then the non-finite check of GRAD and the scaler update: on a saturated gradient plane
 * or a non-finite gradient the step is skipped and the scale halves (per network with "loss_scale_per_network": that network's), else
 * Adam runs with grad_scale = 1 / (scale x nranks) per optimizer and the scale doubles after "loss_scale_growth_interval" good steps.
 * Then the weight-plane refresh; the parameter generation advances even when the step was skipped.  The Adam count t stays on the
 * device, and nothing synchronises the host; cgvc_loss_scale_state reports the step as after a train step.  The counters and the
 * non-finite flag of the next accumulation are cleared by its first tape backward (or by this call, when none ran).
 * Errors, before anything is enqueued: the option off, or no scale yet (neither a tape backward nor cgvc_set_loss_scale_state since
 * "loss_scale" became 2): CGVC_ERR_ARG; PARAM, GRAD, ADAM_M or ADAM_V unbound: CGVC_ERR_UNBOUND. */
int cgvc_apply_gradients(cgvc_handle h, float lr_generator, float lr_discriminator, void* stream);

/* -- replaces CycleGAN.test (model.py:128-137): one generator forward.  direction 0 = 'A2B', 1 = 'B2A';
 * anything else returns CGVC_ERR_DIRECTION ("Conversion direction must be specified.", model.py:135). */
int cgvc_generator_forward(cgvc_handle h, int direction, const float* in_dev, float* out_dev,
                           int batch, int frames, void* stream);
/* generator forward of n utterances of different lengths in one call (conversion): utterance u is the row-major
 * [num_features][len_u] block at element num_features * offsets_host[u] of in_dev, and its converted block lands at the same place
 * in out_dev -- the corpus layout of cgvc_sample_plan.  offsets_host: n + 1 int64 frame prefix sums, offsets_host[0] = 0, every
 * len_u = offsets_host[u+1] - offsets_host[u] a positive multiple of 4.  Needs n <= max_batch and offsets_host[n] <= max_batch *
 * max_frames.  Every utterance's result is what cgvc_generator_forward gives for it alone, up to the summation order of its
 * instance-norm statistics.  Bad offsets, n or capacity return CGVC_ERR_ARG naming the offending utterance; the offsets are copied
 * to the device on the stream before the call returns.  With "debug_taps" a tap holds the concatenated rows of all utterances at
 * that layer's resolution (d2: offsets_host[n] / 4 x 512 elements). */
int cgvc_generator_forward_packed(cgvc_handle h, int direction, const float* in_dev, float* out_dev,
                                  const long long* offsets_host, int n, void* stream);
/* discriminator forward, which 0 = discriminator_A, 1 = discriminator_B: out [batch, 6, frames/16] (module.py:188-213) */
int cgvc_discriminator_forward(cgvc_handle h, int which, const float* in_dev, float* out_dev,
                               int batch, int frames, void* stream);
/* discriminator forward of n utterances of different lengths in one call: utterance u is the row-major [num_features][len_u] block at
 * element num_features * offsets_host[u] of in_dev (the layout cgvc_generator_forward_packed writes), and its probabilities are the
 * row-major [num_features / 4][len_u / 16] block at element (num_features / 4) * offsets_host[u] / 16 of prob_dev.  Every len_u must
 * be a positive multiple of 16 (the four stride-2 stages along time).  Every layer keeps to its utterance: each convolution pads with
 * zeros at the utterance's own edges and each instance norm takes its statistics over the utterance alone, so every utterance's result
 * is what cgvc_discriminator_forward gives for it alone, up to the summation order.  Argument checks and errors are those of
 * cgvc_generator_forward_packed (n <= max_batch, offsets_host[n] <= max_batch * max_frames, CGVC_ERR_ARG naming a bad utterance), all
 * before anything is enqueued.  Inside, every level of the network is stored utterance after utterance: utterance u owns rows
 * H_l * offsets[u] / d_l ... H_l * offsets[u+1] / d_l of a level with H_l rows at time divisor d_l, as [y][x][channel]. */
int cgvc_discriminator_forward_packed(cgvc_handle h, int which, const float* in_dev, float* prob_dev,
                                      const long long* offsets_host, int n, void* stream);

/* -- activation tapes: the two networks as differentiable operators (the reference composes module.py:148-213 into its loss graph,
 * model.py:44-108; here a caller composes them into any objective and runs each application's backward itself).
 * A tape is caller-owned device memory (256-byte aligned, at least cgvc_tape_bytes) that a forward fills with what the backward of that
 * one network application reads: its input and its layers' pre-norm outputs, statistics, outputs and operand planes, as a train step
 * keeps them.  kind 0 = generator, 1 = discriminator; batch <= max_batch, frames <= max_frames (a multiple of 4 / 16).  kind 2 = packed
 * generator (cgvc_generator_forward_packed_tape): cgvc_tape_bytes(h, 2, n, rows, &bytes) with n utterances of rows = offsets[n] frames in
 * all, n <= max_batch and rows <= max_batch x max_frames as cgvc_generator_forward_packed takes them.
 *   - Forward: the same outputs, bit for bit, as cgvc_generator_forward / cgvc_discriminator_forward.  A tape starts with a header
 *     written by the forward (kind, direction or which, batch, frames, the writing engine and its parameter generation); the engine
 *     keeps a copy, so that a backward checks its tape without reading the device.  cgvc_params_updated, cgvc_bind_arena and every Adam
 *     update (cgvc_adam_step, cgvc_train_step) advance the parameter generation.
 *   - Backward: from d out [batch, 24, frames] (generator) or d prob [batch, 6, frames/16] (discriminator), the network's kernel / bias /
 *     beta / gamma gradients are ADDED into its GRAD range and d in [batch, 24, frames] is written to din_dev (NULL = none).  It does not
 *     modify the tape: a tape can be back-propagated any number of times (each adds its gradients again).  cgvc_generator_backward_tape
 *     takes kinds 0 and 2; of a packed tape, d out and d in have the packed layout of cgvc_generator_forward_packed (utterance u is the
 *     [24][len_u] block at element 24 * offsets[u]), and every tap, instance norm and edge-layer sum stays inside its utterance, as in
 *     the forward.  The tape holds its own copy of the offsets: a later call that reuses WORK does not change what its backward reads.
 *   - Errors, all before anything is enqueued: a tape this engine did not write, one written before the parameters last changed or one
 *     of the other kind: CGVC_ERR_ARG.  A tape buffer smaller than cgvc_tape_bytes: CGVC_ERR_UNBOUND.  A backward on an engine without
 *     GRAD or without a training WORK arena (train = 0): CGVC_ERR_UNBOUND.
 *   - Scratch: the backward borrows the backward scratch of a train step at max_batch in WORK; WORK is not enlarged for it.
 *   - Loss scaling (F16F8): the upstream gradient is multiplied by the static loss scale of the tape's batch (of a packed tape: of a
 *     batch of n, its utterance count) before its gradient planes
 *     are formed and d in is returned with it removed (exact: a power of two); the GRAD contributions keep it (see cgvc_adam_step).
 *     With "loss_scale" = 1 the backward counts its saturated gradient-plane groups into the counters of cgvc_loss_scale_state (and the
 *     per-network ones: the generator's into index 0, the discriminator's into index 1), adding to them until the next train step clears
 *     them.  With "loss_scale" = 2 and "tape_loss_scale" = 0 (the default) tape calls use the static scale and are not counted.
 *   - "tape_loss_scale" = 1 (needs "loss_scale" = 2): the dynamic policy acts on tape calls.  The upstream gradient is multiplied by the
 *     scaler's current scale, read on the device: s_G for a generator tape and s_D for a discriminator tape with
 *     "loss_scale_per_network", else the one scale.  d in is returned with that scale removed, and the backward counts its gradient
 *     planes (per network: into that network's block) for cgvc_apply_gradients, which checks, skips or applies the step and is the only
 *     call that changes the scale, so that every tape backward between two of them uses one scale per network.  The first tape
 *     backward before any scale was set starts the scaler from the static scale of its tape's batch, as a first train step does.  A
 *     discriminator tape uses s_D also when back-propagated as part of a generator loss; its d in leaves unscaled, and the generator tape
 *     then applies s_G.  A saturation in that pass therefore halves s_D and skips the step, even if its discriminator gradients are
 *     discarded afterwards.  A train step in between discards the accumulation (it zeroes GRAD and the counters).
 *   - Options: "deterministic" makes repeated forward / backward sequences give the same GRAD bits; the kernel-choice options act as in a
 *     train step.  Tape calls run eagerly on `stream`, never as captured graphs.
 * Kind 3 = packed discriminator (cgvc_discriminator_forward_packed_tape): cgvc_tape_bytes(h, 3, n, rows, &bytes) as for kind 2, every length a
 * multiple of 16; cgvc_discriminator_backward_tape takes kinds 1 and 3, with d prob and d in in the packed layouts of
 * cgvc_discriminator_forward_packed, every tap and instance norm inside its utterance; the generator backward refuses kind 3.
 * Not covered: loss scales the caller passes per call; without "tape_loss_scale", data-parallel reduction (cgvc_allreduce_grads sums
 * GRAD over ranks; cgvc_apply_gradients all-reduces). */
int cgvc_tape_bytes(cgvc_handle h, int kind, int batch, int frames, size_t* bytes);
/* cgvc_discriminator_forward_packed with a kind 3 tape: the same argument checks and errors, all before anything is enqueued, then the
 * tape checks above; prob_dev bit for bit what cgvc_discriminator_forward_packed writes.  The offsets and the row prefix sums of the
 * network's levels are copied into the tape. */
int cgvc_discriminator_forward_packed_tape(cgvc_handle h, int which, const float* in_dev, float* prob_dev, const long long* offsets_host,
                                           int n, void* tape_dev, size_t tape_bytes, void* stream);
int cgvc_generator_forward_tape(cgvc_handle h, int direction, const float* in_dev, float* out_dev, int batch, int frames,
                                void* tape_dev, size_t tape_bytes, void* stream);
/* cgvc_generator_forward_packed with a kind 2 tape: the same argument checks and errors (all before anything is enqueued), then the
 * tape checks above; out_dev bit for bit what cgvc_generator_forward_packed writes.  The offsets are copied into the tape. */
int cgvc_generator_forward_packed_tape(cgvc_handle h, int direction, const float* in_dev, float* out_dev, const long long* offsets_host,
                                       int n, void* tape_dev, size_t tape_bytes, void* stream);
int cgvc_discriminator_forward_tape(cgvc_handle h, int which, const float* in_dev, float* prob_dev, int batch, int frames,
                                    void* tape_dev, size_t tape_bytes, void* stream);
int cgvc_generator_backward_tape(cgvc_handle h, const void* tape_dev, const float* dout_dev, float* din_dev, void* stream);
int cgvc_discriminator_backward_tape(cgvc_handle h, const void* tape_dev, const float* dprob_dev, float* din_dev, void* stream);

/* Debug/parity taps: copy a named layer-boundary activation of the most recent cgvc_generator_forward /
 * cgvc_discriminator_forward (channels-last, fp32) into out_dev.  The generator forward only keeps them when the option
 * "debug_taps" is 1 (default 0: the inference path writes neither fp32 layer outputs nor anything for a backward pass).  Names: h1_glu d1 d2 r1..r6 u1 u2 (generator),
 * h1_glu d1 d2 d3 (discriminator).  n_out receives the element count. */
int cgvc_debug_activation(cgvc_handle h, const char* name, float* out_dev, size_t capacity, size_t* n_out, void* stream);

/* Read-only view of the tensor-core weight store: the reduced-precision copies of PARAM in GEMM layout ("weight planes") that every
 * tensor-core GEMM reads instead of PARAM, rebuilt whenever PARAM changes (tests/test_gpu_weight_planes.py checks them against
 * tests/weight_planes_ref.py).  Layers are numbered in registration order, 0 .. n_layers - 1 (no layers: CGVC_PREC_FP32_SIMT).
 * Extents: *_k rounded up to 64, *_n and *_q to 128; Ntot = cout * (gated ? 2 : 1). */
typedef struct cgvc_weight_layer_info {
  int n_layers;                     /* layers in the store */
  int kh, kw, cin, cout, gated;     /* the registered shape: TF kernel [kh, kw, cin, cout] per branch */
  int shuffle;                      /* 2: the output goes through the pixel shuffler (forward rows then in the shuffle order) */
  int fold;                         /* > 0: a 1 x 1 layer whose cout columns are the (tap, channel) pairs of a [1, fold, cin, cout / fold] kernel */
  long long ka, kg, ba, bg;         /* PARAM offsets (elements) of kernel_a / kernel_g / bias_a / bias_g */
  int nt_n, cin_k, cin_n, nt_k, cin_q, nt_q;   /* padded extents of the planes below */
  int q_ok;                         /* the layer's shape has F16F8 planes (cin a multiple of 4) */
} cgvc_weight_layer_info;
/* cgvc_weight_planes: *info (may be NULL) receives layer `layer`'s registration; with `plane` non-NULL, *bytes_out the size of that
 * plane (padding included) and, when out_dev is non-NULL, a copy of it enqueued on `stream` (capacity: bytes at out_dev).  Planes:
 *   "wf_hi", "wf_lo"    bf16 [taps][nt_n][cin_k]   forward layout (row order: see tc_gemm.cu perm_row)
 *   "wd_hi", "wd_lo"    bf16 [taps][cin_n][nt_k]   data-gradient layout (gate branch at column offset cout)
 *   "wq16", "wq8hi", "wq8lo"      fp16 / e4m3 / e4m3 [taps][nt_n][cin_q]   F16F8, forward layout, weight-role scales
 *   "wdq16", "wdq8hi", "wdq8lo"   fp16 / e4m3 / e4m3 [taps][cin_n][nt_q]   F16F8, data-gradient layout (training engines)
 *   "bias"              fp32 [nt_n] in forward row order (zero for tap-folded layers)
 * A plane the engine does not keep is refused with CGVC_ERR_ARG: the F16F8 planes outside CGVC_PREC_F16F8, the F16F8 data-gradient
 * planes of a forward-only engine, and in CGVC_PREC_F16F8 the bf16 planes of a layer with F16F8 planes.  Launches no kernel; refused
 * while `stream` is capturing a graph. */
int cgvc_weight_planes(cgvc_handle h, int layer, cgvc_weight_layer_info* info, const char* plane, void* out_dev, size_t capacity,
                       size_t* bytes_out, void* stream);

/* -- device-resident training data (replaces the per-step host feed of train.py:90-107 / preprocess.py:207-238) ---------------
 * The caller uploads each speaker's normalised MCEP corpus once: utterance u as a row-major [num_features][len_u] block at element
 * num_features * offsets[u] of corpus_X_dev, offsets_X_dev = n_X + 1 frame prefix sums (int64).
 * cgvc_sample_plan draws one epoch: both utterance lists shuffled independently, truncated to num_pairs = min(n_A, n_B), one uniform
 * crop start per utterance, from a counter-based generator keyed by (seed, epoch) -- the exact contract is stated in
 * csrc/simt_kernels.cu and mirrored on the host by cgvc.preprocess.counter_sample_plan.  plan_dev = int[4][num_pairs]
 * (utt_A, start_A, utt_B, start_B); *err_dev becomes non-zero (utterance index + 1, bit 30 set for speaker B) if an utterance is
 * shorter than crop_frames (the reference asserts this, preprocess.py:217).
 * cgvc_gather_minibatch writes pairs [first_pair, first_pair + batch) as A_out / B_out [batch][num_features][crop_frames]. */
int cgvc_sample_plan(cgvc_handle h, const long long* offsets_A_dev, int n_A, const long long* offsets_B_dev, int n_B,
                     unsigned long long seed, long long epoch, int crop_frames, int* plan_dev, int* err_dev, void* stream);
int cgvc_gather_minibatch(cgvc_handle h, const float* corpus_A_dev, const long long* offsets_A_dev, const float* corpus_B_dev,
                          const long long* offsets_B_dev, const int* plan_dev, int num_pairs, int first_pair, int batch, int crop_frames,
                          float* A_out_dev, float* B_out_dev, void* stream);

/* -- multi-GPU (no counterpart in the reference, which is single-device: model.py:22) --------------------
 * One process per GPU.  Rank 0 obtains a 128-byte NCCL unique id, the host side distributes it, every rank
 * calls cgvc_comm_init; cgvc_train_step then does ONE fp32 sum-all-reduce of the GRAD arena per step. */
int cgvc_comm_unique_id(cgvc_handle h, void* id128_host);
int cgvc_comm_init(cgvc_handle h, const void* id128_host, int rank, int nranks);
int cgvc_comm_destroy(cgvc_handle h);
int cgvc_allreduce_grads(cgvc_handle h, void* stream);

/* -- measurement hooks (bench.py) ----------------------------------------------------------------------------
 * cgvc_kernel_launches: number of CUDA kernels this library has launched so far (process-wide).
 * cgvc_profile_enable(1) starts recording a CUDA-event pair around every tensor-core kernel launch;
 * cgvc_profile_collect synchronises and returns, per kernel class (arrays of 3: 0 = forward/data-gradient
 * gather-GEMM with the plain epilogue, 1 = weight-gradient gather-GEMM, 2 = forward gather-GEMM with the fused instance-norm
 * epilogue), the summed device time [ms], algorithmic FLOPs (2*M*N*K, counted once, whatever the bf16 split multiplies it by)
 * and launch count since the enable call. */
int cgvc_kernel_launches(unsigned long long* count);
/* options.  Every option belongs to its handle: it changes what that engine launches and no other engine's, and a call that changes
 * an option's value drops that handle's captured step graphs (the next step captures anew).  The options below that are flags take
 * any value, non-zero meaning 1; a value outside an option's range is refused with CGVC_ERR_ARG.
 * "two_streams" (default 1): run the two symmetric halves of a train step on two internal streams; 0 enqueues
 * everything on the caller's stream (used while per-kernel timings are taken).
 * "fuse_in" (default 1): instance norm + GLU / + residual fused into the forward conv kernel's epilogue where the shape
 * allows (generator layers whose 128-row tiles hold whole samples); 0 always uses the separate streaming kernels.
 * "fuse_bwd" (default 0): GLU / instance-norm backward of the generator's residual stack fused into the epilogue of the
 * data-gradient kernel that produces its upstream gradient (one kernel per layer backward instead of three); correct and tested, opt-in.
 * "side_wgrad" (default 0): the weight-gradient GEMMs of a train step run on a side stream per lane, off the critical path of the
 * data-gradient chain (needs two_streams; not combined with fuse_bwd).  Correct and tested.
 * "pipelined_comm" (default 1): with a communicator attached, cgvc_train_step all-reduces the gradients network by network on a
 * communication stream and runs Adam + the weight-plane refresh of each network as soon as its all-reduce is done (0: one all-reduce
 * of the whole arena, then Adam).
 * "fuse_c1" (default 1): the discriminator's input layer (one input channel, K = 9, gate without instance norm) as fused HBM-bound kernels:
 * forward = convolution + GLU in one pass (the pre-gate outputs are written for the backward pass but not read back by a second kernel),
 * backward = the GLU backward recomputed inside its weight-gradient / data-gradient kernels instead of a dP tensor written to and read
 * from HBM.
 * "edge_lower" (default 1): the generator's two 15-tap layers with 24 channels on one side (h1: 24 -> 2 x 128, o1: 256 -> 24;
 * module.py:85-86,148) as dense 1 x 1 GEMMs -- h1 over the im2col of the 24-channel input (K = 360), o1 with its taps folded into the
 * output columns (N = 360) followed by the tap-shifted sum; forward, data gradient and weight gradient.  0 = 15-tap gather-GEMMs with the
 * 24-channel side padded to a 64 / 128-channel line per tap (forward / data gradient on a 32-wide tile).
 * "wgrad_f16" (CGVC_PREC_F16F8 only, default 1): weight-gradient GEMMs from the fp16 planes alone, one MMA unit per product; every
 * gradient tensor stays within 3.6e-4 of the float64 oracle (tolerance 1e-3; 1.8e-4 with 0 = fp16 + two e4m3 cross terms, 2 units).
 * "prep_batched" (CGVC_PREC_F16F8 only, default 1): the fp16 + e4m3 weight planes of all layers (forward and data-gradient
 * layouts, biases) are rebuilt after Adam by ONE kernel that walks a job table in 32 x 64 tiles (one per network range in the pipelined
 * data-parallel schedule); 0 = three small kernels per layer branch (~210 launches per step).  Bit-identical planes.
 * "post_onepass" (default 1): GLU / instance-norm backward of samples with <= 64 positions in one kernel that keeps the
 * sample's rows in registers (reads dY and the pre-norm outputs once); 0 = always the sums + apply kernel pair.
 * "post_stream" (default 1): gated layers without pixel shuffle whose samples have 32, 48 or 64 positions take the streaming
 * form of the one-pass GLU / instance-norm backward: persistent CTAs walk (sample, channel block) items through a cp.async double buffer
 * in shared memory instead of holding a sample's rows in registers (needs post_onepass = 1).
 * "loss_scale" (default 0; 0, 1 or 2), "loss_scale_growth_interval" (default 2000; >= 1) and "loss_scale_per_network" (default 0): see
 * cgvc_loss_scale_state.  Switching "loss_scale_per_network" on while a dynamic scale is in use starts both networks from it.
 * "tape_loss_scale" (default 0): 1 puts the tape backward calls on the dynamic scaler (see the activation tapes and
 * cgvc_apply_gradients).  Setting it to 1 outside "loss_scale" = 2, or moving "loss_scale" away from 2 while it is 1: CGVC_ERR_ARG.
 * "deterministic" (default 0): 1 makes cgvc_train_step and cgvc_compute_gradients bitwise reproducible on one GPU.  The same inputs,
 * PARAM, ADAM_M / ADAM_V, Adam step, loss-scaler state, batch, frames, precision and options give the same bits of PARAM, GRAD, ADAM_M,
 * ADAM_V, the 8 losses, gen_A / gen_B and the scaler state, in every precision and loss_scale mode, on repeated calls and fresh
 * engines, and whatever "two_streams" and "cuda_graph" are.  Every kernel that adds into GRAD or a loss slot from many CTAs then stores
 * per-CTA partials to a slab in WORK and a second kernel adds them in a fixed order, one add per element (DESIGN.md section 11).
 * "fuse_bwd" and "side_wgrad" are ignored while it is on.  It enlarges WORK (cgvc_arena_bytes): bind the larger arena after setting
 * it, or the calls return CGVC_ERR_UNBOUND; cgvc_conv_backward and cgvc_in_glu_backward(_planes) honour it too and then need WORK
 * bound.  With a communicator attached each rank's gradients are deterministic; the NCCL all-reduce that sums them is not covered.
 * "debug_taps" (default 0): see cgvc_debug_activation.
 * "tc_debug" (default 0; 0 to 7): timing-experiment knobs of the tensor-core kernels (results become garbage): 1 = the
 * forward/data-gradient epilogue skips global stores, 2 = also skips the accumulator reads, 4 = the producers of every gather-GEMM,
 * the weight gradient's included, skip the activation loads.  The plain epilogue stores straight from the accumulator registers, so
 * for it 2 acts as 1. */
int cgvc_set_option(cgvc_handle h, const char* name, int value);
int cgvc_profile_enable(int on);
int cgvc_profile_collect(double* ms3, double* flops3, long long* launches3);
/* every recorded tensor-core launch in launch order: ms[i], flops[i], meta4[4i..4i+3] = (class, M rows, N columns,
 * K = taps * channels); *n_out = launches recorded (may exceed capacity; only `capacity` entries are written). */
int cgvc_profile_launches(double* ms, double* flops, long long* meta4, int capacity, int* n_out);

/* -- per-kernel entry points (unit parity against the oracle's primitives) -------------------------------
 * cgvc_conv_forward: channels-last TF-'SAME' cross-correlation (module.py:22-64), y = conv(x, w) + bias.
 *   x [B,H,W,Cin], w [kh,kw,Cin,Cout] (TF layout), y [B,Ho,Wo,Cout]; 1-D convs use H = kh = 1.
 *   precision: CGVC_PREC_*; shapes the tensor-core path cannot take fall back to CGVC_ERR_UNSUPPORTED. */
int cgvc_conv_forward(cgvc_handle h, int precision, const float* x, const float* w, const float* bias, float* y,
                      int B, int H, int W, int Cin, int kh, int kw, int Cout, int sh, int sw, void* stream);
/* gradients of the above: dx (may be NULL), dw and dbias are ACCUMULATED into (like the GRAD arena). */
int cgvc_conv_backward(cgvc_handle h, int precision, const float* x, const float* w, const float* dy,
                       float* dx, float* dw, float* dbias,
                       int B, int H, int W, int Cin, int kh, int kw, int Cout, int sh, int sw, void* stream);
/* fused instance-norm (+ optional pixel-shuffle view) + GLU (module.py:3-20,85-146):
 *   p [B, R/shuffle, 2*C*shuffle]: conv outputs, 'a' branch in columns [0,C*shuffle), gates after;
 *   y [B, R, C] = IN(a; beta_a, gamma_a) * sigmoid(IN(g; beta_g, gamma_g)); stats [B,4,C] = mean_a,rstd_a,mean_g,rstd_g */
int cgvc_in_glu_forward(cgvc_handle h, const float* p, const float* beta_a, const float* gamma_a,
                        const float* beta_g, const float* gamma_g, float* y, float* stats,
                        int B, int R, int C, int shuffle, void* stream);
int cgvc_in_glu_backward(cgvc_handle h, const float* dy, const float* p, const float* stats,
                         const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                         float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                         int B, int R, int C, int shuffle, void* stream);
/* The operand-plane writers of a train step, one call each, so that their planes and saturation counts can be checked against a
 * host reference (tests/f16f8_ref.py).  precision CGVC_PREC_BF16X3 or CGVC_PREC_BF16: bf16 planes hi = bf16(x), lo = bf16(x - hi);
 * CGVC_PREC_F16F8: hi = q16 = fp16(x), lo = q8hi followed by q8lo (e4m3 bytes, activation-role scales; kernels.cuh cgvc_quant4).
 * sat: a device counter the call ADDS the saturated 4-value groups of F16F8 planes to (kernels.cuh cgvc_sat4), or NULL.
 * cgvc_split_planes: x [rows, C] -> planes [rows, Cpad], Cpad = C rounded up to 64 (bf16) / 128 (F16F8), zero columns [C, Cpad):
 *   the input and output-gradient splits of the generator. */
int cgvc_split_planes(cgvc_handle h, int precision, const float* x, long long rows, int C, void* hi, void* lo,
                      unsigned long long* sat, void* stream);
/* cgvc_im2col_planes: the tap lowering of a stride-1 1-D TF-'SAME' convolution (option "edge_lower"): x [rows, C] holds rows / T
 *   samples of T positions; planes [rows, Cpad], Cpad = kw * C rounded up to 128, column t * C + c of row m = x[m + dir * (t - (kw-1)/2), c]
 *   when that row lies in the same sample, else 0.  dir = +1: the h1 input, -1: the o1 output gradient. */
int cgvc_im2col_planes(cgvc_handle h, int precision, const float* x, long long rows, int T, int C, int kw, int dir, void* hi, void* lo,
                       unsigned long long* sat, void* stream);
/* cgvc_set_plane_counters: ufl_groups_dev (device, 2 counters; NULL: none) receives, while it is set, what the F16F8 plane writers of
 *   cgvc_split_planes, cgvc_im2col_planes, cgvc_in_glu_*_planes, cgvc_glu_*_planes and cgvc_disc_input_forward add to the
 *   underflow counts of a train step with "loss_scale_per_network": [0] += groups below the fp16 lower edge, [1] += groups counted. */
int cgvc_set_plane_counters(cgvc_handle h, unsigned long long* ufl_groups_dev);
/* cgvc_in_glu_forward / _backward with the planes of y [B, R, C] / of dp (layout of p) written by the same kernels:
 *   precision CGVC_PREC_FP32_SIMT writes no planes (hi, lo, sat ignored: the two calls above);
 *   gate 1: the gated form above; gate 0: the residual block's h2 form, p [B, R/shuffle, C*shuffle], y = IN(a) (+ resid [B, R, C] if
 *   not NULL), beta_g / gamma_g / dbeta_g / dgamma_g unused. */
int cgvc_in_glu_forward_planes(cgvc_handle h, const float* p, const float* beta_a, const float* gamma_a,
                               const float* beta_g, const float* gamma_g, float* y, float* stats,
                               int B, int R, int C, int shuffle, int precision, int gate, const float* resid,
                               void* hi, void* lo, unsigned long long* sat, void* stream);
int cgvc_in_glu_backward_planes(cgvc_handle h, const float* dy, const float* p, const float* stats,
                                const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                                float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                                int B, int R, int C, int shuffle, int precision, int gate,
                                void* hi, void* lo, unsigned long long* sat, void* stream);
/* cgvc_in_glu_forward_planes over packed utterances, as cgvc_generator_forward_packed normalises them: p holds R / shuffle conv rows
 *   in all, of which utterance u owns [offsets[u] / div, offsets[u + 1] / div).  offsets (device): n_utt + 1 frame prefix sums, each
 *   length a multiple of 4; div = 1, 2 or 4 (P's level), a multiple of shuffle; max_len: the longest utterance in frames.  Each
 *   utterance is normalised over its own positions; stats is [n_utt, 4, C]. */
int cgvc_in_glu_forward_packed(cgvc_handle h, const float* p, const float* beta_a, const float* gamma_a,
                               const float* beta_g, const float* gamma_g, float* y, float* stats,
                               int R, int C, int shuffle, int precision, int gate, const float* resid,
                               const long long* offsets, int n_utt, int div, int max_len,
                               void* hi, void* lo, unsigned long long* sat, void* stream);
/* cgvc_in_glu_backward_planes that also accumulates the conv-bias gradients dbias_a, dbias_g [C * shuffle] (the column sums of dp, as
 *   the train step does; dbias_g needs dbias_a and is unused when gate is 0). */
int cgvc_in_glu_backward_bias(cgvc_handle h, const float* dy, const float* p, const float* stats,
                              const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                              float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                              float* dbias_a, float* dbias_g, int B, int R, int C, int shuffle, int precision, int gate,
                              void* hi, void* lo, unsigned long long* sat, void* stream);
/* One generator layer with its instance norm, as a train step or a conversion runs it, so that the fused gather-GEMM epilogues can be
 * checked against float64 and against the separate kernels.  precision CGVC_PREC_BF16X3, _BF16 or _F16F8 (planes as above).
 * fuse = 1: the instance norm runs in the GEMM epilogue where the shape allows (1-D layer, R = 32, 64 or 128 positions per sample);
 * fuse = 0, or a shape it refuses: the plain epilogue writes P and the instance-norm kernels follow.  *fused (may be NULL) tells which
 * ran.  Both paths take the same arguments and write the same outputs.
 * cgvc_conv_in_forward: the 1-D TF-'SAME' convolution of x [B, W, Cin] with stride sw, R = ceil(W / sw) positions per sample, then
 *   gated (w_g given): y = IN(a; beta_a, gamma_a) * sigmoid(IN(g; beta_g, gamma_g)), shuffle 1 or 2 (the pixel shuffle of the upsample
 *   blocks: IN over the shuffled view, module.py:115-146);
 *   residual (w_g NULL, shuffle 1): y = resid [B, R, Cout] + IN(a; beta_a, gamma_a).
 *   w_a / w_g [kw, Cin, Cout] and b_a / b_g [Cout] (TF layout).  Outputs, each NULL to skip: p [B, R, Ntot] the pre-norm convolution
 *   (a in columns [0, Cout), g after; Ntot = Cout or 2 Cout), stats [B, 4, C] (mean_a, rstd_a, mean_g, rstd_g; C = Cout / shuffle),
 *   y [B, R * shuffle, C] fp32; hi / lo, the planes of y, are required.  p = stats = NULL is the inference form.
 * cgvc_conv_in_backward: dY = dgrad(dp) (+ dx when accumulate) of a stride-1 1-D layer L (w_a / w_g [kw, Cin, Cout] as above, no bias),
 *   dp [B, R, Ntot] fp32; then the instance-norm backward of the upstream layer U whose output L read: bp [B, R, Cin or 2 Cin] its
 *   pre-norm output, stats [B, 4, Cin] its statistics.
 *   gate 1: U is gated (y = IN(a) * sigmoid(IN(g))); dx is only read (dY's accumulate term, or NULL).
 *   gate 0: U is the residual h2 form (y = resid + IN(a)); dx (+)= dgrad(dp), so that dx = dY, the skip gradient.
 *   hi / lo receive U's dP planes (layout of bp).  dbeta_a, dgamma_a (and dbeta_g, dgamma_g for gate 1): all NULL or all given, then
 *   accumulated.  Never fused in CGVC_PREC_F16F8 or with the option "deterministic" on (which also needs WORK bound, as
 *   cgvc_in_glu_backward). */
int cgvc_conv_in_forward(cgvc_handle h, int precision, const float* x, const float* w_a, const float* w_g, const float* b_a,
                         const float* b_g, const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                         const float* resid, float* p, float* stats, float* y, void* hi, void* lo,
                         int B, int W, int Cin, int kw, int Cout, int sw, int shuffle, int fuse, int* fused, void* stream);
int cgvc_conv_in_backward(cgvc_handle h, int precision, const float* dp, const float* w_a, const float* w_g, const float* bp,
                          const float* stats, const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                          float* dx, void* hi, void* lo, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                          int B, int R, int Cin, int kw, int Cout, int gate, int accumulate, int fuse, int* fused, void* stream);
/* The layers without an instance norm and the loss heads, as a train step runs them, so that they can be checked against float64
 * (tests/test_gpu_glu_layers.py).  Planes and sat as cgvc_split_planes; precision CGVC_PREC_FP32_SIMT writes no planes (hi, lo, sat
 * ignored).  The calls that add into their outputs from many CTAs honour the option "deterministic" (then WORK must be bound, as for
 * cgvc_in_glu_backward).
 * cgvc_glu_forward_planes: the gated form without instance norm (generator h1, discriminator h1): p [B, R, 2C] = [a | g],
 *   y [B, R, C] = a * sigmoid(g) (y may be NULL when hi / lo are given).  C a multiple of 4, B <= 65535.
 * cgvc_glu_backward_planes: dy [B, R, C], p as above -> dp [B, R, 2C] (= dy s(g), dy a s(g) (1 - s(g)); may be NULL when hi / lo are
 *   given) and its planes; dbias_a, dbias_g [C] (both NULL or both given) += the column sums of dp. */
int cgvc_glu_forward_planes(cgvc_handle h, const float* p, float* y, int B, int R, int C, int precision, void* hi, void* lo,
                            unsigned long long* sat, void* stream);
int cgvc_glu_backward_planes(cgvc_handle h, const float* dy, const float* p, float* dp, float* dbias_a, float* dbias_g, int B, int R, int C,
                             int precision, void* hi, void* lo, unsigned long long* sat, void* stream);
/* cgvc_disc_input_forward: the discriminator's input layer (one input channel, kh * kw <= 9 taps, Cout = 128, gate without instance norm;
 *   module.py:196-203): x [B, H, W], w_a / w_g [kh, kw, 1, Cout], b_a / b_g [Cout], strides sh, sw, M = B * ceil(H / sh) * ceil(W / sw)
 *   output rows.  p [M, 2 Cout] = [a | g] = conv(x) + bias (required: the backward pass reads it), y [M, Cout] = a * sigmoid(g) and
 *   its planes (y may be NULL when hi / lo are given).  fuse = 1: one pass (option "fuse_c1", the default); 0: the convolution, then
 *   the GLU kernels of cgvc_glu_forward_planes.  *fused (may be NULL) tells which ran.
 * cgvc_disc_input_backward: dy [M, Cout], the saved p, x and the weights -> dw_a, dw_g [kh, kw, 1, Cout], db_a, db_g [Cout] (all four
 *   NULL or all given, then accumulated) and dx [B, H, W] (NULL: no data gradient).  fuse = 1: dP is formed inside the weight-gradient
 *   and data-gradient kernels; 0: the GLU backward writes an fp32 dP that they read. */
int cgvc_disc_input_forward(cgvc_handle h, int precision, const float* x, const float* w_a, const float* w_g, const float* b_a, const float* b_g,
                            float* p, float* y, void* hi, void* lo, unsigned long long* sat,
                            int B, int H, int W, int kh, int kw, int Cout, int sh, int sw, int fuse, int* fused, void* stream);
int cgvc_disc_input_backward(cgvc_handle h, const float* dy, const float* p, const float* x, const float* w_a, const float* w_g,
                             float* dw_a, float* dw_g, float* db_a, float* db_g, float* dx,
                             int B, int H, int W, int kh, int kw, int Cout, int sh, int sw, int fuse, int* fused, void* stream);
/* cgvc_head_forward: the discriminator's dense head (module.py:211): prob[r] = sigmoid(y[r, :] . w + b[0]), y [rows, 1024].
 * cgvc_head_loss_backward: the LSGAN loss of those probabilities (model.py:68-69,81-86): *loss += coef * mean((prob - target)^2) (loss
 *   may be NULL); with dz = g coef 2 (prob - target) / rows * prob (1 - prob), g = *grad_mult (NULL: 1): dy [rows, 1024] = dz w (NULL:
 *   not written), dw [1024] += sum dz y, db [1] += sum dz (both NULL or both given; then y is required).
 * cgvc_l1_loss_grad: the L1 loss (utils.py:6-8): *loss += mean |yhat - y| over n elements (loss may be NULL); d[i] (+)= s sign(yhat[i] -
 *   y[i]) with s = (*gscale / n) * *grad_mult (a NULL pointer stands for 1), added to d when accumulate (d NULL: not written). */
int cgvc_head_forward(cgvc_handle h, const float* y, long long rows, const float* w, const float* b, float* prob, void* stream);
int cgvc_head_loss_backward(cgvc_handle h, const float* prob, const float* y, long long rows, const float* w, float target, float coef,
                            const float* grad_mult, float* loss, float* dy, float* dw, float* db, void* stream);
/* cgvc_head_backward: the same head from an upstream gradient dprob [rows] instead of the loss (cgvc_discriminator_backward_tape):
 *   dz = g dprob[r] prob[r] (1 - prob[r]), g = *grad_mult (NULL: 1); dy, dw, db as above. */
int cgvc_head_backward(cgvc_handle h, const float* prob, const float* y, long long rows, const float* w, const float* dprob,
                       const float* grad_mult, float* dy, float* dw, float* db, void* stream);
int cgvc_l1_loss_grad(cgvc_handle h, const float* yhat, const float* y, long long n, const float* gscale, const float* grad_mult, float* loss,
                      float* d, int accumulate, void* stream);
/* The generator's two 15-tap edge layers as the step runs them with option "edge_lower" (module.py:85-86 h1, module.py:148 o1): dense
 * 1 x 1 GEMMs over an im2col of the 24-channel side.  They act on the handle's generator `direction` (0 = A2B, 1 = B2A): weights
 * from PARAM through the planes cgvc_params_updated prepares, kernel and bias gradients accumulated into that generator's GRAD
 * ranges.  Rows are B samples of T positions, or for the forwards (offsets, host, not NULL) B packed utterances with the offsets
 * contract of cgvc_generator_forward_packed (T ignored).  F = 24 features, K = 15 taps; plane buffers hold [rows, 384] values in the
 * engine's precision (bf16 hi / lo; F16F8 fp16 hi, then lo = the two e4m3 planes one after the other).  CGVC_ERR_UNSUPPORTED when
 * the layers are not lowered (edge_lower 0, CGVC_PREC_FP32_SIMT, or before cgvc_params_updated).  The backward calls honour
 * "deterministic" (WORK bound).
 * cgvc_edge_h1_forward: x [rows, F] -> p [rows, 256] = [a | g] (the GEMM over im2col(x) [rows, K F], bias included), y [rows, 128]
 *   = a * sigmoid(g) and, when hi / lo are given, y's planes.
 * cgvc_edge_o1_forward: u [rows, 256] (its planes are written here) -> z [rows, K F] = u . W' with column t F + c the tap t product
 *   for output channel c (may be NULL), out [rows, F] = bias + sum_t z[r + t - 7, t F + c] over the rows of r's sample.
 * cgvc_edge_o1_backward: u, d_out [rows, F] -> GRAD o1 kernel += u^T dZ, bias += column sums of d_out; du [rows, 256] = dZ . W'^T;
 *   dZ [rows, K F] = d_out shifted by tap (dZ[r, t F + c] = d_out[r - t + 7, c] within the sample) as planes into dz_hi / dz_lo
 *   (both NULL: scratch).
 * cgvc_edge_h1_backward: x, p and dy [rows, 128] (d loss / d y) -> GRAD h1 a and g kernels += im2col(x)^T dP and biases += column
 *   sums of dP, dP [rows, 256] the GLU backward; dp = that dP (may be NULL), dz [rows, K F] = dP . W^T (may be NULL), dx [rows, F] =
 *   sum_t dz[r - t + 7, t F + c] within the sample (may be NULL). */
int cgvc_edge_h1_forward(cgvc_handle h, int direction, const float* x, int B, int T, const long long* offsets, float* p, float* y,
                         void* hi, void* lo, void* stream);
int cgvc_edge_o1_forward(cgvc_handle h, int direction, const float* u, int B, int T, const long long* offsets, float* z, float* out,
                         void* stream);
int cgvc_edge_o1_backward(cgvc_handle h, int direction, const float* u, const float* d_out, int B, int T, float* du, void* dz_hi,
                          void* dz_lo, void* stream);
int cgvc_edge_h1_backward(cgvc_handle h, int direction, const float* x, const float* p, const float* dy, int B, int T, float* dp, float* dz,
                          float* dx, void* stream);

/* error codes */
enum {
  CGVC_OK = 0,
  CGVC_ERR_ARG = -1,
  CGVC_ERR_CUDA = -2,
  CGVC_ERR_UNBOUND = -3,      /* an arena needed by the call is not bound / too small */
  CGVC_ERR_DIRECTION = -4,    /* model.py:135 */
  CGVC_ERR_UNSUPPORTED = -5,
  CGVC_ERR_NCCL = -6
};

#ifdef __cplusplus
}
#endif
#endif /* CGVC_H */
