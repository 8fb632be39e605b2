// libcgvc.so engine: parameter table, workspace planner, forward/backward schedules and the C ABI.
//
// Replaces the TensorFlow-1 session behind CycleGAN.train/test (model.py:110-137 of /root/reference):
// the graph wiring below follows model.py:44-90, the network shapes module.py:148-213.
#include "../../include/cgvc.h"
#include "kernels.cuh"
#include "tc_gemm.cuh"
#include "geom.h"

#include <atomic>
#include <dlfcn.h>
#include <limits.h>
#include <stddef.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <utility>
#include <vector>

static thread_local std::string g_create_error;

#define ADAM_B1 0.5f        // model.py:107-108
#define ADAM_B2 0.999f
#define ADAM_EPS 1e-8f

// ---------------------------------------------------------------------------------------------------
// parameter table (TF variable names / creation order; SURVEY.md Appendix A.4, A.5)
// ---------------------------------------------------------------------------------------------------
struct TensorInfo { std::string name; size_t off; int ndim; int shape[4]; size_t numel; };
struct ConvW { size_t k, b; int kh, kw, cin, cout; };
struct InW { size_t beta, gamma; int c; };
// One layer: convolution a, in the gated layers beside convolution g over the same input (P = [a | g]), then optionally instance
// norm (of each branch), the GLU of the two branches and the pixel shuffle.  The residual blocks' h2 is a layer without gate whose
// normalised output is added to the block input.
struct Layer {
  ConvW a, g; InW ina, ing; int has_in; int sh, sw; int shuffle; int tc_slot = -1;
  bool gated() const { return g.cout != 0; }
  int width() const { return gated() ? 2 * a.cout : a.cout; }       // columns of P
};
struct ResBlock { Layer h1, h2; };
struct GenNet { Layer h1; Layer d[2]; ResBlock r[6]; Layer u[2]; Layer o1; size_t begin, end;
                int h1c_slot = -1, o1f_slot = -1; };      // the tap-lowered forms of the two 15-tap edge layers (`edge_lower`, see edge_on)
struct DiscNet { Layer h1; Layer d[3]; size_t dense_k, dense_b; size_t begin, end; };

// per-layer activations kept for backward: pre-norm conv output, instance-norm statistics, output (fp32 and operand planes)
struct GLAct { float* P; float* stats; float* Y; __nv_bfloat16 *Yhi, *Ylo; };
struct GenActs {
  int n, T;
  const long long* off;         // packed utterances (cgvc_generator_forward_packed): n + 1 device frame prefix sums, else null
  long long rows;               // rows at full resolution: n * T, or off[n]
  int max_len;                  // packed: the longest utterance
  const float* x_cl; __nv_bfloat16 *xhi, *xlo;
  __nv_bfloat16 *xchi, *xclo;   // im2col of the input over h1's taps: operand planes [n*T, ru128(kw*F)] (edge_lower)
  float* z;                     // o1's per-tap products [n*T, kw*F] before the tap-shifted sum (edge_lower)
  GLAct h1, d[2];
  struct { GLAct h1, h2; } r[6];
  GLAct u[2];
  float* out_cl;
  float* post;                  // scratch for the instance-norm sums [n,4,1024]
};
struct DiscActs {
  int n, T; const float* x; GLAct h1, d[3]; float* prob; float* post;
  // packed utterances (cgvc_discriminator_forward_packed): n + 1 device frame prefix sums, else null; then every level is a packed 2-D
  // grid (kernels.cuh PackGeom2) and seg[i] holds the n + 1 row prefix sums of d[i]'s output grid (its instance-norm segments)
  const long long* off; const long long* seg[3];
  long long rows;               // frames in all: n * T, or off[n]
  int max_len;                  // packed: the longest utterance
};

struct GraphKey {
  int batch, frames, id_off, kind;
  bool operator<(const GraphKey& o) const { return memcmp(this, &o, sizeof(GraphKey)) < 0; }
};
struct GraphEntry { cudaGraphExec_t exec; unsigned long long launches; };

// What one network application (a forward of the C ABI, or an activation tape) runs over.  kind 0: the generator over n samples of
// T frames; 1: the discriminator likewise; 2: the generator over n packed utterances (T = 0); 3: the discriminator over n packed
// utterances (T = 0).  which: the generator's direction, or the discriminator
struct NetGeom {
  int kind, which, n, T;
  long long rows;               // rows at full resolution: n * T, or (kinds 2, 3) offsets[n]
  int max_len;                  // kinds 2, 3: the longest utterance
};
static bool packed_kind(int kind) { return kind == 2 || kind == 3; }
static bool disc_kind(int kind) { return kind == 1 || kind == 3; }
static NetGeom net_geom(int kind, int which, int n, int T) { return NetGeom{kind, which, n, T, (long long)n * T, 0}; }

// The header at the start of an activation tape (cgvc_*_forward_tape), also kept by the engine that wrote it, keyed by the tape's
// address: a backward call checks its tape against that copy, so that it needs no device-to-host read before it enqueues anything
struct TapeHeader {
  unsigned long long magic;     // kTapeMagic
  unsigned long long engine;    // cgvc_engine::id of the writer
  unsigned long long gen;       // cgvc_engine::param_gen when it was written
  NetGeom geom;                 // what the forward applied the network to
};
static const unsigned long long kTapeMagic = 0x45504154435647ull;   // "GVCTAPE"
static const size_t kTapeHead = 256;                                // the activations start 256 bytes in
static std::atomic<unsigned long long> g_engine_ids{0};

struct Bump {
  char* base = nullptr; size_t cap = 0, off = 0; bool overflow = false;
  void reset(void* b, size_t c) { base = (char*)b; cap = c; off = 0; overflow = false; }
  template <class T> T* take(size_t n) {
    size_t bytes = (n * sizeof(T) + 255) & ~(size_t)255;
    if (off + bytes > cap) { overflow = true; off += bytes; return (T*)base; }
    T* p = (T*)(base + off); off += bytes; return p;
  }
};

// NCCL through dlopen: no link-time dependency, single-GPU use never touches it.
struct Id128 { char b[128]; };   // ncclUniqueId (passed by value)
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, Id128, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};

// Weight-gradient launches leave the critical path: a layer's backward is  (GLU / instance-norm backward -> dP planes) -> {weight gradient,
// data gradient}, and only the data gradient feeds the next layer.  With `on`, the weight-gradient GEMMs are enqueued on a side stream
// (a side branch of the captured graph) behind an event on their dP planes, so the tensor cores have them to run while the main chain
// is in its elementwise kernels.  The dP planes ping-pong between two buffers; a buffer is rewritten only after the weight gradient that
// read it has finished (`done`).
struct SideQ {
  cudaStream_t side = nullptr;
  cudaEvent_t ready[2] = {nullptr, nullptr}, done[2] = {nullptr, nullptr};
  bool used[2] = {false, false};
  int cur = 0;
  bool on = false;
};

// The engine's options (cgvc_set_option, include/cgvc.h) with their defaults.  Those that only the tensor-core module reads
// (wgrad_f16, prep_batched, tc_debug) live in TcWeights.
struct Options {
  int fuse_in = 1;              // fuse instance norm (+GLU / +residual) into the forward GEMM epilogue where the shape allows
  int fuse_bwd = 0;             // fuse the instance-norm (+GLU) backward into the upstream data-gradient GEMM's epilogue likewise.
                                // Off by default: unlike the streaming kernels, that epilogue work cannot overlap the other lane's
                                // tensor-core kernels
  int edge_lower = 1;           // the generator's 15-tap, 24-channel edge layers as dense 1 x 1 GEMMs (taps moved into the channel / column dimension)
  int side_wgrad = 0;           // weight-gradient GEMMs on a side stream per lane (see SideQ); needs two_streams, excludes fuse_bwd.  Off by default
  int fuse_c1 = 1;              // discriminator input layer backward: GLU backward fused into its weight / data gradient kernels
  int two_streams = 1;          // 0: both lanes are enqueued on the caller's stream (clean per-kernel timing for profiling)
  int pipelined_comm = 1;       // data parallel: all-reduce, Adam and plane refresh network by network (see comm_stream)
  int deterministic = 0;        // bit-reproducible steps: fixed-order reductions into GRAD and the loss slots (DESIGN.md section 11);
                                // ignores fuse_bwd and side_wgrad
  int debug_taps = 0;           // cgvc_generator_forward also writes the fp32 copy of every layer output (cgvc_debug_activation)
  int use_graphs = 1;           // "cuda_graph": replay the step as a CUDA graph (turned off when a capture fails)
  int ls_mode = 0;              // "loss_scale": 0 static, 1 monitor (static scale, counters collected), 2 dynamic
  int ls_growth = 2000;         // "loss_scale_growth_interval"
  int ls_nets = 0;              // "loss_scale_per_network": one scale for the generators' passes, one for the discriminators' D-loss pass
  int tape_ls = 0;              // "tape_loss_scale" (needs ls_mode 2): tape backwards scale by the scaler and count; cgvc_apply_gradients
  PostForms post = {1, 1};      // "post_onepass", "post_stream": the forms the instance-norm kernels may take (kernels.cuh)
};

struct cgvc_engine {
  cgvc_config cfg;
  Options opt;
  std::string err;
  std::vector<TensorInfo> tensors;
  size_t n_params = 0;        // arena length in elements (tensors padded to 16-byte boundaries)
  size_t n_real_params = 0;   // 119,787,058 trainable scalars
  GenNet gen[2];     // 0 = generator_A2B, 1 = generator_B2A
  DiscNet disc[2];   // 0 = discriminator_A, 1 = discriminator_B
  void* arena[CGVC_ARENA_COUNT] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t arena_bytes[CGVC_ARENA_COUNT] = {0, 0, 0, 0, 0};
  long long adam_t = 0;
  // small device buffers owned by the engine
  float* d_scalars = nullptr;   // [0..1] lambdas, [2..3] adam hyper G (lr_t, gscale), [4..5] adam hyper D, [8..15] losses
  // tensor-core weight planes (owned; derived from PARAM)
  TcWeights tcw;
  // communicator
  NcclApi nccl; void* comm = nullptr; int rank = 0, nranks = 1;
  // the two lanes of a training step run on their own streams (forked from / joined into the caller's stream)
  cudaStream_t lane_stream[2] = {nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  std::map<GraphKey, GraphEntry> graphs;
  float* stage = nullptr;       // [2][max_batch,num_features,max_frames]: fixed-address copies of the step's inputs for the graphs
  cudaStream_t graph_stream = nullptr; cudaEvent_t ev_bridge = nullptr, ev_bridge2 = nullptr;
  // data-parallel step: the gradient all-reduce runs per network on its own stream; Adam and the weight-plane refresh of a network
  // start as soon as its all-reduce has finished, while the next network's is still on the wire
  cudaStream_t comm_stream = nullptr; cudaEvent_t ev_grads = nullptr, ev_ar[4] = {nullptr, nullptr, nullptr, nullptr};
  SideQ sideq[2];
  // loss scaling (opt.ls_mode).  ls: the device state; d_scalars[16 + l] holds the static scale of batches [2^l, 2^(l+1)) (loss_scale),
  // so that the loss kernels always read a pointer
  LossScaler* ls = nullptr;
  bool ls_ready = false;        // dynamic mode: ls->scale holds a scale (set on the first step from the static one, or by the caller)
  int ls_batch = 0;             // monitor mode: the batch whose static scale ls->scale reports
  bool counting = false;        // a train step is being enqueued: the plane writers count saturation (ls_mode != 0, F16F8)
  int ls_net = 0;               // per-network loss scale: the network whose pass is being enqueued (0 generators, 1 discriminators);
                                // it picks the scale of the loss gradients and the counter block of the gradient-plane writers
  unsigned long long* plane_ufl = nullptr;   // cgvc_set_plane_counters: [ufl, groups] the per-kernel plane entry points add into
  cudaEvent_t ev_ls = nullptr;  // data parallel: the saturation all-reduce and the GRAD check are done (comm stream)
  bool tape_open = false;       // "tape_loss_scale": the counters of the gradients accumulating for cgvc_apply_gradients were cleared
  // debug taps of the last forward
  std::map<std::string, std::pair<const float*, size_t>> taps;
  // the instance-norm sums scratch of the calls outside a train step (which has its WORK slices): conversions, cgvc_in_glu_*
  float* post_buf = nullptr; size_t post_elems = 0;
  // activation tapes: this engine's id, the parameter generation (advanced whenever PARAM may have changed: cgvc_params_updated,
  // cgvc_bind_arena, every Adam update) and the headers of the tapes written since the parameters last changed
  unsigned long long id = 0, param_gen = 0;
  std::map<const void*, TapeHeader> tapes;

  float* P() const { return (float*)arena[CGVC_ARENA_PARAM]; }
  float* G() const { return (float*)arena[CGVC_ARENA_GRAD]; }
};

static int fail(cgvc_engine* e, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
  if (e) e->err = buf; else g_create_error = buf;
  return code;
}

#define CK(call)                                                                                   \
  do { cudaError_t _e = (call);                                                                    \
       if (_e != cudaSuccess) return fail(e, CGVC_ERR_CUDA, "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); } while (0)
#define RET(call) do { int _r = (call); if (_r != 0) return _r; } while (0)

// Captured step graphs hold the kernels, options and addresses of the moment they were captured: dropped whenever one of those changes
static void drop_graphs(cgvc_engine* e) {
  for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second.exec);
  e->graphs.clear();
}

// e->post_buf with room for `elems` floats (on the engine's device: called under its DeviceGuard)
static cudaError_t grow_post_buf(cgvc_engine* e, size_t elems, float** out) {
  if (elems > e->post_elems) {
    cudaFree(e->post_buf);
    const size_t want = elems < (size_t)(1 << 22) ? (size_t)(1 << 22) : elems * 2;
    cudaError_t ce = cudaMalloc(&e->post_buf, want * sizeof(float));
    if (ce != cudaSuccess) { e->post_buf = nullptr; e->post_elems = 0; return ce; }
    e->post_elems = want;
  }
  *out = e->post_buf;
  return cudaSuccess;
}

// Every entry point runs on the engine's device and leaves the caller's current device as it found it (a single process may
// drive several GPUs through torch, whose current device must not change behind its back).
struct DeviceGuard {
  int prev = -1;
  cudaError_t set(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev == dev) { prev = -1; return cudaSuccess; }
    return cudaSetDevice(dev);
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// ---- table construction ------------------------------------------------------------------------------
struct TableBuilder {
  std::vector<TensorInfo>& t; size_t off = 0; std::string scope;
  size_t real = 0;
  size_t add(const std::string& name, std::initializer_list<int> shp) {
    off = (off + 3) & ~(size_t)3;     // every tensor starts 16-byte aligned (float4 / red.v4 / cp.async paths rely on it)
    TensorInfo ti; ti.name = scope + "/" + name; ti.off = off; ti.ndim = (int)shp.size(); ti.numel = 1;
    int i = 0; for (int s : shp) { ti.shape[i++] = s; ti.numel *= (size_t)s; }
    for (; i < 4; ++i) ti.shape[i] = 1;
    t.push_back(ti); off += ti.numel; real += ti.numel; return ti.off;
  }
  ConvW conv1d(const std::string& name, int k, int cin, int cout) {
    ConvW c; c.kh = 1; c.kw = k; c.cin = cin; c.cout = cout;
    c.k = add(name + "/kernel", {k, cin, cout}); c.b = add(name + "/bias", {cout}); return c;
  }
  ConvW conv2d(const std::string& name, int kh, int kw, int cin, int cout) {
    ConvW c; c.kh = kh; c.kw = kw; c.cin = cin; c.cout = cout;
    c.k = add(name + "/kernel", {kh, kw, cin, cout}); c.b = add(name + "/bias", {cout}); return c;
  }
  InW inorm(int idx, int c) {
    std::string n = idx == 0 ? "InstanceNorm" : "InstanceNorm_" + std::to_string(idx);
    InW w; w.c = c; w.beta = add(n + "/beta", {c}); w.gamma = add(n + "/gamma", {c}); return w;
  }
};

static void build_generator(TableBuilder& tb, GenNet& g, int nf) {
  g.begin = tb.off;
  g.h1 = Layer{}; g.h1.a = tb.conv1d("h1_conv", 15, nf, 128); g.h1.g = tb.conv1d("h1_conv_gates", 15, nf, 128);
  g.h1.has_in = 0; g.h1.sh = 1; g.h1.sw = 1; g.h1.shuffle = 1;
  int idx = 0, cin = 128;
  const int dco[2] = {256, 512};
  for (int i = 0; i < 2; ++i) {
    std::string p = "downsample1d_block" + std::to_string(i + 1) + "_";
    Layer& L = g.d[i]; L = Layer{};
    L.a = tb.conv1d(p + "h1_conv", 5, cin, dco[i]); L.ina = tb.inorm(idx++, dco[i]);
    L.g = tb.conv1d(p + "h1_gates", 5, cin, dco[i]); L.ing = tb.inorm(idx++, dco[i]);
    L.has_in = 1; L.sh = 1; L.sw = 2; L.shuffle = 1; cin = dco[i];
  }
  for (int i = 0; i < 6; ++i) {
    std::string p = "residual1d_block" + std::to_string(i + 1) + "_";
    ResBlock& R = g.r[i]; R = ResBlock{};
    R.h1.a = tb.conv1d(p + "h1_conv", 3, 512, 1024); R.h1.ina = tb.inorm(idx++, 1024);
    R.h1.g = tb.conv1d(p + "h1_gates", 3, 512, 1024); R.h1.ing = tb.inorm(idx++, 1024);
    R.h1.has_in = 1; R.h1.sh = 1; R.h1.sw = 1; R.h1.shuffle = 1;
    R.h2.a = tb.conv1d(p + "h2_conv", 3, 1024, 512); R.h2.ina = tb.inorm(idx++, 512);
    R.h2.has_in = 1; R.h2.sh = 1; R.h2.sw = 1; R.h2.shuffle = 1;
  }
  cin = 512;
  const int uco[2] = {1024, 512};
  for (int i = 0; i < 2; ++i) {
    std::string p = "upsample1d_block" + std::to_string(i + 1) + "_";
    Layer& L = g.u[i]; L = Layer{};
    L.a = tb.conv1d(p + "h1_conv", 5, cin, uco[i]); L.ina = tb.inorm(idx++, uco[i] / 2);
    L.g = tb.conv1d(p + "h1_gates", 5, cin, uco[i]); L.ing = tb.inorm(idx++, uco[i] / 2);
    L.has_in = 1; L.sh = 1; L.sw = 1; L.shuffle = 2; cin = uco[i] / 2;
  }
  g.o1 = Layer{}; g.o1.a = tb.conv1d("o1_conv", 15, 256, nf);
  g.o1.has_in = 0; g.o1.sh = 1; g.o1.sw = 1; g.o1.shuffle = 1;
  g.end = tb.off;
}

static void build_discriminator(TableBuilder& tb, DiscNet& d) {
  d.begin = tb.off;
  d.h1 = Layer{}; d.h1.a = tb.conv2d("h1_conv", 3, 3, 1, 128); d.h1.g = tb.conv2d("h1_conv_gates", 3, 3, 1, 128);
  d.h1.has_in = 0; d.h1.sh = 1; d.h1.sw = 2; d.h1.shuffle = 1;
  int idx = 0, cin = 128;
  const int kh[3] = {3, 3, 6}, co[3] = {256, 512, 1024}, sh[3] = {2, 2, 1};
  for (int i = 0; i < 3; ++i) {
    std::string p = "downsample2d_block" + std::to_string(i + 1) + "_";
    Layer& L = d.d[i]; L = Layer{};
    L.a = tb.conv2d(p + "h1_conv", kh[i], 3, cin, co[i]); L.ina = tb.inorm(idx++, co[i]);
    L.g = tb.conv2d(p + "h1_gates", kh[i], 3, cin, co[i]); L.ing = tb.inorm(idx++, co[i]);
    L.has_in = 1; L.sh = sh[i]; L.sw = 2; L.shuffle = 1; cin = co[i];
  }
  d.dense_k = tb.add("dense/kernel", {1024, 1}); d.dense_b = tb.add("dense/bias", {1});
  d.end = tb.off;
}

// ---- conv building blocks (dispatch: tensor cores where the layer is registered, else fp32 SIMT) ---------------------
struct ConvIO {               // one convolution application
  const float* x; const __nv_bfloat16 *xhi, *xlo;   // input [n,H,W,Cin] fp32 (may be null on the tensor-core path) + bf16 planes
  int n, H, W;
  PackGeom pk{};              // packed utterances (pk.off != null): n = H = 1, W = rows at the level of divisor pk.div; or with H > 1
                              // packed 2-D grids (kernels.cuh PackGeom2): n = 1, W = all frames / pk.div
  const long long* seg_out{}; // packed 2-D grids: the n + 1 row prefix sums of the layer's output grid (instance-norm segments)
};
static const PackGeom* packed(const ConvIO& io) { return io.pk.off ? &io.pk : nullptr; }

struct PlanePair { __nv_bfloat16 *hi, *lo; };

static int conv_out_dims(const ConvW& c, int sh, int sw, int H, int W, int& Ho, int& Wo) {
  int p; same_pad(H, c.kh, sh, p, Ho); same_pad(W, c.kw, sw, p, Wo); return 0;
}

// y[., coff:coff+cout] = conv(x, w) + b  into a row-major [rows, ld] buffer
static int conv_fwd_simt(cgvc_engine* e, const float* w, const float* bias, const ConvW& c, int sh, int sw, const ConvIO& io,
                         float* dst, int ld, int coff, cudaStream_t st) {
  if (!io.x) return fail(e, CGVC_ERR_UNSUPPORTED, "fp32 activations were not kept for a layer that fell back to the SIMT path");
  GatherGeom g = fwd_geom(io.n, io.H, io.W, c.kh, c.kw, sh, sw);
  GemmOperands op; memset(&op, 0, sizeof op);
  op.src = io.x; op.s_ld = c.cin; op.s_coff = 0; op.C = c.cin;
  op.w = w; op.w_ts = (long long)c.cin * c.cout; op.w_cs = c.cout; op.w_ns = 1; op.N = c.cout;
  op.dst = dst; op.d_ld = ld; op.d_coff = coff; op.bias = bias; op.accumulate = 0;
  if (io.pk.off) CK(launch_gg_simt_packed(g, op, io.pk, st));
  else CK(launch_gg_simt(g, op, st));
  return 0;
}

// dx (+)= dgrad(dy[., coff:coff+cout], w)
// pk: packed utterances (n = H = 1, pk->div the input level's divisor): every parity class reads dy at the output level, of divisor
// pk->div * sw (DESIGN.md section 12)
static int conv_dgrad_simt(cgvc_engine* e, const float* w, const ConvW& c, int sh, int sw, int n, int H, int W,
                           const float* dy, int ld, int coff, float* dx, int accumulate, cudaStream_t st, const PackGeom* pk = nullptr) {
  if (!dy) return fail(e, CGVC_ERR_UNSUPPORTED, "fp32 gradients were not kept for a layer that fell back to the SIMT path");
  std::vector<GatherGeom> gs = dgrad_geoms(n, H, W, c.kh, c.kw, sh, sw);
  for (const GatherGeom& g : gs) {
    GemmOperands op; memset(&op, 0, sizeof op);
    op.src = dy; op.s_ld = ld; op.s_coff = coff; op.C = c.cout;
    op.w = w; op.w_ts = (long long)c.cin * c.cout; op.w_cs = 1; op.w_ns = c.cout; op.N = c.cin;
    op.dst = dx; op.d_ld = c.cin; op.d_coff = 0; op.bias = nullptr; op.accumulate = accumulate;
    if (pk) { PackGeom q = *pk; q.div = pk->div * sw; CK(launch_gg_simt_packed(g, op, q, st)); }
    else CK(launch_gg_simt(g, op, st));
  }
  return 0;
}

// dW += x^T * dy (forward geometry); the bias gradient comes from the IN/GLU backward kernel (or launch_colsum for o1)
static int conv_wgrad_simt(cgvc_engine* e, float* dw, const ConvW& c, int sh, int sw, const ConvIO& io,
                           const float* dy, int ld, int coff, cudaStream_t st, const DetSlab* det) {
  if (!io.x || !dy) return fail(e, CGVC_ERR_UNSUPPORTED, "fp32 tensors were not kept for a layer that fell back to the SIMT path");
  GatherGeom g = fwd_geom(io.n, io.H, io.W, c.kh, c.kw, sh, sw);
  CK(launch_wgrad_simt(g, io.x, c.cin, 0, c.cin, dy, ld, coff, c.cout, dw, (long long)c.cin * c.cout, c.cout, 1, st, det != nullptr, packed(io)));
  return 0;
}

// Loss scale of the F16F8 gradient planes (DESIGN.md section 10): gradients shrink as 1 / batch, and their fp16 + e4m3 planes have a
// window of about 8 binades in which the result does not depend on the scale; 2^(9 + floor(log2(batch))) sits in its middle
// (2^10 at batch 2 ... 2^17 at batch 256).  Applied where the loss gradients are formed, removed by Adam's grad_scale.  1 otherwise.
static float loss_scale(const cgvc_engine* e, int batch) {
  if (e->cfg.precision != CGVC_PREC_F16F8) return 1.f;
  int l = 0; while ((2 << l) <= batch && l < 9) ++l;       // floor(log2(batch)), capped
  return ldexpf(1.f, 9 + l);
}
// option "loss_scale_per_network" in effect: it applies in loss_scale modes 1 and 2, and only F16F8 has a scale other than 1
static bool ls_nets(const cgvc_engine* e) { return e->opt.ls_nets && e->opt.ls_mode && e->cfg.precision == CGVC_PREC_F16F8; }
// the device copy of loss_scale(e, batch): d_scalars[16 + floor(log2 batch)], written at creation
static const float* static_scale_dev(const cgvc_engine* e, int batch) {
  int l = 0; while ((2 << l) <= batch && l < 9) ++l;
  return e->d_scalars + 16 + l;
}
// ... or in dynamic mode the scaler's current scale (per network: that of the pass being enqueued, e->ls_net): what the loss-gradient
// kernels multiply by
static const float* loss_scale_dev(const cgvc_engine* e, int batch) {
  if (e->opt.ls_mode == 2) return ls_nets(e) ? &e->ls->net[e->ls_net].scale : &e->ls->scale;
  return static_scale_dev(e, batch);
}
// saturation counters of the plane writers (null: not counted): only F16F8 has reduced-range planes, only train steps are counted.
// Per network, the gradient planes count into the block of the pass being enqueued, which also takes their underflow counts
static unsigned long long* sat_grad(const cgvc_engine* e) {
  if (!(e->counting && e->opt.ls_mode && e->cfg.precision == CGVC_PREC_F16F8)) return nullptr;
  return ls_nets(e) ? e->ls->cnt[e->ls_net] : &e->ls->sat_grad;
}
static unsigned long long* ufl_grad(const cgvc_engine* e) {
  return e->counting && ls_nets(e) ? e->ls->cnt[e->ls_net] + 1 : nullptr;
}
static unsigned long long* sat_act(const cgvc_engine* e) {
  return e->counting && e->opt.ls_mode && e->cfg.precision == CGVC_PREC_F16F8 ? &e->ls->sat_act : nullptr;
}

static bool tc_enabled(const cgvc_engine* e) { return e->cfg.precision != CGVC_PREC_FP32_SIMT && e->tcw.ready; }
static bool use_tc(const cgvc_engine* e, int slot) { return slot >= 0 && tc_enabled(e); }

// One layer's tensors by pointer, so that the train step, the conversions, the tapes and the test entry points run the same launches:
// kernels, biases and instance-norm affine parameters of branches a and g (null where the layer has none), their gradients (null: no
// gradient), and the tensor-core layer whose planes the convolutions read (null: the fp32 SIMT path) with the precision and the store
// options (TcWeights::debug, TcWeights::wgrad16) it runs with
struct LayerTensors {
  const float *ka, *kg, *ba, *bg, *beta_a, *gamma_a, *beta_g, *gamma_g;
  float *dka, *dkg, *dba, *dbg, *dbeta_a, *dgamma_a, *dbeta_g, *dgamma_g;
  const TcLayer* tc;
  int precision, debug, wgrad16;
};

// ... of registered layer L: PARAM, with grads GRAD, and the engine's tensor-core store
static LayerTensors layer_tensors(const cgvc_engine* e, const Layer& L, bool grads) {
  LayerTensors t; memset(&t, 0, sizeof t);
  const float* Pm = e->P();
  t.ka = Pm + L.a.k; t.ba = Pm + L.a.b;
  if (L.gated()) { t.kg = Pm + L.g.k; t.bg = Pm + L.g.b; }
  if (L.has_in) { t.beta_a = Pm + L.ina.beta; t.gamma_a = Pm + L.ina.gamma; }
  if (L.has_in && L.gated()) { t.beta_g = Pm + L.ing.beta; t.gamma_g = Pm + L.ing.gamma; }
  if (grads) {
    float* Gm = e->G();
    t.dka = Gm + L.a.k; t.dba = Gm + L.a.b;
    if (L.gated()) { t.dkg = Gm + L.g.k; t.dbg = Gm + L.g.b; }
    if (L.has_in) { t.dbeta_a = Gm + L.ina.beta; t.dgamma_a = Gm + L.ina.gamma; }
    if (L.has_in && L.gated()) { t.dbeta_g = Gm + L.ing.beta; t.dgamma_g = Gm + L.ing.gamma; }
  }
  t.tc = use_tc(e, L.tc_slot) ? &e->tcw.layers[L.tc_slot] : nullptr;
  t.precision = e->cfg.precision; t.debug = e->tcw.debug; t.wgrad16 = e->tcw.wgrad16;
  return t;
}

// How a tensor-core call on layer c ended: done (*done = true); unsupported (TC_UNSUPPORTED, nothing
// launched): the caller falls back to SIMT where it passes `done`, else CGVC_ERR_UNSUPPORTED; or failed: CGVC_ERR_CUDA
static int tc_result(cgvc_engine* e, int r, const ConvW* c, const char* what, bool* done = nullptr) {
  if (r == 0) { if (done) *done = true; return 0; }
  if (r == TC_UNSUPPORTED && done) return 0;
  std::string where = what;
  for (const TensorInfo& t : e->tensors) if (t.off == c->k) where = t.name + " " + what;
  if (r == TC_UNSUPPORTED) return fail(e, CGVC_ERR_UNSUPPORTED, "%s: shape not supported by the tensor-core path", where.c_str());
  return fail(e, CGVC_ERR_CUDA, "%s on the tensor cores: %s", where.c_str(), cudaGetErrorString((cudaError_t)r));
}

// P = conv(x) + bias, plain epilogue (gated: conv_a || conv_g -> P [rows, 2*cout])
static int conv_fwd(cgvc_engine* e, const Layer& L, const LayerTensors& t, const ConvIO& io, float* P, cudaStream_t st) {
  bool done = false;
  if (t.tc && io.xhi)
    RET(tc_result(e, tc_conv_fwd(*t.tc, t.precision, t.debug, io.xhi, io.xlo, io.n, io.H, io.W, L.sh, L.sw, P, st, nullptr, nullptr, packed(io)),
                  &L.a, "forward", &done));
  if (done) return 0;
  if (L.gated() && L.a.cin == 1 && io.x && !io.pk.off && L.a.cout % 4 == 0 && 256 % (L.a.cout / 2) == 0) {   // discriminator h1: HBM-bound special
    GatherGeom g = fwd_geom(io.n, io.H, io.W, L.a.kh, L.a.kw, L.sh, L.sw);
    CK(launch_conv_c1_fwd(g, io.x, t.ka, t.kg, t.ba, t.bg, L.a.cout, P, st));
    return 0;
  }
  RET(conv_fwd_simt(e, t.ka, t.ba, L.a, L.sh, L.sw, io, P, L.width(), 0, st));
  if (L.gated()) RET(conv_fwd_simt(e, t.kg, t.bg, L.g, L.sh, L.sw, io, P, L.width(), L.a.cout, st));
  return 0;
}

// dx[io's n,H,W] (+)= dgrad(dP); fuse: see tc_conv_dgrad
static int conv_dgrad(cgvc_engine* e, const Layer& L, const LayerTensors& t, const ConvIO& io, const float* dP, PlanePair dp, float* dx,
                      int accumulate, cudaStream_t st, const TcBwdFuse* fuse = nullptr, bool* fused = nullptr) {
  bool done = false;
  if (t.tc && dp.hi)
    RET(tc_result(e, tc_conv_dgrad(*t.tc, t.precision, t.debug, dp.hi, dp.lo, io.n, io.H, io.W, L.sh, L.sw, dx, accumulate, st, fuse, fused,
                                   packed(io)), &L.a, "data gradient", &done));
  if (done) return 0;
  RET(conv_dgrad_simt(e, t.ka, L.a, L.sh, L.sw, io.n, io.H, io.W, dP, L.width(), 0, dx, accumulate, st, packed(io)));
  if (L.gated()) RET(conv_dgrad_simt(e, t.kg, L.g, L.sh, L.sw, io.n, io.H, io.W, dP, L.width(), L.a.cout, dx, 1, st, packed(io)));
  return 0;
}

// det: deterministic mode (the lane's partials slab), else null
static int conv_wgrad(cgvc_engine* e, const Layer& L, const LayerTensors& t, const ConvIO& io, const float* dP, PlanePair dp, cudaStream_t st,
                      const DetSlab* det) {
  bool done = false;
  if (t.tc && dp.hi && io.xhi)
    RET(tc_result(e, tc_conv_wgrad(*t.tc, t.precision, t.debug, t.wgrad16, io.xhi, io.xlo, dp.hi, dp.lo, io.n, io.H, io.W, L.sh, L.sw, t.dka, t.dkg,
                                   st, det, packed(io)), &L.a, "weight gradient", &done));
  if (done) return 0;
  RET(conv_wgrad_simt(e, t.dka, L.a, L.sh, L.sw, io, dP, L.width(), 0, st, det));
  if (L.gated()) RET(conv_wgrad_simt(e, t.dkg, L.g, L.sh, L.sw, io, dP, L.width(), L.a.cout, st, det));
  return 0;
}

// instance norm (+ GLU | + resid) and pixel shuffle of A.P, the output of L's convolution over io (rows_per_sample_out rows per sample)
static PostParams post_params(const cgvc_engine* e, const Layer& L, const LayerTensors& t, const ConvIO& io, const GLAct& A,
                              int rows_per_sample_out, bool keep_y, float* scratch, const float* resid = nullptr) {
  PostParams q; memset(&q, 0, sizeof q);
  q.scratch = scratch;
  q.p = A.P; q.ldp = L.width(); q.Cc = L.a.cout; q.B = io.n; q.sh = L.shuffle;
  q.R = rows_per_sample_out * L.shuffle; q.C = L.a.cout / L.shuffle;
  q.has_in = L.has_in; q.has_gate = L.gated();
  q.beta_a = t.beta_a; q.gamma_a = t.gamma_a; q.beta_g = t.beta_g; q.gamma_g = t.gamma_g;
  q.resid = resid;
  q.y = (keep_y || !A.Yhi) ? A.Y : nullptr;      // without planes the fp32 activation is the only copy
  q.stats = L.has_in ? A.stats : nullptr; q.y_hi = A.Yhi; q.y_lo = A.Ylo;
  q.qmode = t.precision == CGVC_PREC_F16F8;
  q.sat = sat_act(e);
  if (io.pk.off && L.has_in && io.seg_out) {
    // packed 2-D grids: instance norm per utterance over its rows of the output grid, H_out x len_u / d_out of them
    const long long frames = (long long)io.pk.div * io.W, view_rows = q.R;
    q.B = io.pk.n; q.R = (int)(view_rows * io.pk.max_len / frames);
    q.seg = PackGeom{io.seg_out, io.pk.n, 1, q.R}; q.seg_rows = view_rows;
  } else if (io.pk.off && L.has_in) {
    // packed utterances: q describes one sample holding all q.R view rows; instance norm runs per utterance over its own view rows
    // (the GLU-only layer is row-local and keeps that view)
    const long long view_rows = q.R;
    const int div = (int)((long long)io.pk.div * io.W / view_rows);
    q.seg = PackGeom{io.pk.off, io.pk.n, div, io.pk.max_len}; q.seg_rows = view_rows;
    q.B = io.pk.n; q.R = io.pk.max_len / div;
  }
  return q;
}

// One layer's forward: convolution, then instance norm (+ GLU | + resid) and pixel shuffle into A.  The paths, in order: tensor
// cores with the norm fused into the GEMM epilogue (1-D layer, not packed, whole samples per 128-row tile); else tensor cores with
// the plain epilogue, or SIMT, then the instance-norm kernels.  keep_y: also write the fp32 output.  save_pre = false (inference):
// the fused epilogue need not write the pre-norm output and statistics, as nothing runs backward.  fuse: the fused epilogue may run
// (option fuse_in); *fused (may be null) is set when it did
static int layer_forward(cgvc_engine* e, const Layer& L, const LayerTensors& t, const ConvIO& io, const GLAct& A, int rows_per_sample_out,
                         bool keep_y, bool save_pre, bool fuse, float* post_scratch, cudaStream_t st, const float* resid = nullptr,
                         bool* fused = nullptr) {
  bool done = false;
  if (t.tc && io.xhi && !io.pk.off && L.has_in && (L.shuffle == 1 || L.shuffle == 2) && io.H == 1 && A.Yhi && fuse) {
    TcFuse f; memset(&f, 0, sizeof f);
    f.R = rows_per_sample_out;
    f.gamma_a = t.gamma_a; f.beta_a = t.beta_a; f.gamma_g = t.gamma_g; f.beta_g = t.beta_g;
    f.stats = save_pre ? A.stats : nullptr; f.resid = resid; f.y = keep_y ? A.Y : nullptr; f.y_hi = A.Yhi; f.y_lo = A.Ylo;
    bool in_epi = false;
    int r = tc_conv_fwd(*t.tc, t.precision, t.debug, io.xhi, io.xlo, io.n, io.H, io.W, L.sh, L.sw, save_pre ? A.P : nullptr, st, &f, &in_epi);
    if (r != 0 && !save_pre)                                  // shape not fusable: the two-kernel path needs P as its intermediate
      r = tc_conv_fwd(*t.tc, t.precision, t.debug, io.xhi, io.xlo, io.n, io.H, io.W, L.sh, L.sw, A.P, st, &f, &in_epi);
    RET(tc_result(e, r, &L.a, "forward", &done));
    if (in_epi) { if (fused) *fused = true; return 0; }
  }
  if (!done) RET(conv_fwd(e, L, t, io, A.P, st));
  PostParams q = post_params(e, L, t, io, A, rows_per_sample_out, keep_y, post_scratch, resid);
  CK(launch_post_fwd(q, e->opt.post, st));
  return 0;
}

// ---- generator -------------------------------------------------------------------------------------------
// Tap lowering of the two 15-tap edge layers (module.py:85-86 h1, module.py:148 o1; kernels and rationale in simt_kernels.cu above
// im2col_taps_kernel): h1 becomes a 1 x 1 gated layer over the im2col of the 24-channel input (TF's [1,15,24,128] kernel is that
// [360,128] matrix as it lies in memory, so forward, data and weight gradient address the same PARAM / GRAD ranges), o1 a 1 x 1 layer
// with the taps folded into its output columns (TcLayer::fold) followed by the tap-shifted sum.
static inline int edge_cpad(int c) { return (c + 127) / 128 * 128; }      // operand-plane width of kw * F channels (a multiple of 128 serves both precisions)
static bool edge_on(const cgvc_engine* e, const GenNet& N) { return e->opt.edge_lower && use_tc(e, N.h1c_slot) && use_tc(e, N.o1f_slot); }

static void plan_gated(Bump& ws, GLAct& a, long long rows_out, int cout2, int n, int Cstat, bool planes, long long y_elems) {
  a.P = ws.take<float>((size_t)rows_out * cout2);
  a.stats = ws.take<float>((size_t)n * 4 * Cstat);
  a.Y = ws.take<float>((size_t)y_elems);
  a.Yhi = a.Ylo = nullptr;
  if (planes) { a.Yhi = ws.take<__nv_bfloat16>((size_t)y_elems); a.Ylo = ws.take<__nv_bfloat16>((size_t)y_elems); }
}

// activations of n samples of r1 rows in all (n x T, or n packed utterances)
static void plan_generator_rows(cgvc_engine* e, Bump& ws, GenActs& A, int n, long long r1) {
  const bool pl = e->cfg.precision != CGVC_PREC_FP32_SIMT;
  A.n = n; A.T = 0; A.off = nullptr; A.rows = r1; A.max_len = 0; A.xhi = A.xlo = nullptr; A.post = nullptr;
  long long r2 = r1 / 2, r4 = r1 / 4;
  if (pl) { A.xhi = ws.take<__nv_bfloat16>((size_t)r1 * 128); A.xlo = ws.take<__nv_bfloat16>((size_t)r1 * 128); }   // input planes, channels padded to 64 (128: F16F8)
  A.xchi = A.xclo = nullptr; A.z = nullptr;
  if (pl) {                                                    // tap-lowered edge layers (edge_on)
    const size_t cp = (size_t)edge_cpad(e->gen[0].h1.a.kw * e->cfg.num_features);
    A.xchi = ws.take<__nv_bfloat16>((size_t)r1 * cp); A.xclo = ws.take<__nv_bfloat16>((size_t)r1 * cp);
    A.z = ws.take<float>((size_t)r1 * e->gen[0].o1.a.kw * e->cfg.num_features);
  }
  plan_gated(ws, A.h1, r1, 256, n, 128, pl, r1 * 128);
  plan_gated(ws, A.d[0], r2, 512, n, 256, pl, r2 * 256);
  plan_gated(ws, A.d[1], r4, 1024, n, 512, pl, r4 * 512);
  for (int i = 0; i < 6; ++i) {
    plan_gated(ws, A.r[i].h1, r4, 2048, n, 1024, pl, r4 * 1024);
    plan_gated(ws, A.r[i].h2, r4, 512, n, 512, pl, r4 * 512);
  }
  plan_gated(ws, A.u[0], r4, 2048, n, 512, pl, r2 * 512);
  plan_gated(ws, A.u[1], r2, 1024, n, 256, pl, r1 * 256);
  A.out_cl = ws.take<float>((size_t)r1 * e->cfg.num_features);
}

static void plan_generator(cgvc_engine* e, Bump& ws, GenActs& A, int n, int T) {
  plan_generator_rows(e, ws, A, n, (long long)n * T);
  A.T = T;
}

// The tap-lowered edge layers (edge_on) by pointer, so that the walks and the test entry points (cgvc_edge_*) run the same launches.
// Rows: n samples of T, or (off) one sequence of T rows holding n_off packed utterances (n = 1).
// h1: the im2col planes xc of x [n*T, F], P [n*T, 256] = [a | g] = xc . W + bias, then the GLU that q describes (q.p = P)
static int h1_edge_forward(cgvc_engine* e, const GenNet& N, const float* x, int n, int T, const long long* off, int n_off,
                           __nv_bfloat16* xchi, __nv_bfloat16* xclo, float* P, const PostParams& q, cudaStream_t st) {
  const int nf = e->cfg.num_features;
  CK(launch_im2col_taps(x, (long long)n * T, T, nf, N.h1.a.kw, +1, edge_cpad(N.h1.a.kw * nf), e->cfg.precision == CGVC_PREC_F16F8,
                        xchi, xclo, st, off, n_off, sat_act(e)));
  RET(tc_result(e, tc_conv_fwd(e->tcw.layers[N.h1c_slot], e->cfg.precision, e->tcw.debug, xchi, xclo, n, 1, T, 1, 1, P, st), &N.h1.a,
                "forward (tap-lowered)"));
  CK(launch_post_fwd(q, e->opt.post, st));
  return 0;
}

// o1: Z [n*W, kw*F] = U . W' (the taps folded into the columns) from U's planes, then out [n*W, F] = bias + the tap-shifted sum of Z
static int o1_edge_forward(cgvc_engine* e, const GenNet& N, const __nv_bfloat16* uhi, const __nv_bfloat16* ulo, int n, int W,
                           const long long* off, int n_off, float* z, float* out, cudaStream_t st) {
  const int nf = e->cfg.num_features;
  RET(tc_result(e, tc_conv_fwd(e->tcw.layers[N.o1f_slot], e->cfg.precision, e->tcw.debug, uhi, ulo, n, 1, W, 1, 1, z, st), &N.o1.a,
                "forward (tap-lowered)"));
  CK(launch_col2im_taps(z, N.o1.a.kw * nf, (long long)n * W, W, nf, N.o1.a.kw, +1, e->P() + N.o1.a.b, out, st, off, n_off));
  return 0;
}

// keep_y: also write the fp32 copy of every activation (debug taps / SIMT path); the tensor-core training path only
// needs fp32 where a residual add or the discriminator head reads it.
// save_pre = false (inference): the fused layers do not write their pre-norm outputs / statistics (nothing runs backward)
static int generator_forward(cgvc_engine* e, const GenNet& N, GenActs& A, const float* x_cl, cudaStream_t st, bool keep_y, bool save_pre = true) {
  // packed utterances (A.off): the geometry is one sequence of all rows, n = 1 and T = the row count; every layer's taps, instance
  // norms and edge-layer tap lowering then follow the utterance boundaries of A.off instead
  const bool packed = A.off != nullptr;
  const int n = packed ? 1 : A.n, T = packed ? (int)A.rows : A.T, nf = e->cfg.num_features;
  auto at = [&](const float* x, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int W) {
    ConvIO io; io.x = x; io.xhi = hi; io.xlo = lo; io.n = n; io.H = 1; io.W = W;
    if (packed) io.pk = PackGeom{A.off, A.n, (int)(A.rows / W), A.max_len};
    return io;
  };
  auto of = [&](const GLAct& a, int W) { return at((keep_y || !a.Yhi) ? a.Y : nullptr, a.Yhi, a.Ylo, W); };   // a layer output as input
  auto fwd = [&](const Layer& L, const ConvIO& in, const GLAct& a, int W, bool y, const float* resid = nullptr) {
    return layer_forward(e, L, layer_tensors(e, L, false), in, a, W, y, save_pre, e->opt.fuse_in, A.post, st, resid);
  };
  A.x_cl = x_cl;
  const bool edge = edge_on(e, N) && A.xchi && A.z;
  ConvIO io = at(x_cl, A.xhi, A.xlo, T);
  if (edge) {
    // h1 = dense [n*T, kw*F] x [kw*F, 2*128] GEMM on the im2col of the input
    const PostParams q = post_params(e, N.h1, layer_tensors(e, N.h1, false), io, A.h1, T, keep_y, A.post);
    RET(h1_edge_forward(e, N, x_cl, n, T, A.off, A.n, A.xchi, A.xclo, A.h1.P, q, st));
  } else {
    if (A.xhi && tc_enabled(e)) CK(tc_split_planes(e->cfg.precision, x_cl, (long long)n * T, nf, A.xhi, A.xlo, st, sat_act(e)));
    RET(fwd(N.h1, io, A.h1, T, keep_y));
  }
  const GLAct* cur = &A.h1;
  int W = T;
  for (int i = 0; i < 2; ++i) {
    io = of(*cur, W);
    W /= 2;
    RET(fwd(N.d[i], io, A.d[i], W, keep_y || i == 1));   // d2's fp32 output is the first residual input
    cur = &A.d[i];
  }
  for (int i = 0; i < 6; ++i) {       // cur: the block input, whose fp32 copy is always written
    RET(fwd(N.r[i].h1, at(cur->Y, cur->Yhi, cur->Ylo, W), A.r[i].h1, W, keep_y));
    RET(fwd(N.r[i].h2, of(A.r[i].h1, W), A.r[i].h2, W, true, cur->Y));
    cur = &A.r[i].h2;
  }
  io = at(cur->Y, cur->Yhi, cur->Ylo, W);
  for (int i = 0; i < 2; ++i) {
    RET(fwd(N.u[i], io, A.u[i], W, keep_y));      // W = conv rows per sample; the shuffle doubles them
    W *= 2;
    io = of(A.u[i], W);
  }
  if (edge && io.xhi) {
    // o1: Z[m, (t, c)] = U[m, :] . W[t][:, c] as one dense GEMM, then out[m, c] = b[c] + sum_t Z[m + t - 7, (t, c)]
    RET(o1_edge_forward(e, N, io.xhi, io.xlo, n, W, A.off, A.n, A.z, A.out_cl, st));
  } else {
    RET(conv_fwd(e, N.o1, layer_tensors(e, N.o1, false), io, A.out_cl, st));
  }
  if (keep_y) {
    e->taps.clear();
    size_t r1 = (size_t)n * T;
    e->taps["h1_glu"] = {A.h1.Y, r1 * 128}; e->taps["d1"] = {A.d[0].Y, r1 / 2 * 256}; e->taps["d2"] = {A.d[1].Y, r1 / 4 * 512};
    for (int i = 0; i < 6; ++i) e->taps["r" + std::to_string(i + 1)] = {A.r[i].h2.Y, r1 / 4 * 512};
    e->taps["u1"] = {A.u[0].Y, r1 / 2 * 512}; e->taps["u2"] = {A.u[1].Y, r1 * 256};
    e->taps["out_cl"] = {A.out_cl, r1 * (size_t)nf};
  }
  return 0;
}

// ---- backward -----------------------------------------------------------------------------------------------
struct BwdScratch { float *bufA, *bufB, *dP; __nv_bfloat16 *dPhi, *dPlo; float* post;
                    __nv_bfloat16 *dP2hi, *dP2lo;      // second plane pair: a fused dgrad epilogue writes the next layer's dP while reading this one's
                    __nv_bfloat16 *dPbhi, *dPblo;      // ping-pong partner of dPhi / dPlo (same size) for the side-stream weight gradients
                    SideQ* sq;
                    DetSlab det; };                    // deterministic mode: the lane's partials slab (det.p null otherwise)

static bool side_on(const BwdScratch& S) { return S.sq && S.sq->on && S.dPbhi; }
static const DetSlab* det_of(const BwdScratch& S) { return S.det.p ? &S.det : nullptr; }

// The dP planes of one backward walk.  Fused backward (tensor-core path, fuse_bwd): a stride-1 data-gradient launch whose result is
// d loss / d (output of an instance-normed layer) runs that layer's instance-norm (+GLU) backward in its epilogue and writes the
// layer's dP planes directly, reading one plane pair while writing the other.
struct BwdWalk {
  const BwdScratch& S;
  bool fuse;                  // fuse_bwd in effect
  PlanePair pb[2];            // [0]: the planes a GLU / instance-norm backward writes (side_wgrad off), [1]: its fused-epilogue partner
  int have = -1;              // pb[have] already holds the dP planes of the layer differentiated next, or -1
  int cur = 0;                // the pb index of the planes handed out last
  BwdWalk(const BwdScratch& s, bool f) : S(s), fuse(f), pb{{s.dPhi, s.dPlo}, {s.dP2hi, s.dP2lo}} {}
};

// The dP plane pair of the next layer: the one the previous data-gradient launch's fused epilogue wrote (*written), else the pair for
// its GLU / instance-norm backward to write: with side_wgrad the ping-pong buffer, once the weight gradient that last read it (on the
// side stream) has finished
static PlanePair dp_planes(BwdWalk& w, cudaStream_t st, bool* written = nullptr) {
  if (written) *written = w.have >= 0;
  if (w.have >= 0) { w.cur = w.have; w.have = -1; return w.pb[w.cur]; }
  w.cur = 0;
  if (!side_on(w.S)) return w.pb[0];
  SideQ* q = w.S.sq;
  q->cur ^= 1;
  if (q->used[q->cur]) cudaStreamWaitEvent(st, q->done[q->cur], 0);
  return q->cur ? PlanePair{w.S.dPbhi, w.S.dPblo} : PlanePair{w.S.dPhi, w.S.dPlo};
}

// Runs wgrad(stream), a weight gradient of the planes handed out last.  With side_wgrad and planes, on the side stream behind an
// event on them, recording when it is done with them; else on st
template <class F> static int run_wgrad(const BwdScratch& S, bool planes, cudaStream_t st, F&& wgrad) {
  if (!planes || !side_on(S)) return wgrad(st);
  SideQ* q = S.sq;
  cudaEventRecord(q->ready[q->cur], st);
  cudaStreamWaitEvent(q->side, q->ready[q->cur], 0);
  const int r = wgrad(q->side);
  cudaEventRecord(q->done[q->cur], q->side);
  q->used[q->cur] = true;
  return r;
}

// every side-stream weight gradient of this lane has finished before st continues
static void side_join(const BwdScratch& S, cudaStream_t st) {
  SideQ* q = S.sq;
  if (!q) return;
  for (int b = 0; b < 2; ++b) if (q->used[b]) { cudaStreamWaitEvent(st, q->done[b], 0); q->used[b] = false; }
}

// GLU / instance-norm backward of a layer into dP planes `out`, with the parameter gradients t holds; fp32 dP is only materialised when
// a SIMT kernel will read it.  in (may be null): the layer's input; when it is packed and L has an instance norm, *seg receives the
// utterance segments the norm follows (launch_post_bwd's PostBwdSeg), else seg->seg.off stays null
static PostBwdParams post_bwd_params(const cgvc_engine* e, const Layer& L, const LayerTensors& t, const float* dy, const GLAct& A, int n,
                                     int rows_per_sample_out, const BwdScratch& S, bool need_fp32, PlanePair out,
                                     const ConvIO* in = nullptr, PostBwdSeg* seg = nullptr) {
  PostBwdParams q; memset(&q, 0, sizeof q);
  q.dy1 = dy; q.p = A.P; q.ldp = L.width(); q.Cc = L.a.cout; q.B = n; q.sh = L.shuffle;
  q.R = rows_per_sample_out * L.shuffle; q.C = L.a.cout / L.shuffle;
  q.has_in = L.has_in; q.has_gate = L.gated(); q.stats = A.stats;
  q.beta_a = t.beta_a; q.gamma_a = t.gamma_a; q.beta_g = t.beta_g; q.gamma_g = t.gamma_g;
  q.dbeta_a = t.dbeta_a; q.dgamma_a = t.dgamma_a; q.dbeta_g = t.dbeta_g; q.dgamma_g = t.dgamma_g;
  q.dbias_a = t.dba; q.dbias_g = t.dbg;
  q.scratch = S.post;
  const bool tc = t.tc && S.dPhi;
  q.dp = (!tc || need_fp32) ? S.dP : nullptr;
  if (tc) { q.dp_hi = out.hi; q.dp_lo = out.lo; }
  q.qmode = t.precision == CGVC_PREC_F16F8;
  q.sat = sat_grad(e); q.ufl = ufl_grad(e);
  if (t.dba || t.dbeta_a) q.det = S.det;    // passes without parameter gradients keep the faster (equally deterministic) forms
  if (seg) seg->seg.off = nullptr;
  if (seg && in && in->pk.off && L.has_in && in->seg_out) {
    // packed 2-D grids, as post_params: per utterance over its rows of the output grid (n + 1 row prefix sums in->seg_out, div 1)
    const long long frames = (long long)in->pk.div * in->W, view_rows = q.R;
    q.B = in->pk.n; q.R = (int)(view_rows * in->pk.max_len / frames);
    *seg = PostBwdSeg{PackGeom{in->seg_out, in->pk.n, 1, q.R}, view_rows};
  } else if (seg && in && in->pk.off && L.has_in) {
    // packed utterances, as post_params: per utterance over its own view rows (the GLU-only layer is row-local and keeps one sample)
    const long long view_rows = q.R;
    const int div = (int)((long long)in->pk.div * in->W / view_rows);
    *seg = PostBwdSeg{PackGeom{in->pk.off, in->pk.n, div, in->pk.max_len}, view_rows};
    q.B = in->pk.n; q.R = in->pk.max_len / div;
  }
  return q;
}

// the fused backward epilogue (tc_conv_dgrad) of L's instance norm (+ GLU; no pixel shuffle), writing its dP planes into `out`
static TcBwdFuse bwd_fuse(const Layer& L, const LayerTensors& t, const GLAct& A, int rows_per_sample, PlanePair out) {
  TcBwdFuse f; memset(&f, 0, sizeof f);
  f.R = (L.has_in && L.shuffle == 1) ? rows_per_sample : 0;      // R = 0: not fusable
  f.gated = L.gated(); f.bp = A.P; f.bp_ld = L.width(); f.stats = A.stats;
  f.gamma_a = t.gamma_a; f.beta_a = t.beta_a; f.gamma_g = t.gamma_g; f.beta_g = t.beta_g;
  f.dp_hi = out.hi; f.dp_lo = out.lo; f.dp_ld = L.width();
  f.dgamma_a = t.dgamma_a; f.dbeta_a = t.dbeta_a; f.dgamma_g = t.dgamma_g; f.dbeta_g = t.dbeta_g;
  return f;
}

// dP of a layer: the GLU / instance-norm backward kernel, unless the previous data-gradient launch's fused epilogue wrote it
static int layer_dp(cgvc_engine* e, BwdWalk& w, const Layer& L, const LayerTensors& t, const GLAct& A, const float* dy, int n,
                    int rows_per_sample_out, cudaStream_t st, PostBwdParams& q, const ConvIO* in = nullptr) {
  bool written = false;
  const PlanePair out = dp_planes(w, st, &written);
  PostBwdSeg seg;
  q = post_bwd_params(e, L, t, dy, A, n, rows_per_sample_out, w.S, false, out, in, &seg);
  if (!written) CK(launch_post_bwd(q, e->opt.post, st, seg.seg.off ? &seg : nullptr));
  return 0;
}

// dx (+)= the data gradient of L from its dP (fp32 dP, planes dp), with the instance-norm backward of `up` (tensors ut, activations upA)
// -- the layer whose output was L's input -- fused into its epilogue under w.fuse where the shape allows; the fused epilogue writes up's
// dP planes into the walk's other plane pair, which up's layer_dp then takes without a launch
static int layer_dx(cgvc_engine* e, BwdWalk& w, const Layer& L, const LayerTensors& t, const ConvIO& in, const float* dP, PlanePair dp,
                    float* dx, int accumulate, cudaStream_t st, const Layer* up, const LayerTensors* ut, const GLAct* upA) {
  const int other = 1 - w.cur;
  TcBwdFuse f;
  const bool fuse = up && w.fuse && dp.hi;
  if (fuse) f = bwd_fuse(*up, *ut, *upA, in.W, w.pb[other]);
  bool fused = false;
  RET(conv_dgrad(e, L, t, in, dP, dp, dx, accumulate, st, fuse ? &f : nullptr, &fused));
  if (fused) w.have = other;
  return 0;
}

// Backward through one layer, whose input was `in` and upstream gradient is dy: (1) dP (layer_dp); (2) with wgrad, the weight
// gradient (run_wgrad); (3) with dx, layer_dx (up, upA: the layer whose output is `in` and its activations)
static int layer_backward(cgvc_engine* e, BwdWalk& w, const Layer& L, const GLAct& A, const ConvIO& in, const float* dy,
                          int rows_per_sample_out, bool wgrad, float* dx, int accumulate, cudaStream_t st,
                          const Layer* up = nullptr, const GLAct* upA = nullptr) {
  const LayerTensors t = layer_tensors(e, L, wgrad);
  PostBwdParams q;
  RET(layer_dp(e, w, L, t, A, dy, in.n, rows_per_sample_out, st, q, &in));
  const PlanePair dp{q.dp_hi, q.dp_lo};
  if (wgrad) RET(run_wgrad(w.S, dp.hi != nullptr, st, [&](cudaStream_t ws) { return conv_wgrad(e, L, t, in, q.dp, dp, ws, det_of(w.S)); }));
  if (!dx) return 0;
  LayerTensors ut{};
  if (up) ut = layer_tensors(e, *up, wgrad);
  return layer_dx(e, w, L, t, in, q.dp, dp, dx, accumulate, st, up, &ut, upA);
}

// The tap-lowered edge layers' backward (see h1_edge_forward), n samples of T rows.
// o1 from d_out [n*T, F]: its dZ planes (the im2col of d_out, dir -1), the kernel gradient U^T dZ into GRAD (run_wgrad, folded columns
// scattered by tn_dst) and du [n*T, 256] = dZ . W'^T.  The bias gradient, the column sums of d_out, is the caller's
// (off, n_off: packed utterances, as o1_edge_forward)
static int o1_edge_backward(cgvc_engine* e, const GenNet& N, const float* d_out, const __nv_bfloat16* uhi, const __nv_bfloat16* ulo, int n,
                            int T, PlanePair dz, float* du, const BwdScratch& S, cudaStream_t st, const long long* off = nullptr, int n_off = 0) {
  const int nf = e->cfg.num_features;
  float* Gm = e->G();
  const TcLayer& O = e->tcw.layers[N.o1f_slot];
  CK(launch_im2col_taps(d_out, (long long)n * T, T, nf, N.o1.a.kw, -1, edge_cpad(N.o1.a.kw * nf), e->cfg.precision == CGVC_PREC_F16F8,
                        dz.hi, dz.lo, st, off, n_off, sat_grad(e), ufl_grad(e)));
  RET(run_wgrad(S, true, st, [&](cudaStream_t ws) {
    return tc_result(e, tc_conv_wgrad(O, e->cfg.precision, e->tcw.debug, e->tcw.wgrad16, uhi, ulo, dz.hi, dz.lo, n, 1, T, 1, 1, Gm + N.o1.a.k, nullptr, ws,
                                      det_of(S)),
                     &N.o1.a, "weight gradient (tap-lowered)"); }));
  RET(tc_result(e, tc_conv_dgrad(O, e->cfg.precision, e->tcw.debug, dz.hi, dz.lo, n, 1, T, 1, 1, du, 0, st), &N.o1.a,
                "data gradient (tap-lowered)"));
  return 0;
}

// h1 from its dP planes (written by the GLU backward, which also takes the bias gradients): the kernel gradients xc^T dP straight into
// the [15,24,128] a and g ranges of GRAD (run_wgrad); with dz, dz [n*T, kw*F] = dP . W^T, and with dx too, dx [n*T, F] = the
// tap-shifted sum of dz (dir -1)
static int h1_edge_backward(cgvc_engine* e, const GenNet& N, const __nv_bfloat16* xchi, const __nv_bfloat16* xclo, PlanePair dp, int n,
                            int T, float* dz, float* dx, const BwdScratch& S, cudaStream_t st, const long long* off = nullptr, int n_off = 0) {
  const int nf = e->cfg.num_features;
  float* Gm = e->G();
  const TcLayer& H = e->tcw.layers[N.h1c_slot];
  RET(run_wgrad(S, true, st, [&](cudaStream_t ws) {
    return tc_result(e, tc_conv_wgrad(H, e->cfg.precision, e->tcw.debug, e->tcw.wgrad16, xchi, xclo, dp.hi, dp.lo, n, 1, T, 1, 1, Gm + N.h1.a.k,
                                      Gm + N.h1.g.k, ws, det_of(S)),
                     &N.h1.a, "weight gradient (tap-lowered)"); }));
  if (dz) RET(tc_result(e, tc_conv_dgrad(H, e->cfg.precision, e->tcw.debug, dp.hi, dp.lo, n, 1, T, 1, 1, dz, 0, st), &N.h1.a,
                        "data gradient (tap-lowered)"));
  if (dz && dx) CK(launch_col2im_taps(dz, N.h1.a.kw * nf, (long long)n * T, T, nf, N.h1.a.kw, -1, nullptr, dx, st, off, n_off));
  return 0;
}

// Backward through one generator application.  d_out_cl: [n*T, 24] gradient w.r.t. the channels-last output.
// Weight gradients are accumulated into the GRAD arena; d_in_cl (optional) receives d loss / d input (channels-last).
static int generator_backward(cgvc_engine* e, const GenNet& N, const GenActs& A, const float* d_out_cl, float* d_in_cl,
                              const BwdScratch& S, cudaStream_t st) {
  // packed utterances (A.off), as generator_forward: one sequence of all rows whose taps, instance norms and edge-layer tap lowering
  // follow the utterance boundaries
  const bool packed = A.off != nullptr;
  const int n = packed ? 1 : A.n, T = packed ? (int)A.rows : A.T, nf = e->cfg.num_features;
  float* Gm = e->G();
  auto at = [&](const float* x, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int W) {
    ConvIO io; io.x = x; io.xhi = hi; io.xlo = lo; io.n = n; io.H = 1; io.W = W;
    if (packed) io.pk = PackGeom{A.off, A.n, (int)(A.rows / W), A.max_len};
    return io;
  };
  auto of = [&](const GLAct& a, int W) { return at(a.Y, a.Yhi, a.Ylo, W); };
  // the fused backward epilogues do not count saturation: a step whose planes are counted takes the separate kernels.  Nor do they
  // take packed rows: they need whole equal-length samples per 128-row tile
  BwdWalk w(S, e->opt.fuse_bwd && !packed && !e->opt.deterministic && !sat_grad(e) && !side_on(S) && tc_enabled(e) && S.dPhi && S.dP2hi &&
               A.r[0].h1.Yhi && A.r[0].h2.Yhi);
  const bool edge = edge_on(e, N) && A.xchi && A.z;
  // o1 (no norm, no gate): bias gradient = column sums of d_out
  CK(launch_colsum(d_out_cl, (long long)n * T, nf, 0, nf, Gm + N.o1.a.b, st, det_of(S)));
  const ConvIO u2 = of(A.u[1], T);
  if (edge && u2.xhi && S.dPhi) {
    // tap-lowered o1: dZ[m, (t, c)] = d_out[m - t + 7, c] (im2col of the 24-channel gradient), then dense weight and data gradients
    RET(o1_edge_backward(e, N, d_out_cl, u2.xhi, u2.xlo, n, T, dp_planes(w, st), S.bufA, S, st, A.off, A.n));
  } else {
    const LayerTensors t = layer_tensors(e, N.o1, true);
    PlanePair dp{nullptr, nullptr};
    if (t.tc && u2.xhi && S.dPhi) {
      dp = dp_planes(w, st);
      CK(tc_split_planes(e->cfg.precision, d_out_cl, (long long)n * T, nf, dp.hi, dp.lo, st, sat_grad(e), ufl_grad(e)));
    }
    RET(run_wgrad(S, dp.hi != nullptr, st, [&](cudaStream_t ws) { return conv_wgrad(e, N.o1, t, u2, d_out_cl, dp, ws, det_of(S)); }));
    RET(conv_dgrad(e, N.o1, t, u2, d_out_cl, dp, S.bufA, 0, st));
  }
  float* cur = S.bufA; float* oth = S.bufB;
  // up-sampling blocks, convolutions at T/2 and T/4 (the shuffle doubles the rows).  u1's data gradient is d loss / d (residual block
  // 6 output), so its launch can run that block's h2 instance-norm backward
  RET(layer_backward(e, w, N.u[1], A.u[1], of(A.u[0], T / 2), cur, T / 2, true, oth, 0, st));
  std::swap(cur, oth);
  RET(layer_backward(e, w, N.u[0], A.u[0], of(A.r[5].h2, T / 4), cur, T / 4, true, oth, 0, st, &N.r[5].h2, &A.r[5].h2));
  std::swap(cur, oth);
  // residual blocks (width T/4); cur holds d(block output).  h2's data gradient is d loss / d (h1's GLU output); h1's is added to cur
  // in place (the skip), making it d loss / d (previous block's output) -- or, for the first block, of the second down-sampling
  // layer's output
  for (int i = 5; i >= 0; --i) {
    const Layer& Lin = i > 0 ? N.r[i - 1].h2 : N.d[1];
    const GLAct& Ain = i > 0 ? A.r[i - 1].h2 : A.d[1];
    RET(layer_backward(e, w, N.r[i].h2, A.r[i].h2, of(A.r[i].h1, T / 4), cur, T / 4, true, oth, 0, st, &N.r[i].h1, &A.r[i].h1));
    RET(layer_backward(e, w, N.r[i].h1, A.r[i].h1, of(Ain, T / 4), oth, T / 4, true, cur, 1, st, &Lin, &Ain));
  }
  // down-sampling blocks (stride 2)
  RET(layer_backward(e, w, N.d[1], A.d[1], of(A.d[0], T / 2), cur, T / 4, true, oth, 0, st));
  std::swap(cur, oth);
  RET(layer_backward(e, w, N.d[0], A.d[0], of(A.h1, T), cur, T / 2, true, oth, 0, st));
  std::swap(cur, oth);
  // h1 (no IN)
  const ConvIO x = at(A.x_cl, A.xhi, A.xlo, T);
  if (!edge) return layer_backward(e, w, N.h1, A.h1, x, cur, T, true, d_in_cl, 0, st);
  // tap-lowered h1: the weight gradient is im2col(x)^T dP straight into the [15,24,128] kernels' GRAD ranges; the data gradient
  // (cycle passes only) is the dense dP . W^T [n*T, kw*F] followed by the tap-shifted sum
  PostBwdParams q;
  RET(layer_dp(e, w, N.h1, layer_tensors(e, N.h1, true), A.h1, cur, n, T, st, q, &x));
  return h1_edge_backward(e, N, A.xchi, A.xclo, PlanePair{q.dp_hi, q.dp_lo}, n, T, d_in_cl ? oth : nullptr, d_in_cl, S, st, A.off, A.n);
}

// ---- discriminator ---------------------------------------------------------------------------------------
// activations of n samples of `frames` frames in all (n x T, or n packed utterances: every length a multiple of 16)
static void plan_discriminator_rows(cgvc_engine* e, Bump& ws, DiscActs& A, int n, long long frames) {
  const bool pl = e->cfg.precision != CGVC_PREC_FP32_SIMT;
  A.n = n; A.T = 0; A.post = nullptr; A.off = nullptr; A.seg[0] = A.seg[1] = A.seg[2] = nullptr; A.rows = frames; A.max_len = 0;
  const int H = e->cfg.num_features;
  long long r0 = H * (frames / 2), r1 = (H / 2) * (frames / 4), r2 = (H / 4) * (frames / 8), r3 = (H / 4) * (frames / 16);
  plan_gated(ws, A.h1, r0, 256, n, 128, pl, r0 * 128);
  plan_gated(ws, A.d[0], r1, 512, n, 256, pl, r1 * 256);
  plan_gated(ws, A.d[1], r2, 1024, n, 512, pl, r2 * 512);
  plan_gated(ws, A.d[2], r3, 2048, n, 1024, false, r3 * 1024);
  A.prob = ws.take<float>((size_t)r3);
}

static void plan_discriminator(cgvc_engine* e, Bump& ws, DiscActs& A, int n, int T) {
  plan_discriminator_rows(e, ws, A, n, (long long)n * T);
  A.T = T;
}

// The discriminator's input layer L (one input channel, <= 9 taps, gate without instance norm: module.py:196-203), its tensors t by
// pointer, so that the walk and the test entry points (cgvc_disc_input_forward / _backward) run the same launches.
// P [n * Ho * Wo, 2 cout] = [a | g] = conv(x [n, H, W]) + bias, and the GLU that q describes (q.p = P: y, its planes and their count).
// fuse: convolution + GLU in one HBM-bound pass (P is written for the backward pass but not read back); else the convolution, then the
// GLU-only post kernels
// pk (may be null): x and P are packed 2-D grids (n = 1, W = all frames)
static int disc_input_forward(cgvc_engine* e, const Layer& L, const LayerTensors& t, const float* x, int n, int H, int W, float* P,
                              const PostParams& q, bool fuse, cudaStream_t st, const PackGeom* pk = nullptr) {
  const GatherGeom g = fwd_geom(n, H, W, L.a.kh, L.a.kw, L.sh, L.sw);
  if (fuse) {
    CK(launch_conv_c1_glu_fwd(g, x, t.ka, t.kg, t.ba, t.bg, L.a.cout, P, q.y, q.y_hi, q.y_lo, q.qmode, st, q.sat, q.ufl, pk));
    return 0;
  }
  CK(launch_conv_c1_fwd(g, x, t.ka, t.kg, t.ba, t.bg, L.a.cout, P, st, pk));
  CK(launch_post_fwd(q, e->opt.post, st));
  return 0;
}

// Backward of the same layer from dy [n * Ho * Wo, cout] and the saved P: t's weight and bias gradients += (t.dka null: none), dx [n, H, W]
// = the data gradient (null: none), Z scratch [n * Ho * Wo, taps].  fuse: dP = (dy s(g), dy a s(g) (1 - s(g))) formed in registers inside
// the weight-gradient and data-gradient kernels; else the GLU-only backward q (bias gradients included) writes the fp32 dP q.dp, which
// wgrad_c1 and dgrad_c1 read.  det: deterministic mode's partials slab, else null
// pk (may be null): packed 2-D grids, as disc_input_forward
static int disc_input_backward(cgvc_engine* e, const Layer& L, const LayerTensors& t, const float* x, const float* dy, const float* P, int n,
                               int H, int W, float* dx, float* Z, bool fuse, const PostBwdParams& q, const DetSlab* det, cudaStream_t st,
                               const PackGeom* pk = nullptr) {
  const int kh = L.a.kh, kw = L.a.kw, cout = L.a.cout;
  const GatherGeom g = fwd_geom(n, H, W, kh, kw, L.sh, L.sw);
  if (fuse) {
    if (t.dka) CK(launch_glu_bwd_wgrad_c1(g, x, dy, P, cout, t.dka, t.dkg, t.dba, t.dbg, st, det, pk));
    if (dx) CK(launch_glu_bwd_dgrad_c1(dy, P, cout, t.ka, t.kg, Z, dx, n, H, W, kh, kw, L.sh, L.sw, st, pk));
    return 0;
  }
  CK(launch_post_bwd(q, e->opt.post, st));
  if (t.dka) CK(launch_wgrad_c1(g, x, q.dp, 2 * cout, 2 * cout, t.dka, t.dkg, cout, nullptr, nullptr, st, det, pk));
  if (dx) CK(launch_dgrad_c1(q.dp, 2 * cout, t.ka, t.kg, cout, Z, dx, n, H, W, kh, kw, L.sh, L.sw, st, pk));
  return 0;
}

// the input layer takes the fused kernels (option fuse_c1)
static bool c1_fused(const cgvc_engine* e, const Layer& L) {
  return e->opt.fuse_c1 && !use_tc(e, L.tc_slot) && L.a.cin == 1 && !L.has_in && L.a.kh * L.a.kw <= 9 && L.a.cout == 128;
}

// Packed utterances (A.off): the walk runs over one sample of all A.rows frames whose levels are packed 2-D grids, so n = 1 and T =
// A.rows below; each convolution keeps to its utterance and each instance norm takes its statistics over its utterance (A.seg)
static int discriminator_forward(cgvc_engine* e, const DiscNet& N, DiscActs& A, const float* x, cudaStream_t st, bool keep_y) {
  const int n = A.off ? 1 : A.n, T = A.off ? (int)A.rows : A.T, H0 = e->cfg.num_features;
  const float* Pm = e->P();
  A.x = x;
  ConvIO io; io.x = x; io.xhi = nullptr; io.xlo = nullptr; io.n = n; io.H = H0; io.W = T;
  if (A.off) io.pk = PackGeom{A.off, A.n, 1, A.max_len};
  int H = H0, W = T / 2;
  // input layer: one input channel, K = 9, gate without norm; P is kept for the backward pass
  const LayerTensors t1 = layer_tensors(e, N.h1, false);
  RET(disc_input_forward(e, N.h1, t1, x, n, H0, T, A.h1.P, post_params(e, N.h1, t1, io, A.h1, H * W, keep_y, A.post), c1_fused(e, N.h1), st,
                         packed(io)));
  const GLAct* cur = &A.h1;
  for (int i = 0; i < 3; ++i) {
    io.x = (keep_y || !cur->Yhi) ? cur->Y : nullptr; io.xhi = cur->Yhi; io.xlo = cur->Ylo; io.H = H; io.W = W;
    if (A.off) { io.pk.div = T / W; io.seg_out = A.seg[i]; }
    int Ho, Wo; conv_out_dims(N.d[i].a, N.d[i].sh, N.d[i].sw, H, W, Ho, Wo); H = Ho; W = Wo;
    // d3 has no planes: its fp32 output feeds the head
    RET(layer_forward(e, N.d[i], layer_tensors(e, N.d[i], false), io, A.d[i], H * W, keep_y, true, e->opt.fuse_in, A.post, st));
    cur = &A.d[i];
  }
  CK(launch_head_fwd(cur->Y, (long long)n * H * W, 1024, Pm + N.dense_k, Pm + N.dense_b, A.prob, st));
  if (keep_y) {
    e->taps.clear();
    e->taps["h1_glu"] = {A.h1.Y, (size_t)n * H0 * (T / 2) * 128};
    e->taps["d1"] = {A.d[0].Y, (size_t)n * (H0 / 2) * (T / 4) * 256};
    e->taps["d2"] = {A.d[1].Y, (size_t)n * (H0 / 4) * (T / 8) * 512};
    e->taps["d3"] = {A.d[2].Y, (size_t)n * (H0 / 4) * (T / 16) * 1024};
  }
  return 0;
}

// view of samples [s0, s0+ns) of a DiscActs
static DiscActs disc_view(const cgvc_engine* e, const DiscActs& A, int s0, int ns) {
  DiscActs V = A; V.n = ns;
  const int H = e->cfg.num_features, T = A.T;
  long long rows[4] = {(long long)H * (T / 2), (long long)(H / 2) * (T / 4), (long long)(H / 4) * (T / 8), (long long)(H / 4) * (T / 16)};
  const int co[4] = {128, 256, 512, 1024};
  GLAct* src[4] = {const_cast<GLAct*>(&A.h1), const_cast<GLAct*>(&A.d[0]), const_cast<GLAct*>(&A.d[1]), const_cast<GLAct*>(&A.d[2])};
  GLAct* dst[4] = {&V.h1, &V.d[0], &V.d[1], &V.d[2]};
  for (int i = 0; i < 4; ++i) {
    dst[i]->P = src[i]->P + (long long)s0 * rows[i] * 2 * co[i];
    dst[i]->stats = src[i]->stats + (long long)s0 * 4 * co[i];
    dst[i]->Y = src[i]->Y + (long long)s0 * rows[i] * co[i];
    dst[i]->Yhi = src[i]->Yhi ? src[i]->Yhi + (long long)s0 * rows[i] * co[i] : nullptr;
    dst[i]->Ylo = src[i]->Ylo ? src[i]->Ylo + (long long)s0 * rows[i] * co[i] : nullptr;
  }
  V.x = A.x + (long long)s0 * H * T;
  V.prob = A.prob + (long long)s0 * rows[3];
  return V;
}

// dY3: gradient w.r.t. the d3 GLU output [n*48, 1024].  wgrad: accumulate weight gradients.  d_in: optional [n,24,T].
// Packed utterances (A.off): over one sample of all A.rows frames, as discriminator_forward
static int discriminator_backward(cgvc_engine* e, const DiscNet& N, const DiscActs& A, const float* dY3, bool wgrad, float* d_in,
                                  const BwdScratch& S, cudaStream_t st) {
  const int n = A.off ? 1 : A.n, T = A.off ? (int)A.rows : A.T, H0 = e->cfg.num_features;
  int Hs[4] = {H0, H0 / 2, H0 / 4, H0 / 4}, Ws[4] = {T / 2, T / 4, T / 8, T / 16};   // output dims of h1, d1, d2, d3
  const float* dy = dY3;
  float* bufs[2] = {S.bufA, S.bufB};
  int flip = 0;
  BwdWalk w(S, false);
  for (int i = 2; i >= 0; --i) {
    const GLAct& in = (i == 0) ? A.h1 : A.d[i - 1];
    ConvIO io; io.x = in.Y; io.xhi = in.Yhi; io.xlo = in.Ylo; io.n = n; io.H = Hs[i]; io.W = Ws[i];
    if (A.off) { io.pk = PackGeom{A.off, A.n, T / Ws[i], A.max_len}; io.seg_out = A.seg[i]; }
    RET(layer_backward(e, w, N.d[i], A.d[i], io, dy, Hs[i + 1] * Ws[i + 1], wgrad, bufs[flip], 0, st));
    dy = bufs[flip]; flip ^= 1;
  }
  // h1: one input channel (K = 9), gate without instance norm.  Fused form: the GLU backward is recomputed inside the weight-gradient /
  // data-gradient kernels, dP never goes to HBM.  D.h1 has no tensor-core slot, so the unfused form's dP is fp32 (no planes)
  const LayerTensors t = layer_tensors(e, N.h1, wgrad);
  const PostBwdParams q = post_bwd_params(e, N.h1, t, dy, A.h1, n, Hs[0] * Ws[0], S, true, PlanePair{S.dPhi, S.dPlo});
  const PackGeom pk{A.off, A.n, 1, A.max_len};
  return disc_input_backward(e, N.h1, t, A.x, dy, A.h1.P, n, H0, T, d_in, bufs[flip], c1_fused(e, N.h1), q, det_of(S), st,
                             A.off ? &pk : nullptr);
}

// ---- workspace sizing ---------------------------------------------------------------------------------------
// The step is two symmetric, data-independent lanes that only meet in the (atomically accumulated) gradient arena and
// loss slots:   lane 0:  G_A2B([A;B]) -> [gen_B; id_B],  G_B2A(gen_B) -> cycle_A,  D_B([B; gen_B])
//               lane 1:  G_B2A([B;A]) -> [gen_A; id_A],  G_A2B(gen_A) -> cycle_B,  D_A([A; gen_A])
// They run on two streams so that one lane's HBM-bound kernels overlap the other lane's tensor-bound kernels.
struct LanePlan {
  GenActs gfirst, gcyc;         // batch 2B and B
  DiscActs d;                   // batch 2B
  float* in;                    // channels-last generator input [2B,T,24] = [X; Y]
  float* din;                   // discriminator input [2B,24,T] = [Y_real; gen_Y]
  float* d_cyc;                 // d cycle loss / d cycle_X, channels-last [B,T,24] (later reused as transpose scratch)
  float* d_out;                 // upstream gradient of the first pass [2B,T,24] = [d gen_Y; d id_Y]
  float* d_adv;                 // d G-adv / d gen_Y, [B,24,T]
  float* dY3;                   // [2B*48, 1024]
  BwdScratch S;
};
struct TrainPlan { LanePlan lane[2]; };

static void plan_train(cgvc_engine* e, Bump& ws, TrainPlan& P, int B, int T) {
  const int nf = e->cfg.num_features;
  const bool pl = e->cfg.precision != CGVC_PREC_FP32_SIMT;
  size_t img = (size_t)B * nf * T;
  size_t n2 = 2 * (size_t)B;
  size_t buf = n2 * (size_t)nf * (T / 2) * 128;            // largest dY: discriminator h1 output
  size_t bufg = n2 * (size_t)T * 256; if (bufg > buf) buf = bufg;
  size_t dp = n2 * (size_t)nf * (T / 2) * 256;             // largest dP: discriminator h1 conv output
  size_t dpg = n2 * (size_t)T * 512; if (dpg > dp) dp = dpg;
  for (int l = 0; l < 2; ++l) {
    LanePlan& L = P.lane[l];
    L.in = ws.take<float>(2 * img); L.din = ws.take<float>(2 * img);
    L.d_cyc = ws.take<float>(img); L.d_out = ws.take<float>(2 * img); L.d_adv = ws.take<float>(img);
    L.dY3 = ws.take<float>((size_t)2 * B * (nf / 4) * (T / 16) * 1024);
    L.S.bufA = ws.take<float>(buf); L.S.bufB = ws.take<float>(buf); L.S.dP = ws.take<float>(dp);
    L.S.dPhi = L.S.dPlo = L.S.dP2hi = L.S.dP2lo = nullptr;
    if (pl) {
      L.S.dPhi = ws.take<__nv_bfloat16>(dp); L.S.dPlo = ws.take<__nv_bfloat16>(dp);
      L.S.dP2hi = ws.take<__nv_bfloat16>(dpg); L.S.dP2lo = ws.take<__nv_bfloat16>(dpg);     // generator layers only
    }
    L.S.dPbhi = L.S.dPblo = nullptr;
    if (pl) { L.S.dPbhi = ws.take<__nv_bfloat16>(dp); L.S.dPblo = ws.take<__nv_bfloat16>(dp); }
    L.S.sq = &e->sideq[l];
    L.S.det = DetSlab{nullptr, 0};
    if (e->opt.deterministic) {
      // the weight-gradient partials are capped by CGVC_DET_SLAB_FLOATS (launch_tn lowers the split); the GLU / instance-norm bias partials,
      // one row of 2 x (conv columns) per 32 positions of a sample, grow with the batch and stay below dp / 8
      const long long slab = CGVC_DET_SLAB_FLOATS > (long long)(dp / 8) ? CGVC_DET_SLAB_FLOATS : (long long)(dp / 8);
      L.S.det = DetSlab{ws.take<float>((size_t)slab), slab};
    }
    L.S.post = ws.take<float>(n2 * 4 * 1024);
    plan_generator(e, ws, L.gfirst, 2 * B, T); plan_generator(e, ws, L.gcyc, B, T);
    plan_discriminator(e, ws, L.d, 2 * B, T);
    L.gfirst.post = L.gcyc.post = L.d.post = L.S.post;
  }
}

// The buffers of one network application: its input, kind 2's device offsets and the activations of its network (g or d)
struct AppPlan { GenActs g; DiscActs d; float* x; long long* off; };

// Lays out the buffers of application a from base: for a tape first the TapeHeader's kTapeHead bytes, then for kind 2 the n + 1
// device frame offsets (off), the input x (generator: channels-last rows [rows, 24]; discriminator: [n, 24, T]) and the activations,
// as a train step keeps them.  Returns the bytes it takes from base; a null base sizes it
static size_t plan_app(cgvc_engine* e, const NetGeom& a, void* base, bool tape, AppPlan& P) {
  const size_t head = tape ? kTapeHead : 0;
  Bump ws; ws.reset((char*)base + head, (size_t)1 << 62);
  // kind 3: the frame offsets, then the row prefix sums of the outputs of d1, d2 and d3 (DiscActs::seg), (n + 1) each
  P.off = packed_kind(a.kind) ? ws.take<long long>((size_t)(a.kind == 3 ? 4 : 1) * (a.n + 1)) : nullptr;
  P.x = ws.take<float>((size_t)a.rows * e->cfg.num_features);
  if (disc_kind(a.kind)) {
    plan_discriminator_rows(e, ws, P.d, a.n, a.rows);
    P.d.T = a.T; P.d.x = P.x;
    if (a.kind == 3) {
      P.d.off = P.off; P.d.max_len = a.max_len;
      for (int i = 0; i < 3; ++i) P.d.seg[i] = P.off + (size_t)(i + 1) * (a.n + 1);
    }
  } else {
    plan_generator_rows(e, ws, P.g, a.n, a.rows);
    P.g.T = a.T; P.g.off = P.off; P.g.max_len = a.max_len; P.g.x_cl = P.x;
  }
  return head + ws.off;
}

static size_t work_bytes_needed(cgvc_engine* e) {
  Bump ws; ws.reset(nullptr, 0);
  size_t need = 0;
  if (e->cfg.train) { TrainPlan P; plan_train(e, ws, P, e->cfg.max_batch, e->cfg.max_frames); need = ws.off; }
  for (int kind = 0; kind < 4; ++kind) {      // the forwards at their largest (kinds 2, 3: max_batch utterances of max_batch x max_frames rows)
    AppPlan F;
    const size_t fwd = plan_app(e, net_geom(kind, 0, e->cfg.max_batch, e->cfg.max_frames), nullptr, false, F);
    if (fwd > need) need = fwd;
  }
  if (e->opt.deterministic) {                 // the per-kernel entry points' slab (plan_entry_det)
    ws.reset(nullptr, 0); ws.take<float>((size_t)CGVC_DET_SLAB_FLOATS);
    if (ws.off > need) need = ws.off;
  }
  return need + 4096;
}

// Deterministic mode in a per-kernel entry point: the partials slab at the start of WORK, which work_bytes_needed reserves.  *det stays
// null outside deterministic mode; CGVC_ERR_UNBOUND when WORK is missing or too small
static int plan_entry_det(cgvc_engine* e, DetSlab* slab, const DetSlab** det) {
  *det = nullptr;
  if (!e->opt.deterministic) return 0;
  if (!e->arena[CGVC_ARENA_WORK]) return fail(e, CGVC_ERR_UNBOUND, "deterministic mode needs the WORK arena bound");
  Bump ws; ws.reset(e->arena[CGVC_ARENA_WORK], e->arena_bytes[CGVC_ARENA_WORK]);
  *slab = DetSlab{ws.take<float>((size_t)CGVC_DET_SLAB_FLOATS), CGVC_DET_SLAB_FLOATS};
  if (ws.overflow) return fail(e, CGVC_ERR_UNBOUND, "WORK arena too small for the deterministic partials slab");
  *det = slab;
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------
extern "C" {

int cgvc_abi_version(void) { return CGVC_ABI_VERSION; }

const char* cgvc_last_error(cgvc_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int cgvc_create(const cgvc_config* cfg, cgvc_handle* out) {
  if (!cfg || !out) return fail(nullptr, CGVC_ERR_ARG, "cgvc_create: null argument");
  if (cfg->num_features != 24) return fail(nullptr, CGVC_ERR_ARG, "only num_features = 24 is supported (got %d)", cfg->num_features);
  if (cfg->max_batch < 1 || cfg->max_frames < 16 || cfg->max_frames % 4 != 0)
    return fail(nullptr, CGVC_ERR_ARG, "max_batch must be >= 1 and max_frames a multiple of 4, >= 16");
  if (cfg->precision < 0 || cfg->precision > 3) return fail(nullptr, CGVC_ERR_ARG, "unknown precision %d", cfg->precision);
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(nullptr, CGVC_ERR_CUDA, "no CUDA device available (%s): libcgvc has no CPU fallback", cudaGetErrorString(ce));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, CGVC_ERR_ARG, "device %d out of range (%d devices)", cfg->device, ndev);
  DeviceGuard dguard;
  ce = dguard.set(cfg->device);
  if (ce != cudaSuccess) return fail(nullptr, CGVC_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(ce));
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, cfg->device);
  if (prop.major != 9 || prop.minor != 0) return fail(nullptr, CGVC_ERR_CUDA, "libcgvc is built for sm_90a only; device is sm_%d%d", prop.major, prop.minor);
  cgvc_engine* e = new cgvc_engine();
  e->cfg = *cfg;
  e->id = ++g_engine_ids;
  TableBuilder tb{e->tensors};
  const char* gn[2] = {"generator_A2B", "generator_B2A"}; const char* dn[2] = {"discriminator_A", "discriminator_B"};
  for (int i = 0; i < 2; ++i) { tb.scope = gn[i]; build_generator(tb, e->gen[i], cfg->num_features); }
  for (int i = 0; i < 2; ++i) { tb.scope = dn[i]; build_discriminator(tb, e->disc[i]); }
  e->n_params = (tb.off + 3) & ~(size_t)3;
  e->n_real_params = tb.real;
  ce = post_init_kernels();
  if (ce != cudaSuccess) { delete e; return fail(nullptr, CGVC_ERR_CUDA, "post_init_kernels: %s", cudaGetErrorString(ce)); }
  ce = cudaMalloc(&e->d_scalars, 64 * sizeof(float));
  if (ce != cudaSuccess) { delete e; return fail(nullptr, CGVC_ERR_CUDA, "cudaMalloc scalars: %s", cudaGetErrorString(ce)); }
  cudaMemset(e->d_scalars, 0, 64 * sizeof(float));
  {
    float st[10];
    for (int l = 0; l < 10; ++l) st[l] = loss_scale(e, 1 << l);
    cudaMemcpy(e->d_scalars + 16, st, sizeof st, cudaMemcpyHostToDevice);
  }
  ce = cudaMalloc(&e->ls, sizeof(LossScaler));
  if (ce != cudaSuccess) { cudaFree(e->d_scalars); delete e; return fail(nullptr, CGVC_ERR_CUDA, "cudaMalloc loss scaler: %s", cudaGetErrorString(ce)); }
  cudaMemset(e->ls, 0, sizeof(LossScaler));
  cudaEventCreateWithFlags(&e->ev_ls, cudaEventDisableTiming);
  for (int l = 0; l < 2; ++l) { cudaStreamCreateWithFlags(&e->lane_stream[l], cudaStreamNonBlocking); cudaEventCreateWithFlags(&e->ev_join[l], cudaEventDisableTiming); }
  cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming);
  { int lo = 0, hi = 0; cudaDeviceGetStreamPriorityRange(&lo, &hi); cudaStreamCreateWithPriority(&e->comm_stream, cudaStreamNonBlocking, hi); }
  cudaEventCreateWithFlags(&e->ev_grads, cudaEventDisableTiming);
  for (int k = 0; k < 4; ++k) cudaEventCreateWithFlags(&e->ev_ar[k], cudaEventDisableTiming);
  for (int l = 0; l < 2; ++l) {
    cudaStreamCreateWithFlags(&e->sideq[l].side, cudaStreamNonBlocking);
    for (int b = 0; b < 2; ++b) { cudaEventCreateWithFlags(&e->sideq[l].ready[b], cudaEventDisableTiming); cudaEventCreateWithFlags(&e->sideq[l].done[b], cudaEventDisableTiming); }
  }
  cudaStreamCreateWithFlags(&e->graph_stream, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&e->ev_bridge, cudaEventDisableTiming); cudaEventCreateWithFlags(&e->ev_bridge2, cudaEventDisableTiming);
  if (cfg->precision != CGVC_PREC_FP32_SIMT) {
    // register every dense layer with the tensor-core weight store (in this order: the F16F8 plane jobs of a network are contiguous)
    auto reg = [&](Layer& L) {
      L.tc_slot = tc_register(e->tcw, L.a.k, L.g.k, L.a.b, L.g.b, L.a.kh, L.a.kw, L.a.cin, L.a.cout, L.gated(), L.shuffle);
    };
    for (int i = 0; i < 2; ++i) {
      GenNet& g = e->gen[i];
      // the 24-channel edge layers run on the tensor cores too (channel dims zero-padded to 64 / 128 inside the planes)
      reg(g.h1); reg(g.o1);
      // ... and, preferred (edge_lower), as dense 1 x 1 layers with the taps in the channel (h1) / column (o1) dimension: see edge_on
      const ConvW &h1 = g.h1.a, &o1 = g.o1.a;
      if ((h1.kw * h1.cin) % 4 == 0 && o1.cout % 4 == 0) {
        g.h1c_slot = tc_register(e->tcw, h1.k, g.h1.g.k, h1.b, g.h1.g.b, 1, 1, h1.kw * h1.cin, h1.cout, 1);
        g.o1f_slot = tc_register(e->tcw, o1.k, 0, o1.b, 0, 1, 1, o1.cin, o1.kw * o1.cout, 0, 1, o1.kw);
      }
      for (Layer& L : g.d) reg(L);
      for (ResBlock& R : g.r) { reg(R.h1); reg(R.h2); }
      for (Layer& L : g.u) reg(L);
      for (Layer& L : e->disc[i].d) reg(L);
    }
    int r = tc_alloc(e->tcw, cfg->precision, cfg->train);
    if (r != 0) { std::string m = cudaGetErrorString((cudaError_t)r); cudaFree(e->d_scalars); cudaFree(e->ls); delete e; return fail(nullptr, CGVC_ERR_CUDA, "tc_alloc: %s", m.c_str()); }
  }
  *out = e;
  return 0;
}

int cgvc_destroy(cgvc_handle e) {
  if (!e) return 0;
  DeviceGuard dguard; dguard.set(e->cfg.device);
  if (e->comm && e->nccl.CommDestroy) e->nccl.CommDestroy(e->comm);
  tc_free(e->tcw);
  for (int l = 0; l < 2; ++l) { if (e->lane_stream[l]) cudaStreamDestroy(e->lane_stream[l]); if (e->ev_join[l]) cudaEventDestroy(e->ev_join[l]); }
  if (e->ev_fork) cudaEventDestroy(e->ev_fork);
  if (e->comm_stream) cudaStreamDestroy(e->comm_stream);
  if (e->ev_grads) cudaEventDestroy(e->ev_grads);
  for (int k = 0; k < 4; ++k) if (e->ev_ar[k]) cudaEventDestroy(e->ev_ar[k]);
  for (int l = 0; l < 2; ++l) {
    if (e->sideq[l].side) cudaStreamDestroy(e->sideq[l].side);
    for (int b = 0; b < 2; ++b) { if (e->sideq[l].ready[b]) cudaEventDestroy(e->sideq[l].ready[b]); if (e->sideq[l].done[b]) cudaEventDestroy(e->sideq[l].done[b]); }
  }
  drop_graphs(e);
  if (e->stage) cudaFree(e->stage);
  cudaFree(e->post_buf);
  if (e->graph_stream) cudaStreamDestroy(e->graph_stream);
  if (e->ev_bridge) cudaEventDestroy(e->ev_bridge);
  if (e->ev_bridge2) cudaEventDestroy(e->ev_bridge2);
  cudaFree(e->d_scalars);
  cudaFree(e->ls);
  if (e->ev_ls) cudaEventDestroy(e->ev_ls);
  delete e;
  return 0;
}

int cgvc_arena_bytes(cgvc_handle e, int arena, size_t* bytes) {
  if (!e || !bytes || arena < 0 || arena >= CGVC_ARENA_COUNT) return fail(e, CGVC_ERR_ARG, "cgvc_arena_bytes: bad argument");
  if (arena == CGVC_ARENA_WORK) *bytes = work_bytes_needed(e);
  else *bytes = ((e->n_params * sizeof(float)) + 255) & ~(size_t)255;
  return 0;
}

int cgvc_bind_arena(cgvc_handle e, int arena, void* p, size_t bytes) {
  if (!e || arena < 0 || arena >= CGVC_ARENA_COUNT) return fail(e, CGVC_ERR_ARG, "cgvc_bind_arena: bad argument");
  size_t need; cgvc_arena_bytes(e, arena, &need);
  if (!p || bytes < need) return fail(e, CGVC_ERR_UNBOUND, "arena %d needs %zu bytes, got %zu", arena, need, bytes);
  if ((uintptr_t)p & 255) return fail(e, CGVC_ERR_ARG, "arena %d must be 256-byte aligned", arena);
  e->arena[arena] = p; e->arena_bytes[arena] = bytes;
  drop_graphs(e);
  ++e->param_gen;
  return 0;
}

int cgvc_param_count(cgvc_handle e, int* n_tensors, size_t* n_elements) {
  if (!e) return CGVC_ERR_ARG;
  if (n_tensors) *n_tensors = (int)e->tensors.size();
  if (n_elements) *n_elements = e->n_real_params;
  return 0;
}

int cgvc_param_info(cgvc_handle e, int index, const char** name, size_t* offset, int* ndim, int shape_out[4]) {
  if (!e || index < 0 || index >= (int)e->tensors.size()) return fail(e, CGVC_ERR_ARG, "cgvc_param_info: index out of range");
  const TensorInfo& t = e->tensors[index];
  if (name) *name = t.name.c_str();
  if (offset) *offset = t.off;
  if (ndim) *ndim = t.ndim;
  if (shape_out) for (int i = 0; i < 4; ++i) shape_out[i] = t.shape[i];
  return 0;
}

static int need_arenas(cgvc_engine* e, bool train) {
  if (!e->arena[CGVC_ARENA_PARAM] || !e->arena[CGVC_ARENA_WORK]) return fail(e, CGVC_ERR_UNBOUND, "PARAM and WORK arenas must be bound");
  if (train && (!e->arena[CGVC_ARENA_GRAD])) return fail(e, CGVC_ERR_UNBOUND, "GRAD arena must be bound");
  return 0;
}

int cgvc_params_updated(cgvc_handle e, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if (!e->arena[CGVC_ARENA_PARAM]) return fail(e, CGVC_ERR_UNBOUND, "PARAM arena must be bound");
  ++e->param_gen;
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  if (e->cfg.precision != CGVC_PREC_FP32_SIMT) {
    int r = tc_refresh_weights(e->tcw, e->P(), (cudaStream_t)stream);
    if (r != 0) return fail(e, CGVC_ERR_CUDA, "tc_refresh_weights: %s", cudaGetErrorString((cudaError_t)r));
  }
  return 0;
}

// in dynamic loss-scale mode the step count lives on the device (the scaler advances it): these two synchronise the device
int cgvc_set_adam_step(cgvc_handle e, long long t) {
  if (!e || t < 0) return CGVC_ERR_ARG;
  e->adam_t = t;
  if (e->opt.ls_mode == 2) {
    DeviceGuard dguard; CK(dguard.set(e->cfg.device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(&e->ls->t, &t, sizeof t, cudaMemcpyHostToDevice));
  }
  return 0;
}
int cgvc_get_adam_step(cgvc_handle e, long long* t) {
  if (!e || !t) return CGVC_ERR_ARG;
  if (e->opt.ls_mode == 2) {
    DeviceGuard dguard; CK(dguard.set(e->cfg.device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(&e->adam_t, &e->ls->t, sizeof e->adam_t, cudaMemcpyDeviceToHost));
  }
  *t = e->adam_t;
  return 0;
}

static_assert(sizeof(cgvc_loss_scale_info) == offsetof(LossScaler, t) && offsetof(cgvc_loss_scale_info, sat_act) == offsetof(LossScaler, sat_act) &&
              offsetof(cgvc_loss_scale_info, nonfinite) == offsetof(LossScaler, nonfinite) && offsetof(cgvc_loss_scale_info, skipped) == offsetof(LossScaler, skipped),
              "cgvc_loss_scale_info is the head of LossScaler");
int cgvc_loss_scale_state(cgvc_handle e, cgvc_loss_scale_info* out_dev, void* stream) {
  if (!e || !out_dev) return fail(e, CGVC_ERR_ARG, "null argument");
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(cudaMemcpyAsync(out_dev, e->ls, sizeof(cgvc_loss_scale_info), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}
int cgvc_set_loss_scale_state(cgvc_handle e, float scale, int good_steps, long long skipped, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if (!(scale >= 1.f && scale <= 16777216.f) || good_steps < 0 || skipped < 0)
    return fail(e, CGVC_ERR_ARG, "cgvc_set_loss_scale_state: scale %g outside [1, 2^24] or negative counts", (double)scale);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  const cgvc_loss_scale_info v{scale, good_steps, skipped, 0, 0, 0, 0};     // the last step's flag and counters cleared
  const LossScaler::Net n{scale, good_steps};                                  // both networks' scales (per-network option)
  CK(cudaMemcpyAsync(e->ls, &v, sizeof v, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  for (int k = 0; k < 2; ++k) CK(cudaMemcpyAsync(&e->ls->net[k], &n, sizeof n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  CK(cudaMemsetAsync(e->ls->cnt, 0, sizeof e->ls->cnt, (cudaStream_t)stream));
  CK(cudaStreamSynchronize((cudaStream_t)stream));           // v and n live on this stack frame
  e->ls_ready = true;
  return 0;
}

static_assert(sizeof(cgvc_loss_scale_net_info) == sizeof(LossScaler::Net) + sizeof(unsigned long long[3]) &&
              offsetof(cgvc_loss_scale_net_info, good_steps) == offsetof(LossScaler::Net, good_steps) &&
              offsetof(cgvc_loss_scale_net_info, sat_grad) == sizeof(LossScaler::Net) &&
              offsetof(cgvc_loss_scale_info, good_steps) == offsetof(LossScaler::Net, good_steps),
              "cgvc_loss_scale_net_info is a LossScaler::Net followed by that network's counters");
int cgvc_loss_scale_net_state(cgvc_handle e, cgvc_loss_scale_net_info* out_dev, void* stream) {
  if (!e || !out_dev) return fail(e, CGVC_ERR_ARG, "null argument");
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  for (int k = 0; k < 2; ++k) {
    CK(cudaMemcpyAsync(&out_dev[k], &e->ls->net[k], sizeof(LossScaler::Net), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    CK(cudaMemcpyAsync(&out_dev[k].sat_grad, e->ls->cnt[k], sizeof e->ls->cnt[k], cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  }
  return 0;
}
int cgvc_set_loss_scale_net_state(cgvc_handle e, int net, float scale, int good_steps, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if ((net != 0 && net != 1) || !(scale >= 1.f && scale <= 16777216.f) || good_steps < 0)
    return fail(e, CGVC_ERR_ARG, "cgvc_set_loss_scale_net_state: net %d not 0 or 1, scale %g outside [1, 2^24] or negative count", net,
                (double)scale);
  // no scale set yet: the other network starts from the same one
  if (!e->ls_ready) RET(cgvc_set_loss_scale_state(e, scale, good_steps, 0, stream));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  const LossScaler::Net n{scale, good_steps};
  CK(cudaMemcpyAsync(&e->ls->net[net], &n, sizeof n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  if (net == 0) CK(cudaMemcpyAsync(&e->ls->scale, &scale, sizeof scale, cudaMemcpyHostToDevice, (cudaStream_t)stream));   // scale is s_G
  CK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}
int cgvc_set_plane_counters(cgvc_handle e, unsigned long long* ufl_groups_dev) {
  if (!e) return CGVC_ERR_ARG;
  e->plane_ufl = ufl_groups_dev;
  return 0;
}

static int check_bt(cgvc_engine* e, int batch, int frames, int mult) {
  if (batch < 1 || batch > e->cfg.max_batch) return fail(e, CGVC_ERR_ARG, "batch %d outside [1, %d]", batch, e->cfg.max_batch);
  if (frames < mult || frames % mult != 0 || frames > e->cfg.max_frames)
    return fail(e, CGVC_ERR_ARG, "frames %d must be a multiple of %d in [%d, %d]", frames, mult, mult, e->cfg.max_frames);
  return 0;
}

int cgvc_debug_activation(cgvc_handle e, const char* name, float* out_dev, size_t capacity, size_t* n_out, void* stream) {
  if (!e || !name) return CGVC_ERR_ARG;
  auto it = e->taps.find(name);
  if (it == e->taps.end()) return fail(e, CGVC_ERR_ARG, "no activation tap named '%s' (generator taps need the 'debug_taps' option set before the forward call)", name);
  if (n_out) *n_out = it->second.second;
  if (out_dev) {
    if (capacity < it->second.second) return fail(e, CGVC_ERR_ARG, "tap '%s' needs %zu elements", name, it->second.second);
    CK(cudaMemcpyAsync(out_dev, it->second.first, it->second.second * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  }
  return 0;
}

int cgvc_weight_planes(cgvc_handle e, int layer, cgvc_weight_layer_info* info, const char* plane, void* out_dev, size_t capacity,
                       size_t* bytes_out, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  const int n = (int)e->tcw.layers.size();
  if (layer < 0 || layer >= n) return fail(e, CGVC_ERR_ARG, "cgvc_weight_planes: layer %d outside [0, %d)", layer, n);
  const TcLayer& L = e->tcw.layers[layer];
  if (info) {
    int d[7]; tc_layer_dims(e->tcw, layer, d);
    *info = cgvc_weight_layer_info{n, L.kh, L.kw, L.cin, L.cout, L.gated, L.shuffle, L.fold,
                                   (long long)L.ka, (long long)L.kg, (long long)L.ba, (long long)L.bg, d[0], d[1], d[2], d[3], d[4], d[5], d[6]};
  }
  if (!plane) return 0;
  const void* src = nullptr; size_t bytes = 0;
  if (tc_layer_plane(e->tcw, layer, plane, &src, &bytes) != 0) return fail(e, CGVC_ERR_ARG, "cgvc_weight_planes: unknown plane '%s'", plane);
  if (!src) return fail(e, CGVC_ERR_ARG, "cgvc_weight_planes: layer %d keeps no plane '%s' in this engine", layer, plane);
  if (bytes_out) *bytes_out = bytes;
  if (!out_dev) return 0;
  if (capacity < bytes) return fail(e, CGVC_ERR_ARG, "cgvc_weight_planes: plane '%s' of layer %d needs %zu bytes", plane, layer, bytes);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CK(cudaStreamIsCapturing((cudaStream_t)stream, &cs));
  if (cs != cudaStreamCaptureStatusNone) return fail(e, CGVC_ERR_ARG, "cgvc_weight_planes: stream is capturing a graph");
  CK(cudaMemcpyAsync(out_dev, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

// forward + losses + backward of one training step; leaves gradients in GRAD (model.py:44-90,107-108)
// one lane of the step (see LanePlan), enqueued on stream st
static int run_lane(cgvc_engine* e, LanePlan& L, int lane, const float* Yreal_dev, int B, int T, float lambda_identity,
                    float* gen_out_dev, cudaStream_t st) {
  const int nf = e->cfg.num_features;
  const size_t img = (size_t)B * nf * T;
  float* Gm = e->G(); const float* Pm = e->P();
  float* sc = e->d_scalars; float* Ls = sc + 8;
  const GenNet& Gfirst = e->gen[lane];          // lane 0: generator_A2B ; lane 1: generator_B2A
  const GenNet& Gcyc = e->gen[1 - lane];
  const DiscNet& DN = e->disc[1 - lane];        // lane 0 judges domain B (discriminator_B); lane 1 domain A
  const float* X_cl = L.in; const float* Y_cl = L.in + img;
  // ---- forward (model.py:44-54,75-78) ----
  RET(generator_forward(e, Gfirst, L.gfirst, L.in, st, false));             // [gen_Y ; id_Y]
  const float* genY_cl = L.gfirst.out_cl; const float* idY_cl = L.gfirst.out_cl + img;
  RET(generator_forward(e, Gcyc, L.gcyc, genY_cl, st, false));              // cycle_X
  CK(cudaMemcpyAsync(L.din, Yreal_dev, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CK(launch_transpose_ft(genY_cl, L.din + img, B, T, nf, st));
  if (gen_out_dev) CK(cudaMemcpyAsync(gen_out_dev, L.din + img, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
  RET(discriminator_forward(e, DN, L.d, L.din, st, false));
  // ---- losses and their gradients (model.py:57-90) ----
  // the loss scale multiplies every gradient of the step (not the loss values); Adam divides it out.  Per network, the D-loss pass
  // (its heads and everything they back-propagate) takes s_D, the generators' losses s_G
  e->ls_net = 0;
  const float* ls = loss_scale_dev(e, B);
  e->ls_net = 1;
  const float* lsD = loss_scale_dev(e, B);
  const DetSlab* det = det_of(L.S);
  CK(launch_l1_loss_grad(L.gcyc.out_cl, X_cl, (long long)img, Ls + 0, sc + 0, L.d_cyc, 0, st, ls, det));     // cycle term
  CK(launch_l1_loss_grad(idY_cl, Y_cl, (long long)img, Ls + 1, sc + 1, L.d_out + img, 0, st, ls, det));      // identity term
  const long long hrows = (long long)B * (nf / 4) * (T / 16);   // head rows per half
  const float* Y3 = L.d.d[2].Y;
  float* Dslot = Ls + (lane == 0 ? 6 : 5);                      // discriminator_loss_B / _A
  float* Gslot = Ls + (lane == 0 ? 2 : 3);                      // generator_loss_A2B / _B2A
  // discriminator loss: real half -> target 1, fake half -> target 0, each weighted 1/2 (model.py:81-88)
  CK(launch_head_loss_bwd(L.d.prob, Y3, hrows, 1024, Pm + DN.dense_k, 1.f, 0.5f, Dslot, L.dY3, Gm + DN.dense_k, Gm + DN.dense_b, st, lsD, det));
  CK(launch_head_loss_bwd(L.d.prob + hrows, Y3 + hrows * 1024, hrows, 1024, Pm + DN.dense_k, 0.f, 0.5f, Dslot,
                          L.dY3 + hrows * 1024, Gm + DN.dense_k, Gm + DN.dense_b, st, lsD, det));
  RET(discriminator_backward(e, DN, L.d, L.dY3, true, nullptr, L.S, st));
  e->ls_net = 0;                                                // the rest of the lane is the generators' pass
  // generator adversarial loss on the fake half: target 1 (model.py:68-69); the gradient flows to the fake only
  DiscActs V = disc_view(e, L.d, B, B);
  CK(launch_head_loss_bwd(V.prob, V.d[2].Y, hrows, 1024, Pm + DN.dense_k, 1.f, 1.f, Gslot, L.dY3, nullptr, nullptr, st, ls, det));
  RET(discriminator_backward(e, DN, V, L.dY3, false, L.d_adv, L.S, st));
  // ---- generator backward ----
  // cycle pass: G_{Y->X}(gen_Y) <- d cycle_X ; its input gradient is the first half of the first pass's upstream
  RET(generator_backward(e, Gcyc, L.gcyc, L.d_cyc, L.d_out, L.S, st));
  CK(launch_transpose_ft(L.d_adv, L.d_cyc, B, nf, T, st));      // adversarial gradient [B,24,T] -> channels-last (d_cyc is free now)
  CK(launch_add(L.d_out, L.d_cyc, L.d_out, (long long)img, st));
  if (lambda_identity == 0.f) {
    // train.py:98-99 switches the identity loss off after 10k iterations (it is still computed and logged, model.py:157):
    // its upstream gradient is then exactly zero, so only the gen_Y half of the first pass is back-propagated
    GenActs half = L.gfirst; half.n = B;
    RET(generator_backward(e, Gfirst, half, L.d_out, nullptr, L.S, st));
  } else {
    RET(generator_backward(e, Gfirst, L.gfirst, L.d_out, nullptr, L.S, st));
  }
  side_join(L.S, st);                                        // the side-stream weight gradients rejoin the lane
  return 0;
}

// forward + losses + backward of one training step; leaves gradients in GRAD (model.py:44-90,107-108)
static int forward_backward(cgvc_engine* e, const float* A_dev, const float* B_dev, int B, int T, float lc, float li,
                            float* gen_A_dev, float* gen_B_dev, float* losses_dev, cudaStream_t st) {
  const int nf = e->cfg.num_features;
  RET(check_bt(e, B, T, 16));
  if (!e->cfg.train) return fail(e, CGVC_ERR_ARG, "engine was created with train = 0");
  RET(need_arenas(e, true));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  Bump ws; ws.reset(e->arena[CGVC_ARENA_WORK], e->arena_bytes[CGVC_ARENA_WORK]);
  TrainPlan P; plan_train(e, ws, P, B, T);
  if (ws.overflow) return fail(e, CGVC_ERR_UNBOUND, "WORK arena too small for batch %d x %d frames", B, T);
  const size_t img = (size_t)B * nf * T;
  float* sc = e->d_scalars; float* L = sc + 8;
  (void)lc;                                                  // lambdas are already in d_scalars[0..1] (set_step_scalars)
  CK(cudaMemsetAsync(L, 0, 8 * sizeof(float), st));
  if (e->opt.ls_mode) CK(cudaMemsetAsync(&e->ls->nonfinite, 0, (char*)(&e->ls->sat_act + 1) - (char*)&e->ls->nonfinite, st));   // this step's counters
  if (ls_nets(e)) CK(cudaMemsetAsync(e->ls->cnt, 0, sizeof e->ls->cnt, st));
  struct Counting { cgvc_engine* e; ~Counting() { e->counting = false; } } counting{e};
  e->counting = true;
  CK(cudaMemsetAsync(e->G(), 0, e->n_params * sizeof(float), st));
  // channels-last copies of the real samples: lane 0 reads [A;B], lane 1 [B;A]
  CK(launch_transpose_ft(A_dev, P.lane[0].in, B, nf, T, st));
  CK(launch_transpose_ft(B_dev, P.lane[0].in + img, B, nf, T, st));
  CK(cudaMemcpyAsync(P.lane[1].in, P.lane[0].in + img, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(P.lane[1].in + img, P.lane[0].in, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
  for (int l = 0; l < 2; ++l) {
    SideQ& q = e->sideq[l];
    q.on = e->opt.side_wgrad && e->opt.two_streams && !e->opt.fuse_bwd && !e->opt.deterministic && !tc_profile_is_on() && q.side != nullptr;
    q.used[0] = q.used[1] = false; q.cur = 0;
  }
  if (e->opt.two_streams) {
    // fork
    CK(cudaEventRecord(e->ev_fork, st));
    for (int l = 0; l < 2; ++l) CK(cudaStreamWaitEvent(e->lane_stream[l], e->ev_fork, 0));
    RET(run_lane(e, P.lane[0], 0, B_dev, B, T, li, gen_B_dev, e->lane_stream[0]));
    RET(run_lane(e, P.lane[1], 1, A_dev, B, T, li, gen_A_dev, e->lane_stream[1]));
    // join
    for (int l = 0; l < 2; ++l) { CK(cudaEventRecord(e->ev_join[l], e->lane_stream[l])); CK(cudaStreamWaitEvent(st, e->ev_join[l], 0)); }
  } else {
    RET(run_lane(e, P.lane[0], 0, B_dev, B, T, li, gen_B_dev, st));
    RET(run_lane(e, P.lane[1], 1, A_dev, B, T, li, gen_A_dev, st));
  }
  CK(launch_finalize_losses(L, sc, st));
  if (losses_dev) CK(cudaMemcpyAsync(losses_dev, L, 8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // extern "C"

// d_scalars: [0..1] lambda_cycle, lambda_identity; [2..3] generator Adam (lr_t, grad_scale); [4..5] discriminator Adam
static int set_lambdas(cgvc_engine* e, float lc, float li, cudaStream_t st) {
  float v[6] = {lc, li, 0, 0, 0, 0};
  CK(launch_set_scalars(e->d_scalars, 0, 2, v, st));
  return 0;
}
// deferred (a train step in dynamic loss-scale mode): see below
static int set_adam_scalars(cgvc_engine* e, float lr_g, float lr_d, float grad_scale, cudaStream_t st, bool deferred = false) {
  e->adam_t += 1;                                            // both optimizers advance once per train() (Appendix A.6)
  if (deferred) {
    // dynamic loss scale: t lives on the device and only the scaler knows whether this step goes through; it turns these raw values
    // into lr_t and the grad_scale (loss_scale_update_kernel)
    float v[6] = {lr_g, grad_scale, lr_d, grad_scale, 0, 0};
    CK(launch_set_scalars(e->d_scalars, 2, 4, v, st));
    return 0;
  }
  double t = (double)e->adam_t;
  double corr = sqrt(1.0 - pow((double)ADAM_B2, t)) / (1.0 - pow((double)ADAM_B1, t));
  float v[6] = {(float)(lr_g * corr), grad_scale, (float)(lr_d * corr), grad_scale, 0, 0};
  CK(launch_set_scalars(e->d_scalars, 2, 4, v, st));
  return 0;
}
// the capturable part of the optimizer step: two Adam ranges + refresh of the tensor-core weight planes
static int adam_body(cgvc_engine* e, cudaStream_t st, const int* skip = nullptr) {
  float* p = e->P(); float* g = e->G(); float* m = (float*)e->arena[CGVC_ARENA_ADAM_M]; float* v = (float*)e->arena[CGVC_ARENA_ADAM_V];
  size_t gend = e->gen[1].end;   // generators occupy [0, gend), discriminators [gend, n_params)  (model.py:94-95)
  CK(launch_adam(p, g, m, v, (long long)gend, e->d_scalars + 2, ADAM_B1, ADAM_B2, ADAM_EPS, st, skip));
  CK(launch_adam(p + gend, g + gend, m + gend, v + gend, (long long)(e->n_params - gend), e->d_scalars + 4, ADAM_B1, ADAM_B2, ADAM_EPS, st, skip));
  return cgvc_params_updated(e, (void*)st);
}

// Loss scaling after the gradients are complete (and summed over ranks): the non-finite check of GRAD per optimizer range, then in
// dynamic mode the scaler update, whose skip word the Adam kernels read
static int ls_check_grads(cgvc_engine* e, cudaStream_t st) {
  CK(launch_check_finite(e->G(), (long long)e->n_params, (long long)e->gen[1].end, &e->ls->nonfinite, st));
  return 0;
}
// dynamic mode; per network also monitor mode, where it only sums the networks' counts into sat_grad
static int ls_update(cgvc_engine* e, cudaStream_t st) {
  const int nets = ls_nets(e) ? (e->opt.ls_mode == 2 ? 1 : 2) : 0;
  CK(launch_loss_scale_update(e->ls, e->d_scalars + 2, e->cfg.precision == CGVC_PREC_F16F8, e->opt.ls_growth, ADAM_B1, ADAM_B2, st, nets));
  return 0;
}
// the saturation counts summed over ranks, so that every rank takes the same decision (dynamic mode): per network both blocks at once
static int ls_allreduce_counts(cgvc_engine* e, cudaStream_t st) {
  unsigned long long* c = ls_nets(e) ? e->ls->cnt[0] : &e->ls->sat_grad;
  const size_t n = ls_nets(e) ? sizeof e->ls->cnt / sizeof(unsigned long long) : 1;
  int r = e->nccl.AllReduce(c, c, n, 5, 0, e->comm, st);                                                    // ncclUint64, ncclSum
  if (r != 0) return fail(e, CGVC_ERR_NCCL, "ncclAllReduce: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(r) : "?");
  return 0;
}
static const int* ls_skip(const cgvc_engine* e) { return e->opt.ls_mode == 2 ? &e->ls->last_skipped : nullptr; }

// Before a step is enqueued: dynamic mode starts from the static scale of the step's batch unless the caller set one
// (cgvc_set_loss_scale_state); monitor mode reports the static scale in use
static int ls_prepare(cgvc_engine* e, int batch, cudaStream_t st) {
  const bool dyn = e->opt.ls_mode == 2 && !e->ls_ready, mon = e->opt.ls_mode == 1 && e->ls_batch != batch;
  if (!dyn && !mon) return 0;
  const float v[6] = {loss_scale(e, batch), 0, 0, 0, 0, 0};
  CK(launch_set_scalars(&e->ls->scale, 0, 1, v, st));
  if (ls_nets(e)) for (int k = 0; k < 2; ++k) CK(launch_set_scalars(&e->ls->net[k].scale, 0, 1, v, st));
  e->ls_ready = e->opt.ls_mode == 2; e->ls_batch = e->opt.ls_mode == 1 ? batch : 0;
  return 0;
}

// ---- CUDA graphs: the ~650 launches of a step are captured once per (buffers, batch, frames, identity-on/off) and replayed.
// Everything inside the captured bodies reads its per-step scalars from d_scalars (written by the eager set_scalars kernel),
// so a replay is exact.  Capture needs a non-legacy stream: work arriving on the legacy default stream is bridged with events.
template <class Body>
static int run_captured(cgvc_engine* e, const GraphKey& key, cudaStream_t user, Body body) {
  if (!e->opt.use_graphs || tc_profile_is_on()) return body(user);
  cudaStream_t st = user;
  const bool bridge = (user == nullptr || user == cudaStreamLegacy || user == cudaStreamPerThread);
  if (bridge) { st = e->graph_stream; CK(cudaEventRecord(e->ev_bridge, user)); CK(cudaStreamWaitEvent(st, e->ev_bridge, 0)); }
  auto it = e->graphs.find(key);
  GraphEntry ent{nullptr, 0};
  if (it != e->graphs.end()) ent = it->second;
  else {
    if (e->graphs.size() >= 16) drop_graphs(e);
    cudaGraph_t graph = nullptr;
    const unsigned long long before = g_cgvc_launches;
    cudaError_t ce = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) { cudaGetLastError(); e->opt.use_graphs = 0; return body(user); }
    int rc = body(st);
    ce = cudaStreamEndCapture(st, &graph);
    ent.launches = g_cgvc_launches - before;                 // kernels recorded, not run: counted per replay below
    g_cgvc_launches = before;
    if (rc != 0 || ce != cudaSuccess || !graph) {
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      if (rc != 0 && ce == cudaSuccess) return rc;           // the body itself refused (bad argument, arena too small): not a capture problem
      e->opt.use_graphs = 0;                                     // fall back to eager launches for the rest of this engine's life
      return body(user);
    }
    ce = cudaGraphInstantiate(&ent.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) { cudaGetLastError(); e->opt.use_graphs = 0; return body(user); }
    e->graphs[key] = ent;
  }
  cudaGraphExec_t exec = ent.exec;
  g_cgvc_launches += ent.launches;
  CK(cudaGraphLaunch(exec, st));
  if (bridge) { CK(cudaEventRecord(e->ev_bridge2, st)); CK(cudaStreamWaitEvent(user, e->ev_bridge2, 0)); }
  return 0;
}

// The step's WORK plan fits the bound arena (checked before anything is enqueued: a call refused for a short WORK -- e.g. after
// "deterministic" was switched on without re-binding -- launches nothing)
static int check_work_train(cgvc_engine* e, int batch, int frames) {
  RET(check_bt(e, batch, frames, 16));
  if (!e->cfg.train) return fail(e, CGVC_ERR_ARG, "engine was created with train = 0");
  RET(need_arenas(e, true));
  Bump ws; ws.reset(e->arena[CGVC_ARENA_WORK], e->arena_bytes[CGVC_ARENA_WORK]);
  TrainPlan P; plan_train(e, ws, P, batch, frames);
  if (ws.overflow) return fail(e, CGVC_ERR_UNBOUND, "WORK arena too small for batch %d x %d frames", batch, frames);
  return 0;
}

// "tape_loss_scale": the gradients that tape backward calls accumulate for cgvc_apply_gradients are checked against counters of their own.
// The first tape backward after a step (or cgvc_apply_gradients, when none ran) clears the counters and the non-finite flag, so that
// those of the step before stay readable (cgvc_loss_scale_state) until the next accumulation starts
static int tape_counts_open(cgvc_engine* e, cudaStream_t st) {
  if (e->tape_open) return 0;
  CK(cudaMemsetAsync(&e->ls->nonfinite, 0, (char*)(&e->ls->sat_act + 1) - (char*)&e->ls->nonfinite, st));
  CK(cudaMemsetAsync(e->ls->cnt, 0, sizeof e->ls->cnt, st));
  e->tape_open = true;
  return 0;
}

// The optimizer tail of a step, behind the gradients in GRAD on stream st: with a communicator the gradient all-reduce (per network and
// pipelined with each network's Adam and plane refresh when "pipelined_comm" is on), then with "loss_scale" != 0 the GRAD check and the
// scaler update, then Adam (skipped by the scaler in dynamic mode) and the refresh of the tensor-core weight planes.  The Adam scalars
// are already written (set_adam_scalars).  cgvc_train_step and cgvc_apply_gradients
static int optimizer_tail(cgvc_engine* e, cudaStream_t st) {
  if (e->comm && e->opt.pipelined_comm && e->comm_stream) {
    // one all-reduce per network (arena order), all enqueued on the communication stream behind the step's gradients; the caller's
    // stream then takes the networks one by one: wait for its all-reduce, Adam over its range, refresh of its tensor-core planes
    // the four networks in arena order; every tensor starts on a 16-byte boundary, so the ranges are cut at the aligned start of each
    // network's first tensor (the up-to-3 padding floats in front of it belong to the previous range and hold zero gradients)
    auto al4 = [](size_t v) { return (v + 3) & ~(size_t)3; };
    const size_t cut[5] = {0, al4(e->gen[1].begin), al4(e->disc[0].begin), al4(e->disc[1].begin), e->n_params};
    struct Range { size_t b, n; const float* hyper; } rg[4];
    for (int k = 0; k < 4; ++k) { rg[k].b = cut[k]; rg[k].n = cut[k + 1] - cut[k]; rg[k].hyper = e->d_scalars + (k < 2 ? 2 : 4); }
    CK(cudaEventRecord(e->ev_grads, st));
    CK(cudaStreamWaitEvent(e->comm_stream, e->ev_grads, 0));
    for (int k = 0; k < 4; ++k) {
      int r = e->nccl.AllReduce(e->G() + rg[k].b, e->G() + rg[k].b, rg[k].n, 7, 0, e->comm, e->comm_stream);     // ncclFloat32, ncclSum
      if (r != 0) return fail(e, CGVC_ERR_NCCL, "ncclAllReduce: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(r) : "?");
      CK(cudaEventRecord(e->ev_ar[k], e->comm_stream));
    }
    if (e->opt.ls_mode) {
      // every rank takes the same decision: the saturation counts are summed like the gradients (the GRAD check after the sum is
      // consistent by construction), and in dynamic mode each network's Adam waits for the scaler
      if (e->opt.ls_mode == 2) RET(ls_allreduce_counts(e, e->comm_stream));
      RET(ls_check_grads(e, e->comm_stream));
      if (e->opt.ls_mode == 1 && ls_nets(e)) RET(ls_update(e, e->comm_stream));
      CK(cudaEventRecord(e->ev_ls, e->comm_stream));
      if (e->opt.ls_mode == 2) { CK(cudaStreamWaitEvent(st, e->ev_ls, 0)); RET(ls_update(e, st)); }
    }
    float* pp = e->P(); float* gg = e->G(); float* mm = (float*)e->arena[CGVC_ARENA_ADAM_M]; float* vv = (float*)e->arena[CGVC_ARENA_ADAM_V];
    for (int k = 0; k < 4; ++k) {
      CK(cudaStreamWaitEvent(st, e->ev_ar[k], 0));
      GraphKey kk; memset(&kk, 0, sizeof kk); kk.kind = 2 + k;
      const Range R = rg[k];
      RET(run_captured(e, kk, st, [&](cudaStream_t s) {
        CK(launch_adam(pp + R.b, gg + R.b, mm + R.b, vv + R.b, (long long)R.n, R.hyper, ADAM_B1, ADAM_B2, ADAM_EPS, s, ls_skip(e)));
        if (e->cfg.precision != CGVC_PREC_FP32_SIMT) {
          int r = tc_refresh_weights_range(e->tcw, pp, R.b, R.b + R.n, s);
          if (r != 0) return fail(e, CGVC_ERR_CUDA, "tc_refresh_weights: %s", cudaGetErrorString((cudaError_t)r));
        }
        return 0;
      }));
    }
    if (e->opt.ls_mode == 1) CK(cudaStreamWaitEvent(st, e->ev_ls, 0));
    return 0;
  }
  if (e->comm) {
    RET(cgvc_allreduce_grads(e, (void*)st));
    if (e->opt.ls_mode == 2) RET(ls_allreduce_counts(e, st));
  }
  GraphKey k2; memset(&k2, 0, sizeof k2); k2.kind = 1;
  RET(run_captured(e, k2, st, [&](cudaStream_t s) {
    if (e->opt.ls_mode) RET(ls_check_grads(e, s));
    if (e->opt.ls_mode == 2 || ls_nets(e)) RET(ls_update(e, s));
    return adam_body(e, s, ls_skip(e));
  }));
  return 0;
}

extern "C" {

int cgvc_compute_gradients(cgvc_handle e, const float* A_dev, const float* B_dev, int batch, int frames,
                           float lambda_cycle, float lambda_identity, float* gen_A_dev, float* gen_B_dev, float* losses_dev, void* stream) {
  if (!e || !A_dev || !B_dev) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(check_work_train(e, batch, frames));
  e->tape_open = false;
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  RET(set_lambdas(e, lambda_cycle, lambda_identity, (cudaStream_t)stream));
  RET(ls_prepare(e, batch, (cudaStream_t)stream));
  RET(forward_backward(e, A_dev, B_dev, batch, frames, lambda_cycle, lambda_identity, gen_A_dev, gen_B_dev, losses_dev, (cudaStream_t)stream));
  // the gradients are handed out, not fed to Adam: remove the loss scale here (in dynamic mode the device scale they were formed with)
  if (e->opt.ls_mode == 2 && ls_nets(e)) {                 // each GRAD range its own network's scale
    const long long gend = (long long)e->gen[1].end;
    CK(launch_scale(e->G(), gend, 1.f, (cudaStream_t)stream, &e->ls->net[0].scale));
    CK(launch_scale(e->G() + gend, (long long)e->n_params - gend, 1.f, (cudaStream_t)stream, &e->ls->net[1].scale));
  } else if (e->opt.ls_mode == 2) CK(launch_scale(e->G(), (long long)e->n_params, 1.f, (cudaStream_t)stream, &e->ls->scale));
  else if (loss_scale(e, batch) != 1.f) CK(launch_scale(e->G(), (long long)e->n_params, 1.f / loss_scale(e, batch), (cudaStream_t)stream));
  return 0;
}

int cgvc_adam_step(cgvc_handle e, float lr_g, float lr_d, float grad_scale, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  for (int a = 0; a < 4; ++a) if (!e->arena[a]) return fail(e, CGVC_ERR_UNBOUND, "PARAM/GRAD/ADAM_M/ADAM_V arenas must be bound");
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  // dynamic loss-scale mode keeps t on the device: bring it to the host (synchronises), step with the host's lr_t like the other
  // modes, and write the advanced t back (synchronises again).  No skip: the caller decides on this step
  if (e->opt.ls_mode == 2) { long long t; RET(cgvc_get_adam_step(e, &t)); }
  const long long t_before = e->adam_t;
  RET(set_adam_scalars(e, lr_g, lr_d, grad_scale, (cudaStream_t)stream));
  int r = adam_body(e, (cudaStream_t)stream);
  if (r != 0) { e->adam_t = t_before; return r; }
  if (e->opt.ls_mode == 2) RET(cgvc_set_adam_step(e, e->adam_t));
  return 0;
}

int cgvc_train_step(cgvc_handle e, const float* A_dev, const float* B_dev, int batch, int frames,
                    float lambda_cycle, float lambda_identity, float lr_g, float lr_d,
                    float* gen_A_dev, float* gen_B_dev, float* losses_dev, void* stream) {
  if (!e || !A_dev || !B_dev) return fail(e, CGVC_ERR_ARG, "null argument");
  for (int a = 0; a < 4; ++a) if (!e->arena[a]) return fail(e, CGVC_ERR_UNBOUND, "PARAM/GRAD/ADAM_M/ADAM_V arenas must be bound");
  RET(check_work_train(e, batch, frames));
  ++e->param_gen;                                            // a replayed graph does not run adam_body's host code
  e->tape_open = false;                                      // the step zeroes GRAD and the counters: a tape accumulation starts anew
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const float gscale = (e->comm ? 1.f / (float)e->nranks : 1.f) / loss_scale(e, batch);
  RET(set_lambdas(e, lambda_cycle, lambda_identity, st));
  // the Adam step counter advances only if the whole step was enqueued: a call that is refused further down (WORK arena too small,
  // capture failure, NCCL error) must not change the bias correction of the next one
  const long long adam_t_before = e->adam_t;
  struct Rollback { cgvc_engine* e; long long t; bool armed; ~Rollback() { if (armed) e->adam_t = t; } } rollback{e, adam_t_before, true};
  RET(set_adam_scalars(e, lr_g, lr_d, e->opt.ls_mode == 2 ? (e->comm ? 1.f / (float)e->nranks : 1.f) : gscale, st, e->opt.ls_mode == 2));
  RET(ls_prepare(e, batch, st));
  if (e->opt.use_graphs && !tc_profile_is_on()) {
    // the graphs read the inputs from fixed staging buffers and leave the results in the WORK arena / d_scalars, so one
    // captured graph serves any caller pointers; the copies either side are eager
    const size_t img = (size_t)batch * e->cfg.num_features * frames;
    const size_t cap = (size_t)e->cfg.max_batch * e->cfg.num_features * e->cfg.max_frames;
    if (!e->stage) CK(cudaMalloc(&e->stage, 2 * cap * sizeof(float)));
    float* sA = e->stage; float* sB = e->stage + cap;
    CK(cudaMemcpyAsync(sA, A_dev, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(sB, B_dev, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
    GraphKey key; memset(&key, 0, sizeof key);
    key.batch = batch; key.frames = frames; key.id_off = lambda_identity == 0.f; key.kind = 0;
    RET(run_captured(e, key, st, [&](cudaStream_t s) {
      return forward_backward(e, sA, sB, batch, frames, lambda_cycle, lambda_identity, nullptr, nullptr, nullptr, s);
    }));
    if (gen_A_dev || gen_B_dev) {
      Bump ws; ws.reset(e->arena[CGVC_ARENA_WORK], e->arena_bytes[CGVC_ARENA_WORK]);
      TrainPlan P; plan_train(e, ws, P, batch, frames);
      if (gen_B_dev) CK(cudaMemcpyAsync(gen_B_dev, P.lane[0].din + img, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
      if (gen_A_dev) CK(cudaMemcpyAsync(gen_A_dev, P.lane[1].din + img, img * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (losses_dev) CK(cudaMemcpyAsync(losses_dev, e->d_scalars + 8, 8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  } else {
    RET(forward_backward(e, A_dev, B_dev, batch, frames, lambda_cycle, lambda_identity, gen_A_dev, gen_B_dev, losses_dev, st));
  }
  RET(optimizer_tail(e, st));
  rollback.armed = false;
  return 0;
}

int cgvc_apply_gradients(cgvc_handle e, float lr_g, float lr_d, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if (!e->opt.tape_ls) return fail(e, CGVC_ERR_ARG, "cgvc_apply_gradients needs the option tape_loss_scale = 1 (else: cgvc_adam_step)");
  for (int a = 0; a < 4; ++a) if (!e->arena[a]) return fail(e, CGVC_ERR_UNBOUND, "PARAM/GRAD/ADAM_M/ADAM_V arenas must be bound");
  if (!e->ls_ready)
    return fail(e, CGVC_ERR_ARG, "no loss scale yet: a tape backward or cgvc_set_loss_scale_state sets it before cgvc_apply_gradients");
  ++e->param_gen;                                            // a replayed graph does not run adam_body's host code
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  RET(tape_counts_open(e, st));                              // no tape backward since the last step: nothing was counted
  RET(set_adam_scalars(e, lr_g, lr_d, e->comm ? 1.f / (float)e->nranks : 1.f, st, true));
  RET(optimizer_tail(e, st));
  e->tape_open = false;
  return 0;
}

// ---- NCCL --------------------------------------------------------------------------------------------------
static int load_nccl(cgvc_engine* e) {
  if (e->nccl.lib) return 0;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* lib = nullptr;
  for (const char* n : names) { lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
  if (!lib) return fail(e, CGVC_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
  e->nccl.lib = lib;
  *(void**)&e->nccl.GetUniqueId = dlsym(lib, "ncclGetUniqueId");
  *(void**)&e->nccl.CommInitRank = dlsym(lib, "ncclCommInitRank");
  *(void**)&e->nccl.CommDestroy = dlsym(lib, "ncclCommDestroy");
  *(void**)&e->nccl.AllReduce = dlsym(lib, "ncclAllReduce");
  *(void**)&e->nccl.GetErrorString = dlsym(lib, "ncclGetErrorString");
  if (!e->nccl.GetUniqueId || !e->nccl.CommInitRank || !e->nccl.AllReduce || !e->nccl.CommDestroy)
    return fail(e, CGVC_ERR_NCCL, "libnccl is missing required symbols");
  return 0;
}

int cgvc_comm_unique_id(cgvc_handle e, void* id128_host) {
  if (!e || !id128_host) return CGVC_ERR_ARG;
  RET(load_nccl(e));
  int r = e->nccl.GetUniqueId(id128_host);
  if (r != 0) return fail(e, CGVC_ERR_NCCL, "ncclGetUniqueId: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(r) : "?");
  return 0;
}

int cgvc_comm_init(cgvc_handle e, const void* id128_host, int rank, int nranks) {
  if (!e || !id128_host || nranks < 1 || rank < 0 || rank >= nranks) return fail(e, CGVC_ERR_ARG, "cgvc_comm_init: bad argument");
  RET(load_nccl(e));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  Id128 id; memcpy(id.b, id128_host, 128);
  int r = e->nccl.CommInitRank(&e->comm, nranks, id, rank);
  if (r != 0) { e->comm = nullptr; return fail(e, CGVC_ERR_NCCL, "ncclCommInitRank: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(r) : "?"); }
  e->rank = rank; e->nranks = nranks;
  return 0;
}

int cgvc_comm_destroy(cgvc_handle e) {
  if (!e) return CGVC_ERR_ARG;
  if (e->comm) { e->nccl.CommDestroy(e->comm); e->comm = nullptr; e->nranks = 1; e->rank = 0; }
  return 0;
}

int cgvc_allreduce_grads(cgvc_handle e, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if (!e->comm) return fail(e, CGVC_ERR_NCCL, "no communicator attached");
  if (!e->arena[CGVC_ARENA_GRAD]) return fail(e, CGVC_ERR_UNBOUND, "GRAD arena must be bound");
  // ncclFloat32 = 7, ncclSum = 0
  int r = e->nccl.AllReduce(e->G(), e->G(), e->n_params, 7, 0, e->comm, (cudaStream_t)stream);
  if (r != 0) return fail(e, CGVC_ERR_NCCL, "ncclAllReduce: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(r) : "?");
  return 0;
}

// Every option: its name, valid range and home.  A flag (range [0, 1]) takes any value, non-zero meaning 1
struct OptionDef { const char* name; int lo, hi; int* (*field)(cgvc_engine*); };
#define OPT(name, lo, hi, member) {name, lo, hi, [](cgvc_engine* e) { return &e->member; }}
static const OptionDef kOptions[] = {
  OPT("two_streams", 0, 1, opt.two_streams),        OPT("fuse_in", 0, 1, opt.fuse_in),
  OPT("fuse_bwd", 0, 1, opt.fuse_bwd),              OPT("edge_lower", 0, 1, opt.edge_lower),
  OPT("side_wgrad", 0, 1, opt.side_wgrad),          OPT("deterministic", 0, 1, opt.deterministic),
  OPT("pipelined_comm", 0, 1, opt.pipelined_comm),  OPT("fuse_c1", 0, 1, opt.fuse_c1),
  OPT("debug_taps", 0, 1, opt.debug_taps),          OPT("cuda_graph", 0, 1, opt.use_graphs),
  OPT("post_onepass", 0, 1, opt.post.onepass),      OPT("post_stream", 0, 1, opt.post.stream),
  OPT("loss_scale", 0, 2, opt.ls_mode),             OPT("loss_scale_growth_interval", 1, INT_MAX, opt.ls_growth),
  OPT("loss_scale_per_network", 0, 1, opt.ls_nets),  OPT("tape_loss_scale", 0, 1, opt.tape_ls),
  OPT("wgrad_f16", 0, 1, tcw.wgrad16),              OPT("prep_batched", 0, 1, tcw.prep_batched),
  OPT("tc_debug", 0, 7, tcw.debug),
};
#undef OPT

int cgvc_set_option(cgvc_handle e, const char* name, int value) {
  if (!e || !name) return CGVC_ERR_ARG;
  const OptionDef* d = nullptr;
  for (const OptionDef& o : kOptions) if (!strcmp(o.name, name)) d = &o;
  if (!d) return fail(e, CGVC_ERR_ARG, "unknown option '%s'", name);
  if (d->lo == 0 && d->hi == 1) value = value != 0;
  if (value < d->lo || value > d->hi) return fail(e, CGVC_ERR_ARG, "option %s: bad value %d", name, value);
  int* field = d->field(e);
  if (*field == value) return 0;
  if (field == &e->opt.tape_ls && value && e->opt.ls_mode != 2)
    return fail(e, CGVC_ERR_ARG, "option tape_loss_scale = 1 needs loss_scale = 2 (dynamic)");
  if (field == &e->opt.ls_mode && e->opt.tape_ls)
    return fail(e, CGVC_ERR_ARG, "loss_scale must stay 2 while tape_loss_scale = 1");
  if (field == &e->opt.ls_mode) {
    DeviceGuard dguard; CK(dguard.set(e->cfg.device));
    long long t = 0;
    RET(cgvc_get_adam_step(e, &t));                          // the step count moves between host and device with the mode
    e->opt.ls_mode = value;
    RET(cgvc_set_adam_step(e, t));
    e->ls_ready = false; e->ls_batch = 0;
  }
  if (field == &e->opt.ls_nets && value && e->ls_ready) {
    // a dynamic scale in use: both networks continue from it ({scale, good_steps} is the head's layout)
    DeviceGuard dguard; CK(dguard.set(e->cfg.device));
    for (int k = 0; k < 2; ++k) CK(cudaMemcpy(&e->ls->net[k], e->ls, sizeof(LossScaler::Net), cudaMemcpyDeviceToDevice));
  }
  if (field == &e->opt.ls_nets) e->ls_batch = 0;            // monitor mode writes the networks' static scales on the next step
  *field = value;
  drop_graphs(e);
  return 0;
}
int cgvc_kernel_launches(unsigned long long* count) { if (!count) return CGVC_ERR_ARG; *count = g_cgvc_launches; return 0; }
int cgvc_profile_enable(int on) { tc_profile_enable(on); return 0; }
int cgvc_profile_launches(double* ms, double* flops, long long* meta4, int capacity, int* n_out) {
  if (!ms || !flops || !meta4 || capacity < 0) return CGVC_ERR_ARG;
  return tc_profile_launches(ms, flops, meta4, capacity, n_out) == 0 ? 0 : CGVC_ERR_CUDA;
}
int cgvc_profile_collect(double* ms3, double* flops3, long long* launches3) {
  if (!ms3 || !flops3 || !launches3) return CGVC_ERR_ARG;
  return tc_profile_collect(ms3, flops3, launches3) == 0 ? 0 : CGVC_ERR_CUDA;
}

// ---- device-resident training data ---------------------------------------------------------------------------
int cgvc_sample_plan(cgvc_handle e, const long long* offsets_A_dev, int n_A, const long long* offsets_B_dev, int n_B,
                     unsigned long long seed, long long epoch, int crop_frames, int* plan_dev, int* err_dev, void* stream) {
  if (!e || !offsets_A_dev || !offsets_B_dev || !plan_dev || !err_dev) return fail(e, CGVC_ERR_ARG, "null argument");
  if (n_A < 1 || n_B < 1 || crop_frames < 1 || epoch < 0) return fail(e, CGVC_ERR_ARG, "cgvc_sample_plan: empty corpus or bad crop / epoch");
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(cudaMemsetAsync(err_dev, 0, sizeof(int), (cudaStream_t)stream));
  CK(launch_sample_plan(offsets_A_dev, n_A, offsets_B_dev, n_B, seed, epoch, crop_frames, plan_dev, err_dev, (cudaStream_t)stream));
  return 0;
}

int cgvc_gather_minibatch(cgvc_handle e, const float* corpus_A_dev, const long long* offsets_A_dev, const float* corpus_B_dev,
                          const long long* offsets_B_dev, const int* plan_dev, int num_pairs, int first_pair, int batch, int crop_frames,
                          float* A_out_dev, float* B_out_dev, void* stream) {
  if (!e || !corpus_A_dev || !corpus_B_dev || !offsets_A_dev || !offsets_B_dev || !plan_dev || !A_out_dev || !B_out_dev)
    return fail(e, CGVC_ERR_ARG, "null argument");
  if (batch < 1 || first_pair < 0 || first_pair + batch > num_pairs || crop_frames < 1)
    return fail(e, CGVC_ERR_ARG, "cgvc_gather_minibatch: pairs [%d, %d) outside the epoch's %d", first_pair, first_pair + batch, num_pairs);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_gather_minibatch(corpus_A_dev, offsets_A_dev, corpus_B_dev, offsets_B_dev, plan_dev, num_pairs, first_pair, batch,
                             e->cfg.num_features, crop_frames, A_out_dev, B_out_dev, (cudaStream_t)stream));
  return 0;
}

}  // extern "C"

// ---- per-kernel entry points ---------------------------------------------------------------------------------
// the entry points' scratch, carved from the per-engine buffer: carve(ws) runs once on a null base to size it, then on the buffer
template <class F> static cudaError_t entry_scratch(cgvc_engine* e, F&& carve) {
  Bump ws; ws.reset(nullptr, 0);
  carve(ws);
  float* buf;
  cudaError_t ce = grow_post_buf(e, ws.off / sizeof(float) + 1, &buf);
  if (ce != cudaSuccess) return ce;
  ws.reset(buf, e->post_elems * sizeof(float));
  carve(ws);
  return cudaSuccess;
}

// room for the operand planes of `rows` rows of c channels in any precision: bf16 hi / lo [rows, ru64(c)], F16F8 fp16 + two e4m3 [rows, ru128(c)]
static void take_planes(Bump& ws, long long rows, int c, __nv_bfloat16** hi, __nv_bfloat16** lo) {
  const size_t n = (size_t)rows * edge_cpad(c);
  *hi = ws.take<__nv_bfloat16>(n); *lo = ws.take<__nv_bfloat16>(n);
}

// One convolution layer in the engine's own description for the convolution entry points, whose tensors they take by pointer
// (a.k = b = -1: no PARAM tensor, which tc_result would name)
static Layer conv_layer(int kh, int kw, int cin, int cout, bool gated, int sh, int sw, int shuffle = 1) {
  Layer L{}; L.a = ConvW{(size_t)-1, (size_t)-1, kh, kw, cin, cout}; if (gated) L.g = L.a;
  L.sh = sh; L.sw = sw; L.shuffle = shuffle;
  return L;
}

// The tensor-core planes of such a layer in t.precision: a one-layer store, refreshed from t's weights (null biases read as the zeros
// `zero` [cout] is set to) on st, which the call synchronises before the store is freed.  Sets t.tc and the store options
struct EntryStore {
  TcWeights w;
  ~EntryStore() { tc_free(w); }
};
static int entry_store(cgvc_engine* e, EntryStore& S, const Layer& L, LayerTensors& t, float* zero, cudaStream_t st) {
  tc_register(S.w, 0, 0, 0, 0, L.a.kh, L.a.kw, L.a.cin, L.a.cout, L.gated(), L.shuffle);
  int r = tc_alloc(S.w, t.precision, true);
  if (r != 0) return fail(e, CGVC_ERR_CUDA, "tc_alloc: %s", cudaGetErrorString((cudaError_t)r));
  CK(cudaStreamSynchronize(nullptr));                   // tc_alloc zeroes the planes' padding on the legacy stream
  if (!t.ba || (L.gated() && !t.bg)) CK(cudaMemsetAsync(zero, 0, L.a.cout * sizeof(float), st));
  TcLayer& T = S.w.layers[0];
  r = tc_refresh_layer(T, t.ka, t.kg, t.ba ? t.ba : zero, t.bg ? t.bg : zero, st);
  if (r != 0) return fail(e, CGVC_ERR_CUDA, "tc_refresh_layer: %s", cudaGetErrorString((cudaError_t)r));
  t.tc = &T; t.debug = e->tcw.debug; t.wgrad16 = e->tcw.wgrad16;
  return 0;
}

extern "C" {

int cgvc_conv_forward(cgvc_handle e, int precision, const float* x, const float* w, const float* bias, float* y,
                      int B, int H, int W, int Cin, int kh, int kw, int Cout, int sh, int sw, void* stream) {
  if (!e || !x || !w || !y) return fail(e, CGVC_ERR_ARG, "null argument");
  if (kh * kw > CGVC_MAX_TAPS) return fail(e, CGVC_ERR_UNSUPPORTED, "at most %d filter taps", CGVC_MAX_TAPS);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const Layer L = conv_layer(kh, kw, Cin, Cout, false, sh, sw);
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w; t.ba = bias; t.precision = precision;
  ConvIO io{}; io.x = x; io.n = B; io.H = H; io.W = W;
  if (precision == CGVC_PREC_FP32_SIMT) return conv_fwd(e, L, t, io, y, st);
  // the tensor-core path reads x through its planes only (as a train step does), so that a shape it refuses is CGVC_ERR_UNSUPPORTED
  float* zero;
  __nv_bfloat16 *xhi, *xlo;
  CK(entry_scratch(e, [&](Bump& ws) { take_planes(ws, (long long)B * H * W, Cin, &xhi, &xlo); zero = ws.take<float>(Cout); }));
  EntryStore S;
  RET(entry_store(e, S, L, t, zero, st));
  CK(tc_split_planes(precision, x, (long long)B * H * W, Cin, xhi, xlo, st));
  io.x = nullptr; io.xhi = xhi; io.xlo = xlo;
  RET(conv_fwd(e, L, t, io, y, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

int cgvc_conv_backward(cgvc_handle e, int precision, const float* x, const float* w, const float* dy,
                       float* dx, float* dw, float* dbias, int B, int H, int W, int Cin, int kh, int kw, int Cout, int sh, int sw, void* stream) {
  if (!e || !x || !w || !dy) return fail(e, CGVC_ERR_ARG, "null argument");
  if (kh * kw > CGVC_MAX_TAPS) return fail(e, CGVC_ERR_UNSUPPORTED, "at most %d filter taps", CGVC_MAX_TAPS);
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const Layer L = conv_layer(kh, kw, Cin, Cout, false, sh, sw);
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w; t.dka = dw; t.precision = precision;
  ConvIO io{}; io.x = x; io.n = B; io.H = H; io.W = W;
  const GatherGeom g = fwd_geom(B, H, W, kh, kw, sh, sw);
  const long long rows = (long long)B * H * W, orows = (long long)g.B * g.Hy * g.Wx;
  const float* dP = dy;
  PlanePair dp{nullptr, nullptr};
  EntryStore S;
  if (precision != CGVC_PREC_FP32_SIMT) {                // planes only, as in cgvc_conv_forward
    __nv_bfloat16 *xhi, *xlo;
    float* zero;
    CK(entry_scratch(e, [&](Bump& ws) {
      take_planes(ws, rows, Cin, &xhi, &xlo); take_planes(ws, orows, Cout, &dp.hi, &dp.lo); zero = ws.take<float>(Cout);
    }));
    RET(entry_store(e, S, L, t, zero, st));
    CK(tc_split_planes(precision, x, rows, Cin, xhi, xlo, st));
    CK(tc_split_planes(precision, dy, orows, Cout, dp.hi, dp.lo, st));
    io.x = nullptr; io.xhi = xhi; io.xlo = xlo; dP = nullptr;
  }
  if (dx) RET(conv_dgrad(e, L, t, io, dP, dp, dx, 0, st));
  if (dw) {
    RET(conv_wgrad(e, L, t, io, dP, dp, st, det));
    if (dbias) CK(launch_colsum(dy, orows, Cout, 0, Cout, dbias, st, det));
  }
  if (precision != CGVC_PREC_FP32_SIMT) CK(cudaStreamSynchronize(st));
  return 0;
}

// ---- operand-plane writers (test entry points: exact planes and saturation counts against a host reference) --------------
static int plane_precision(cgvc_engine* e, int precision, const void* hi, const void* lo) {
  if (precision != CGVC_PREC_BF16X3 && precision != CGVC_PREC_BF16 && precision != CGVC_PREC_F16F8)
    return fail(e, CGVC_ERR_ARG, "operand planes: precision %d has none", precision);
  if (!hi || !lo) return fail(e, CGVC_ERR_ARG, "null argument");
  return 0;
}

int cgvc_split_planes(cgvc_handle e, int precision, const float* x, long long rows, int C, void* hi, void* lo,
                      unsigned long long* sat, void* stream) {
  if (!e || !x) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(plane_precision(e, precision, hi, lo));
  if (rows < 0 || C < 1) return fail(e, CGVC_ERR_ARG, "cgvc_split_planes: bad shape [%lld, %d]", rows, C);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(tc_split_planes(precision, x, rows, C, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, (cudaStream_t)stream, sat, e->plane_ufl));
  return 0;
}

int cgvc_im2col_planes(cgvc_handle e, int precision, const float* x, long long rows, int T, int C, int kw, int dir, void* hi, void* lo,
                       unsigned long long* sat, void* stream) {
  if (!e || !x) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(plane_precision(e, precision, hi, lo));
  if (T < 1 || rows < 0 || rows % T || C < 4 || C % 4 || kw < 1 || kw > CGVC_MAX_TAPS || (dir != 1 && dir != -1))
    return fail(e, CGVC_ERR_ARG, "cgvc_im2col_planes: bad shape (rows %lld, T %d, C %d, kw %d, dir %d)", rows, T, C, kw, dir);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_im2col_taps(x, rows, T, C, kw, dir, edge_cpad(kw * C), precision == CGVC_PREC_F16F8, hi, lo, (cudaStream_t)stream,
                        nullptr, 0, sat, e->plane_ufl));
  return 0;
}

// An instance-normed layer in the engine's own description, for the entry points below: gated or residual (the h2 form), shuffle 1
// or 2, C channels after the pixel-shuffle view.  post_params / post_bwd_params build its launch parameters as a train step does; the
// entry points then point the affine, plane and counter fields at the caller's buffers.
static Layer in_layer(int C, int gate, int shuffle) {
  Layer L{}; L.a.cout = C * shuffle; L.g.cout = gate ? C * shuffle : 0; L.a.cin = L.g.cin = 1; L.has_in = 1; L.sh = L.sw = 1;
  L.shuffle = shuffle;
  return L;
}

// the forward of such a layer over B samples of R positions, or (offsets != null) over packed utterances
static int in_glu_forward(cgvc_engine* e, const float* p, const float* beta_a, const float* gamma_a, const float* beta_g,
                          const float* gamma_g, float* y, float* stats, int B, int R, int C, int shuffle, int precision, int gate,
                          const float* resid, const long long* offsets, int n_utt, int div, int max_len, void* hi, void* lo,
                          unsigned long long* sat, void* stream) {
  if (!e || !p || !y || !stats) return fail(e, CGVC_ERR_ARG, "null argument");
  if (C % 32 != 0 || shuffle < 1 || R % shuffle != 0) return fail(e, CGVC_ERR_UNSUPPORTED, "C must be a multiple of 32 and R of shuffle");
  if (offsets && (B != 1 || n_utt < 1 || n_utt > 65535 || (div != 1 && div != 2 && div != 4) || div % shuffle || max_len < 4 || max_len % 4))
    return fail(e, CGVC_ERR_ARG, "cgvc_in_glu_forward_packed: bad packed geometry (B %d, n_utt %d, div %d, max_len %d)", B, n_utt, div, max_len);
  if (precision != CGVC_PREC_FP32_SIMT) RET(plane_precision(e, precision, hi, lo));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  ConvIO io{}; io.n = B;
  if (offsets) { io.n = io.H = 1; io.W = R / shuffle; io.pk = PackGeom{offsets, n_utt, div, max_len}; }
  const GLAct A{const_cast<float*>(p), stats, y, nullptr, nullptr};
  LayerTensors t; memset(&t, 0, sizeof t);
  t.beta_a = beta_a; t.gamma_a = gamma_a; t.beta_g = gate ? beta_g : nullptr; t.gamma_g = gate ? gamma_g : nullptr;
  PostParams q = post_params(e, in_layer(C, gate, shuffle), t, io, A, R / shuffle, true, nullptr, resid);
  q.sat = q.ufl = nullptr;
  if (precision != CGVC_PREC_FP32_SIMT) {
    q.y_hi = (__nv_bfloat16*)hi; q.y_lo = (__nv_bfloat16*)lo; q.qmode = precision == CGVC_PREC_F16F8; q.sat = q.qmode ? sat : nullptr;
    q.ufl = q.qmode ? e->plane_ufl : nullptr;
  }
  CK(grow_post_buf(e, (size_t)q.B * 4 * C, &q.scratch));
  CK(launch_post_fwd(q, e->opt.post, (cudaStream_t)stream));
  return 0;
}

// its backward, with the conv-bias gradients when dbias_a is given
static int in_glu_backward(cgvc_engine* e, const float* dy, const float* p, const float* stats,
                           const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                           float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g, float* dbias_a, float* dbias_g,
                           int B, int R, int C, int shuffle, int precision, int gate, void* hi, void* lo, unsigned long long* sat,
                           void* stream) {
  if (!e || !dy || !p || !stats || !dp) return fail(e, CGVC_ERR_ARG, "null argument");
  if (C % 32 != 0 || shuffle < 1 || R % shuffle != 0) return fail(e, CGVC_ERR_UNSUPPORTED, "C must be a multiple of 32 and R of shuffle");
  if (!dbias_a && dbias_g) return fail(e, CGVC_ERR_ARG, "cgvc_in_glu_backward_bias: dbias_g needs dbias_a");
  if (precision != CGVC_PREC_FP32_SIMT) RET(plane_precision(e, precision, hi, lo));
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  const GLAct A{const_cast<float*>(p), const_cast<float*>(stats), nullptr, nullptr, nullptr};
  BwdScratch S; memset(&S, 0, sizeof S); S.dP = dp;
  if (det) S.det = *det;
  LayerTensors t; memset(&t, 0, sizeof t);
  t.beta_a = beta_a; t.gamma_a = gamma_a; t.beta_g = gate ? beta_g : nullptr; t.gamma_g = gate ? gamma_g : nullptr;
  t.dbeta_a = dbeta_a; t.dgamma_a = dgamma_a; t.dbeta_g = gate ? dbeta_g : nullptr; t.dgamma_g = gate ? dgamma_g : nullptr;
  t.dba = dbias_a; t.dbg = gate ? dbias_g : nullptr;
  PostBwdParams q = post_bwd_params(e, in_layer(C, gate, shuffle), t, dy, A, B, R / shuffle, S, true, PlanePair{nullptr, nullptr});
  if (det) q.det = *det;
  q.sat = q.ufl = nullptr;
  if (precision != CGVC_PREC_FP32_SIMT) {
    q.dp_hi = (__nv_bfloat16*)hi; q.dp_lo = (__nv_bfloat16*)lo; q.qmode = precision == CGVC_PREC_F16F8; q.sat = q.qmode ? sat : nullptr;
    q.ufl = q.qmode ? e->plane_ufl : nullptr;
  }
  CK(grow_post_buf(e, (size_t)B * 4 * C, &q.scratch));
  CK(launch_post_bwd(q, e->opt.post, (cudaStream_t)stream));
  return 0;
}

// ---- one generator layer with its instance norm, fused into the gather-GEMM epilogue or not (test entry points) ----------------
int cgvc_conv_in_forward(cgvc_handle e, int precision, const float* x, const float* w_a, const float* w_g, const float* b_a, const float* b_g,
                         const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g, const float* resid,
                         float* p, float* stats, float* y, void* hi, void* lo,
                         int B, int W, int Cin, int kw, int Cout, int sw, int shuffle, int fuse, int* fused, void* stream) {
  if (fused) *fused = 0;
  if (!e || !x || !w_a || !b_a || !beta_a || !gamma_a) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(plane_precision(e, precision, hi, lo));
  const bool gated = w_g != nullptr;
  if (gated ? (!b_g || !beta_g || !gamma_g) : (!resid || shuffle != 1))
    return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_forward: a gated layer needs b_g, beta_g and gamma_g; a residual one resid and shuffle 1");
  if (B < 1 || W < 1 || Cin < 1 || kw < 1 || kw > CGVC_MAX_TAPS || sw < 1 || (shuffle != 1 && shuffle != 2) || Cout % (32 * shuffle))
    return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_forward: bad shape (B %d, W %d, Cin %d, kw %d, Cout %d, sw %d, shuffle %d)", B, W, Cin, kw, Cout, sw, shuffle);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  Layer L = conv_layer(1, kw, Cin, Cout, gated, 1, sw, shuffle);
  L.has_in = 1;
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w_a; t.kg = w_g; t.ba = b_a; t.bg = b_g; t.beta_a = beta_a; t.gamma_a = gamma_a; t.precision = precision;
  if (gated) { t.beta_g = beta_g; t.gamma_g = gamma_g; }
  // p and stats may be null: the inference form (neither) runs as a conversion does, with scratch for the fallback's intermediates
  const int Wo = (W + sw - 1) / sw, C = Cout / shuffle;
  __nv_bfloat16 *xhi, *xlo;
  float *ps, *ss, *post;
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, (long long)B * W, Cin, &xhi, &xlo);
    ps = ws.take<float>((size_t)B * Wo * L.width()); ss = ws.take<float>((size_t)B * 4 * C); post = ws.take<float>((size_t)B * 4 * C);
  }));
  EntryStore S;
  RET(entry_store(e, S, L, t, nullptr, st));
  CK(tc_split_planes(precision, x, (long long)B * W, Cin, xhi, xlo, st));
  ConvIO io{}; io.xhi = xhi; io.xlo = xlo; io.n = B; io.H = 1; io.W = W;
  const GLAct A{p ? p : ps, stats ? stats : ss, y, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo};
  bool f = false;
  RET(layer_forward(e, L, t, io, A, Wo, true, p || stats, fuse != 0, post, st, resid, &f));
  CK(cudaStreamSynchronize(st));
  if (fused) *fused = f;
  return 0;
}

int cgvc_conv_in_backward(cgvc_handle e, int precision, const float* dp, const float* w_a, const float* w_g, const float* bp, const float* stats,
                          const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g, float* dx, void* hi, void* lo,
                          float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                          int B, int R, int Cin, int kw, int Cout, int gate, int accumulate, int fuse, int* fused, void* stream) {
  if (fused) *fused = 0;
  if (!e || !dp || !w_a || !bp || !stats || !beta_a || !gamma_a) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(plane_precision(e, precision, hi, lo));
  if (gate ? (!beta_g || !gamma_g) : !dx)
    return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_backward: the gated form needs beta_g and gamma_g; the residual form dx");
  if (accumulate && !dx) return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_backward: accumulate needs dx");
  const bool some = dbeta_a || dgamma_a || dbeta_g || dgamma_g, all = dbeta_a && dgamma_a && (!gate || (dbeta_g && dgamma_g));
  if (some && !all) return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_backward: the affine gradients are all given or none");
  if (B < 1 || R < 1 || Cin < 1 || Cin % 32 || kw < 1 || kw > CGVC_MAX_TAPS || Cout < 1)
    return fail(e, CGVC_ERR_ARG, "cgvc_conv_in_backward: bad shape (B %d, R %d, Cin %d, kw %d, Cout %d)", B, R, Cin, kw, Cout);
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  // L: the stride-1 layer whose data gradient this is; U: the upstream layer whose output L read, whose dP planes are hi / lo
  const Layer L = conv_layer(1, kw, Cin, Cout, w_g != nullptr, 1, 1);
  const Layer U = in_layer(Cin, gate, 1);
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w_a; t.kg = w_g; t.precision = precision;
  const long long rows = (long long)B * R;
  __nv_bfloat16 *dphi, *dplo;
  float *zero, *dY = dx;
  BwdScratch S; memset(&S, 0, sizeof S);
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, rows, L.width(), &dphi, &dplo);
    zero = ws.take<float>(Cout); S.post = ws.take<float>((size_t)B * 4 * Cin);
    if (gate) dY = ws.take<float>((size_t)rows * Cin);
  }));
  EntryStore store;
  RET(entry_store(e, store, L, t, zero, st));
  LayerTensors u; memset(&u, 0, sizeof u);
  u.beta_a = beta_a; u.gamma_a = gamma_a; u.dbeta_a = dbeta_a; u.dgamma_a = dgamma_a;
  if (gate) { u.beta_g = beta_g; u.gamma_g = gamma_g; u.dbeta_g = dbeta_g; u.dgamma_g = dgamma_g; }
  u.tc = t.tc; u.precision = precision;                   // (tc: U's dP goes to operand planes)
  CK(tc_split_planes(precision, dp, rows, L.width(), dphi, dplo, st));
  // dY = dgrad(dp) (+ dx): the residual form keeps it in dx; the gated form works on a copy, so that dx is only read
  if (gate && accumulate) CK(cudaMemcpyAsync(dY, dx, (size_t)rows * Cin * sizeof(float), cudaMemcpyDeviceToDevice, st));
  S.dPhi = S.dP2hi = (__nv_bfloat16*)hi; S.dPlo = S.dP2lo = (__nv_bfloat16*)lo;
  if (det) S.det = *det;
  BwdWalk w(S, fuse && !det);
  ConvIO in{}; in.n = B; in.H = 1; in.W = R;
  const GLAct UA{const_cast<float*>(bp), const_cast<float*>(stats), nullptr, nullptr, nullptr};
  RET(layer_dx(e, w, L, t, in, nullptr, PlanePair{dphi, dplo}, dY, accumulate, st, &U, &u, &UA));
  const bool f = w.have >= 0;
  PostBwdParams q;
  RET(layer_dp(e, w, U, u, UA, dY, B, R, st, q));
  CK(cudaStreamSynchronize(st));
  if (fused) *fused = f;
  return 0;
}

int cgvc_in_glu_forward_planes(cgvc_handle e, const float* p, const float* beta_a, const float* gamma_a, const float* beta_g,
                               const float* gamma_g, float* y, float* stats, int B, int R, int C, int shuffle, int precision, int gate,
                               const float* resid, void* hi, void* lo, unsigned long long* sat, void* stream) {
  return in_glu_forward(e, p, beta_a, gamma_a, beta_g, gamma_g, y, stats, B, R, C, shuffle, precision, gate, resid, nullptr, 0, 0, 0,
                        hi, lo, sat, stream);
}

int cgvc_in_glu_forward_packed(cgvc_handle e, const float* p, const float* beta_a, const float* gamma_a, const float* beta_g,
                               const float* gamma_g, float* y, float* stats, int R, int C, int shuffle, int precision, int gate,
                               const float* resid, const long long* offsets, int n_utt, int div, int max_len, void* hi, void* lo,
                               unsigned long long* sat, void* stream) {
  if (!offsets) return fail(e, CGVC_ERR_ARG, "null argument");
  return in_glu_forward(e, p, beta_a, gamma_a, beta_g, gamma_g, y, stats, 1, R, C, shuffle, precision, gate, resid, offsets, n_utt, div,
                        max_len, hi, lo, sat, stream);
}

int cgvc_in_glu_backward_planes(cgvc_handle e, const float* dy, const float* p, const float* stats,
                                const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                                float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                                int B, int R, int C, int shuffle, int precision, int gate, void* hi, void* lo, unsigned long long* sat,
                                void* stream) {
  return in_glu_backward(e, dy, p, stats, beta_a, gamma_a, beta_g, gamma_g, dp, dbeta_a, dgamma_a, dbeta_g, dgamma_g, nullptr, nullptr,
                         B, R, C, shuffle, precision, gate, hi, lo, sat, stream);
}

int cgvc_in_glu_backward_bias(cgvc_handle e, const float* dy, const float* p, const float* stats,
                              const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                              float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g, float* dbias_a, float* dbias_g,
                              int B, int R, int C, int shuffle, int precision, int gate, void* hi, void* lo, unsigned long long* sat,
                              void* stream) {
  return in_glu_backward(e, dy, p, stats, beta_a, gamma_a, beta_g, gamma_g, dp, dbeta_a, dgamma_a, dbeta_g, dgamma_g, dbias_a, dbias_g,
                         B, R, C, shuffle, precision, gate, hi, lo, sat, stream);
}

int cgvc_in_glu_forward(cgvc_handle e, const float* p, const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                        float* y, float* stats, int B, int R, int C, int shuffle, void* stream) {
  return cgvc_in_glu_forward_planes(e, p, beta_a, gamma_a, beta_g, gamma_g, y, stats, B, R, C, shuffle, CGVC_PREC_FP32_SIMT, 1, nullptr,
                                    nullptr, nullptr, nullptr, stream);
}

int cgvc_in_glu_backward(cgvc_handle e, const float* dy, const float* p, const float* stats,
                         const float* beta_a, const float* gamma_a, const float* beta_g, const float* gamma_g,
                         float* dp, float* dbeta_a, float* dgamma_a, float* dbeta_g, float* dgamma_g,
                         int B, int R, int C, int shuffle, void* stream) {
  return cgvc_in_glu_backward_planes(e, dy, p, stats, beta_a, gamma_a, beta_g, gamma_g, dp, dbeta_a, dgamma_a, dbeta_g, dgamma_g,
                                     B, R, C, shuffle, CGVC_PREC_FP32_SIMT, 1, nullptr, nullptr, nullptr, stream);
}

// ---- the layers without an instance norm and the loss heads (test entry points) --------------------------------------------------
// A gated layer without instance norm or shuffle (generator h1, discriminator h1) over P [B * R, 2C], in the engine's own description
static Layer glu_layer(int C) {
  Layer L{}; L.a.cout = C; L.g.cout = C; L.a.cin = L.g.cin = 1; L.has_in = 0; L.sh = L.sw = 1; L.shuffle = 1;
  return L;
}
static ConvIO rows_io(int B) { ConvIO io{}; io.n = B; return io; }

// post_params / post_bwd_params of that layer; the fields they take from the engine's precision and train-step state (plane format,
// saturation counter, arena gradients, partials slab) come from the caller's arguments instead
static PostParams glu_fwd_params(cgvc_engine* e, const float* p, float* y, int B, int R, int C, int precision, void* hi, void* lo,
                                 unsigned long long* sat) {
  const GLAct A{const_cast<float*>(p), nullptr, y, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo};
  LayerTensors t; memset(&t, 0, sizeof t);
  t.precision = precision;
  PostParams q = post_params(e, glu_layer(C), t, rows_io(B), A, R, true, nullptr);
  q.sat = q.qmode && hi ? sat : nullptr;
  q.ufl = q.qmode && hi ? e->plane_ufl : nullptr;
  return q;
}
static PostBwdParams glu_bwd_params(cgvc_engine* e, const float* dy, const float* p, float* dp, float* dbias_a, float* dbias_g, int B, int R,
                                    int C, int precision, void* hi, void* lo, unsigned long long* sat, const DetSlab* det) {
  const GLAct A{const_cast<float*>(p), nullptr, nullptr, nullptr, nullptr};
  BwdScratch S; memset(&S, 0, sizeof S); S.dP = dp;
  LayerTensors t; memset(&t, 0, sizeof t);
  t.dba = dbias_a; t.dbg = dbias_g; t.precision = precision;
  PostBwdParams q = post_bwd_params(e, glu_layer(C), t, dy, A, B, R, S, true, PlanePair{nullptr, nullptr});
  q.dp_hi = (__nv_bfloat16*)hi; q.dp_lo = (__nv_bfloat16*)lo;
  q.sat = q.qmode && hi ? sat : nullptr;
  q.ufl = q.qmode && hi ? e->plane_ufl : nullptr;
  if (dbias_a && det) q.det = *det;
  return q;
}

static int glu_shape(cgvc_engine* e, const char* what, long long B, long long R, int C) {
  if (B < 1 || B > 65535 || R < 1 || C < 4 || C % 4) return fail(e, CGVC_ERR_ARG, "%s: bad shape (B %lld, R %lld, C %d)", what, B, R, C);
  return 0;
}

int cgvc_glu_forward_planes(cgvc_handle e, const float* p, float* y, int B, int R, int C, int precision, void* hi, void* lo,
                            unsigned long long* sat, void* stream) {
  if (!e || !p || (!y && !hi)) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(glu_shape(e, "cgvc_glu_forward_planes", B, R, C));
  if (precision != CGVC_PREC_FP32_SIMT) RET(plane_precision(e, precision, hi, lo));
  else hi = lo = nullptr;
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_post_fwd(glu_fwd_params(e, p, y, B, R, C, precision, hi, lo, sat), e->opt.post, (cudaStream_t)stream));
  return 0;
}

int cgvc_glu_backward_planes(cgvc_handle e, const float* dy, const float* p, float* dp, float* dbias_a, float* dbias_g, int B, int R, int C,
                             int precision, void* hi, void* lo, unsigned long long* sat, void* stream) {
  if (!e || !dy || !p || (!dp && !hi) || (!dbias_a != !dbias_g)) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(glu_shape(e, "cgvc_glu_backward_planes", B, R, C));
  if (precision != CGVC_PREC_FP32_SIMT) RET(plane_precision(e, precision, hi, lo));
  else hi = lo = nullptr;
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_post_bwd(glu_bwd_params(e, dy, p, dp, dbias_a, dbias_g, B, R, C, precision, hi, lo, sat, det), e->opt.post, (cudaStream_t)stream));
  return 0;
}

static int c1_shape(cgvc_engine* e, const char* what, int B, int H, int W, int kh, int kw, int Cout, int sh, int sw) {
  if (B < 1 || H < 1 || W < 1 || kh < 1 || kw < 1 || kh * kw > 9 || Cout != 128 || sh < 1 || sw < 1)
    return fail(e, CGVC_ERR_ARG, "%s: bad shape (B %d, H %d, W %d, kh %d, kw %d, Cout %d, sh %d, sw %d)", what, B, H, W, kh, kw, Cout, sh, sw);
  const long long rows = (long long)((H + sh - 1) / sh) * ((W + sw - 1) / sw);
  return glu_shape(e, what, B, rows, Cout);
}

int cgvc_disc_input_forward(cgvc_handle e, int precision, const float* x, const float* w_a, const float* w_g, const float* b_a, const float* b_g,
                            float* p, float* y, void* hi, void* lo, unsigned long long* sat,
                            int B, int H, int W, int kh, int kw, int Cout, int sh, int sw, int fuse, int* fused, void* stream) {
  if (fused) *fused = 0;
  if (!e || !x || !w_a || !w_g || !b_a || !b_g || !p || (!y && !hi)) return fail(e, CGVC_ERR_ARG, "null argument");
  RET(c1_shape(e, "cgvc_disc_input_forward", B, H, W, kh, kw, Cout, sh, sw));
  if (precision != CGVC_PREC_FP32_SIMT) RET(plane_precision(e, precision, hi, lo));
  else hi = lo = nullptr;
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  const int R = ((H + sh - 1) / sh) * ((W + sw - 1) / sw);
  const Layer L = conv_layer(kh, kw, 1, Cout, true, sh, sw);
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w_a; t.kg = w_g; t.ba = b_a; t.bg = b_g;
  RET(disc_input_forward(e, L, t, x, B, H, W, p, glu_fwd_params(e, p, y, B, R, Cout, precision, hi, lo, sat), fuse != 0, (cudaStream_t)stream));
  if (fused) *fused = fuse != 0;
  return 0;
}

int cgvc_disc_input_backward(cgvc_handle e, const float* dy, const float* p, const float* x, const float* w_a, const float* w_g,
                             float* dw_a, float* dw_g, float* db_a, float* db_g, float* dx,
                             int B, int H, int W, int kh, int kw, int Cout, int sh, int sw, int fuse, int* fused, void* stream) {
  if (fused) *fused = 0;
  if (!e || !dy || !p || !x || !w_a || !w_g) return fail(e, CGVC_ERR_ARG, "null argument");
  const bool some = dw_a || dw_g || db_a || db_g;
  if (some && !(dw_a && dw_g && db_a && db_g))
    return fail(e, CGVC_ERR_ARG, "cgvc_disc_input_backward: the weight and bias gradients are all given or none");
  RET(c1_shape(e, "cgvc_disc_input_backward", B, H, W, kh, kw, Cout, sh, sw));
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  const long long rows = (long long)B * ((H + sh - 1) / sh) * ((W + sw - 1) / sw);
  // scratch: the fp32 dP of the unfused form [rows, 2 Cout], then Z [rows, taps]
  const long long ndp = fuse ? 0 : rows * 2 * Cout;
  float* buf;
  CK(grow_post_buf(e, (size_t)(ndp + rows * kh * kw), &buf));
  const Layer L = conv_layer(kh, kw, 1, Cout, true, sh, sw);
  LayerTensors t; memset(&t, 0, sizeof t);
  t.ka = w_a; t.kg = w_g; t.dka = dw_a; t.dkg = dw_g; t.dba = db_a; t.dbg = db_g;
  const PostBwdParams q = glu_bwd_params(e, dy, p, fuse ? nullptr : buf, db_a, db_g, B, (int)(rows / B), Cout, CGVC_PREC_FP32_SIMT, nullptr,
                                         nullptr, nullptr, det);
  RET(disc_input_backward(e, L, t, x, dy, p, B, H, W, dx, buf + ndp, fuse != 0, q, det, (cudaStream_t)stream));
  if (fused) *fused = fuse != 0;
  return 0;
}

int cgvc_head_forward(cgvc_handle e, const float* y, long long rows, const float* w, const float* b, float* prob, void* stream) {
  if (!e || !y || !w || !b || !prob) return fail(e, CGVC_ERR_ARG, "null argument");
  if (rows < 0) return fail(e, CGVC_ERR_ARG, "cgvc_head_forward: rows %lld", rows);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_head_fwd(y, rows, 1024, w, b, prob, (cudaStream_t)stream));
  return 0;
}

int cgvc_head_loss_backward(cgvc_handle e, const float* prob, const float* y, long long rows, const float* w, float target, float coef,
                            const float* grad_mult, float* loss, float* dy, float* dw, float* db, void* stream) {
  if (!e || !prob || !w || ((dw || db) && !y) || (!dw != !db)) return fail(e, CGVC_ERR_ARG, "null argument");
  if (rows < 0) return fail(e, CGVC_ERR_ARG, "cgvc_head_loss_backward: rows %lld", rows);
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_head_loss_bwd(prob, y, rows, 1024, w, target, coef, loss, dy, dw, db, (cudaStream_t)stream, grad_mult, det));
  return 0;
}

int cgvc_head_backward(cgvc_handle e, const float* prob, const float* y, long long rows, const float* w, const float* dprob,
                       const float* grad_mult, float* dy, float* dw, float* db, void* stream) {
  if (!e || !prob || !w || !dprob || ((dw || db) && !y) || (!dw != !db)) return fail(e, CGVC_ERR_ARG, "null argument");
  if (rows < 0) return fail(e, CGVC_ERR_ARG, "cgvc_head_backward: rows %lld", rows);
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_head_loss_bwd(prob, y, rows, 1024, w, 0.f, 0.f, nullptr, dy, dw, db, (cudaStream_t)stream, grad_mult, det, dprob));
  return 0;
}

int cgvc_l1_loss_grad(cgvc_handle e, const float* yhat, const float* y, long long n, const float* gscale, const float* grad_mult, float* loss,
                      float* d, int accumulate, void* stream) {
  if (!e || !yhat || !y) return fail(e, CGVC_ERR_ARG, "null argument");
  if (n < 0) return fail(e, CGVC_ERR_ARG, "cgvc_l1_loss_grad: n %lld", n);
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  CK(launch_l1_loss_grad(yhat, y, n, loss, gscale, d, accumulate, (cudaStream_t)stream, grad_mult, det));
  return 0;
}

}  // extern "C"

// ---- the generator's tap-lowered edge layers (test entry points) -----------------------------------------------------------------
// What every cgvc_edge_* call checks: the handle's generator `direction` runs its edge layers tap-lowered (edge_on: option edge_lower,
// a tensor-core precision, weights prepared by cgvc_params_updated), the arenas it reads and writes are bound, and the rows are B
// samples of T or (offsets, host) B packed utterances with the contract of cgvc_generator_forward_packed.  *rows: the row count
static int edge_entry(cgvc_engine* e, const char* what, int direction, int B, int T, const long long* offsets, bool grad, long long* rows) {
  if (direction != 0 && direction != 1) return fail(e, CGVC_ERR_DIRECTION, "Conversion direction must be specified.");
  if (!e->arena[CGVC_ARENA_PARAM] || (grad && !e->arena[CGVC_ARENA_GRAD]))
    return fail(e, CGVC_ERR_UNBOUND, "%s: the PARAM%s arena must be bound", what, grad ? " and GRAD" : "");
  if (!edge_on(e, e->gen[direction]))
    return fail(e, CGVC_ERR_UNSUPPORTED, "%s: the edge layers are not tap-lowered here (option edge_lower, a tensor-core precision and "
                "cgvc_params_updated are needed)", what);
  if (B < 1 || B > 65535) return fail(e, CGVC_ERR_ARG, "%s: %d samples outside [1, 65535]", what, B);
  if (offsets) {
    if (offsets[0] != 0) return fail(e, CGVC_ERR_ARG, "%s: offsets[0] is %lld, must be 0", what, offsets[0]);
    for (int u = 0; u < B; ++u) {
      const long long len = offsets[u + 1] - offsets[u];
      if (len <= 0 || len % 4 != 0)
        return fail(e, CGVC_ERR_ARG, "%s: utterance %d: length %lld must be a positive multiple of 4", what, u, len);
    }
    *rows = offsets[B];
  } else {
    if (T < 1) return fail(e, CGVC_ERR_ARG, "%s: T %d", what, T);
    *rows = (long long)B * T;
  }
  if (*rows > INT_MAX / 512) return fail(e, CGVC_ERR_ARG, "%s: %lld rows exceed %d", what, *rows, INT_MAX / 512);
  return 0;
}

extern "C" {

int cgvc_edge_h1_forward(cgvc_handle e, int direction, const float* x, int B, int T, const long long* offsets, float* p, float* y,
                         void* hi, void* lo, void* stream) {
  if (!e || !x || !p || !y || (!hi != !lo)) return fail(e, CGVC_ERR_ARG, "null argument");
  long long rows;
  RET(edge_entry(e, "cgvc_edge_h1_forward", direction, B, T, offsets, false, &rows));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const GenNet& N = e->gen[direction];
  __nv_bfloat16 *xchi, *xclo; long long* off = nullptr;
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, rows, N.h1.a.kw * e->cfg.num_features, &xchi, &xclo);
    if (offsets) off = ws.take<long long>((size_t)B + 1);
  }));
  if (offsets) CK(cudaMemcpyAsync(off, offsets, ((size_t)B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  const int n = offsets ? 1 : B, W = offsets ? (int)rows : T;
  const GLAct A{p, nullptr, y, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo};
  const PostParams q = post_params(e, N.h1, layer_tensors(e, N.h1, false), rows_io(n), A, W, true, nullptr);
  return h1_edge_forward(e, N, x, n, W, off, offsets ? B : 0, xchi, xclo, p, q, st);
}

int cgvc_edge_o1_forward(cgvc_handle e, int direction, const float* u, int B, int T, const long long* offsets, float* z, float* out,
                         void* stream) {
  if (!e || !u || !out) return fail(e, CGVC_ERR_ARG, "null argument");
  long long rows;
  RET(edge_entry(e, "cgvc_edge_o1_forward", direction, B, T, offsets, false, &rows));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const GenNet& N = e->gen[direction];
  __nv_bfloat16 *uhi, *ulo; long long* off = nullptr; float* zs = nullptr;
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, rows, N.o1.a.cin, &uhi, &ulo);
    if (offsets) off = ws.take<long long>((size_t)B + 1);
    if (!z) zs = ws.take<float>((size_t)rows * N.o1.a.kw * N.o1.a.cout);
  }));
  if (offsets) CK(cudaMemcpyAsync(off, offsets, ((size_t)B + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  CK(tc_split_planes(e->cfg.precision, u, rows, N.o1.a.cin, uhi, ulo, st));
  const int n = offsets ? 1 : B, W = offsets ? (int)rows : T;
  return o1_edge_forward(e, N, uhi, ulo, n, W, off, offsets ? B : 0, z ? z : zs, out, st);
}

int cgvc_edge_o1_backward(cgvc_handle e, int direction, const float* u, const float* d_out, int B, int T, float* du, void* dz_hi,
                          void* dz_lo, void* stream) {
  if (!e || !u || !d_out || !du || (!dz_hi != !dz_lo)) return fail(e, CGVC_ERR_ARG, "null argument");
  long long rows;
  RET(edge_entry(e, "cgvc_edge_o1_backward", direction, B, T, nullptr, true, &rows));
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const GenNet& N = e->gen[direction];
  const int nf = e->cfg.num_features;
  __nv_bfloat16 *uhi, *ulo, *zhi = (__nv_bfloat16*)dz_hi, *zlo = (__nv_bfloat16*)dz_lo;
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, rows, N.o1.a.cin, &uhi, &ulo);
    if (!dz_hi) take_planes(ws, rows, N.o1.a.kw * nf, &zhi, &zlo);
  }));
  CK(tc_split_planes(e->cfg.precision, u, rows, N.o1.a.cin, uhi, ulo, st));
  BwdScratch S; memset(&S, 0, sizeof S);
  if (det) S.det = *det;
  CK(launch_colsum(d_out, rows, nf, 0, nf, e->G() + N.o1.a.b, st, det));
  return o1_edge_backward(e, N, d_out, uhi, ulo, B, T, PlanePair{zhi, zlo}, du, S, st);
}

int cgvc_edge_h1_backward(cgvc_handle e, int direction, const float* x, const float* p, const float* dy, int B, int T, float* dp, float* dz,
                          float* dx, void* stream) {
  if (!e || !x || !p || !dy) return fail(e, CGVC_ERR_ARG, "null argument");
  long long rows;
  RET(edge_entry(e, "cgvc_edge_h1_backward", direction, B, T, nullptr, true, &rows));
  DetSlab slab; const DetSlab* det;
  RET(plan_entry_det(e, &slab, &det));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const GenNet& N = e->gen[direction];
  const int nf = e->cfg.num_features, kc = N.h1.a.kw * nf;
  __nv_bfloat16 *xchi, *xclo, *dphi, *dplo; float* zs = nullptr;
  BwdScratch S; memset(&S, 0, sizeof S);
  CK(entry_scratch(e, [&](Bump& ws) {
    take_planes(ws, rows, kc, &xchi, &xclo);
    take_planes(ws, rows, N.h1.width(), &dphi, &dplo);
    S.post = ws.take<float>((size_t)B * 4 * 1024);
    if (dx && !dz) zs = ws.take<float>((size_t)rows * kc);
  }));
  CK(launch_im2col_taps(x, rows, T, nf, N.h1.a.kw, +1, edge_cpad(kc), e->cfg.precision == CGVC_PREC_F16F8, xchi, xclo, st));
  S.dP = dp; S.dPhi = dphi; S.dPlo = dplo;
  if (det) S.det = *det;
  const GLAct A{const_cast<float*>(p), nullptr, nullptr, nullptr, nullptr};
  const PostBwdParams q = post_bwd_params(e, N.h1, layer_tensors(e, N.h1, true), dy, A, B, T, S, dp != nullptr, PlanePair{dphi, dplo});
  CK(launch_post_bwd(q, e->opt.post, st));
  return h1_edge_backward(e, N, xchi, xclo, PlanePair{q.dp_hi, q.dp_lo}, B, T, dz ? dz : zs, dx, S, st);
}

}  // extern "C"

// ---- network applications: the forwards of the C ABI, and the activation tapes that record what a backward reads ----------------
// A forward checks its geometry, plans its buffers (plan_app) in WORK or in the caller's tape, runs its network and, into a tape,
// records the header.  A tape backward re-plans the tape from that header and borrows a train step's backward scratch from WORK.

// The geometry checks of every call that takes one: the forwards, their tapes and cgvc_tape_bytes.  Kind 2 with the host offsets off
// checks them and sets a.rows and a.max_len; without them (cgvc_tape_bytes) it checks the a.rows given
static int check_geom(cgvc_engine* e, NetGeom& a, const long long* off) {
  if (a.which != 0 && a.which != 1)
    return disc_kind(a.kind) ? fail(e, CGVC_ERR_ARG, "which must be 0 (discriminator_A) or 1 (discriminator_B)")
                       : fail(e, CGVC_ERR_DIRECTION, "Conversion direction must be specified.");
  if (!packed_kind(a.kind)) return check_bt(e, a.n, a.T, a.kind == 0 ? 4 : 16);
  const int mult = a.kind == 3 ? 16 : 4;     // the discriminator halves time four times, the generator twice
  if (a.n < 1 || a.n > e->cfg.max_batch) return fail(e, CGVC_ERR_ARG, "%d utterances outside [1, %d]", a.n, e->cfg.max_batch);
  if (off) {
    if (off[0] != 0) return fail(e, CGVC_ERR_ARG, "offsets[0] is %lld, must be 0", off[0]);
    for (int u = 0; u < a.n; ++u) {
      const long long len = off[u + 1] - off[u];
      if (len <= 0 || len % mult != 0)
        return fail(e, CGVC_ERR_ARG, "utterance %d: length %lld (offsets %lld .. %lld) must be a positive multiple of %d", u, len, off[u],
                    off[u + 1], mult);
      if (len > a.max_len) a.max_len = (int)len;
    }
    a.rows = off[a.n];
  }
  const long long cap = (long long)e->cfg.max_batch * e->cfg.max_frames;
  if (a.rows < (long long)mult * a.n || a.rows % mult != 0 || a.rows > cap)
    return fail(e, CGVC_ERR_ARG, "%lld frames of %d utterances: must be a multiple of %d in [%d, %lld] (max_batch x max_frames)", a.rows,
                a.n, mult, mult * a.n, cap);
  return 0;
}

// A generator's input or output between the caller's layout ([n, 24, T], or kind 2 the [24][len_u] block of utterance u at element
// 24 offsets[u]) and channels-last rows: into the rows (to_rows) or out of them
static cudaError_t transpose_app(const cgvc_engine* e, const NetGeom& a, const GenActs& g, const float* in, float* out, bool to_rows,
                                 cudaStream_t st) {
  const int nf = e->cfg.num_features;
  if (a.kind == 2) return launch_transpose_packed(in, out, g.off, a.n, a.rows, nf, to_rows, st);
  return to_rows ? launch_transpose_ft(in, out, a.n, nf, a.T, st) : launch_transpose_ft(in, out, a.n, a.T, nf, st);
}

// The generator from in to out.  A conversion keeps the fp32 layer outputs only for the debug taps and no pre-norm outputs; a tape
// forward keeps what the backward reads
static int generator_app(cgvc_engine* e, const NetGeom& a, AppPlan& P, const long long* off, const float* in, float* out, bool tape,
                         cudaStream_t st) {
  CK(grow_post_buf(e, (size_t)a.n * 4 * 1024, &P.g.post));
  if (P.off) CK(cudaMemcpyAsync(P.off, off, ((size_t)a.n + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  CK(transpose_app(e, a, P.g, in, P.x, true, st));
  const bool keep_y = !tape && e->opt.debug_taps;
  if (!tape && !keep_y) e->taps.clear();
  RET(generator_forward(e, e->gen[a.which], P.g, P.x, st, keep_y, tape));
  CK(transpose_app(e, a, P.g, P.g.out_cl, out, false, st));
  return 0;
}

// The discriminator from in to the probabilities out.  cgvc_discriminator_forward reads in where it is and keeps every fp32 layer
// output (its taps); a tape forward copies in into the tape, where the input layer's backward reads it.  Kind 3 (off: the host
// offsets) also copies the offsets and the instance-norm segments of its levels, computed here, in front of its plan
static int discriminator_app(cgvc_engine* e, const NetGeom& a, AppPlan& P, const long long* off, const float* in, float* out, bool tape,
                             cudaStream_t st) {
  const int nf = e->cfg.num_features;
  CK(grow_post_buf(e, (size_t)a.n * 4 * 1024, &P.d.post));
  if (P.off) {
    const int Hl[3] = {nf / 2, nf / 4, nf / 4}, dl[3] = {4, 8, 16};      // (H, divisor) of the outputs of d1, d2, d3
    std::vector<long long> h((size_t)4 * (a.n + 1));
    for (int u = 0; u <= a.n; ++u) {
      h[u] = off[u];
      for (int i = 0; i < 3; ++i) h[(size_t)(i + 1) * (a.n + 1) + u] = Hl[i] * off[u] / dl[i];
    }
    CK(cudaMemcpyAsync(P.off, h.data(), h.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  }
  if (tape) CK(cudaMemcpyAsync(P.x, in, (size_t)a.rows * nf * sizeof(float), cudaMemcpyDeviceToDevice, st));
  RET(discriminator_forward(e, e->disc[a.which], P.d, tape ? P.x : in, st, !tape));
  CK(cudaMemcpyAsync(out, P.d.prob, (size_t)(nf / 4) * (a.rows / 16) * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// The header is written behind the forward on its stream; the engine's copy replaces any earlier tape at that address, and the tapes of
// older parameters are forgotten (their backward is refused either way)
static int tape_record(cgvc_engine* e, void* tape, const TapeHeader& hd, cudaStream_t st) {
  CK(cudaMemcpyAsync(tape, &hd, sizeof hd, cudaMemcpyHostToDevice, st));
  for (auto it = e->tapes.begin(); it != e->tapes.end();) it = it->second.gen != e->param_gen ? e->tapes.erase(it) : std::next(it);
  e->tapes[tape] = hd;
  return 0;
}

struct TapeBuf { void* p; size_t bytes; };   // the caller's tape of a tape forward

// Every forward of the C ABI: application a from in to out, in WORK, or with tape in that tape.  off: kind 2's host offsets.  Every
// refusal comes before anything is enqueued
static int forward_app(cgvc_engine* e, NetGeom a, const long long* off, const float* in, float* out, const TapeBuf* tape, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  if (!in || !out || (packed_kind(a.kind) && !off) || (tape && !tape->p)) return fail(e, CGVC_ERR_ARG, "null buffer");
  RET(check_geom(e, a, off));
  if (tape && ((uintptr_t)tape->p & 255)) return fail(e, CGVC_ERR_ARG, "a tape must be 256-byte aligned");
  RET(need_arenas(e, false));
  AppPlan P;
  const size_t need = plan_app(e, a, tape ? tape->p : e->arena[CGVC_ARENA_WORK], tape != nullptr, P);
  const size_t have = tape ? tape->bytes : e->arena_bytes[CGVC_ARENA_WORK];
  if (need > have)
    return fail(e, CGVC_ERR_UNBOUND, "%s of %zu bytes: %d %s of %lld frames in all need %zu", tape ? "tape" : "WORK arena", have, a.n,
                packed_kind(a.kind) ? "utterances" : "samples", a.rows, need);
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  RET(disc_kind(a.kind) ? discriminator_app(e, a, P, off, in, out, tape != nullptr, st) : generator_app(e, a, P, off, in, out, tape != nullptr, st));
  return tape ? tape_record(e, tape->p, TapeHeader{kTapeMagic, e->id, e->param_gen, a}, st) : 0;
}

// What a tape backward checks before it launches anything: the tape is one this engine wrote for `kind` under its current parameters,
// GRAD is bound and WORK holds a train step's plan at max_batch, whose lane-0 BwdScratch (sized for 2 max_batch samples) and upstream
// buffers the backward borrows.  *a and *P receive the tape's geometry and plan, *L the lane plan for its d_out / in / dY3 buffers
static int tape_backward_entry(cgvc_engine* e, int kind, const void* tape, const void* dout, NetGeom* a, AppPlan* P, LanePlan* L) {
  if (!tape || !dout) return fail(e, CGVC_ERR_ARG, "null buffer");
  auto it = e->tapes.find(tape);
  if (it == e->tapes.end())
    return fail(e, CGVC_ERR_ARG, "%p is not a tape written by this engine's cgvc_*_forward_tape since its parameters last changed", tape);
  const TapeHeader& hd = it->second;
  if (hd.gen != e->param_gen) return fail(e, CGVC_ERR_ARG, "stale tape: the parameters changed after its forward");
  static const char* const names[4] = {"generator", "discriminator", "packed generator", "packed discriminator"};
  if (disc_kind(hd.geom.kind) != (kind == 1))    // the generator backward takes kinds 0 and 2, the discriminator's 1 and 3
    return fail(e, CGVC_ERR_ARG, "a %s tape given to the %s backward", names[hd.geom.kind], names[kind]);
  if (!e->cfg.train || !e->arena[CGVC_ARENA_GRAD])
    return fail(e, CGVC_ERR_UNBOUND, "a tape backward needs the GRAD arena and a WORK arena sized for training (train = 1)");
  RET(need_arenas(e, true));
  Bump ws; ws.reset(e->arena[CGVC_ARENA_WORK], e->arena_bytes[CGVC_ARENA_WORK]);
  TrainPlan TP; plan_train(e, ws, TP, e->cfg.max_batch, e->cfg.max_frames);
  if (ws.overflow) return fail(e, CGVC_ERR_UNBOUND, "WORK arena too small for the backward scratch");
  *L = TP.lane[0];
  L->S.sq = nullptr;                                        // the weight gradients stay on the caller's stream
  *a = hd.geom;
  plan_app(e, *a, const_cast<void*>(tape), true, *P);
  P->g.post = P->d.post = L->S.post;
  return 0;
}

// the upstream gradient is counted like a train step's in monitor mode (loss_scale = 1), and in dynamic mode with "tape_loss_scale",
// into network `net`'s block
struct TapeCounting {
  cgvc_engine* e;
  TapeCounting(cgvc_engine* en, int net) : e(en) { e->counting = e->opt.ls_mode == 1 || e->opt.tape_ls; e->ls_net = net; }
  ~TapeCounting() { e->counting = false; e->ls_net = 0; }
};

// The loss scale of a tape backward's gradient planes: with "tape_loss_scale" the scaler's current scale of the network being enqueued
// (e->ls_net), read on the device (dev), after the first such call set the scaler from the static scale of its tape's batch (as a first
// train step does) and cleared the accumulation's counters; else the static scale s of the tape's batch (1 outside F16F8)
struct TapeScale { float s; const float* dev; };
static int tape_scale(cgvc_engine* e, const NetGeom& a, cudaStream_t st, TapeScale* ts) {
  if (!e->opt.tape_ls) { *ts = TapeScale{loss_scale(e, a.n), nullptr}; return 0; }
  RET(ls_prepare(e, a.n, st));
  RET(tape_counts_open(e, st));
  *ts = TapeScale{1.f, loss_scale_dev(e, a.n)};
  return 0;
}

// d in of a tape backward to the caller (din null: none): a generator's out of the channels-last rows, with the loss scale s of the
// gradient planes taken out (exact: a power of two)
static int tape_din(cgvc_engine* e, const NetGeom& a, const AppPlan& P, const float* rows, float* din, const TapeScale& s, cudaStream_t st) {
  if (!din) return 0;
  if (!disc_kind(a.kind)) CK(transpose_app(e, a, P.g, rows, din, false, st));
  if (s.dev) CK(launch_scale(din, a.rows * e->cfg.num_features, 1.f, st, s.dev));
  else if (s.s != 1.f) CK(launch_scale(din, a.rows * e->cfg.num_features, 1.f / s.s, st));
  return 0;
}

extern "C" {

int cgvc_generator_forward(cgvc_handle e, int direction, const float* in_dev, float* out_dev, int batch, int frames, void* stream) {
  return forward_app(e, net_geom(0, direction, batch, frames), nullptr, in_dev, out_dev, nullptr, stream);
}

int cgvc_generator_forward_packed(cgvc_handle e, int direction, const float* in_dev, float* out_dev,
                                  const long long* offsets_host, int n, void* stream) {
  return forward_app(e, net_geom(2, direction, n, 0), offsets_host, in_dev, out_dev, nullptr, stream);
}

int cgvc_discriminator_forward(cgvc_handle e, int which, const float* in_dev, float* out_dev, int batch, int frames, void* stream) {
  return forward_app(e, net_geom(1, which, batch, frames), nullptr, in_dev, out_dev, nullptr, stream);
}

int cgvc_discriminator_forward_packed(cgvc_handle e, int which, const float* in_dev, float* prob_dev, const long long* offsets_host, int n,
                                      void* stream) {
  return forward_app(e, net_geom(3, which, n, 0), offsets_host, in_dev, prob_dev, nullptr, stream);
}

int cgvc_tape_bytes(cgvc_handle e, int kind, int batch, int frames, size_t* bytes) {
  if (!e || !bytes || kind < 0 || kind > 3) return fail(e, CGVC_ERR_ARG, "cgvc_tape_bytes: bad argument");
  // kinds 2, 3: batch = n utterances, frames = rows = offsets[n]
  NetGeom a = packed_kind(kind) ? NetGeom{kind, 0, batch, 0, frames, 0} : net_geom(kind, 0, batch, frames);
  RET(check_geom(e, a, nullptr));
  AppPlan P;
  *bytes = plan_app(e, a, nullptr, true, P);
  return 0;
}

int cgvc_generator_forward_tape(cgvc_handle e, int direction, const float* in_dev, float* out_dev, int batch, int frames, void* tape_dev,
                                size_t tape_bytes, void* stream) {
  const TapeBuf tape{tape_dev, tape_bytes};
  return forward_app(e, net_geom(0, direction, batch, frames), nullptr, in_dev, out_dev, &tape, stream);
}

int cgvc_generator_forward_packed_tape(cgvc_handle e, int direction, const float* in_dev, float* out_dev, const long long* offsets_host, int n,
                                       void* tape_dev, size_t tape_bytes, void* stream) {
  const TapeBuf tape{tape_dev, tape_bytes};
  return forward_app(e, net_geom(2, direction, n, 0), offsets_host, in_dev, out_dev, &tape, stream);
}

int cgvc_discriminator_forward_packed_tape(cgvc_handle e, int which, const float* in_dev, float* prob_dev, const long long* offsets_host,
                                           int n, void* tape_dev, size_t tape_bytes, void* stream) {
  const TapeBuf tape{tape_dev, tape_bytes};
  return forward_app(e, net_geom(3, which, n, 0), offsets_host, in_dev, prob_dev, &tape, stream);
}

int cgvc_discriminator_forward_tape(cgvc_handle e, int which, const float* in_dev, float* prob_dev, int batch, int frames, void* tape_dev,
                                    size_t tape_bytes, void* stream) {
  const TapeBuf tape{tape_dev, tape_bytes};
  return forward_app(e, net_geom(1, which, batch, frames), nullptr, in_dev, prob_dev, &tape, stream);
}

int cgvc_generator_backward_tape(cgvc_handle e, const void* tape_dev, const float* dout_dev, float* din_dev, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  NetGeom a; AppPlan P; LanePlan L;
  RET(tape_backward_entry(e, 0, tape_dev, dout_dev, &a, &P, &L));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  // the upstream gradient channels-last, times the loss scale of the F16F8 gradient planes; a packed tape of n utterances takes the
  // static scale of a batch of n
  TapeCounting counting(e, 0);
  TapeScale s;
  RET(tape_scale(e, a, st, &s));
  CK(transpose_app(e, a, P.g, dout_dev, L.d_out, true, st));
  if (s.dev) CK(launch_scale_by(L.d_out, a.rows * e->cfg.num_features, 1.f, s.dev, st));
  else if (s.s != 1.f) CK(launch_scale(L.d_out, a.rows * e->cfg.num_features, s.s, st));
  RET(generator_backward(e, e->gen[a.which], P.g, L.d_out, din_dev ? L.in : nullptr, L.S, st));
  return tape_din(e, a, P, L.in, din_dev, s, st);
}

int cgvc_discriminator_backward_tape(cgvc_handle e, const void* tape_dev, const float* dprob_dev, float* din_dev, void* stream) {
  if (!e) return CGVC_ERR_ARG;
  NetGeom a; AppPlan P; LanePlan L;
  RET(tape_backward_entry(e, 1, tape_dev, dprob_dev, &a, &P, &L));
  DeviceGuard dguard; CK(dguard.set(e->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const DiscNet& DN = e->disc[a.which];
  const float* Pm = e->P(); float* Gm = e->G();
  TapeCounting counting(e, 1);
  TapeScale s;
  RET(tape_scale(e, a, st, &s));
  // dz = s dprob p (1 - p) through the head: dY3 and the dense kernel / bias gradients
  CK(launch_head_loss_bwd(P.d.prob, P.d.d[2].Y, (long long)(e->cfg.num_features / 4) * (a.rows / 16), 1024, Pm + DN.dense_k, 0.f,
                          0.f, nullptr, L.dY3, Gm + DN.dense_k, Gm + DN.dense_b, st, s.dev ? s.dev : static_scale_dev(e, a.n), det_of(L.S),
                          dprob_dev));
  RET(discriminator_backward(e, DN, P.d, L.dY3, true, din_dev, L.S, st));
  return tape_din(e, a, P, nullptr, din_dev, s, st);
}

}  // extern "C"
