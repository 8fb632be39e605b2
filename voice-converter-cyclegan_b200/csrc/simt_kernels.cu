// fp32 SIMT kernels of libcgvc.so (sm_90a).
//
// These are (a) the reference-arithmetic path used as the on-GPU cross-check of the tensor-core kernels and
// (b) the permanent path for everything that is not a dense contraction with K >= 64: the K=9 discriminator
// input layer (HBM-bound), the 24-channel generator input/output convs, instance-norm / GLU / residual
// elementwise passes, the discriminator head, the losses and Adam.
//
// Semantics follow /root/reference module.py:3-213, utils.py:6-12, model.py:57-108 as restated in
// SURVEY.md Appendix A.
#include "kernels.cuh"
#include <math.h>

#define IN_EPS 1e-6f   // module.py:11

unsigned long long g_cgvc_launches = 0;   // kernels launched by this library (bench.py reports it)

// ------------------------------------------------------------------------------------------------
// gather-GEMM, forward / data-gradient form
// ------------------------------------------------------------------------------------------------
// Packed variable-length utterances (launch_gg_simt_packed; VEC only): the instantiations with one trailing PackGeom argument.  Their
// A-row slots keep (first source row of the utterance, its length at the source level, local position * stride) where the dense form
// keeps (b, y, x).  The dense instantiations take no such argument.  With a trailing PackGeom2 (packed 2-D grids) the slots keep
// (first source row of the utterance, y * sy, x * sx) and the utterance's source width, and the epilogue stores into the row's own
// utterance of the destination grid.
__device__ __forceinline__ const PackGeom& pack_arg(const PackGeom& p) { return p; }
__device__ __forceinline__ const PackGeom& pack_arg(const PackGeom2& p) { return p.pk; }
template <class... PKs> struct pack_is_2d { static constexpr bool value = false; };
template <> struct pack_is_2d<PackGeom2> { static constexpr bool value = true; };
template <int BM, int BK, bool VEC, class... PKs>
__global__ void __launch_bounds__(256)
gg_simt_kernel(const __grid_constant__ GatherGeom g, const __grid_constant__ GemmOperands op, const PKs... pks) {
  constexpr bool PK = sizeof...(PKs) > 0;
  constexpr bool PK2 = pack_is_2d<PKs...>::value;
  static_assert(VEC || !PK, "the packed form gathers 4-channel quads");
  constexpr int BN = 64;
  constexpr int TM = BM / 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int HW = g.Hy * g.Wx;

  float acc[TM][4];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  if constexpr (VEC) {
    // each thread owns fixed (row, 4-channel quad) slots of the A tile
    constexpr int QPR = BK / 4;                       // quads per row
    constexpr int SLOTS = (BM * QPR + 255) / 256;
    int rb[SLOTS], ry[SLOTS], rx[SLOTS], rrow[SLOTS], rkq[SLOTS];
    int rw[PK2 ? SLOTS : 1];                          // PK2: the source width of the row's utterance
    long long rb2[PK2 ? SLOTS : 1];                   // PK2: the first source row of the row's utterance
    bool rvalid[SLOTS];
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) {
      int idx = tid + s * 256;
      int row = idx / QPR;
      rrow[s] = row; rkq[s] = (idx % QPR) * 4;
      long long m = m0 + row;
      rvalid[s] = (idx < BM * QPR) && (m < M);
      long long mm = rvalid[s] ? m : 0;
      if constexpr (PK2) {
        const PackGeom& pk = pack_arg(pks...);
        const Pack2Pos o = pack2_pos(pk, g.Hy, pk.div * g.sx, mm);
        rb2[s] = g.Hs * o.o0 / pk.div; rw[s] = (int)((o.o1 - o.o0) / pk.div); ry[s] = o.y * g.sy; rx[s] = o.x * g.sx;
      } else if constexpr (PK) {
        const PackGeom& pk = pack_arg(pks...);
        const int dout = pk.div * g.sx;
        const int u = pack_find(pk.off, pk.n, mm * dout);
        const long long o0 = __ldg(pk.off + u), o1 = __ldg(pk.off + u + 1);
        rb[s] = (int)(o0 / pk.div); ry[s] = (int)((o1 - o0) / pk.div); rx[s] = (int)(mm - o0 / dout) * g.sx;
      } else {
        int b = (int)(mm / HW); int rem = (int)(mm - (long long)b * HW);
        int y = rem / g.Wx; int x = rem - y * g.Wx;
        rb[s] = b; ry[s] = y * g.sy; rx[s] = x * g.sx;
      }
    }
    for (int t = 0; t < g.ntaps; ++t) {
      const float* aptr[SLOTS];
#pragma unroll
      for (int s = 0; s < SLOTS; ++s) {
        if constexpr (PK2) {
          const int yy = ry[s] + g.oy[t], xx = rx[s] + g.ox[t];
          const bool ok = rvalid[s] && yy >= 0 && yy < g.Hs && xx >= 0 && xx < rw[s];
          aptr[s] = ok ? op.src + (rb2[s] + (long long)yy * rw[s] + xx) * op.s_ld + op.s_coff + rkq[s] : nullptr;
        } else if constexpr (PK) {
          const int xx = rx[s] + g.ox[t];
          aptr[s] = rvalid[s] && xx >= 0 && xx < ry[s] ? op.src + (long long)(rb[s] + xx) * op.s_ld + op.s_coff + rkq[s] : nullptr;
        } else {
          int yy = ry[s] + g.oy[t], xx = rx[s] + g.ox[t];
          bool ok = rvalid[s] && yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws;
          aptr[s] = ok ? op.src + ((long long)(rb[s] * g.Hs + yy) * g.Ws + xx) * op.s_ld + op.s_coff + rkq[s] : nullptr;
        }
      }
      const float* wt = op.w + (long long)g.widx[t] * op.w_ts;
      for (int c0 = 0; c0 < op.C; c0 += BK) {
#pragma unroll
        for (int s = 0; s < SLOTS; ++s) {
          if (tid + s * 256 < BM * QPR) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (aptr[s]) v = *reinterpret_cast<const float4*>(aptr[s] + c0);
            As[rkq[s] + 0][rrow[s]] = v.x; As[rkq[s] + 1][rrow[s]] = v.y;
            As[rkq[s] + 2][rrow[s]] = v.z; As[rkq[s] + 3][rrow[s]] = v.w;
          }
        }
#pragma unroll
        for (int s = 0; s < (BK * BN) / 256; ++s) {
          int idx = tid + s * 256;
          int kk, n;
          if (op.w_ns == 1) { n = idx % BN; kk = idx / BN; } else { kk = idx % BK; n = idx / BK; }
          float v = 0.f;
          if (n0 + n < op.N) v = wt[(long long)(c0 + kk) * op.w_cs + (long long)(n0 + n) * op.w_ns];
          Bs[kk][n] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
          float a[TM];
#pragma unroll
          for (int i = 0; i < TM; i += 4) {
            float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
            a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
          }
          float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
#pragma unroll
          for (int i = 0; i < TM; ++i) {
            acc[i][0] = fmaf(a[i], bv.x, acc[i][0]); acc[i][1] = fmaf(a[i], bv.y, acc[i][1]);
            acc[i][2] = fmaf(a[i], bv.z, acc[i][2]); acc[i][3] = fmaf(a[i], bv.w, acc[i][3]);
          }
        }
        __syncthreads();
      }
    }
  } else {
    // generic path: flattened contraction index kf = t*C + c, scalar gathers (tiny layers only)
    const int Ktot = g.ntaps * op.C;
    for (int k0 = 0; k0 < Ktot; k0 += BK) {
      for (int idx = tid; idx < BM * BK; idx += 256) {
        int kk = idx % BK, row = idx / BK;
        int kf = k0 + kk;
        long long m = m0 + row;
        float v = 0.f;
        if (kf < Ktot && m < M) {
          int t = kf / op.C, c = kf - t * op.C;
          int b = (int)(m / HW); int rem = (int)(m - (long long)b * HW);
          int y = rem / g.Wx; int x = rem - y * g.Wx;
          int yy = y * g.sy + g.oy[t], xx = x * g.sx + g.ox[t];
          if (yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws)
            v = op.src[((long long)(b * g.Hs + yy) * g.Ws + xx) * op.s_ld + op.s_coff + c];
        }
        As[kk][row] = v;
      }
      for (int idx = tid; idx < BK * BN; idx += 256) {
        int n = idx % BN, kk = idx / BN;
        int kf = k0 + kk;
        float v = 0.f;
        if (kf < Ktot && n0 + n < op.N) {
          int t = kf / op.C, c = kf - t * op.C;
          v = op.w[(long long)g.widx[t] * op.w_ts + (long long)c * op.w_cs + (long long)(n0 + n) * op.w_ns];
        }
        Bs[kk][n] = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM];
#pragma unroll
        for (int i = 0; i < TM; i += 4) {
          float4 v = *reinterpret_cast<const float4*>(&As[kk][ty * TM + i]);
          a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
        }
        float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          acc[i][0] = fmaf(a[i], bv.x, acc[i][0]); acc[i][1] = fmaf(a[i], bv.y, acc[i][1]);
          acc[i][2] = fmaf(a[i], bv.z, acc[i][2]); acc[i][3] = fmaf(a[i], bv.w, acc[i][3]);
        }
      }
      __syncthreads();
    }
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + ty * TM + i;
    if (m >= M) continue;
    long long drow;
    if constexpr (PK2) {
      const PackGeom& pk = pack_arg(pks...);
      const int dout = pk.div * g.sx;
      const Pack2Pos o = pack2_pos(pk, g.Hy, dout, m);
      drow = pack2_row(o.o0, o.o1, g.Hd, dout / g.dsx, o.y * g.dsy + g.doy, o.x * g.dsx + g.dox);
      if (drow < 0) continue;                         // (a data-gradient class row always lies inside its utterance)
    } else {
      int b = (int)(m / HW); int rem = (int)(m - (long long)b * HW);
      int y = rem / g.Wx; int x = rem - y * g.Wx;
      drow = ((long long)(b * g.Hd + y * g.dsy + g.doy) * g.Wd + x * g.dsx + g.dox);
    }
    float* d = op.dst + drow * op.d_ld + op.d_coff;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < op.N) {
        float v = acc[i][j];
        if (op.bias) v += op.bias[n];
        if (op.accumulate) v += d[n];
        d[n] = v;
      }
    }
  }
}

cudaError_t launch_gg_simt_packed(const GatherGeom& g, const GemmOperands& op, const PackGeom& pk, cudaStream_t st) {
  const long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0 || op.N == 0) return cudaSuccess;
  const bool aligned = (op.s_ld % 4 == 0) && (op.s_coff % 4 == 0) && ((reinterpret_cast<uintptr_t>(op.src) & 15) == 0);
  if (!pk.off || g.B != 1 || !aligned || op.C % 8) return cudaErrorInvalidValue;
  ++g_cgvc_launches;
  const dim3 block(256);
  if (g.Hy > 1 || g.Hs > 1 || g.Hd > 1) {                   // packed 2-D grids
    const PackGeom2 p2{pk};
    if (op.C % 16 == 0) {
      if (M >= 4096) gg_simt_kernel<128, 16, true, PackGeom2><<<dim3((unsigned)((M + 127) / 128), (op.N + 63) / 64), block, 0, st>>>(g, op, p2);
      else           gg_simt_kernel<64, 16, true, PackGeom2><<<dim3((unsigned)((M + 63) / 64), (op.N + 63) / 64), block, 0, st>>>(g, op, p2);
    } else {
      if (M >= 4096) gg_simt_kernel<128, 8, true, PackGeom2><<<dim3((unsigned)((M + 127) / 128), (op.N + 63) / 64), block, 0, st>>>(g, op, p2);
      else           gg_simt_kernel<64, 8, true, PackGeom2><<<dim3((unsigned)((M + 63) / 64), (op.N + 63) / 64), block, 0, st>>>(g, op, p2);
    }
  } else if (op.C % 16 == 0) {
    if (M >= 4096) gg_simt_kernel<128, 16, true, PackGeom><<<dim3((unsigned)((M + 127) / 128), (op.N + 63) / 64), block, 0, st>>>(g, op, pk);
    else           gg_simt_kernel<64, 16, true, PackGeom><<<dim3((unsigned)((M + 63) / 64), (op.N + 63) / 64), block, 0, st>>>(g, op, pk);
  } else {
    if (M >= 4096) gg_simt_kernel<128, 8, true, PackGeom><<<dim3((unsigned)((M + 127) / 128), (op.N + 63) / 64), block, 0, st>>>(g, op, pk);
    else           gg_simt_kernel<64, 8, true, PackGeom><<<dim3((unsigned)((M + 63) / 64), (op.N + 63) / 64), block, 0, st>>>(g, op, pk);
  }
  return cudaGetLastError();
}

cudaError_t launch_gg_simt(const GatherGeom& g, const GemmOperands& op, cudaStream_t st) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0 || op.N == 0) return cudaSuccess;
  ++g_cgvc_launches;
  bool aligned = (op.s_ld % 4 == 0) && (op.s_coff % 4 == 0) && ((reinterpret_cast<uintptr_t>(op.src) & 15) == 0);
  dim3 block(256);
  if (aligned && op.C % 16 == 0) {
    if (M >= 4096) { dim3 grid((unsigned)((M + 127) / 128), (op.N + 63) / 64); gg_simt_kernel<128, 16, true><<<grid, block, 0, st>>>(g, op); }
    else           { dim3 grid((unsigned)((M + 63) / 64), (op.N + 63) / 64);   gg_simt_kernel<64, 16, true><<<grid, block, 0, st>>>(g, op); }
  } else if (aligned && op.C % 8 == 0) {
    if (M >= 4096) { dim3 grid((unsigned)((M + 127) / 128), (op.N + 63) / 64); gg_simt_kernel<128, 8, true><<<grid, block, 0, st>>>(g, op); }
    else           { dim3 grid((unsigned)((M + 63) / 64), (op.N + 63) / 64);   gg_simt_kernel<64, 8, true><<<grid, block, 0, st>>>(g, op); }
  } else {
    dim3 grid((unsigned)((M + 63) / 64), (op.N + 63) / 64);
    gg_simt_kernel<64, 16, false><<<grid, block, 0, st>>>(g, op);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// weight gradient (forward geometry), split over rows with atomic accumulation into the GRAD arena
// ------------------------------------------------------------------------------------------------
// Packed variable-length utterances (launch_wgrad_simt with pk; VEC only): the instantiation with one trailing PackGeom argument.  Row m
// (an output row of all packed rows) reads its source row from its own utterance; a tap outside it contributes a zero row.
template <bool VEC, class... PKs>
__global__ void __launch_bounds__(256)
wgrad_simt_kernel(const __grid_constant__ GatherGeom g, const float* __restrict__ src, int s_ld, int s_coff, int C,
                  const float* __restrict__ grad, int g_ld, int g_coff, int N,
                  float* __restrict__ dw, long long w_ts, int w_cs, int w_ns, int ksplit, const PKs... pks) {
  constexpr bool PK = sizeof...(PKs) > 0;
  constexpr bool PK2 = pack_is_2d<PKs...>::value;
  static_assert(VEC || !PK, "the packed form reads 4-channel quads");
  __shared__ __align__(16) float As[16][64 + 4];
  __shared__ __align__(16) float Gs[16][64 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const int t = blockIdx.z % g.ntaps, ks = blockIdx.z / g.ntaps;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  const int HW = g.Hy * g.Wx;
  long long chunk = (M + ksplit - 1) / ksplit;
  chunk = (chunk + 15) / 16 * 16;
  const long long mbeg = (long long)ks * chunk;
  const long long mend = (mbeg + chunk < M) ? mbeg + chunk : M;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int lrow = tid >> 4, lq = (tid & 15) * 4;
  for (long long mb = mbeg; mb < mend; mb += 16) {
    long long m = mb + lrow;
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f), gv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < mend) {
      if constexpr (PK2) {                           // packed 2-D grids: a tap outside the row's utterance gives a zero row
        const PackGeom& pk = pack_arg(pks...);
        const Pack2Pos o = pack2_pos(pk, g.Hy, pk.div * g.sx, m);
        const long long r = pack2_row(o.o0, o.o1, g.Hs, pk.div, o.y * g.sy + g.oy[t], o.x * g.sx + g.ox[t]);
        if (r >= 0 && c0 + lq < C) av = *reinterpret_cast<const float4*>(src + r * s_ld + s_coff + c0 + lq);
      } else if constexpr (PK) {
        const PackGeom& pk = pack_arg(pks...);
        const int dout = pk.div * g.sx;
        const int u = pack_find(pk.off, pk.n, m * dout);
        const long long o0 = __ldg(pk.off + u), o1 = __ldg(pk.off + u + 1);
        const int xx = (int)(m - o0 / dout) * g.sx + g.ox[t];
        if (xx >= 0 && xx < (int)((o1 - o0) / pk.div) && c0 + lq < C)
          av = *reinterpret_cast<const float4*>(src + (o0 / pk.div + xx) * s_ld + s_coff + c0 + lq);
      } else {
      int b = (int)(m / HW); int rem = (int)(m - (long long)b * HW);
      int y = rem / g.Wx; int x = rem - y * g.Wx;
      int yy = y * g.sy + g.oy[t], xx = x * g.sx + g.ox[t];
      if (yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws) {
        const float* sp = src + ((long long)(b * g.Hs + yy) * g.Ws + xx) * s_ld + s_coff;
        if (VEC) { if (c0 + lq < C) av = *reinterpret_cast<const float4*>(sp + c0 + lq); }
        else {
          if (c0 + lq + 0 < C) av.x = sp[c0 + lq + 0];
          if (c0 + lq + 1 < C) av.y = sp[c0 + lq + 1];
          if (c0 + lq + 2 < C) av.z = sp[c0 + lq + 2];
          if (c0 + lq + 3 < C) av.w = sp[c0 + lq + 3];
        }
      }
      }
      const float* gp = grad + m * g_ld + g_coff;
      if (VEC) { if (n0 + lq < N) gv = *reinterpret_cast<const float4*>(gp + n0 + lq); }
      else {
        if (n0 + lq + 0 < N) gv.x = gp[n0 + lq + 0];
        if (n0 + lq + 1 < N) gv.y = gp[n0 + lq + 1];
        if (n0 + lq + 2 < N) gv.z = gp[n0 + lq + 2];
        if (n0 + lq + 3 < N) gv.w = gp[n0 + lq + 3];
      }
    }
    *reinterpret_cast<float4*>(&As[lrow][lq]) = av;
    *reinterpret_cast<float4*>(&Gs[lrow][lq]) = gv;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Gs[kk][tx * 4]);
      float aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* wt = dw + (long long)g.widx[t] * w_ts;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int c = c0 + ty * 4 + i;
    if (c >= C) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < N) atomicAdd(wt + (long long)c * w_cs + (long long)n * w_ns, acc[i][j]);
    }
  }
}

cudaError_t launch_wgrad_simt(const GatherGeom& g, const float* src, int s_ld, int s_coff, int C,
                              const float* grad, int g_ld, int g_coff, int N,
                              float* dw, long long w_ts, int w_cs, int w_ns, cudaStream_t st, int det, const PackGeom* pk) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0) return cudaSuccess;
  if (pk && (!pk->off || g.B != 1)) return cudaErrorInvalidValue;
  ++g_cgvc_launches;
  int tiles = ((N + 63) / 64) * ((C + 63) / 64) * g.ntaps;
  int ksplit = det ? 1 : (592 + tiles - 1) / tiles;       // det: one CTA, one thread and one add per element
  long long maxsplit = (M + 63) / 64;
  if (ksplit > maxsplit) ksplit = (int)maxsplit;
  if (ksplit < 1) ksplit = 1;
  if ((long long)g.ntaps * ksplit > 65535) ksplit = 65535 / g.ntaps;
  dim3 grid((N + 63) / 64, (C + 63) / 64, g.ntaps * ksplit);
  bool vec = (C % 4 == 0) && (N % 4 == 0) && (s_ld % 4 == 0) && (s_coff % 4 == 0) && (g_ld % 4 == 0) && (g_coff % 4 == 0) &&
             ((reinterpret_cast<uintptr_t>(src) & 15) == 0) && ((reinterpret_cast<uintptr_t>(grad) & 15) == 0);
  if (pk && (g.Hy > 1 || g.Hs > 1)) {                       // packed 2-D grids
    if (!vec) return cudaErrorInvalidValue;
    wgrad_simt_kernel<true, PackGeom2><<<grid, 256, 0, st>>>(g, src, s_ld, s_coff, C, grad, g_ld, g_coff, N, dw, w_ts, w_cs, w_ns, ksplit,
                                                             PackGeom2{*pk});
  } else if (pk) {
    if (!vec) return cudaErrorInvalidValue;
    wgrad_simt_kernel<true, PackGeom><<<grid, 256, 0, st>>>(g, src, s_ld, s_coff, C, grad, g_ld, g_coff, N, dw, w_ts, w_cs, w_ns, ksplit, *pk);
  }
  else if (vec) wgrad_simt_kernel<true><<<grid, 256, 0, st>>>(g, src, s_ld, s_coff, C, grad, g_ld, g_coff, N, dw, w_ts, w_cs, w_ns, ksplit);
  else     wgrad_simt_kernel<false><<<grid, 256, 0, st>>>(g, src, s_ld, s_coff, C, grad, g_ld, g_coff, N, dw, w_ts, w_cs, w_ns, ksplit);
  return cudaGetLastError();
}

// db[n] += sum over rows
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ grad, long long rows, int g_ld, int g_coff, int N, float* __restrict__ db, int rows_per_block,
              float* __restrict__ part) {
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  long long r0 = (long long)blockIdx.y * rows_per_block;
  long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
  float s = 0.f;
  if (n < N)
    for (long long r = r0 + warp; r < r1; r += 8) s += grad[r * g_ld + g_coff + n];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && n < N) {
    float tsum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tsum += red[w][lane];
    if (part) part[(long long)blockIdx.y * N + n] = tsum;
    else atomicAdd(db + n, tsum);
  }
}

cudaError_t launch_colsum(const float* grad, long long rows, int g_ld, int g_coff, int N, float* db, cudaStream_t st, const DetSlab* det) {
  if (rows == 0) return cudaSuccess;
  int rpb = 2048;
  dim3 grid((N + 31) / 32, (unsigned)((rows + rpb - 1) / rpb));
  float* part = det ? det->p : nullptr;
  if (part && (long long)grid.y * N > det->cap) return cudaErrorInvalidValue;
  ++g_cgvc_launches; colsum_kernel<<<grid, 256, 0, st>>>(grad, rows, g_ld, g_coff, N, db, rpb, part);
  if (!part) return cudaGetLastError();
  return launch_reduce_parts(part, grid.y, N, DetSegs{{db}, {0}, {N}}, st);
}

// deterministic mode: dst[i][j] += the rows' values summed in row order, one atomic add per element (the other lane may add into the
// same GRAD element concurrently; with one add per lane the result does not depend on which comes first)
__global__ void __launch_bounds__(256)
reduce_parts_kernel(const float* __restrict__ part, long long nparts, long long row, const DetSegs s, long long total) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  int k = 0; long long j = i;
  while (j >= s.len[k]) { j -= s.len[k]; ++k; }
  if (!s.dst[k]) return;
  const float* p = part + s.off[k] + j;
  float acc = p[0];
  for (long long r = 1; r < nparts; ++r) acc += p[r * row];
  atomicAdd(s.dst[k] + j, acc);
}

cudaError_t launch_reduce_parts(const float* part, long long nparts, long long row, const DetSegs& s, cudaStream_t st) {
  long long total = 0;
  for (int k = 0; k < 4; ++k) {
    if (s.len[k] < 0 || (s.len[k] && s.off[k] + s.len[k] > row)) return cudaErrorInvalidValue;
    total += s.len[k];
  }
  if (total == 0 || nparts < 1) return cudaSuccess;
  ++g_cgvc_launches; reduce_parts_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(part, nparts, row, s, total);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// instance norm + GLU (+ pixel-shuffle view, + residual) forward
// one CTA per (sample, 32-channel group): lane = channel, the 8 warps stride over positions
// ------------------------------------------------------------------------------------------------
// sigmoid with the hardware exp2 / reciprocal units (relative error ~1e-6, far inside the 1e-3 parity budget); the post
// kernels are instruction-issue bound (ncu: 60-65 % issue-active at 27-56 % DRAM), so the IEEE expf + division mattered
__device__ __forceinline__ float sigmoidf_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }

__device__ __forceinline__ float block_sum8(float v, float (*red)[32], int warp, int lane) {
  __syncthreads();
  red[warp][lane] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w][lane];
  return s;
}

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// The instance-norm "post" kernels are streaming kernels: CTA = (128-channel group, 32-position chunk, sample);
// thread = (position lane rl = warp 0..7, channel quad cq = lane): 16-byte accesses, 128 channels x 4 positions per thread
// sweep.  The per-(sample, channel) reductions of instance norm are split off into a first streaming kernel that
// accumulates SHIFTED sums (x - x[first position], robust against |mean| >> std) with one atomicAdd per channel per CTA;
// the second kernel is purely elementwise.  Both are HBM-bound; nothing is cached across kernels except via L2.
struct F4 { float v[4]; };
__device__ __forceinline__ F4 ld4(const float* p) { float4 t = *reinterpret_cast<const float4*>(p); return F4{{t.x, t.y, t.z, t.w}}; }
__device__ __forceinline__ void st4(float* p, const F4& a) { *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]); }
__device__ __forceinline__ void st4_split(__nv_bfloat16* hi, __nv_bfloat16* lo, const F4& a) {
  // packed conversions: 2 x cvt.rn.bf16x2.f32 for hi, 2 for lo
  __nv_bfloat162 h01 = __floats2bfloat162_rn(a.v[0], a.v[1]), h23 = __floats2bfloat162_rn(a.v[2], a.v[3]);
  float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  __nv_bfloat162 l01 = __floats2bfloat162_rn(a.v[0] - f01.x, a.v[1] - f01.y), l23 = __floats2bfloat162_rn(a.v[2] - f23.x, a.v[3] - f23.y);
  uint2 hv, lv;
  hv.x = *reinterpret_cast<uint32_t*>(&h01); hv.y = *reinterpret_cast<uint32_t*>(&h23);
  lv.x = *reinterpret_cast<uint32_t*>(&l01); lv.y = *reinterpret_cast<uint32_t*>(&l23);
  *reinterpret_cast<uint2*>(hi) = hv;
  *reinterpret_cast<uint2*>(lo) = lv;
}
// F16F8 planes of 4 consecutive activation values (o = element offset, n = elements per plane); sat, ufl: see cgvc_count_planes
__device__ __forceinline__ void st4_quant(__nv_bfloat16* q16, __nv_bfloat16* q8, long long o, long long n, const F4& a,
                                          unsigned long long* sat = nullptr, unsigned long long* ufl = nullptr) {
  uint2 h; uint32_t b_hi, b_lo;
  cgvc_quant4(a.v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO, h, b_hi, b_lo);
  *reinterpret_cast<uint2*>(q16 + o) = h;
  uint8_t* base = reinterpret_cast<uint8_t*>(q8);
  *reinterpret_cast<uint32_t*>(base + o) = b_hi;
  *reinterpret_cast<uint32_t*>(base + n + o) = b_lo;
  cgvc_count_planes(sat, ufl, a.v);
}
__device__ __forceinline__ F4 zero4() { return F4{{0.f, 0.f, 0.f, 0.f}}; }
__device__ __forceinline__ F4 one4() { return F4{{1.f, 1.f, 1.f, 1.f}}; }
__device__ __forceinline__ void atomic_add4(float* p, const F4& a) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a.v[0]), "f"(a.v[1]), "f"(a.v[2]), "f"(a.v[3]) : "memory");
}

// saturated groups among the gradient planes of da (and dg): out of line, so that the counting leaves the register allocation of the
// kernel's uncounted path alone
__device__ __noinline__ unsigned sat_groups(const F4 da, const F4 dg, bool gate) {
  return cgvc_sat4(da.v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO) + (gate && cgvc_sat4(dg.v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO));
}
// ... and their groups below the fp16 lower edge (cgvc_ufl4)
__device__ __noinline__ unsigned ufl_groups(const F4 da, const F4 dg, bool gate) {
  return cgvc_ufl4(da.v) + (gate && cgvc_ufl4(dg.v));
}

constexpr int kPostRows = 32;      // positions per CTA
constexpr int kPostChan = 128;     // channels per CTA

struct PostIdx {
  int c, b, r0, rl; bool cvalid;
  __device__ PostIdx(int C) {
    rl = threadIdx.x >> 5; c = blockIdx.x * kPostChan + (threadIdx.x & 31) * 4; b = blockIdx.z;
    r0 = blockIdx.y * kPostRows + rl; cvalid = c < C;
  }
};

// sum NQ per-thread F4 quantities over the 8 position lanes; the result lands in warp 0 (all lanes).  One 4 KB exchange buffer,
// one quantity at a time: these kernels run next to a persistent tensor-core CTA of the other lane, which leaves < 12 KB of the
// SM's shared memory.
template <int NQ>
__device__ __forceinline__ void sum_over_rows(F4 (&x)[NQ], float4 (*red)[32], int rl, int lane) {
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    red[rl][lane] = make_float4(x[q].v[0], x[q].v[1], x[q].v[2], x[q].v[3]);
    __syncthreads();
    if (rl == 0) {
      F4 r = zero4();
#pragma unroll
      for (int w = 0; w < 8; ++w) { float4 t = red[w][lane]; r.v[0] += t.x; r.v[1] += t.y; r.v[2] += t.z; r.v[3] += t.w; }
      x[q] = r;
    }
    __syncthreads();
  }
}

// sample b's first view row and its positions (PK: packed variable-length samples, PostParams::seg)
template <bool PK>
__device__ __forceinline__ void post_sample(const PostParams& q, int b, long long& s0, int& R) {
  if constexpr (PK) {
    const long long o0 = q.seg.off[b], o1 = q.seg.off[b + 1];
    s0 = o0 / q.seg.div; R = (int)((o1 - o0) / q.seg.div);
  } else {
    s0 = (long long)b * q.R; R = q.R;
  }
}

// scratch[b][q][c], q = 0..3: sum(a-ka), sum((a-ka)^2), sum(g-kg), sum((g-kg)^2)
template <bool HAS_GATE, bool PK = false>
__global__ void __launch_bounds__(256)
post_stats_kernel(const __grid_constant__ PostParams q, float* __restrict__ scratch) {
  __shared__ float4 red[8][32];
  const PostIdx ix(q.C);
  const int lane = threadIdx.x & 31;
  long long s0; int R;
  post_sample<PK>(q, ix.b, s0, R);
  const float* pb = q.p + s0 / q.sh * q.ldp;                  // s0 is a multiple of sh (whole conv rows)
  F4 acc[4] = {zero4(), zero4(), zero4(), zero4()};
  if (ix.cvalid) {
    const F4 ka = ld4(pb + ix.c), kg = HAS_GATE ? ld4(pb + q.Cc + ix.c) : zero4();       // shift = value at position 0
    // the whole position range is reduced inside one CTA (grid.y == 1): deterministic, no atomics
#pragma unroll 4
    for (int r = ix.rl; r < R; r += 8) {
      {
        int w = r >> (q.sh - 1); int s = r & (q.sh - 1);
        long long a = (long long)w * q.ldp + s * q.C + ix.c;
        F4 xa = ld4(pb + a);
#pragma unroll
        for (int k = 0; k < 4; ++k) { float d = xa.v[k] - ka.v[k]; acc[0].v[k] += d; acc[1].v[k] += d * d; }
        if (HAS_GATE) {
          F4 xg = ld4(pb + a + q.Cc);
#pragma unroll
          for (int k = 0; k < 4; ++k) { float d = xg.v[k] - kg.v[k]; acc[2].v[k] += d; acc[3].v[k] += d * d; }
        }
      }
    }
  }
  sum_over_rows<4>(acc, red, ix.rl, lane);
  if (ix.rl == 0 && ix.cvalid) {
    float* sc = scratch + (long long)ix.b * 4 * q.C + ix.c;
    st4(sc, acc[0]); st4(sc + q.C, acc[1]);
    if (HAS_GATE) { st4(sc + 2 * q.C, acc[2]); st4(sc + 3 * q.C, acc[3]); }
  }
}

template <bool HAS_IN, bool HAS_GATE, bool PK = false>
__global__ void __launch_bounds__(256)
post_apply_fwd_kernel(const __grid_constant__ PostParams q, const float* __restrict__ scratch) {
  const PostIdx ix(q.C);
  if (!ix.cvalid) return;
  long long s0; int R;
  post_sample<PK>(q, ix.b, s0, R);
  if (PK && (int)blockIdx.y * kPostRows >= R) return;        // past the end of a shorter sample (R >= 1: block y = 0 stays and writes the stats)
  const float* pb = q.p + s0 / q.sh * q.ldp;
  // per channel: norm(x) = x * sc + of  (sc = rstd*gamma, of = beta - mean*sc)
  F4 sca = one4(), ofa = zero4(), scg = one4(), ofg = zero4();
  if (HAS_IN) {
    const float* sc = scratch + (long long)ix.b * 4 * q.C + ix.c;
    const float invR = 1.f / (float)R;
    F4 mean_a, rstd_a, mean_g = zero4(), rstd_g = one4();
    {
      F4 ka = ld4(pb + ix.c), s1 = ld4(sc), s2 = ld4(sc + q.C), ga = ld4(q.gamma_a + ix.c), ba = ld4(q.beta_a + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float m = s1.v[k] * invR; float var = fmaxf(s2.v[k] * invR - m * m, 0.f);
        mean_a.v[k] = ka.v[k] + m; rstd_a.v[k] = 1.f / sqrtf(var + IN_EPS);
        sca.v[k] = rstd_a.v[k] * ga.v[k]; ofa.v[k] = ba.v[k] - mean_a.v[k] * sca.v[k];
      }
    }
    if (HAS_GATE) {
      F4 kg = ld4(pb + q.Cc + ix.c), t1 = ld4(sc + 2 * q.C), t2 = ld4(sc + 3 * q.C), gg = ld4(q.gamma_g + ix.c), bg = ld4(q.beta_g + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float m = t1.v[k] * invR; float var = fmaxf(t2.v[k] * invR - m * m, 0.f);
        mean_g.v[k] = kg.v[k] + m; rstd_g.v[k] = 1.f / sqrtf(var + IN_EPS);
        scg.v[k] = rstd_g.v[k] * gg.v[k]; ofg.v[k] = bg.v[k] - mean_g.v[k] * scg.v[k];
      }
    }
    if (blockIdx.y == 0 && ix.rl == 0 && q.stats) {
      float* s = q.stats + (long long)ix.b * 4 * q.C + ix.c;
      st4(s, mean_a); st4(s + q.C, rstd_a); st4(s + 2 * q.C, mean_g); st4(s + 3 * q.C, rstd_g);
    }
  }
  const int shs = q.sh - 1;                                   // sh is 1 or 2
#pragma unroll
  for (int i = 0; i < kPostRows / 8; ++i) {
    const int r = ix.r0 + 8 * i;
    if (r < R) {
      const int w = r >> shs, s = r & shs;
      const long long a = (long long)w * q.ldp + s * q.C + ix.c;
      F4 xa = ld4(pb + a), xg = HAS_GATE ? ld4(pb + a + q.Cc) : zero4(), y;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float na = HAS_IN ? fmaf(xa.v[k], sca.v[k], ofa.v[k]) : xa.v[k];
        if (HAS_GATE) {
          float ng = HAS_IN ? fmaf(xg.v[k], scg.v[k], ofg.v[k]) : xg.v[k];
          na *= sigmoidf_(ng);
        }
        y.v[k] = na;
      }
      const long long o = (s0 + r) * q.C + ix.c;
      if (q.resid) { F4 rr = ld4(q.resid + o);
#pragma unroll
        for (int k = 0; k < 4; ++k) y.v[k] += rr.v[k]; }
      if (q.y) st4(q.y + o, y);
      if (q.y_hi) {
        if (q.qmode) st4_quant(q.y_hi, q.y_lo, o, PK ? q.seg_rows * q.C : (long long)q.B * q.R * q.C, y, q.sat, q.ufl);
        else st4_split(q.y_hi + o, q.y_lo + o, y);
      }
    }
  }
}

static bool post_aligned(const void* a, const void* b, const void* c, int ldp, int C, int Cc) {
  return ldp % 4 == 0 && C % 4 == 0 && Cc % 4 == 0 && ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}

static bool post_fwd_stream_dispatch(const PostParams& pp, bool stream, cudaStream_t st, cudaError_t* err);   // streaming one-pass form, further down

// packed variable-length samples (PostParams::seg): one CTA column per sample, grid.y sized by the longest
static cudaError_t launch_post_fwd_packed(const PostParams& pp, cudaStream_t st) {
  if (pp.seg.div < 1 || 4 % (pp.seg.div * pp.sh)) return cudaErrorInvalidValue;     // samples start on whole conv rows: off[u] / div % sh == 0
  dim3 grid((pp.C + kPostChan - 1) / kPostChan, (pp.R + kPostRows - 1) / kPostRows, pp.B);
  float* scratch = pp.scratch;
  if (pp.has_in) {
    ++g_cgvc_launches;
    if (pp.has_gate) post_stats_kernel<true, true><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
    else post_stats_kernel<false, true><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
  }
  ++g_cgvc_launches;
  if (pp.has_in) { if (pp.has_gate) post_apply_fwd_kernel<true, true, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_fwd_kernel<true, false, true><<<grid, 256, 0, st>>>(pp, scratch); }
  else           { if (pp.has_gate) post_apply_fwd_kernel<false, true, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_fwd_kernel<false, false, true><<<grid, 256, 0, st>>>(pp, scratch); }
  return cudaGetLastError();
}

cudaError_t launch_post_fwd(const PostParams& pp, PostForms forms, cudaStream_t st) {
  if (pp.B == 0) return cudaSuccess;
  if (!post_aligned(pp.p, pp.y, pp.resid, pp.ldp, pp.C, pp.Cc) || (pp.sh != 1 && pp.sh != 2) || pp.B > 65535 || (pp.has_in && !pp.scratch))
    return cudaErrorInvalidValue;
  if (pp.seg.off) return launch_post_fwd_packed(pp, st);
  { cudaError_t se = cudaSuccess; if (post_fwd_stream_dispatch(pp, forms.stream, st, &se)) return se; }
  dim3 grid((pp.C + kPostChan - 1) / kPostChan, (pp.R + kPostRows - 1) / kPostRows, pp.B);
  float* scratch = pp.scratch;
  if (pp.has_in) {
    ++g_cgvc_launches;
    if (pp.has_gate) post_stats_kernel<true><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
    else post_stats_kernel<false><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
  }
  ++g_cgvc_launches;
  if (pp.has_in) { if (pp.has_gate) post_apply_fwd_kernel<true, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_fwd_kernel<true, false><<<grid, 256, 0, st>>>(pp, scratch); }
  else           { if (pp.has_gate) post_apply_fwd_kernel<false, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_fwd_kernel<false, false><<<grid, 256, 0, st>>>(pp, scratch); }
  return cudaGetLastError();
}

// ---- backward (SURVEY.md Appendix A.7) ----
// scratch[b][q][c], q = 0..3: S1a = sum dna, S2a = sum dna*ahat, S1g, S2g; also accumulates dgamma / dbeta
// Packed variable-length samples (launch_post_bwd with a PostBwdSeg): the instantiations with one trailing PostBwdSeg argument, whose
// sample b is view rows [s0, s0 + R) of post_bwd_seg and has its own statistics.  The equal-length instantiations take no such argument.
// Sample b's first view row, its view rows, its first conv row (Rw: conv rows per equal-length sample) and the rows of the planes.
template <class... Seg> __device__ __forceinline__ long long bwd_first(const PostBwdParams& q, int b, const Seg&... sg) {
  if constexpr (sizeof...(Seg) > 0) { const PostBwdSeg& s = (sg, ...); return s.seg.off[b] / s.seg.div; }
  else return (long long)b * q.R;
}
template <class... Seg> __device__ __forceinline__ int bwd_len(const PostBwdParams& q, int b, const Seg&... sg) {
  if constexpr (sizeof...(Seg) > 0) { const PostBwdSeg& s = (sg, ...); return (int)((s.seg.off[b + 1] - s.seg.off[b]) / s.seg.div); }
  else return q.R;
}
template <class... Seg> __device__ __forceinline__ long long bwd_conv0(const PostBwdParams& q, int b, int Rw, const Seg&... sg) {
  if constexpr (sizeof...(Seg) > 0) return bwd_first(q, b, sg...) / q.sh;         // a multiple of sh: whole conv rows
  else return (long long)b * Rw;
}
template <class... Seg> __device__ __forceinline__ long long bwd_conv_rows(const PostBwdParams& q, int Rw, const Seg&... sg) {
  if constexpr (sizeof...(Seg) > 0) { const PostBwdSeg& s = (sg, ...); return s.rows / q.sh; }
  else return (long long)q.B * Rw;
}

template <bool HAS_GATE, class... Seg>
__global__ void __launch_bounds__(256)
post_bwd_sums_kernel(const __grid_constant__ PostBwdParams q, float* __restrict__ scratch, const Seg... sg) {
  __shared__ float4 red[8][32];
  const PostIdx ix(q.C);
  const int lane = threadIdx.x & 31;
  const int Rw = q.R / q.sh;
  const float* pb = q.p + bwd_conv0(q, ix.b, Rw, sg...) * q.ldp;
  F4 acc[4] = {zero4(), zero4(), zero4(), zero4()};
  if (ix.cvalid) {
    // per channel: xhat = x*r + h ; norm = x*sc + of
    F4 ra, ha, sca, ofa, rg = one4(), hg = zero4(), scg = one4(), ofg = zero4();
    const float* st = q.stats + (long long)ix.b * 4 * q.C + ix.c;
    {
      F4 mean = ld4(st), rstd = ld4(st + q.C), gam = ld4(q.gamma_a + ix.c), bet = ld4(q.beta_a + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) { ra.v[k] = rstd.v[k]; ha.v[k] = -mean.v[k] * rstd.v[k]; sca.v[k] = rstd.v[k] * gam.v[k]; ofa.v[k] = bet.v[k] - mean.v[k] * sca.v[k]; }
    }
    if (HAS_GATE) {
      F4 mean = ld4(st + 2 * q.C), rstd = ld4(st + 3 * q.C), gam = ld4(q.gamma_g + ix.c), bet = ld4(q.beta_g + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) { rg.v[k] = rstd.v[k]; hg.v[k] = -mean.v[k] * rstd.v[k]; scg.v[k] = rstd.v[k] * gam.v[k]; ofg.v[k] = bet.v[k] - mean.v[k] * scg.v[k]; }
    }
    const int shs = q.sh - 1;
#pragma unroll 2
    for (int r = ix.rl; r < bwd_len(q, ix.b, sg...); r += 8) {   // whole position range in one CTA (grid.y == 1): deterministic
      const int w = r >> shs, s = r & shs;
      const long long a = (long long)w * q.ldp + s * q.C + ix.c;
      const long long o = (bwd_first(q, ix.b, sg...) + r) * q.C + ix.c;
      F4 xa = ld4(pb + a), xg = HAS_GATE ? ld4(pb + a + q.Cc) : zero4(), dy = ld4(q.dy1 + o);
      if (q.dy2) { F4 d2 = ld4(q.dy2 + o);
#pragma unroll
        for (int k = 0; k < 4; ++k) dy.v[k] += d2.v[k]; }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float dna = dy.v[k];
        if (HAS_GATE) {
          float na = fmaf(xa.v[k], sca.v[k], ofa.v[k]), ng = fmaf(xg.v[k], scg.v[k], ofg.v[k]);
          float sg = sigmoidf_(ng);
          dna = dy.v[k] * sg;
          float dng = dna * na * (1.f - sg);
          float gh = fmaf(xg.v[k], rg.v[k], hg.v[k]);
          acc[2].v[k] += dng; acc[3].v[k] = fmaf(dng, gh, acc[3].v[k]);
        }
        float ah = fmaf(xa.v[k], ra.v[k], ha.v[k]);
        acc[0].v[k] += dna; acc[1].v[k] = fmaf(dna, ah, acc[1].v[k]);
      }
    }
  }
  sum_over_rows<4>(acc, red, ix.rl, lane);
  if (ix.rl == 0 && ix.cvalid) {
    float* sc = scratch + (long long)ix.b * 4 * q.C + ix.c;
    st4(sc, acc[0]); st4(sc + q.C, acc[1]);
    if (HAS_GATE) { st4(sc + 2 * q.C, acc[2]); st4(sc + 3 * q.C, acc[3]); }
    if (q.dgamma_a && !q.det.p) {                        // null when only the data gradient is wanted (G-step through D); det: see launch_post_bwd
      atomic_add4(q.dbeta_a + ix.c, acc[0]); atomic_add4(q.dgamma_a + ix.c, acc[1]);
      if (HAS_GATE) { atomic_add4(q.dbeta_g + ix.c, acc[2]); atomic_add4(q.dgamma_g + ix.c, acc[3]); }
    }
  }
}

template <bool HAS_IN, bool HAS_GATE>
__global__ void __launch_bounds__(256)
post_apply_bwd_kernel(const __grid_constant__ PostBwdParams q, const float* __restrict__ scratch) {
  __shared__ float4 red[2][8][32];
  const PostIdx ix(q.C);
  const int lane = threadIdx.x & 31;
  const int Rw = q.R / q.sh;
  const float* pb = q.p + (long long)ix.b * Rw * q.ldp;
  const long long dpoff = (long long)ix.b * Rw * q.ldp;
  F4 bsum[2] = {zero4(), zero4()};                      // this thread's share of the conv-bias gradients (a, g)
  unsigned nsat = 0, nufl = 0, ngrp = 0;                 // plane groups counted for q.sat / q.ufl, added to the counters after the loop
  if (ix.cvalid) {
    // per channel (Appendix A.7):  xhat = x*r + h ; norm = x*sc + of ; dx = c1*dn - c2 - xhat*c3
    F4 ra = one4(), ha = zero4(), sca = one4(), ofa = zero4(), c1a = one4(), c2a = zero4(), c3a = zero4();
    F4 rg = one4(), hg = zero4(), scg = one4(), ofg = zero4(), c1g = one4(), c2g = zero4(), c3g = zero4();
    if (HAS_IN) {
      const float* st = q.stats + (long long)ix.b * 4 * q.C + ix.c;
      const float* sc = scratch + (long long)ix.b * 4 * q.C + ix.c;
      const float invR = 1.f / (float)q.R;
      {
        F4 mean = ld4(st), rstd = ld4(st + q.C), gam = ld4(q.gamma_a + ix.c), bet = ld4(q.beta_a + ix.c), S1 = ld4(sc), S2 = ld4(sc + q.C);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ra.v[k] = rstd.v[k]; ha.v[k] = -mean.v[k] * rstd.v[k];
          sca.v[k] = rstd.v[k] * gam.v[k]; ofa.v[k] = bet.v[k] - mean.v[k] * sca.v[k];
          c1a.v[k] = sca.v[k]; c2a.v[k] = sca.v[k] * S1.v[k] * invR; c3a.v[k] = sca.v[k] * S2.v[k] * invR;
        }
      }
      if (HAS_GATE) {
        F4 mean = ld4(st + 2 * q.C), rstd = ld4(st + 3 * q.C), gam = ld4(q.gamma_g + ix.c), bet = ld4(q.beta_g + ix.c), S1 = ld4(sc + 2 * q.C), S2 = ld4(sc + 3 * q.C);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          rg.v[k] = rstd.v[k]; hg.v[k] = -mean.v[k] * rstd.v[k];
          scg.v[k] = rstd.v[k] * gam.v[k]; ofg.v[k] = bet.v[k] - mean.v[k] * scg.v[k];
          c1g.v[k] = scg.v[k]; c2g.v[k] = scg.v[k] * S1.v[k] * invR; c3g.v[k] = scg.v[k] * S2.v[k] * invR;
        }
      }
    }
    const int shs = q.sh - 1;
#pragma unroll
    for (int i = 0; i < kPostRows / 8; ++i) {
      const int r = ix.r0 + 8 * i;
      if (r < q.R) {
        const int w = r >> shs, s = r & shs;
        const long long a = (long long)w * q.ldp + s * q.C + ix.c;
        const long long o = ((long long)ix.b * q.R + r) * q.C + ix.c;
        F4 xa = ld4(pb + a), xg = HAS_GATE ? ld4(pb + a + q.Cc) : zero4(), dy = ld4(q.dy1 + o), da, dg = zero4();
        if (q.dy2) { F4 d2 = ld4(q.dy2 + o);
#pragma unroll
          for (int k = 0; k < 4; ++k) dy.v[k] += d2.v[k]; }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float dna = dy.v[k], dng = 0.f;
          if (HAS_GATE) {
            float na = HAS_IN ? fmaf(xa.v[k], sca.v[k], ofa.v[k]) : xa.v[k];
            float ng = HAS_IN ? fmaf(xg.v[k], scg.v[k], ofg.v[k]) : xg.v[k];
            float sg = sigmoidf_(ng);
            dna = dy.v[k] * sg;
            dng = dna * na * (1.f - sg);                          // dy * na * s * (1 - s)
          }
          float a_ = dna, g_ = dng;
          if (HAS_IN) {
            float ah = fmaf(xa.v[k], ra.v[k], ha.v[k]);
            a_ = fmaf(c1a.v[k], dna, -fmaf(ah, c3a.v[k], c2a.v[k]));
            if (HAS_GATE) { float gh = fmaf(xg.v[k], rg.v[k], hg.v[k]); g_ = fmaf(c1g.v[k], dng, -fmaf(gh, c3g.v[k], c2g.v[k])); }
          }
          da.v[k] = a_; dg.v[k] = g_; bsum[0].v[k] += a_; bsum[1].v[k] += g_;
        }
        if (q.dp) { st4(q.dp + dpoff + a, da); if (HAS_GATE) st4(q.dp + dpoff + a + q.Cc, dg); }
        if (q.dp_hi) {
          if (q.qmode) {                                     // F16F8 gradient planes (activation-role scales): q16, then q8hi | q8lo
            const long long nq = (long long)q.B * Rw * q.ldp;
            st4_quant(q.dp_hi, q.dp_lo, dpoff + a, nq, da);
            if (HAS_GATE) st4_quant(q.dp_hi, q.dp_lo, dpoff + a + q.Cc, nq, dg);
            if (q.sat) nsat += sat_groups(da, dg, HAS_GATE);
            if (q.ufl) { nufl += ufl_groups(da, dg, HAS_GATE); ngrp += HAS_GATE ? 2 : 1; }
          } else {
            st4_split(q.dp_hi + dpoff + a, q.dp_lo + dpoff + a, da);
            if (HAS_GATE) st4_split(q.dp_hi + dpoff + a + q.Cc, q.dp_lo + dpoff + a + q.Cc, dg);
          }
        }
      }
    }
  }
  if (q.sat) cgvc_count_hits(q.sat, nsat);
  if (q.ufl) { cgvc_count_hits(q.ufl, nufl); cgvc_count_hits(q.ufl + 1, ngrp); }
  if (q.dbias_a) {
    // positions of lane rl have shuffle phase rl % sh (chunk size and lane stride are even): reduce per phase
    red[0][ix.rl][lane] = make_float4(bsum[0].v[0], bsum[0].v[1], bsum[0].v[2], bsum[0].v[3]);
    red[1][ix.rl][lane] = make_float4(bsum[1].v[0], bsum[1].v[1], bsum[1].v[2], bsum[1].v[3]);
    __syncthreads();
    if (ix.rl < q.sh && ix.cvalid) {
#pragma unroll
      for (int br = 0; br < 2; ++br) {
        float* db = br == 0 ? q.dbias_a : q.dbias_g;
        if (!db || (br == 1 && !HAS_GATE)) continue;
        F4 t = zero4();
        for (int w = ix.rl; w < 8; w += q.sh) { float4 v = red[br][w][lane]; t.v[0] += v.x; t.v[1] += v.y; t.v[2] += v.z; t.v[3] += v.w; }
        if (q.det.p) st4(q.det.p + ((long long)blockIdx.z * gridDim.y + blockIdx.y) * 2 * q.Cc + br * q.Cc + ix.rl * q.C + ix.c, t);
        else atomic_add4(db + ix.rl * q.C + ix.c, t);
      }
    }
  }
}

// The packed form of post_apply_bwd_kernel (instance-normed layers only): sample b = view rows [bwd_first, + bwd_len) of seg, with its
// own statistics and sums.  An overload of its own, so that the equal-length instantiations keep their code
template <bool HAS_GATE>
__global__ void __launch_bounds__(256)
post_apply_bwd_kernel(const __grid_constant__ PostBwdParams q, const float* __restrict__ scratch, const PostBwdSeg sg) {
  constexpr bool HAS_IN = true;
  __shared__ float4 red[2][8][32];
  const PostIdx ix(q.C);
  const int lane = threadIdx.x & 31;
  const int Rw = q.R / q.sh;
  // past the end of a shorter sample: nothing to do, except in deterministic mode, where every (sample, block) row of bias partials
  // is written (zeros here)
  if ((int)blockIdx.y * kPostRows >= bwd_len(q, ix.b, sg) && !q.det.p) return;
  const float* pb = q.p + bwd_conv0(q, ix.b, Rw, sg) * q.ldp;
  const long long dpoff = bwd_conv0(q, ix.b, Rw, sg) * q.ldp;
  F4 bsum[2] = {zero4(), zero4()};                      // this thread's share of the conv-bias gradients (a, g)
  unsigned nsat = 0, nufl = 0, ngrp = 0;                 // plane groups counted for q.sat / q.ufl, added to the counters after the loop
  if (ix.cvalid) {
    // per channel (Appendix A.7):  xhat = x*r + h ; norm = x*sc + of ; dx = c1*dn - c2 - xhat*c3
    F4 ra = one4(), ha = zero4(), sca = one4(), ofa = zero4(), c1a = one4(), c2a = zero4(), c3a = zero4();
    F4 rg = one4(), hg = zero4(), scg = one4(), ofg = zero4(), c1g = one4(), c2g = zero4(), c3g = zero4();
    if (HAS_IN) {
      const float* st = q.stats + (long long)ix.b * 4 * q.C + ix.c;
      const float* sc = scratch + (long long)ix.b * 4 * q.C + ix.c;
      const float invR = 1.f / (float)bwd_len(q, ix.b, sg);
      {
        F4 mean = ld4(st), rstd = ld4(st + q.C), gam = ld4(q.gamma_a + ix.c), bet = ld4(q.beta_a + ix.c), S1 = ld4(sc), S2 = ld4(sc + q.C);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ra.v[k] = rstd.v[k]; ha.v[k] = -mean.v[k] * rstd.v[k];
          sca.v[k] = rstd.v[k] * gam.v[k]; ofa.v[k] = bet.v[k] - mean.v[k] * sca.v[k];
          c1a.v[k] = sca.v[k]; c2a.v[k] = sca.v[k] * S1.v[k] * invR; c3a.v[k] = sca.v[k] * S2.v[k] * invR;
        }
      }
      if (HAS_GATE) {
        F4 mean = ld4(st + 2 * q.C), rstd = ld4(st + 3 * q.C), gam = ld4(q.gamma_g + ix.c), bet = ld4(q.beta_g + ix.c), S1 = ld4(sc + 2 * q.C), S2 = ld4(sc + 3 * q.C);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          rg.v[k] = rstd.v[k]; hg.v[k] = -mean.v[k] * rstd.v[k];
          scg.v[k] = rstd.v[k] * gam.v[k]; ofg.v[k] = bet.v[k] - mean.v[k] * scg.v[k];
          c1g.v[k] = scg.v[k]; c2g.v[k] = scg.v[k] * S1.v[k] * invR; c3g.v[k] = scg.v[k] * S2.v[k] * invR;
        }
      }
    }
    const int shs = q.sh - 1;
#pragma unroll
    for (int i = 0; i < kPostRows / 8; ++i) {
      const int r = ix.r0 + 8 * i;
      if (r < bwd_len(q, ix.b, sg)) {
        const int w = r >> shs, s = r & shs;
        const long long a = (long long)w * q.ldp + s * q.C + ix.c;
        const long long o = (bwd_first(q, ix.b, sg) + r) * q.C + ix.c;
        F4 xa = ld4(pb + a), xg = HAS_GATE ? ld4(pb + a + q.Cc) : zero4(), dy = ld4(q.dy1 + o), da, dg = zero4();
        if (q.dy2) { F4 d2 = ld4(q.dy2 + o);
#pragma unroll
          for (int k = 0; k < 4; ++k) dy.v[k] += d2.v[k]; }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float dna = dy.v[k], dng = 0.f;
          if (HAS_GATE) {
            float na = HAS_IN ? fmaf(xa.v[k], sca.v[k], ofa.v[k]) : xa.v[k];
            float ng = HAS_IN ? fmaf(xg.v[k], scg.v[k], ofg.v[k]) : xg.v[k];
            float sg = sigmoidf_(ng);
            dna = dy.v[k] * sg;
            dng = dna * na * (1.f - sg);                          // dy * na * s * (1 - s)
          }
          float a_ = dna, g_ = dng;
          if (HAS_IN) {
            float ah = fmaf(xa.v[k], ra.v[k], ha.v[k]);
            a_ = fmaf(c1a.v[k], dna, -fmaf(ah, c3a.v[k], c2a.v[k]));
            if (HAS_GATE) { float gh = fmaf(xg.v[k], rg.v[k], hg.v[k]); g_ = fmaf(c1g.v[k], dng, -fmaf(gh, c3g.v[k], c2g.v[k])); }
          }
          da.v[k] = a_; dg.v[k] = g_; bsum[0].v[k] += a_; bsum[1].v[k] += g_;
        }
        if (q.dp) { st4(q.dp + dpoff + a, da); if (HAS_GATE) st4(q.dp + dpoff + a + q.Cc, dg); }
        if (q.dp_hi) {
          if (q.qmode) {                                     // F16F8 gradient planes (activation-role scales): q16, then q8hi | q8lo
            const long long nq = bwd_conv_rows(q, Rw, sg) * q.ldp;
            st4_quant(q.dp_hi, q.dp_lo, dpoff + a, nq, da);
            if (HAS_GATE) st4_quant(q.dp_hi, q.dp_lo, dpoff + a + q.Cc, nq, dg);
            if (q.sat) nsat += sat_groups(da, dg, HAS_GATE);
            if (q.ufl) { nufl += ufl_groups(da, dg, HAS_GATE); ngrp += HAS_GATE ? 2 : 1; }
          } else {
            st4_split(q.dp_hi + dpoff + a, q.dp_lo + dpoff + a, da);
            if (HAS_GATE) st4_split(q.dp_hi + dpoff + a + q.Cc, q.dp_lo + dpoff + a + q.Cc, dg);
          }
        }
      }
    }
  }
  if (q.sat) cgvc_count_hits(q.sat, nsat);
  if (q.ufl) { cgvc_count_hits(q.ufl, nufl); cgvc_count_hits(q.ufl + 1, ngrp); }
  if (q.dbias_a) {
    // positions of lane rl have shuffle phase rl % sh (chunk size and lane stride are even): reduce per phase
    red[0][ix.rl][lane] = make_float4(bsum[0].v[0], bsum[0].v[1], bsum[0].v[2], bsum[0].v[3]);
    red[1][ix.rl][lane] = make_float4(bsum[1].v[0], bsum[1].v[1], bsum[1].v[2], bsum[1].v[3]);
    __syncthreads();
    if (ix.rl < q.sh && ix.cvalid) {
#pragma unroll
      for (int br = 0; br < 2; ++br) {
        float* db = br == 0 ? q.dbias_a : q.dbias_g;
        if (!db || (br == 1 && !HAS_GATE)) continue;
        F4 t = zero4();
        for (int w = ix.rl; w < 8; w += q.sh) { float4 v = red[br][w][lane]; t.v[0] += v.x; t.v[1] += v.y; t.v[2] += v.z; t.v[3] += v.w; }
        if (q.det.p) st4(q.det.p + ((long long)blockIdx.z * gridDim.y + blockIdx.y) * 2 * q.Cc + br * q.Cc + ix.rl * q.C + ix.c, t);
        else atomic_add4(db + ix.rl * q.C + ix.c, t);
      }
    }
  }
}

// One-pass form for samples of at most 8 * NR positions (the generator's 32- and 64-position layers, the discriminator's last
// block): a CTA owns all positions of one sample for 128 channels, keeps its rows of dY and of the saved pre-norm outputs in
// registers, reduces the four per-(sample, channel) sums through shared memory and applies the instance-norm / GLU backward to the
// resident rows -- dY and P are read once (20 instead of 32 bytes per element) and the sums never touch global memory.
template <bool HAS_GATE, int NR>
__global__ void __launch_bounds__(256)
post_bwd_onepass_kernel(const __grid_constant__ PostBwdParams q) {
  __shared__ float4 red[8][32];                       // 6 KB of shared memory in all: the kernel has to fit beside a persistent
  __shared__ float4 bcast[4][32];                     // tensor-core CTA of the other lane, which leaves < 10 KB of the SM's
  const PostIdx ix(q.C);
  const int lane = threadIdx.x & 31;
  const int Rw = q.R / q.sh;
  const float* pb = q.p + (long long)ix.b * Rw * q.ldp;
  const long long dpoff = (long long)ix.b * Rw * q.ldp;
  const int shs = q.sh - 1;
  F4 ra = one4(), ha = zero4(), sca = one4(), ofa = zero4(), rg = one4(), hg = zero4(), scg = one4(), ofg = zero4();
  F4 xa[NR], xg[NR], dy[NR];
  F4 acc[4] = {zero4(), zero4(), zero4(), zero4()};
  if (ix.cvalid) {
    const float* st = q.stats + (long long)ix.b * 4 * q.C + ix.c;
    {
      F4 mean = ld4(st), rstd = ld4(st + q.C), gam = ld4(q.gamma_a + ix.c), bet = ld4(q.beta_a + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) { ra.v[k] = rstd.v[k]; ha.v[k] = -mean.v[k] * rstd.v[k]; sca.v[k] = rstd.v[k] * gam.v[k]; ofa.v[k] = bet.v[k] - mean.v[k] * sca.v[k]; }
    }
    if (HAS_GATE) {
      F4 mean = ld4(st + 2 * q.C), rstd = ld4(st + 3 * q.C), gam = ld4(q.gamma_g + ix.c), bet = ld4(q.beta_g + ix.c);
#pragma unroll
      for (int k = 0; k < 4; ++k) { rg.v[k] = rstd.v[k]; hg.v[k] = -mean.v[k] * rstd.v[k]; scg.v[k] = rstd.v[k] * gam.v[k]; ofg.v[k] = bet.v[k] - mean.v[k] * scg.v[k]; }
    }
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      const int r = ix.rl + 8 * i;
      xa[i] = zero4(); xg[i] = zero4(); dy[i] = zero4();
      if (r < q.R) {
        const int w = r >> shs, sp = r & shs;
        const long long a = (long long)w * q.ldp + sp * q.C + ix.c;
        const long long o = ((long long)ix.b * q.R + r) * q.C + ix.c;
        xa[i] = ld4(pb + a); if (HAS_GATE) xg[i] = ld4(pb + a + q.Cc); dy[i] = ld4(q.dy1 + o);
        if (q.dy2) { F4 d2 = ld4(q.dy2 + o);
#pragma unroll
          for (int k = 0; k < 4; ++k) dy[i].v[k] += d2.v[k]; }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float dna = dy[i].v[k];
          if (HAS_GATE) {
            const float na = fmaf(xa[i].v[k], sca.v[k], ofa.v[k]), ng = fmaf(xg[i].v[k], scg.v[k], ofg.v[k]);
            const float sg = sigmoidf_(ng);
            dna = dy[i].v[k] * sg;
            const float dng = dna * na * (1.f - sg);
            const float gh = fmaf(xg[i].v[k], rg.v[k], hg.v[k]);
            acc[2].v[k] += dng; acc[3].v[k] = fmaf(dng, gh, acc[3].v[k]);
          }
          const float ah = fmaf(xa[i].v[k], ra.v[k], ha.v[k]);
          acc[0].v[k] += dna; acc[1].v[k] = fmaf(dna, ah, acc[1].v[k]);
        }
      }
    }
  }
  sum_over_rows<4>(acc, red, ix.rl, lane);
  if (ix.rl == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) bcast[j][lane] = make_float4(acc[j].v[0], acc[j].v[1], acc[j].v[2], acc[j].v[3]);
    if (ix.cvalid && q.dgamma_a) {
      atomic_add4(q.dbeta_a + ix.c, acc[0]); atomic_add4(q.dgamma_a + ix.c, acc[1]);
      if (HAS_GATE) { atomic_add4(q.dbeta_g + ix.c, acc[2]); atomic_add4(q.dgamma_g + ix.c, acc[3]); }
    }
  }
  __syncthreads();
  F4 bsum[2] = {zero4(), zero4()};
  if (ix.cvalid) {
    const float invR = 1.f / (float)q.R;
    F4 c2a, c3a, c2g = zero4(), c3g = zero4();
    { const float4 S1 = bcast[0][lane], S2 = bcast[1][lane];
      const float s1[4] = {S1.x, S1.y, S1.z, S1.w}, s2[4] = {S2.x, S2.y, S2.z, S2.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) { c2a.v[k] = sca.v[k] * s1[k] * invR; c3a.v[k] = sca.v[k] * s2[k] * invR; } }
    if (HAS_GATE) {
      const float4 S1 = bcast[2][lane], S2 = bcast[3][lane];
      const float s1[4] = {S1.x, S1.y, S1.z, S1.w}, s2[4] = {S2.x, S2.y, S2.z, S2.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) { c2g.v[k] = scg.v[k] * s1[k] * invR; c3g.v[k] = scg.v[k] * s2[k] * invR; }
    }
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      const int r = ix.rl + 8 * i;
      if (r < q.R) {
        const int w = r >> shs, sp = r & shs;
        const long long a = (long long)w * q.ldp + sp * q.C + ix.c;
        F4 da, dg = zero4();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float dna = dy[i].v[k], dng = 0.f;
          if (HAS_GATE) {
            const float na = fmaf(xa[i].v[k], sca.v[k], ofa.v[k]), ng = fmaf(xg[i].v[k], scg.v[k], ofg.v[k]);
            const float sg = sigmoidf_(ng);
            dna = dy[i].v[k] * sg;
            dng = dna * na * (1.f - sg);
          }
          const float ah = fmaf(xa[i].v[k], ra.v[k], ha.v[k]);
          const float a_ = fmaf(sca.v[k], dna, -fmaf(ah, c3a.v[k], c2a.v[k]));
          float g_ = 0.f;
          if (HAS_GATE) { const float gh = fmaf(xg[i].v[k], rg.v[k], hg.v[k]); g_ = fmaf(scg.v[k], dng, -fmaf(gh, c3g.v[k], c2g.v[k])); }
          da.v[k] = a_; dg.v[k] = g_; bsum[0].v[k] += a_; bsum[1].v[k] += g_;
        }
        if (q.dp) { st4(q.dp + dpoff + a, da); if (HAS_GATE) st4(q.dp + dpoff + a + q.Cc, dg); }
        if (q.dp_hi) {
          if (q.qmode) {                                     // F16F8 gradient planes (activation-role scales): q16, then q8hi | q8lo
            const long long nq = (long long)q.B * Rw * q.ldp;
            st4_quant(q.dp_hi, q.dp_lo, dpoff + a, nq, da, q.sat, q.ufl);
            if (HAS_GATE) st4_quant(q.dp_hi, q.dp_lo, dpoff + a + q.Cc, nq, dg, q.sat, q.ufl);
          } else {
            st4_split(q.dp_hi + dpoff + a, q.dp_lo + dpoff + a, da);
            if (HAS_GATE) st4_split(q.dp_hi + dpoff + a + q.Cc, q.dp_lo + dpoff + a + q.Cc, dg);
          }
        }
      }
    }
  }
  if (q.dbias_a) {
    // conv-bias gradients: positions of lane rl have shuffle phase rl % sh; one branch at a time through the 4 KB buffer
#pragma unroll
    for (int br = 0; br < 2; ++br) {
      float* db = br == 0 ? q.dbias_a : q.dbias_g;
      if (!db || (br == 1 && !HAS_GATE)) continue;             // CTA-uniform
      __syncthreads();
      red[ix.rl][lane] = make_float4(bsum[br].v[0], bsum[br].v[1], bsum[br].v[2], bsum[br].v[3]);
      __syncthreads();
      if (ix.rl < q.sh && ix.cvalid) {
        F4 t = zero4();
        for (int w = ix.rl; w < 8; w += q.sh) { float4 v = red[w][lane]; t.v[0] += v.x; t.v[1] += v.y; t.v[2] += v.z; t.v[3] += v.w; }
        atomic_add4(db + ix.rl * q.C + ix.c, t);
      }
    }
  }
}

// Streaming form of the one-pass kernel (round 2): the register-resident kernel above issues its loads, waits, computes, stores -- with
// 128 ... 189 registers per thread one or two CTAs fit on an SM and the memory pipe idles in the compute and store phases (the sums +
// apply pair of the longer samples moves 32 instead of 20 bytes per element).  Here a
// persistent CTA walks (sample, channel block) items through a double buffer in shared memory: every thread copies its own rows of dY
// and of the saved pre-norm outputs (+ the item's statistics / affine parameters) for item i + 1 with 16-byte cp.async while item i is
// reduced and applied out of shared memory, so a CTA always has up to 48 KB (72 KB for 384 positions) of loads in flight and needs few
// registers.  Item = all R positions of one sample x CB = 4 * NQL channels; R = (256 / NQL) * NRT covers every instance-normed layer of
// the model at 128 frames: 32, 48, 64, 96, 128 and 384 positions, with or without the pixel-shuffle view.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int NQL, int NRT>          // channel quads per item (CB = 4 * NQL channels), rows per thread; R = (256 / NQL) * NRT positions
struct StreamCfg {
  static constexpr int CB = NQL * 4, RG = 256 / NQL, R = RG * NRT;
  static constexpr int TILE = R * CB;                       // floats per array (dY, a, g)
  static constexpr int STAGE = 3 * TILE + 8 * CB;           // + mean_a, rstd_a, mean_g, rstd_g, gamma_a, beta_a, gamma_g, beta_g
  static constexpr int RED = 2 * 8 * NQL * 4;               // two float4 quantities x 8 warps x NQL quads
  static constexpr int SMEM = (2 * STAGE + RED) * 4;
  static constexpr int CTAS = SMEM <= 113 * 1024 ? 2 : 1;   // CTAs per SM
};

template <int NQL, int NRT, bool GATE>
__global__ void __launch_bounds__(256, StreamCfg<NQL, NRT>::CTAS)
post_bwd_stream_kernel(const __grid_constant__ PostBwdParams q, int items, int cblocks) {
  using Cfg = StreamCfg<NQL, NRT>;
  constexpr int CB = Cfg::CB, RG = Cfg::RG, R = Cfg::R, TILE = Cfg::TILE;
  static_assert(RG >= 8 && RG % 2 == 0, "coefficient rows are copied by the first 8 row groups; shuffle phases alternate with the row group");
  extern __shared__ __align__(16) float sm[];
  float4* red = reinterpret_cast<float4*>(sm + 2 * Cfg::STAGE);          // [2][8][NQL]
  const int t = threadIdx.x, cq = t % NQL, rg = t / NQL, warp = t >> 5;
  const float invR = 1.f / (float)R;
  const int shs = q.sh - 1, Rw = R >> shs;                                // pixel-shuffle view: position r = conv row r >> shs, column block r & shs
  const long long nplane = (long long)q.B * Rw * q.ldp;                  // elements per gradient plane (F16F8: offset of q8lo)

  auto issue = [&](int item, int s) {
    const int b = item / cblocks, c0 = (item - b * cblocks) * CB + 4 * cq;
    float* S = sm + s * Cfg::STAGE;
    const float* dyb = q.dy1 + (long long)b * R * q.C + c0;
    const float* pb = q.p + (long long)b * Rw * q.ldp + c0;
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int r = rg + RG * i;
      const float* pr = pb + (long long)(r >> shs) * q.ldp + (r & shs) * q.C;
      cp_async16(S + r * CB + 4 * cq, dyb + (long long)r * q.C);
      cp_async16(S + TILE + r * CB + 4 * cq, pr);
      if (GATE) cp_async16(S + 2 * TILE + r * CB + 4 * cq, pr + q.Cc);
    }
    if (rg < 8 && (GATE || (rg & 2) == 0)) {                               // rows 2, 3, 6, 7 belong to the gate branch
      const float* src = rg < 4 ? q.stats + ((long long)b * 4 + rg) * q.C + c0
                                : (rg == 4 ? q.gamma_a : rg == 5 ? q.beta_a : rg == 6 ? q.gamma_g : q.beta_g) + c0;
      cp_async16(S + 3 * TILE + rg * CB + 4 * cq, src);
    }
    cp_async_commit();
  };
  // sum two per-thread float4 quantities over the RG row groups; every thread gets the totals of its channel quad
  auto reduce2 = [&](F4& x0, F4& x1) {
#pragma unroll
    for (int o = NQL; o < 32; o <<= 1) {                                  // row groups that share a warp
#pragma unroll
      for (int k = 0; k < 4; ++k) { x0.v[k] += __shfl_xor_sync(0xffffffffu, x0.v[k], o); x1.v[k] += __shfl_xor_sync(0xffffffffu, x1.v[k], o); }
    }
    __syncthreads();                                                      // previous readers of red are done
    if ((t & 31) < NQL) {
      red[warp * NQL + cq] = make_float4(x0.v[0], x0.v[1], x0.v[2], x0.v[3]);
      red[(8 + warp) * NQL + cq] = make_float4(x1.v[0], x1.v[1], x1.v[2], x1.v[3]);
    }
    __syncthreads();
    F4 a = zero4(), b = zero4();
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float4 u = red[w * NQL + cq], v = red[(8 + w) * NQL + cq];
      a.v[0] += u.x; a.v[1] += u.y; a.v[2] += u.z; a.v[3] += u.w; b.v[0] += v.x; b.v[1] += v.y; b.v[2] += v.z; b.v[3] += v.w;
    }
    x0 = a; x1 = b;
  };

  int it = blockIdx.x, s = 0;
  if (it < items) issue(it, 0);
  for (; it < items; it += gridDim.x, s ^= 1) {
    const int nxt = it + gridDim.x;
    if (nxt < items) { issue(nxt, s ^ 1); cp_async_wait<1>(); } else cp_async_wait<0>();
    __syncthreads();                                                      // the item's coefficient rows were copied by other threads
    const int b = it / cblocks, c = (it - b * cblocks) * CB + 4 * cq;
    const float* S = sm + s * Cfg::STAGE;
    const float* K = S + 3 * TILE + 4 * cq;
    F4 ra, ha, sca, ofa, rgt = one4(), hg = zero4(), scg = one4(), ofg = zero4();
    {
      const F4 mean = ld4(K), rstd = ld4(K + CB), gam = ld4(K + 4 * CB), bet = ld4(K + 5 * CB);
#pragma unroll
      for (int k = 0; k < 4; ++k) { ra.v[k] = rstd.v[k]; ha.v[k] = -mean.v[k] * rstd.v[k]; sca.v[k] = rstd.v[k] * gam.v[k]; ofa.v[k] = bet.v[k] - mean.v[k] * sca.v[k]; }
      if (GATE) {
        const F4 mg = ld4(K + 2 * CB), rsg = ld4(K + 3 * CB), gamg = ld4(K + 6 * CB), betg = ld4(K + 7 * CB);
#pragma unroll
        for (int k = 0; k < 4; ++k) { rgt.v[k] = rsg.v[k]; hg.v[k] = -mg.v[k] * rsg.v[k]; scg.v[k] = rsg.v[k] * gamg.v[k]; ofg.v[k] = betg.v[k] - mg.v[k] * scg.v[k]; }
      }
    }
    F4 acc[4] = {zero4(), zero4(), zero4(), zero4()};
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int o = (rg + RG * i) * CB + 4 * cq;
      const F4 dy = ld4(S + o), xa = ld4(S + TILE + o), xg = GATE ? ld4(S + 2 * TILE + o) : zero4();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float dna = dy.v[k];
        if (GATE) {
          const float na = fmaf(xa.v[k], sca.v[k], ofa.v[k]), ng = fmaf(xg.v[k], scg.v[k], ofg.v[k]);
          const float sg = sigmoidf_(ng);
          dna = dy.v[k] * sg;
          const float dng = dna * na * (1.f - sg);
          const float gh = fmaf(xg.v[k], rgt.v[k], hg.v[k]);
          acc[2].v[k] += dng; acc[3].v[k] = fmaf(dng, gh, acc[3].v[k]);
        }
        const float ah = fmaf(xa.v[k], ra.v[k], ha.v[k]);
        acc[0].v[k] += dna; acc[1].v[k] = fmaf(dna, ah, acc[1].v[k]);
      }
    }
    reduce2(acc[0], acc[1]);
    if (GATE) reduce2(acc[2], acc[3]);
    if (t < NQL && q.dgamma_a) {
      atomic_add4(q.dbeta_a + c, acc[0]); atomic_add4(q.dgamma_a + c, acc[1]);
      if (GATE) { atomic_add4(q.dbeta_g + c, acc[2]); atomic_add4(q.dgamma_g + c, acc[3]); }
    }
    F4 c2a, c3a, c2g = zero4(), c3g = zero4();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c2a.v[k] = sca.v[k] * acc[0].v[k] * invR; c3a.v[k] = sca.v[k] * acc[1].v[k] * invR;
      if (GATE) { c2g.v[k] = scg.v[k] * acc[2].v[k] * invR; c3g.v[k] = scg.v[k] * acc[3].v[k] * invR; }
    }
    F4 bsum[2] = {zero4(), zero4()};
    const long long dpoff = (long long)b * Rw * q.ldp + c;
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int r = rg + RG * i;
      const int o = r * CB + 4 * cq;
      const F4 dy = ld4(S + o), xa = ld4(S + TILE + o), xg = GATE ? ld4(S + 2 * TILE + o) : zero4();
      F4 da, dg = zero4();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float dna = dy.v[k], dng = 0.f;
        if (GATE) {
          const float na = fmaf(xa.v[k], sca.v[k], ofa.v[k]), ng = fmaf(xg.v[k], scg.v[k], ofg.v[k]);
          const float sg = sigmoidf_(ng);
          dna = dy.v[k] * sg;
          dng = dna * na * (1.f - sg);
        }
        const float ah = fmaf(xa.v[k], ra.v[k], ha.v[k]);
        da.v[k] = fmaf(sca.v[k], dna, -fmaf(ah, c3a.v[k], c2a.v[k]));
        if (GATE) { const float gh = fmaf(xg.v[k], rgt.v[k], hg.v[k]); dg.v[k] = fmaf(scg.v[k], dng, -fmaf(gh, c3g.v[k], c2g.v[k])); }
        bsum[0].v[k] += da.v[k]; bsum[1].v[k] += dg.v[k];
      }
      const long long a = dpoff + (long long)(r >> shs) * q.ldp + (r & shs) * q.C;
      if (q.dp) { st4(q.dp + a, da); if (GATE) st4(q.dp + a + q.Cc, dg); }
      if (q.dp_hi) {
        if (q.qmode) { st4_quant(q.dp_hi, q.dp_lo, a, nplane, da, q.sat, q.ufl); if (GATE) st4_quant(q.dp_hi, q.dp_lo, a + q.Cc, nplane, dg, q.sat, q.ufl); }
        else { st4_split(q.dp_hi + a, q.dp_lo + a, da); if (GATE) st4_split(q.dp_hi + a + q.Cc, q.dp_lo + a + q.Cc, dg); }
      }
    }
    if (q.dbias_a) {                                                      // conv-bias gradients (CTA-uniform branch)
      if (shs == 0) {
        reduce2(bsum[0], bsum[1]);
        if (t < NQL) { atomic_add4(q.dbias_a + c, bsum[0]); if (GATE && q.dbias_g) atomic_add4(q.dbias_g + c, bsum[1]); }
      } else {
        // a thread's positions all have shuffle phase rg & 1 (RG is even), and conv channel = phase * C + c: one sum per phase
        const bool odd = (rg & 1) != 0;
#pragma unroll
        for (int br = 0; br < (GATE ? 2 : 1); ++br) {
          F4 e = odd ? zero4() : bsum[br], o = odd ? bsum[br] : zero4();
          reduce2(e, o);
          float* db = br == 0 ? q.dbias_a : q.dbias_g;
          if (t < NQL && db) { atomic_add4(db + c, e); atomic_add4(db + q.C + c, o); }
        }
      }
    }
    __syncthreads();                                                      // stage s is rewritten by the next iteration's copies
  }
}

// The forward counterpart (instance norm + GLU of a gated layer the GEMM epilogue does not fuse: the discriminator's 384-, 96- and
// 48-position blocks, and any generator layer at a frame count whose samples do not tile 128 rows): the item's pre-norm outputs are
// resident in shared memory, so the statistics are an exact two-pass mean / variance and P is read once -- 12 bytes per element
// instead of the 20 of post_stats + post_apply.
template <int NQL, int NRT>
struct StreamFwdCfg {
  static constexpr int CB = NQL * 4, RG = 256 / NQL, R = RG * NRT;
  static constexpr int TILE = R * CB;                       // floats per array (a, g)
  static constexpr int STAGE = 2 * TILE + 4 * CB;           // + gamma_a, beta_a, gamma_g, beta_g
  static constexpr int RED = 2 * 8 * NQL * 4;
  static constexpr int SMEM = (2 * STAGE + RED) * 4;
};

template <int NQL, int NRT>
__global__ void __launch_bounds__(256, 2)
post_fwd_stream_kernel(const __grid_constant__ PostParams q, int items, int cblocks) {
  using Cfg = StreamFwdCfg<NQL, NRT>;
  constexpr int CB = Cfg::CB, RG = Cfg::RG, R = Cfg::R, TILE = Cfg::TILE;
  static_assert(RG >= 4, "coefficient rows are copied by the first 4 row groups");
  extern __shared__ __align__(16) float sm[];
  float4* red = reinterpret_cast<float4*>(sm + 2 * Cfg::STAGE);
  const int t = threadIdx.x, cq = t % NQL, rg = t / NQL, warp = t >> 5;
  const float invR = 1.f / (float)R;
  const int shs = q.sh - 1, Rw = R >> shs;
  const long long nplane = (long long)q.B * R * q.C;

  auto issue = [&](int item, int s) {
    const int b = item / cblocks, c0 = (item - b * cblocks) * CB + 4 * cq;
    float* S = sm + s * Cfg::STAGE;
    const float* pb = q.p + (long long)b * Rw * q.ldp + c0;
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int r = rg + RG * i;
      const float* pr = pb + (long long)(r >> shs) * q.ldp + (r & shs) * q.C;
      cp_async16(S + r * CB + 4 * cq, pr);
      cp_async16(S + TILE + r * CB + 4 * cq, pr + q.Cc);
    }
    if (rg < 4) cp_async16(S + 2 * TILE + rg * CB + 4 * cq, (rg == 0 ? q.gamma_a : rg == 1 ? q.beta_a : rg == 2 ? q.gamma_g : q.beta_g) + c0);
    cp_async_commit();
  };
  auto reduce2 = [&](F4& x0, F4& x1) {
#pragma unroll
    for (int o = NQL; o < 32; o <<= 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) { x0.v[k] += __shfl_xor_sync(0xffffffffu, x0.v[k], o); x1.v[k] += __shfl_xor_sync(0xffffffffu, x1.v[k], o); }
    }
    __syncthreads();
    if ((t & 31) < NQL) {
      red[warp * NQL + cq] = make_float4(x0.v[0], x0.v[1], x0.v[2], x0.v[3]);
      red[(8 + warp) * NQL + cq] = make_float4(x1.v[0], x1.v[1], x1.v[2], x1.v[3]);
    }
    __syncthreads();
    F4 a = zero4(), b = zero4();
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const float4 u = red[w * NQL + cq], v = red[(8 + w) * NQL + cq];
      a.v[0] += u.x; a.v[1] += u.y; a.v[2] += u.z; a.v[3] += u.w; b.v[0] += v.x; b.v[1] += v.y; b.v[2] += v.z; b.v[3] += v.w;
    }
    x0 = a; x1 = b;
  };

  int it = blockIdx.x, s = 0;
  if (it < items) issue(it, 0);
  for (; it < items; it += gridDim.x, s ^= 1) {
    const int nxt = it + gridDim.x;
    if (nxt < items) { issue(nxt, s ^ 1); cp_async_wait<1>(); } else cp_async_wait<0>();
    __syncthreads();
    const int b = it / cblocks, c = (it - b * cblocks) * CB + 4 * cq;
    const float* S = sm + s * Cfg::STAGE;
    F4 ma = zero4(), mg = zero4();
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int o = (rg + RG * i) * CB + 4 * cq;
      const F4 xa = ld4(S + o), xg = ld4(S + TILE + o);
#pragma unroll
      for (int k = 0; k < 4; ++k) { ma.v[k] += xa.v[k]; mg.v[k] += xg.v[k]; }
    }
    reduce2(ma, mg);
#pragma unroll
    for (int k = 0; k < 4; ++k) { ma.v[k] *= invR; mg.v[k] *= invR; }
    F4 va = zero4(), vg = zero4();
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int o = (rg + RG * i) * CB + 4 * cq;
      const F4 xa = ld4(S + o), xg = ld4(S + TILE + o);
#pragma unroll
      for (int k = 0; k < 4; ++k) { const float da = xa.v[k] - ma.v[k], dg = xg.v[k] - mg.v[k]; va.v[k] = fmaf(da, da, va.v[k]); vg.v[k] = fmaf(dg, dg, vg.v[k]); }
    }
    reduce2(va, vg);
    F4 sca, ofa, scg, ofg, rsa, rsg;
    {
      const float* K = S + 2 * TILE + 4 * cq;
      const F4 ga = ld4(K), ba = ld4(K + CB), gg = ld4(K + 2 * CB), bg = ld4(K + 3 * CB);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        rsa.v[k] = 1.f / sqrtf(va.v[k] * invR + IN_EPS); rsg.v[k] = 1.f / sqrtf(vg.v[k] * invR + IN_EPS);
        sca.v[k] = rsa.v[k] * ga.v[k]; ofa.v[k] = ba.v[k] - ma.v[k] * sca.v[k];
        scg.v[k] = rsg.v[k] * gg.v[k]; ofg.v[k] = bg.v[k] - mg.v[k] * scg.v[k];
      }
    }
    if (t < NQL && q.stats) {
      float* st = q.stats + (long long)b * 4 * q.C + c;
      st4(st, ma); st4(st + q.C, rsa); st4(st + 2 * q.C, mg); st4(st + 3 * q.C, rsg);
    }
#pragma unroll
    for (int i = 0; i < NRT; ++i) {
      const int r = rg + RG * i;
      const int o = r * CB + 4 * cq;
      const F4 xa = ld4(S + o), xg = ld4(S + TILE + o);
      F4 y;
#pragma unroll
      for (int k = 0; k < 4; ++k) y.v[k] = fmaf(xa.v[k], sca.v[k], ofa.v[k]) * sigmoidf_(fmaf(xg.v[k], scg.v[k], ofg.v[k]));
      const long long e = ((long long)b * R + r) * q.C + c;
      if (q.y) st4(q.y + e, y);
      if (q.y_hi) {
        if (q.qmode) st4_quant(q.y_hi, q.y_lo, e, nplane, y, q.sat, q.ufl);
        else st4_split(q.y_hi + e, q.y_lo + e, y);
      }
    }
    __syncthreads();
  }
}

#define STREAM_FWD_CONFIGS(X) X(32, 4) X(16, 3) X(16, 4) X(8, 3) X(8, 4) X(4, 6)
template <int NQL, int NRT>
static cudaError_t launch_post_fwd_stream(const PostParams& pp, cudaStream_t st) {
  using Cfg = StreamFwdCfg<NQL, NRT>;
  const int cblocks = pp.C / Cfg::CB;
  const long long items = (long long)pp.B * cblocks;
  const int grid = (int)(items < 2 * CGVC_NUM_SMS ? items : 2 * CGVC_NUM_SMS);
  ++g_cgvc_launches;
  post_fwd_stream_kernel<NQL, NRT><<<grid, 256, Cfg::SMEM, st>>>(pp, (int)items, cblocks);
  return cudaGetLastError();
}

#define STREAM_CONFIGS(X) X(32, 4, true) X(32, 4, false) X(16, 3, true) X(16, 4, true) X(8, 3, true) X(8, 4, true) X(4, 6, true)
cudaError_t post_init_kernels() {
  cudaError_t e;
#define X(NQL_, NRT_, G_) if ((e = cudaFuncSetAttribute(post_bwd_stream_kernel<NQL_, NRT_, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize, StreamCfg<NQL_, NRT_>::SMEM)) != cudaSuccess) return e;
  STREAM_CONFIGS(X)
#undef X
#define X(NQL_, NRT_) if ((e = cudaFuncSetAttribute(post_fwd_stream_kernel<NQL_, NRT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, StreamFwdCfg<NQL_, NRT_>::SMEM)) != cudaSuccess) return e;
  STREAM_FWD_CONFIGS(X)
#undef X
  return cudaSuccess;
}
template <int NQL, int NRT, bool GATE>
static cudaError_t launch_post_bwd_stream(const PostBwdParams& pp, cudaStream_t st) {
  using Cfg = StreamCfg<NQL, NRT>;
  const int cblocks = pp.C / Cfg::CB;
  const long long items = (long long)pp.B * cblocks;
  const int grid = (int)(items < Cfg::CTAS * CGVC_NUM_SMS ? items : Cfg::CTAS * CGVC_NUM_SMS);
  ++g_cgvc_launches;
  post_bwd_stream_kernel<NQL, NRT, GATE><<<grid, 256, Cfg::SMEM, st>>>(pp, (int)items, cblocks);
  return cudaGetLastError();
}
static bool post_fwd_stream_dispatch(const PostParams& pp, bool stream, cudaStream_t st, cudaError_t* err) {
  if (!(pp.has_in && pp.has_gate && !pp.resid && stream && (pp.sh == 1 || pp.sh == 2) && pp.Cc == pp.C * pp.sh &&
        (long long)pp.B * (pp.C / 16) < (1ll << 30)))
    return false;
  const int R = pp.R, C = pp.C;
  if (R == 32 && C % 128 == 0) { *err = launch_post_fwd_stream<32, 4>(pp, st); return true; }
  if (R == 48 && C % 64 == 0) { *err = launch_post_fwd_stream<16, 3>(pp, st); return true; }
  if (R == 64 && C % 64 == 0) { *err = launch_post_fwd_stream<16, 4>(pp, st); return true; }
  if (R == 96 && C % 32 == 0) { *err = launch_post_fwd_stream<8, 3>(pp, st); return true; }
  if (R == 128 && C % 32 == 0) { *err = launch_post_fwd_stream<8, 4>(pp, st); return true; }
  if (R == 384 && C % 16 == 0) { *err = launch_post_fwd_stream<4, 6>(pp, st); return true; }
  return false;
}
// the streaming kernel's configuration for a layer shape, if it has one
static bool post_bwd_stream_dispatch(const PostBwdParams& pp, PostForms forms, cudaStream_t st, cudaError_t* err) {
  if (!(pp.has_in && forms.onepass && forms.stream && !pp.dy2 && pp.stats && (pp.sh == 1 || pp.sh == 2) && pp.Cc == pp.C * pp.sh &&
        (long long)pp.B * (pp.C / 16) < (1ll << 30)))
    return false;
  const int R = pp.R, C = pp.C;
  if (!pp.has_gate) {
    if (R == 32 && C % 128 == 0 && pp.sh == 1) { *err = launch_post_bwd_stream<32, 4, false>(pp, st); return true; }
    return false;
  }
  if (R == 32 && C % 128 == 0) { *err = launch_post_bwd_stream<32, 4, true>(pp, st); return true; }
  if (R == 48 && C % 64 == 0) { *err = launch_post_bwd_stream<16, 3, true>(pp, st); return true; }
  if (R == 64 && C % 64 == 0) { *err = launch_post_bwd_stream<16, 4, true>(pp, st); return true; }
  if (R == 96 && C % 32 == 0) { *err = launch_post_bwd_stream<8, 3, true>(pp, st); return true; }
  if (R == 128 && C % 32 == 0) { *err = launch_post_bwd_stream<8, 4, true>(pp, st); return true; }
  if (R == 384 && C % 16 == 0) { *err = launch_post_bwd_stream<4, 6, true>(pp, st); return true; }
  return false;
}


cudaError_t launch_post_bwd(const PostBwdParams& pp, PostForms forms, cudaStream_t st, const PostBwdSeg* seg) {
  if (pp.B == 0) return cudaSuccess;
  if (!post_aligned(pp.p, pp.dy1, pp.dy2, pp.ldp, pp.C, pp.Cc) || (pp.sh != 1 && pp.sh != 2) || pp.B > 65535 || (pp.has_in && !pp.scratch))
    return cudaErrorInvalidValue;
  dim3 grid((pp.C + kPostChan - 1) / kPostChan, (pp.R + kPostRows - 1) / kPostRows, pp.B);
  // deterministic mode takes the sums + apply form: its per-sample sums are the parameter-gradient contributions, and its bias partials
  // go to one slab row per (sample, position block)
  const bool det = pp.det.p != nullptr;
  const bool det_bias = det && pp.dbias_a;
  if (det_bias && (long long)pp.B * grid.y * 2 * pp.Cc > pp.det.cap) return cudaErrorInvalidValue;
  // packed variable-length samples (seg): the sums + apply form only, one CTA column per sample, grid.y sized by the longest; samples
  // start on whole conv rows (off[u] / div % sh == 0)
  const bool pk = seg && seg->seg.off;
  if (pk && (!pp.has_in || seg->seg.div < 1 || 4 % (seg->seg.div * pp.sh) || seg->seg.n != pp.B)) return cudaErrorInvalidValue;
  if (!det && !pk) { cudaError_t se = cudaSuccess; if (post_bwd_stream_dispatch(pp, forms, st, &se)) return se; }
  if (!det && !pk && pp.has_in && pp.R <= 64 && forms.onepass) {
    ++g_cgvc_launches;
    const dim3 g1(grid.x, 1, grid.z);
#define ONEPASS(NR_) do { if (pp.has_gate) post_bwd_onepass_kernel<true, NR_><<<g1, 256, 0, st>>>(pp); else post_bwd_onepass_kernel<false, NR_><<<g1, 256, 0, st>>>(pp); } while (0)
    if (pp.R <= 32) ONEPASS(4); else if (pp.R <= 48) ONEPASS(6); else ONEPASS(8);
#undef ONEPASS
    return cudaGetLastError();
  }
  float* scratch = pp.scratch;
  if (pp.has_in) {
    ++g_cgvc_launches;
    if (pk) { if (pp.has_gate) post_bwd_sums_kernel<true, PostBwdSeg><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch, *seg);
              else post_bwd_sums_kernel<false, PostBwdSeg><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch, *seg); }
    else if (pp.has_gate) post_bwd_sums_kernel<true><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
    else post_bwd_sums_kernel<false><<<dim3(grid.x, 1, grid.z), 256, 0, st>>>(pp, scratch);
    if (det && pp.dgamma_a) {                            // scratch[b] = [S1a | S2a | S1g | S2g] = sample b's dbeta_a, dgamma_a, dbeta_g, dgamma_g
      const long long C = pp.C, g = pp.has_gate ? C : 0;
      cudaError_t e = launch_reduce_parts(scratch, pp.B, 4 * C, DetSegs{{pp.dbeta_a, pp.dgamma_a, pp.dbeta_g, pp.dgamma_g}, {0, C, 2 * C, 3 * C}, {C, C, g, g}}, st);
      if (e != cudaSuccess) return e;
    }
  }
  ++g_cgvc_launches;
  if (pk) { if (pp.has_gate) post_apply_bwd_kernel<true><<<grid, 256, 0, st>>>(pp, scratch, *seg);
            else post_apply_bwd_kernel<false><<<grid, 256, 0, st>>>(pp, scratch, *seg); }
  else if (pp.has_in) { if (pp.has_gate) post_apply_bwd_kernel<true, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_bwd_kernel<true, false><<<grid, 256, 0, st>>>(pp, scratch); }
  else           { if (pp.has_gate) post_apply_bwd_kernel<false, true><<<grid, 256, 0, st>>>(pp, scratch); else post_apply_bwd_kernel<false, false><<<grid, 256, 0, st>>>(pp, scratch); }
  if (!det_bias) return cudaGetLastError();
  const long long Cc = pp.Cc;
  return launch_reduce_parts(pp.det.p, (long long)pp.B * grid.y, 2 * Cc, DetSegs{{pp.dbias_a, pp.has_gate ? pp.dbias_g : nullptr}, {0, Cc}, {Cc, pp.has_gate ? Cc : 0}}, st);
}

// ------------------------------------------------------------------------------------------------
// discriminator head (module.py:211) + LSGAN loss (model.py:68-69, 81-86)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
head_fwd_kernel(const float* __restrict__ y, long long rows, int C, const float* __restrict__ w, const float* __restrict__ b,
                float* __restrict__ prob) {
  const int lane = threadIdx.x & 31;
  long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* yr = y + row * C;
  float s = 0.f;
  for (int c = lane * 4; c < C; c += 128) {
    float4 a = *reinterpret_cast<const float4*>(yr + c);
    float4 ww = *reinterpret_cast<const float4*>(w + c);
    s += a.x * ww.x + a.y * ww.y + a.z * ww.z + a.w * ww.w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) prob[row] = sigmoidf_(s + b[0]);
}

cudaError_t launch_head_fwd(const float* y, long long rows, int C, const float* w, const float* b, float* prob, cudaStream_t st) {
  if (rows == 0) return cudaSuccess;
  if (C % 128 != 0) return cudaErrorInvalidValue;
  ++g_cgvc_launches; head_fwd_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(y, rows, C, w, b, prob);
  return cudaGetLastError();
}

// C must be 1024 (8 float4 per lane)
__global__ void __launch_bounds__(256)
head_loss_bwd_kernel(const float* __restrict__ prob, const float* __restrict__ y, long long rows, int C,
                     const float* __restrict__ w, float target, float coef, float* __restrict__ loss_slot,
                     float* __restrict__ dy, float* __restrict__ dw, float* __restrict__ db, const float* __restrict__ grad_mult_dev,
                     float* __restrict__ part, const float* __restrict__ dprob) {
  __shared__ float red[8][32];
  float* prow = part ? part + (long long)blockIdx.x * (C + 2) : nullptr;     // det: [dw (C) | db | loss] of this CTA
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float grad_mult = grad_mult_dev ? *grad_mult_dev : 1.f;
  float4 accw[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) accw[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  float lsum = 0.f, dbsum = 0.f;
  const float inv = 1.f / (float)rows;
  for (long long row = (long long)blockIdx.x * 8 + warp; row < rows; row += (long long)gridDim.x * 8) {
    float p = prob[row];
    float dz;
    if (dprob) {                                                        // upstream d prob instead of the LSGAN loss (no loss term)
      dz = grad_mult * dprob[row] * p * (1.f - p);
    } else {
      float d = p - target;
      lsum += d * d;
      dz = grad_mult * coef * 2.f * d * inv * p * (1.f - p);           // grad_mult: loss scale of the reduced-precision gradient planes (1 otherwise)
    }
    dbsum += dz;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int c = lane * 4 + i * 128;
      if (dy) {
        float4 ww = *reinterpret_cast<const float4*>(w + c);
        *reinterpret_cast<float4*>(dy + row * C + c) = make_float4(dz * ww.x, dz * ww.y, dz * ww.z, dz * ww.w);
      }
      if (dw) {
        float4 a = *reinterpret_cast<const float4*>(y + row * C + c);
        accw[i].x += dz * a.x; accw[i].y += dz * a.y; accw[i].z += dz * a.z; accw[i].w += dz * a.w;
      }
    }
  }
  // loss + db: lane 0 of each warp holds the per-warp value (every lane computed the same rows)
  float l = block_sum8(lane == 0 ? lsum : 0.f, red, warp, lane);
  float dbs = block_sum8(lane == 0 ? dbsum : 0.f, red, warp, lane);
  if (threadIdx.x == 0) {
    if (prow) { prow[C] = dbs; prow[C + 1] = coef * l * inv; }
    else {
      if (loss_slot) atomicAdd(loss_slot, coef * l * inv);
      if (db) atomicAdd(db, dbs);
    }
  }
  if (dw) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float vx = block_sum8(accw[i].x, red, warp, lane);
      float vy = block_sum8(accw[i].y, red, warp, lane);
      float vz = block_sum8(accw[i].z, red, warp, lane);
      float vw = block_sum8(accw[i].w, red, warp, lane);
      if (warp == 0) {
        int c = lane * 4 + i * 128;
        if (prow) { prow[c] = vx; prow[c + 1] = vy; prow[c + 2] = vz; prow[c + 3] = vw; }
        else { atomicAdd(dw + c, vx); atomicAdd(dw + c + 1, vy); atomicAdd(dw + c + 2, vz); atomicAdd(dw + c + 3, vw); }
      }
    }
  }
}

cudaError_t launch_head_loss_bwd(const float* prob, const float* y, long long rows, int C, const float* w,
                                 float target, float coef, float* loss_slot,
                                 float* dy, float* dw, float* db, cudaStream_t st, const float* grad_mult_dev, const DetSlab* det,
                                 const float* dprob) {
  if (rows == 0) return cudaSuccess;
  if (C != 1024 || (dprob && loss_slot)) return cudaErrorInvalidValue;
  long long nb = (rows + 7) / 8;
  if (nb > 296) nb = 296;
  float* part = det ? det->p : nullptr;
  if (part && nb * (C + 2) > det->cap) return cudaErrorInvalidValue;
  ++g_cgvc_launches; head_loss_bwd_kernel<<<(unsigned)nb, 256, 0, st>>>(prob, y, rows, C, w, target, coef, loss_slot, dy, dw, db, grad_mult_dev, part,
                                                                      dprob);
  if (!part) return cudaGetLastError();
  return launch_reduce_parts(part, nb, C + 2, DetSegs{{dw, db, loss_slot}, {0, C, C + 1}, {dw ? C : 0, db ? 1 : 0, loss_slot ? 1 : 0}}, st);
}

// ------------------------------------------------------------------------------------------------
// L1 loss + gradient (utils.py:6-8)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
l1_loss_grad_kernel(const float* __restrict__ yhat, const float* __restrict__ y, long long n, float* __restrict__ loss_slot,
                    const float* __restrict__ gscale_dev, float* __restrict__ d, int accumulate, const float* __restrict__ grad_mult_dev,
                    float* __restrict__ part) {
  __shared__ float red[8][32];
  const float inv = 1.f / (float)n;
  const float gs = (gscale_dev ? gscale_dev[0] * inv : inv) * (grad_mult_dev ? *grad_mult_dev : 1.f);
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float e = yhat[i] - y[i];
    s += fabsf(e);
    if (d) {
      float gsign = (e > 0.f) ? gs : ((e < 0.f) ? -gs : 0.f);
      d[i] = accumulate ? d[i] + gsign : gsign;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  float t = block_sum8(lane == 0 ? s : 0.f, red, warp, lane);
  if (threadIdx.x == 0 && part) part[blockIdx.x] = t * inv;
  else if (threadIdx.x == 0 && loss_slot) atomicAdd(loss_slot, t * inv);
}

cudaError_t launch_l1_loss_grad(const float* yhat, const float* y, long long n, float* loss_slot,
                                const float* gscale_dev, float* d, int accumulate, cudaStream_t st, const float* grad_mult_dev, const DetSlab* det) {
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > 592) nb = 592;
  float* part = det && loss_slot ? det->p : nullptr;
  if (part && nb > det->cap) return cudaErrorInvalidValue;
  ++g_cgvc_launches; l1_loss_grad_kernel<<<(unsigned)nb, 256, 0, st>>>(yhat, y, n, loss_slot, gscale_dev, d, accumulate, grad_mult_dev, part);
  if (!part) return cudaGetLastError();
  return launch_reduce_parts(part, nb, 1, DetSegs{{loss_slot}, {0}, {1}}, st);
}

// [B,F,T] -> [B,T,F] (F = 24 features; T frames).  Call with (F,T) swapped for the inverse.
__global__ void __launch_bounds__(256)
transpose_ft_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int F, int T) {
  long long n = (long long)B * F * T;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    int f = (int)(i % F); long long r = i / F; int t = (int)(r % T); int b = (int)(r / T);
    out[i] = in[((long long)b * F + f) * T + t];
  }
}

cudaError_t launch_transpose_ft(const float* in, float* out, int B, int F, int T, cudaStream_t st) {
  long long n = (long long)B * F * T;
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > 2368) nb = 2368;
  ++g_cgvc_launches; transpose_ft_kernel<<<(unsigned)nb, 256, 0, st>>>(in, out, B, F, T);
  return cudaGetLastError();
}

// packed utterances: element (frame m, feature f) is row-major m * F + f, and f * len_u + (m - off[u]) of utterance u's [F][len_u]
// block at F * off[u].  TO_ROWS: blocks -> rows (reads gather, writes coalesce), else rows -> blocks.
template <bool TO_ROWS>
__global__ void __launch_bounds__(256)
transpose_packed_kernel(const float* __restrict__ in, float* __restrict__ out, const long long* __restrict__ off, int n, long long rows, int F) {
  const long long total = rows * F;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long m = i / F; const int f = (int)(i - m * F);
    const int u = pack_find(off, n, m);
    const long long o0 = __ldg(off + u), len = __ldg(off + u + 1) - o0;
    const long long b = F * o0 + f * len + (m - o0);
    if (TO_ROWS) out[i] = in[b]; else out[b] = in[i];
  }
}

cudaError_t launch_transpose_packed(const float* in, float* out, const long long* off, int n, long long rows, int F, int to_rows, cudaStream_t st) {
  const long long total = rows * F;
  if (total == 0) return cudaSuccess;
  if (!off || n < 1) return cudaErrorInvalidValue;
  long long nb = (total + 255) / 256; if (nb > 2368) nb = 2368;
  ++g_cgvc_launches;
  if (to_rows) transpose_packed_kernel<true><<<(unsigned)nb, 256, 0, st>>>(in, out, off, n, rows, F);
  else transpose_packed_kernel<false><<<(unsigned)nb, 256, 0, st>>>(in, out, off, n, rows, F);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) y[i] = a[i] + b[i];
}

cudaError_t launch_add(const float* a, const float* b, float* y, long long n, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > 2368) nb = 2368;
  ++g_cgvc_launches; add_kernel<<<(unsigned)nb, 256, 0, st>>>(a, b, y, n);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// TF Adam (SURVEY.md Appendix A.6): theta -= lr_t * m / (sqrt(v) + eps), eps outside the bias correction
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
            const float* __restrict__ hyper, float beta1, float beta2, float eps, const int* __restrict__ skip) {
  if (skip && *skip) return;                         // a step the loss scaler skipped: p, m and v keep their values
  const float lr_t = hyper[0], gscale = hyper[1];
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float pa[4] = {pv.x, pv.y, pv.z, pv.w}, ga[4] = {gv.x, gv.y, gv.z, gv.w};
    float ma[4] = {mv.x, mv.y, mv.z, mv.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float gk = ga[k] * gscale;
      ma[k] = beta1 * ma[k] + (1.f - beta1) * gk;
      va[k] = beta2 * va[k] + (1.f - beta2) * gk * gk;
      pa[k] = pa[k] - lr_t * ma[k] / (sqrtf(va[k]) + eps);
    }
    reinterpret_cast<float4*>(p)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(ma[0], ma[1], ma[2], ma[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(va[0], va[1], va[2], va[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    long long i = (n4 << 2) + threadIdx.x;
    float gk = g[i] * gscale;
    float mk = beta1 * m[i] + (1.f - beta1) * gk;
    float vk = beta2 * v[i] + (1.f - beta2) * gk * gk;
    m[i] = mk; v[i] = vk;
    p[i] = p[i] - lr_t * mk / (sqrtf(vk) + eps);
  }
}

cudaError_t launch_adam(float* p, const float* g, float* m, float* v, long long n,
                        const float* hyper_dev, float beta1, float beta2, float eps, cudaStream_t st, const int* skip_dev) {
  if (n == 0) return cudaSuccess;
  if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
       reinterpret_cast<uintptr_t>(v)) & 15) return cudaErrorMisalignedAddress;
  long long nb = ((n >> 2) + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16; if (nb < 1) nb = 1;
  ++g_cgvc_launches; adam_kernel<<<(unsigned)nb, 256, 0, st>>>(p, g, m, v, n, hyper_dev, beta1, beta2, eps, skip_dev);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Dynamic loss scaling (DESIGN.md section 10): the GRAD check and the once-per-step scaler update
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
check_finite_kernel(const float* __restrict__ g, long long n, long long cut, unsigned* __restrict__ nonfinite) {
  unsigned bits = 0;
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    const float a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) if (!isfinite(a[k])) bits |= (4 * i + k) < cut ? 1u : 2u;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    if (!isfinite(g[i])) bits |= i < cut ? 1u : 2u;
  }
  bits = __reduce_or_sync(0xffffffffu, bits);
  if ((threadIdx.x & 31) == 0 && bits) atomicOr(nonfinite, bits);
}

cudaError_t launch_check_finite(const float* g, long long n, long long cut, unsigned* nonfinite, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  if (reinterpret_cast<uintptr_t>(g) & 15) return cudaErrorMisalignedAddress;
  long long nb = ((n >> 2) + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16; if (nb < 1) nb = 1;
  ++g_cgvc_launches; check_finite_kernel<<<(unsigned)nb, 256, 0, st>>>(g, n, cut, nonfinite);
  return cudaGetLastError();
}

// One thread.  Overflow (a saturated gradient plane or a non-finite gradient): skip the step, halve the scale (floor 1), reset the
// good-step count.  Otherwise advance Adam's t and, after growth_interval good steps in a row, double the scale (cap 2^24).  adapt = 0
// (the precisions without reduced-range gradient planes): the scale stays where it is and only the skip applies.  lr_t uses the same
// double-precision formula as the host's set_adam_scalars (engine.cu); CUDA's pow is within 2 ulp, not correctly rounded, so the fp32
// result can differ from the host's in the last bit when the double lies at an fp32 rounding boundary.
// nets = 1: one scale per network (option "loss_scale_per_network"; net 0 the generators, 1 the discriminators).  Network k overflowed
// when its planes saturated or its GRAD range (nonfinite bit k) holds a non-finite value: its scale halves (floor 1) and its good-step
// count resets; otherwise that count advances and after growth_interval such steps its scale doubles (cap 2^24).  The step is skipped,
// both optimizers alike, when either network overflowed, and each optimizer's grad_scale divides by its own network's scale.  The head
// of the state keeps its meaning: scale = s_G, sat_grad = both networks' saturated groups, good_steps = consecutive steps not skipped.
// nets = 2 (per network, monitor mode): the sum into sat_grad only.
__device__ void loss_scale_update_nets(LossScaler* s, float* hyper, int nets, int growth_interval, float beta1, float beta2) {
  s->sat_grad = s->cnt[0][0] + s->cnt[1][0];
  if (nets == 2) return;
  const float used[2] = {s->net[0].scale, s->net[1].scale};
  bool skip = false;
  for (int k = 0; k < 2; ++k) {
    LossScaler::Net& n = s->net[k];
    if (s->cnt[k][0] > 0 || ((s->nonfinite >> k) & 1u)) {
      skip = true; n.good_steps = 0; n.scale = fmaxf(1.f, used[k] * 0.5f);
    } else if (++n.good_steps >= growth_interval) {
      n.good_steps = 0; n.scale = fminf(16777216.f, used[k] * 2.f);
    }
  }
  s->scale = s->net[0].scale;
  s->scale_used = used[0];
  if (skip) {
    s->last_skipped = 1; s->good_steps = 0; s->skipped += 1;
    return;
  }
  s->last_skipped = 0;
  s->t += 1;
  s->good_steps += 1;
  const double t = (double)s->t;
  const double corr = sqrt(1.0 - pow((double)beta2, t)) / (1.0 - pow((double)beta1, t));
  hyper[0] = (float)(hyper[0] * corr); hyper[1] = hyper[1] / used[0];   // generator optimizer: lr -> lr_t, 1/nranks -> 1/(nranks s_G)
  hyper[2] = (float)(hyper[2] * corr); hyper[3] = hyper[3] / used[1];   // discriminator optimizer: 1/(nranks s_D)
}

__global__ void loss_scale_update_kernel(LossScaler* s, float* hyper, int adapt, int growth_interval, float beta1, float beta2, int nets) {
  if (nets) { loss_scale_update_nets(s, hyper, nets, growth_interval, beta1, beta2); return; }
  const float used = s->scale;
  s->scale_used = used;
  if (s->sat_grad > 0 || s->nonfinite) {
    s->last_skipped = 1; s->good_steps = 0; s->skipped += 1;
    if (adapt) s->scale = fmaxf(1.f, used * 0.5f);
    return;
  }
  s->last_skipped = 0;
  s->t += 1;
  if (++s->good_steps >= growth_interval) {
    s->good_steps = 0;
    if (adapt) s->scale = fminf(16777216.f, used * 2.f);
  }
  const double t = (double)s->t;
  const double corr = sqrt(1.0 - pow((double)beta2, t)) / (1.0 - pow((double)beta1, t));
  hyper[0] = (float)(hyper[0] * corr); hyper[1] = hyper[1] / used;      // generator optimizer: lr -> lr_t, 1/nranks -> grad_scale
  hyper[2] = (float)(hyper[2] * corr); hyper[3] = hyper[3] / used;      // discriminator optimizer
}

cudaError_t launch_loss_scale_update(LossScaler* s, float* hyper, int adapt, int growth_interval, float beta1, float beta2, cudaStream_t st,
                                     int nets) {
  ++g_cgvc_launches; loss_scale_update_kernel<<<1, 1, 0, st>>>(s, hyper, adapt, growth_interval, beta1, beta2, nets);
  return cudaGetLastError();
}

// losses8: [0] cycle [1] identity [2] G_A2B [3] G_B2A [4] generator [5] D_A [6] D_B [7] discriminator (model.py:57-90)
__global__ void finalize_losses_kernel(float* l, const float* lambdas) {
  if (threadIdx.x == 0) {
    l[4] = l[2] + l[3] + lambdas[0] * l[0] + lambdas[1] * l[1];
    l[7] = l[5] + l[6];
  }
}

cudaError_t launch_finalize_losses(float* losses8, const float* lambdas_dev, cudaStream_t st) {
  ++g_cgvc_launches; finalize_losses_kernel<<<1, 32, 0, st>>>(losses8, lambdas_dev);
  return cudaGetLastError();
}

__global__ void __launch_bounds__(256)
split_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    __nv_bfloat16 h, l; split_bf16(x[i], h, l); hi[i] = h; lo[i] = l;
  }
}

cudaError_t launch_split_bf16(const float* x, __nv_bfloat16* hi, __nv_bfloat16* lo, long long n, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > 2368) nb = 2368;
  ++g_cgvc_launches; split_bf16_kernel<<<(unsigned)nb, 256, 0, st>>>(x, hi, lo, n);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// Discriminator input layer (module.py:201-203: 3x3, stride (1,2), ONE input channel, K = 9): HBM-bound specials.
// ------------------------------------------------------------------------------------------------
// Shared helper of the single-input-channel kernels: gather the taps of `rows` consecutive positions starting at m0 into
// xs[row][tap] (zero outside the image / beyond m1).  All 256 threads participate.
constexpr int kC1Rows = 64;
constexpr int kC1Pad = 20;     // >= CGVC_MAX_TAPS, keeps rows 16-byte aligned
// PKs: an optional trailing PackGeom2 (packed 2-D grids: every tap reads only its own utterance)
template <class... PKs>
__device__ __forceinline__ void c1_stage_taps(const GatherGeom& g, const float* __restrict__ src, long long m0, long long m1, float (*xs)[kC1Pad],
                                              const PKs&... pks) {
  const int HW = g.Hy * g.Wx;
  for (int i = threadIdx.x; i < kC1Rows * g.ntaps; i += 256) {
    int rr = i / g.ntaps, t = i - rr * g.ntaps;
    long long m = m0 + rr;
    float v = 0.f;
    if constexpr (sizeof...(PKs) > 0) {
      if (m < m1) {
        const PackGeom& pk = pack_arg(pks...);
        const Pack2Pos o = pack2_pos(pk, g.Hy, pk.div * g.sx, m);
        const long long r = pack2_row(o.o0, o.o1, g.Hs, pk.div, o.y * g.sy + g.oy[t], o.x * g.sx + g.ox[t]);
        if (r >= 0) v = src[r];
      }
    } else if (m < m1) {
      int b = (int)(m / HW); int rem = (int)(m - (long long)b * HW);
      int y = rem / g.Wx; int x = rem - y * g.Wx;
      int yy = y * g.sy + g.oy[t], xx = x * g.sx + g.ox[t];
      if (yy >= 0 && yy < g.Hs && xx >= 0 && xx < g.Ws) v = src[(long long)(b * g.Hs + yy) * g.Ws + xx];
    }
    xs[rr][t] = v;
  }
}

// weight gradient: dW[t][0][n] += sum_m x[src(m,t)] * G[m, n]   for n in [0, N), N <= 1024 (both branches at once).
// thread = (column quad, position lane): G is streamed exactly once with 16-byte loads; the gathered inputs of 64 positions
// are staged in shared memory per tile.
template <int NT, class... PKs>
__global__ void __launch_bounds__(256)
wgrad_c1_kernel(const __grid_constant__ GatherGeom g, const float* __restrict__ src, const float* __restrict__ grad, int g_ld, int N,
                float* __restrict__ dw_a, float* __restrict__ dw_g, int n_split, float* __restrict__ db_a, float* __restrict__ db_g,
                int rows_per_block, float* __restrict__ part, const PKs... pks) {
  __shared__ __align__(16) float xs[kC1Rows][kC1Pad];
  __shared__ float4 red[256];
  const int nq = N / 4;                                 // host guarantees nq divides 256
  const int cq = threadIdx.x % nq, rl = threadIdx.x / nq, rstep = 256 / nq;
  const int n = cq * 4;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  long long r0 = (long long)blockIdx.x * rows_per_block;
  long long r1 = r0 + rows_per_block < M ? r0 + rows_per_block : M;
  float4 acc[NT + 1];
#pragma unroll
  for (int t = 0; t <= NT; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long mb = r0; mb < r1; mb += kC1Rows) {
    __syncthreads();
    c1_stage_taps(g, src, mb, r1, xs, pks...);
    __syncthreads();
    const int cnt = (int)((r1 - mb) < kC1Rows ? (r1 - mb) : kC1Rows);
    for (int rr = rl; rr < cnt; rr += rstep) {
      float4 gv = *reinterpret_cast<const float4*>(grad + (mb + rr) * g_ld + n);
      acc[NT].x += gv.x; acc[NT].y += gv.y; acc[NT].z += gv.z; acc[NT].w += gv.w;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        if (t < g.ntaps) {
          float v = xs[rr][t];
          acc[t].x = fmaf(v, gv.x, acc[t].x); acc[t].y = fmaf(v, gv.y, acc[t].y); acc[t].z = fmaf(v, gv.z, acc[t].z); acc[t].w = fmaf(v, gv.w, acc[t].w);
        }
      }
    }
  }
  // reduce the position lanes through shared memory (one tap at a time), then one vector atomic per (tap, column quad)
  float* dw = n < n_split ? dw_a : dw_g; float* db = n < n_split ? db_a : db_g;
  const int nn = n < n_split ? n : n - n_split; const int ncols = n < n_split ? n_split : N - n_split;
#pragma unroll
  for (int t = 0; t <= NT; ++t) {
    if (!(t < g.ntaps || t == NT)) continue;             // block-uniform
    __syncthreads();
    red[threadIdx.x] = acc[t];
    __syncthreads();
    if (rl == 0) {
      float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int l = 0; l < rstep; ++l) { float4 v = red[l * nq + cq]; sacc.x += v.x; sacc.y += v.y; sacc.z += v.z; sacc.w += v.w; }
      float* dst = t < NT ? dw + (long long)g.widx[t] * ncols + nn : (db ? db + nn : nullptr);
      if (part) {                                          // det: row [dw_a | dw_g | db_a | db_g] of this CTA
        float* pr = part + (long long)blockIdx.x * (g.ntaps + 1) * N;
        const long long o = n < n_split ? 0 : (long long)g.ntaps * n_split;
        const long long ob = (long long)g.ntaps * N + (n < n_split ? 0 : n_split);
        float* pd = t < NT ? pr + o + (long long)g.widx[t] * ncols + nn : pr + ob + nn;
        *reinterpret_cast<float4*>(pd) = sacc;
      } else if (dst) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(sacc.x), "f"(sacc.y), "f"(sacc.z), "f"(sacc.w) : "memory");
    }
  }
}

cudaError_t launch_wgrad_c1(const GatherGeom& g, const float* src, const float* grad, int g_ld, int N,
                            float* dw_a, float* dw_g, int n_split, float* db_a, float* db_g, cudaStream_t st, const DetSlab* det,
                            const PackGeom* pk) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0) return cudaSuccess;
  int nq = N / 4;
  if (N % 4 != 0 || nq > 256 || 256 % nq != 0 || n_split % 4 != 0 || g_ld % 4 != 0 || (pk && (g.B != 1 || g.ntaps > 9)))
    return cudaErrorInvalidValue;
  int rpb = (int)((M + CGVC_NUM_SMS * 8 - 1) / (CGVC_NUM_SMS * 8)); rpb = (rpb + kC1Rows - 1) / kC1Rows * kC1Rows;
  const long long nb = (M + rpb - 1) / rpb, row = (long long)(g.ntaps + 1) * N, nt = g.ntaps;
  float* part = det ? det->p : nullptr;
  if (part && nb * row > det->cap) return cudaErrorInvalidValue;
  ++g_cgvc_launches;
  if (pk) wgrad_c1_kernel<9, PackGeom2><<<(unsigned)nb, 256, 0, st>>>(g, src, grad, g_ld, N, dw_a, dw_g, n_split, db_a, db_g, rpb, part,
                                                                     PackGeom2{*pk});
  else if (g.ntaps <= 9) wgrad_c1_kernel<9><<<(unsigned)nb, 256, 0, st>>>(g, src, grad, g_ld, N, dw_a, dw_g, n_split, db_a, db_g, rpb, part);
  else wgrad_c1_kernel<CGVC_MAX_TAPS><<<(unsigned)nb, 256, 0, st>>>(g, src, grad, g_ld, N, dw_a, dw_g, n_split, db_a, db_g, rpb, part);
  if (!part) return cudaGetLastError();
  const long long na = n_split, ng = N - n_split;
  return launch_reduce_parts(part, nb, row, DetSegs{{dw_a, dw_g, db_a, db_g}, {0, nt * na, nt * N, nt * N + na},
                                                    {nt * na, nt * ng, db_a ? na : 0, db_g ? ng : 0}}, st);
}

template <class... PKs>
__global__ void gather_taps_kernel(const float* __restrict__ Z, float* __restrict__ dx, int B, int H, int W, int Ho, int Wo, int kh, int kw,
                                   int sh, int sw, int ph, int pw, const PKs... pks);
// ---- discriminator input layer (one input channel, K = 9, no instance norm: module.py:196-199), backward fused --------------------
// Its gated output is the largest activation of the step (805 MB of pre-activations per lane at batch 256), and its backward
// used to be: GLU backward -> dP fp32 written, then read again by the weight gradient and by the data-gradient projection.  The two
// kernels below form dP = (dY s(g), dY a s(g)(1 - s(g))) in registers from dY and the saved P = [a | g] and consume it in place:
//   glu_bwd_wgrad_c1_kernel:  dW[t][n] += sum_m x[src(m,t)] dP[m,n], db[n] += sum_m dP[m,n]      (D-loss pass, all 2B samples)
//   glu_bwd_proj_c1_kernel:   Z[m,t] = sum_n dP[m,n] w[t][n]  (then gather_taps)                 (adversarial pass, the B fakes)
// so dP never touches HBM (-1.6 GB and -0.8 GB per lane).  C = channels per branch (128): thread = (column quad j of BOTH branches,
// position lane).
template <int NT, class... PKs>
__global__ void __launch_bounds__(256)
glu_bwd_wgrad_c1_kernel(const __grid_constant__ GatherGeom g, const float* __restrict__ src, const float* __restrict__ dy,
                        const float* __restrict__ P, int C, float* __restrict__ dw_a, float* __restrict__ dw_g,
                        float* __restrict__ db_a, float* __restrict__ db_g, int rows_per_block, float* __restrict__ part,
                        const PKs... pks) {
  __shared__ __align__(16) float xs[kC1Rows][kC1Pad];
  __shared__ float4 red[256];
  const int nq = C / 4;                                 // column quads per branch; host guarantees nq divides 256
  const int cq = threadIdx.x % nq, rl = threadIdx.x / nq, rstep = 256 / nq;
  const int n = cq * 4;
  const long long M = (long long)g.B * g.Hy * g.Wx;
  long long r0 = (long long)blockIdx.x * rows_per_block;
  long long r1 = r0 + rows_per_block < M ? r0 + rows_per_block : M;
  float4 acc_a[NT + 1], acc_g[NT + 1];                  // [NT] = bias gradient
#pragma unroll
  for (int t = 0; t <= NT; ++t) { acc_a[t] = make_float4(0.f, 0.f, 0.f, 0.f); acc_g[t] = make_float4(0.f, 0.f, 0.f, 0.f); }
  for (long long mb = r0; mb < r1; mb += kC1Rows) {
    __syncthreads();
    c1_stage_taps(g, src, mb, r1, xs, pks...);
    __syncthreads();
    const int cnt = (int)((r1 - mb) < kC1Rows ? (r1 - mb) : kC1Rows);
#pragma unroll 2
    for (int rr = rl; rr < cnt; rr += rstep) {
      const long long m = mb + rr;
      const float4 d = *reinterpret_cast<const float4*>(dy + m * C + n);
      const float4 a = *reinterpret_cast<const float4*>(P + m * 2 * C + n);
      const float4 gg = *reinterpret_cast<const float4*>(P + m * 2 * C + C + n);
      const float dv[4] = {d.x, d.y, d.z, d.w}, av[4] = {a.x, a.y, a.z, a.w}, gv[4] = {gg.x, gg.y, gg.z, gg.w};
      float da[4], dg[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) { const float sg = sigmoidf_(gv[k]); da[k] = dv[k] * sg; dg[k] = da[k] * av[k] * (1.f - sg); }
      acc_a[NT].x += da[0]; acc_a[NT].y += da[1]; acc_a[NT].z += da[2]; acc_a[NT].w += da[3];
      acc_g[NT].x += dg[0]; acc_g[NT].y += dg[1]; acc_g[NT].z += dg[2]; acc_g[NT].w += dg[3];
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        if (t < g.ntaps) {
          const float v = xs[rr][t];
          acc_a[t].x = fmaf(v, da[0], acc_a[t].x); acc_a[t].y = fmaf(v, da[1], acc_a[t].y); acc_a[t].z = fmaf(v, da[2], acc_a[t].z); acc_a[t].w = fmaf(v, da[3], acc_a[t].w);
          acc_g[t].x = fmaf(v, dg[0], acc_g[t].x); acc_g[t].y = fmaf(v, dg[1], acc_g[t].y); acc_g[t].z = fmaf(v, dg[2], acc_g[t].z); acc_g[t].w = fmaf(v, dg[3], acc_g[t].w);
        }
      }
    }
  }
  // reduce the position lanes through shared memory (one quantity at a time), then one vector atomic per (tap, column quad, branch)
#pragma unroll
  for (int br = 0; br < 2; ++br) {
    float* dw = br ? dw_g : dw_a; float* db = br ? db_g : db_a;
#pragma unroll
    for (int t = 0; t <= NT; ++t) {
      if (!(t < g.ntaps || t == NT)) continue;           // block-uniform
      __syncthreads();
      red[threadIdx.x] = br ? acc_g[t] : acc_a[t];
      __syncthreads();
      if (rl == 0) {
        float4 sacc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int l = 0; l < rstep; ++l) { float4 v = red[l * nq + cq]; sacc.x += v.x; sacc.y += v.y; sacc.z += v.z; sacc.w += v.w; }
        float* dst = t < NT ? dw + (long long)g.widx[t] * C + n : (db ? db + n : nullptr);
        if (part) {                                        // det: row [dw_a | dw_g | db_a | db_g] of this CTA
          float* pr = part + (long long)blockIdx.x * 2 * (g.ntaps + 1) * C;
          float* pd = t < NT ? pr + ((long long)br * g.ntaps + g.widx[t]) * C + n : pr + (2ll * g.ntaps + br) * C + n;
          *reinterpret_cast<float4*>(pd) = sacc;
        } else if (dst) asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(sacc.x), "f"(sacc.y), "f"(sacc.z), "f"(sacc.w) : "memory");
      }
    }
  }
}

cudaError_t launch_glu_bwd_wgrad_c1(const GatherGeom& g, const float* src, const float* dy, const float* P, int C,
                                    float* dw_a, float* dw_g, float* db_a, float* db_g, cudaStream_t st, const DetSlab* det,
                                    const PackGeom* pk) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0) return cudaSuccess;
  int nq = C / 4;
  if (C % 4 != 0 || nq > 256 || 256 % nq != 0 || g.ntaps > 9 || (pk && g.B != 1)) return cudaErrorInvalidValue;
  int rpb = (int)((M + CGVC_NUM_SMS * 8 - 1) / (CGVC_NUM_SMS * 8)); rpb = (rpb + kC1Rows - 1) / kC1Rows * kC1Rows;
  const long long nb = (M + rpb - 1) / rpb, nt = g.ntaps, Cl = C, row = 2 * (nt + 1) * Cl;
  float* part = det ? det->p : nullptr;
  if (part && nb * row > det->cap) return cudaErrorInvalidValue;
  ++g_cgvc_launches;
  if (pk) glu_bwd_wgrad_c1_kernel<9, PackGeom2><<<(unsigned)nb, 256, 0, st>>>(g, src, dy, P, C, dw_a, dw_g, db_a, db_g, rpb, part,
                                                                             PackGeom2{*pk});
  else glu_bwd_wgrad_c1_kernel<9><<<(unsigned)nb, 256, 0, st>>>(g, src, dy, P, C, dw_a, dw_g, db_a, db_g, rpb, part);
  if (!part) return cudaGetLastError();
  return launch_reduce_parts(part, nb, row, DetSegs{{dw_a, dw_g, db_a, db_g}, {0, nt * Cl, 2 * nt * Cl, (2 * nt + 1) * Cl},
                                                    {nt * Cl, nt * Cl, db_a ? Cl : 0, db_g ? Cl : 0}}, st);
}

// column sums over the 32 rows of a warp (row = lane): butterfly transpose-reduce, 31 shuffles for 32 columns; lane j ends with column j
__device__ __forceinline__ float warp_colsum32_simt(float (&t)[32], int lane) {
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

// Z[m, t] = sum_n dP[m, n] * w[t][n] with dP formed on the fly; one warp per 3 rows at a time: lane = column quad of both branches
// (C = 128), its 9 x 8 weights in registers; the 27 (row, tap) partial sums of a lane are reduced over the 32 lanes by one butterfly
__global__ void __launch_bounds__(256)
glu_bwd_proj_c1_kernel(const float* __restrict__ dy, const float* __restrict__ P, long long rows, const float* __restrict__ wa,
                       const float* __restrict__ wg, int ntaps, float* __restrict__ Z) {
  constexpr int C = 128;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = lane * 4;
  float4 wav[9], wgv[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    wav[t] = t < ntaps ? *reinterpret_cast<const float4*>(wa + (long long)t * C + n) : make_float4(0.f, 0.f, 0.f, 0.f);
    wgv[t] = t < ntaps ? *reinterpret_cast<const float4*>(wg + (long long)t * C + n) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (long long r = ((long long)blockIdx.x * 8 + warp) * 3; r < rows; r += (long long)gridDim.x * 8 * 3) {
    float part[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) part[k] = 0.f;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const long long m = r + i;
      if (m < rows) {
        const float4 d = *reinterpret_cast<const float4*>(dy + m * C + n);
        const float4 a = *reinterpret_cast<const float4*>(P + m * 2 * C + n);
        const float4 gg = *reinterpret_cast<const float4*>(P + m * 2 * C + C + n);
        const float dv[4] = {d.x, d.y, d.z, d.w}, av[4] = {a.x, a.y, a.z, a.w}, gv[4] = {gg.x, gg.y, gg.z, gg.w};
        float da[4], dg[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float sg = sigmoidf_(gv[k]); da[k] = dv[k] * sg; dg[k] = da[k] * av[k] * (1.f - sg); }
#pragma unroll
        for (int t = 0; t < 9; ++t)
          part[9 * i + t] = da[0] * wav[t].x + da[1] * wav[t].y + da[2] * wav[t].z + da[3] * wav[t].w +
                            dg[0] * wgv[t].x + dg[1] * wgv[t].y + dg[2] * wgv[t].z + dg[3] * wgv[t].w;
      }
    }
    const float tot = warp_colsum32_simt(part, lane);      // lane j = sum over lanes of part[j]; j = 9 * i + t
    if (lane < 27) {
      const int i = lane / 9, t = lane - 9 * i;
      if (r + i < rows && t < ntaps) Z[(r + i) * ntaps + t] = tot;
    }
  }
}

cudaError_t launch_glu_bwd_dgrad_c1(const float* dy, const float* P, int C, const float* wa, const float* wg, float* Z, float* dx,
                                    int B, int H, int W, int kh, int kw, int sh, int sw, cudaStream_t st, const PackGeom* pk) {
  int Ho = (H + sh - 1) / sh, Wo = (W + sw - 1) / sw;
  int th = (Ho - 1) * sh + kh - H; if (th < 0) th = 0; int tw = (Wo - 1) * sw + kw - W; if (tw < 0) tw = 0;
  int ph = th / 2, pw = tw / 2;
  long long rows = (long long)B * Ho * Wo;
  if (rows == 0) return cudaSuccess;
  if (C != 128 || kh * kw > 9) return cudaErrorInvalidValue;
  long long nb = (rows + 23) / 24; if (nb > CGVC_NUM_SMS * 8) nb = CGVC_NUM_SMS * 8;
  g_cgvc_launches += 2;
  glu_bwd_proj_c1_kernel<<<(unsigned)nb, 256, 0, st>>>(dy, P, rows, wa, wg, kh * kw, Z);
  long long n = (long long)B * H * W; long long nb2 = (n + 255) / 256; if (nb2 > CGVC_NUM_SMS * 16) nb2 = CGVC_NUM_SMS * 16;
  if (pk) gather_taps_kernel<PackGeom2><<<(unsigned)nb2, 256, 0, st>>>(Z, dx, B, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, PackGeom2{*pk});
  else gather_taps_kernel<<<(unsigned)nb2, 256, 0, st>>>(Z, dx, B, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw);
  return cudaGetLastError();
}

// data gradient w.r.t. the single input channel, in two HBM-bound steps:
//   (1) Z[m', t] = sum_c G[m', c] * w[t][c]         (G = dP [rows, C] read once; w = [kernel_a | kernel_g] per tap)
//   (2) dx[b,h,w] = sum_taps Z[(b,ho,wo), t]        with ho*sh + i - ph = h, wo*sw + j - pw = w
__global__ void __launch_bounds__(256)
proj_taps_kernel(const float* __restrict__ G, long long rows, int C, const float* __restrict__ wa, const float* __restrict__ wg,
                 int c_split, int ntaps, float* __restrict__ Z) {
  // one warp per row; lane holds channels lane*4 + 128*q
  extern __shared__ float wsm[];                    // [ntaps][C]
  for (int i = threadIdx.x; i < ntaps * C; i += 256) {
    int t = i / C, c = i - t * C;
    wsm[i] = c < c_split ? wa[(long long)t * c_split + c] : wg[(long long)t * (C - c_split) + (c - c_split)];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long r = (long long)blockIdx.x * 8 + warp; r < rows; r += (long long)gridDim.x * 8) {
    float acc[CGVC_MAX_TAPS];
#pragma unroll
    for (int t = 0; t < CGVC_MAX_TAPS; ++t) acc[t] = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
      float4 v = *reinterpret_cast<const float4*>(G + r * C + c);
#pragma unroll
      for (int t = 0; t < CGVC_MAX_TAPS; ++t) {
        if (t < ntaps) {
          float4 w = *reinterpret_cast<const float4*>(wsm + t * C + c);
          acc[t] += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
        }
      }
    }
#pragma unroll
    for (int t = 0; t < CGVC_MAX_TAPS; ++t) {
      if (t < ntaps) {
        float a = acc[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) Z[r * ntaps + t] = a;
      }
    }
  }
}

// PKs: an optional trailing PackGeom2 (packed 2-D grids, B = 1, W = all frames): position idx of the input grid (divisor pk.div)
// sums only the Z rows of its own utterance in the output grid (divisor pk.div * sw)
template <class... PKs>
__global__ void __launch_bounds__(256)
gather_taps_kernel(const float* __restrict__ Z, float* __restrict__ dx, int B, int H, int W, int Ho, int Wo, int kh, int kw,
                   int sh, int sw, int ph, int pw, const PKs... pks) {
  long long n = (long long)B * H * W;
  const int ntaps = kh * kw;
  for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < n; idx += (long long)gridDim.x * 256) {
    if constexpr (sizeof...(PKs) > 0) {
      const PackGeom& pk = pack_arg(pks...);
      const Pack2Pos o = pack2_pos(pk, H, pk.div, idx);
      float a = 0.f;
      for (int i = 0; i < kh; ++i) {
        int ny = o.y + ph - i; if (ny < 0 || ny % sh) continue;
        for (int j = 0; j < kw; ++j) {
          int nx = o.x + pw - j; if (nx < 0 || nx % sw) continue;
          const long long r = pack2_row(o.o0, o.o1, Ho, pk.div * sw, ny / sh, nx / sw);
          if (r >= 0) a += Z[r * ntaps + i * kw + j];
        }
      }
      dx[idx] = a;
      continue;
    }
    int w = (int)(idx % W); long long r = idx / W; int h = (int)(r % H); int b = (int)(r / H);
    float a = 0.f;
    for (int i = 0; i < kh; ++i) {
      int ny = h + ph - i; if (ny < 0 || ny % sh) continue; int ho = ny / sh; if (ho >= Ho) continue;
      for (int j = 0; j < kw; ++j) {
        int nx = w + pw - j; if (nx < 0 || nx % sw) continue; int wo = nx / sw; if (wo >= Wo) continue;
        a += Z[((long long)(b * Ho + ho) * Wo + wo) * ntaps + i * kw + j];
      }
    }
    dx[idx] = a;
  }
}

cudaError_t launch_dgrad_c1(const float* G, int C, const float* wa, const float* wg, int c_split, float* Z, float* dx,
                            int B, int H, int W, int kh, int kw, int sh, int sw, cudaStream_t st, const PackGeom* pk) {
  int Ho = (H + sh - 1) / sh, Wo = (W + sw - 1) / sw;
  int th = (Ho - 1) * sh + kh - H; if (th < 0) th = 0; int tw = (Wo - 1) * sw + kw - W; if (tw < 0) tw = 0;
  int ph = th / 2, pw = tw / 2;
  long long rows = (long long)B * Ho * Wo;
  if (rows == 0) return cudaSuccess;
  if (C % 128 != 0 || kh * kw > CGVC_MAX_TAPS) return cudaErrorInvalidValue;
  size_t smem = (size_t)kh * kw * C * sizeof(float);
  long long nb = (rows + 7) / 8; if (nb > CGVC_NUM_SMS * 8) nb = CGVC_NUM_SMS * 8;
  g_cgvc_launches += 2;
  proj_taps_kernel<<<(unsigned)nb, 256, smem, st>>>(G, rows, C, wa, wg, c_split, kh * kw, Z);
  long long n = (long long)B * H * W; long long nb2 = (n + 255) / 256; if (nb2 > CGVC_NUM_SMS * 16) nb2 = CGVC_NUM_SMS * 16;
  if (pk) gather_taps_kernel<PackGeom2><<<(unsigned)nb2, 256, 0, st>>>(Z, dx, B, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw, PackGeom2{*pk});
  else gather_taps_kernel<<<(unsigned)nb2, 256, 0, st>>>(Z, dx, B, H, W, Ho, Wo, kh, kw, sh, sw, ph, pw);
  return cudaGetLastError();
}

// fp32 rows [M, C] (row stride ld) -> bf16 hi/lo planes [M, Cpad] with zero channels [C, Cpad)
__global__ void __launch_bounds__(256)
pad_split_kernel(const float* __restrict__ x, long long M, int C, int ld, int Cpad, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  long long n = M * Cpad;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    int c = (int)(i % Cpad); long long m = i / Cpad;
    float v = c < C ? x[m * ld + c] : 0.f;
    __nv_bfloat16 h, l; split_bf16(v, h, l); hi[i] = h; lo[i] = l;
  }
}

// fp32 rows [M, C] -> F16F8 planes [M, Cpad] (Cpad a multiple of 4), zero channels [C, Cpad)
__global__ void __launch_bounds__(256)
pad_split_q_kernel(const float* __restrict__ x, long long M, int C, int ld, int Cpad, __half* __restrict__ q16, uint8_t* __restrict__ q8,
                   unsigned long long* __restrict__ sat, unsigned long long* __restrict__ ufl) {
  const long long n = M * Cpad, nq = n / 4;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nq; i += (long long)gridDim.x * 256) {
    const long long e = i * 4; const int c = (int)(e % Cpad); const long long m = e / Cpad;
    float v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = (c + k) < C ? x[m * ld + c + k] : 0.f;
    uint2 h; uint32_t b_hi, b_lo;
    cgvc_quant4(v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO, h, b_hi, b_lo);
    *reinterpret_cast<uint2*>(q16 + e) = h;
    *reinterpret_cast<uint32_t*>(q8 + e) = b_hi;
    *reinterpret_cast<uint32_t*>(q8 + n + e) = b_lo;
    cgvc_count_planes(sat, ufl, v);
  }
}

cudaError_t launch_pad_split_q(const float* x, long long M, int C, int ld, int Cpad, void* q16, void* q8, cudaStream_t st, unsigned long long* sat,
                               unsigned long long* ufl) {
  if (M == 0) return cudaSuccess;
  if (Cpad % 4) return cudaErrorInvalidValue;
  long long n = M * Cpad / 4; long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16;
  ++g_cgvc_launches;
  pad_split_q_kernel<<<(unsigned)nb, 256, 0, st>>>(x, M, C, ld, Cpad, (__half*)q16, (uint8_t*)q8, sat, ufl);
  return cudaGetLastError();
}

cudaError_t launch_pad_split(const float* x, long long M, int C, int ld, int Cpad, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st) {
  if (M == 0) return cudaSuccess;
  long long n = M * Cpad; long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16;
  ++g_cgvc_launches;
  pad_split_kernel<<<(unsigned)nb, 256, 0, st>>>(x, M, C, ld, Cpad, hi, lo);
  return cudaGetLastError();
}

// ---- tap lowering of the generator's two 15-tap edge layers (module.py:85-86 h1: 24 -> 2 x 128 channels; module.py:148 o1: 256 -> 24).
// Both have 24 channels on one side, so as 15-tap gather-GEMMs they waste the tensor cores: the 24-channel operand is padded to a
// 64 / 128-channel line per tap, or the 24 output columns fill a 32-wide tile while the 256-channel operand is streamed 15 times.
// With the taps moved into the GEMM's channel / column dimension they become dense 1 x 1 layers (engine.cu, `edge_lower`):
//   h1:  P = im2col(x) [M, 15*24] . W[(t,c)][n]          -- TF's [1,15,24,128] kernel IS that [360,128] matrix
//   o1:  Z = U [M,256] . W'[c][(t,n)],  out[m,n] = b[n] + sum_t Z[m + t - 7, (t,n)]   (and the transposes of both for the backward pass)
// im2col over the taps of a stride-1 1-D TF-SAME convolution of a NARROW channels-last tensor x [B*T, C] (C % 4 == 0):
//   out[m, t*C + c] = x[m + dir*(t - pl), c]  if that row lies in the same sample, else 0;   columns [kw*C, Cpad) = 0
// Q = 1: F16F8 planes (q16; q8hi followed by q8lo, activation-role scales); Q = 0: bf16 hi / lo planes.
// row m's position in its sample and the sample's length: T-row blocks, or (off != null) the packed utterances [off[u], off[u+1])
__device__ __forceinline__ int tap_sample(long long m, int T, const long long* __restrict__ off, int n_off, int& len) {
  if (off) {
    const int u = pack_find(off, n_off, m);
    const long long o0 = __ldg(off + u);
    len = (int)(__ldg(off + u + 1) - o0);
    return (int)(m - o0);
  }
  len = T;
  return (int)(m % T);
}

template <int Q>
__global__ void __launch_bounds__(256)
im2col_taps_kernel(const float* __restrict__ x, long long M, int T, int C, int kw, int pl, int dir, int Cpad, void* __restrict__ hi, void* __restrict__ lo,
                   const long long* __restrict__ off, int n_off, unsigned long long* __restrict__ sat,
                   unsigned long long* __restrict__ ufl) {
  const long long n = M * Cpad, nq = n / 4;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nq; i += (long long)gridDim.x * 256) {
    const long long e = i * 4; const int col = (int)(e % Cpad); const long long m = e / Cpad;
    const int t = col / C, c = col - t * C;
    int len; const int w = tap_sample(m, T, off, n_off, len), ws = w + dir * (t - pl);
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (t < kw && ws >= 0 && ws < len) {
      const float4 q = *reinterpret_cast<const float4*>(x + (m + (long long)(ws - w)) * C + c);
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    }
    if (Q) {
      uint2 h; uint32_t b_hi, b_lo;
      cgvc_quant4(v, CGVC_Q_ACT_SHI, CGVC_Q_ACT_SLO, h, b_hi, b_lo);
      *reinterpret_cast<uint2*>((__half*)hi + e) = h;
      *reinterpret_cast<uint32_t*>((uint8_t*)lo + e) = b_hi;
      *reinterpret_cast<uint32_t*>((uint8_t*)lo + n + e) = b_lo;
      cgvc_count_planes(sat, ufl, v);
    } else {
      __align__(8) __nv_bfloat16 h[4]; __align__(8) __nv_bfloat16 l[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) split_bf16(v[k], h[k], l[k]);
      *reinterpret_cast<uint2*>((__nv_bfloat16*)hi + e) = *reinterpret_cast<const uint2*>(h);
      *reinterpret_cast<uint2*>((__nv_bfloat16*)lo + e) = *reinterpret_cast<const uint2*>(l);
    }
  }
}

cudaError_t launch_im2col_taps(const float* x, long long M, int T, int C, int kw, int dir, int Cpad, int qmode, void* hi, void* lo, cudaStream_t st,
                               const long long* off, int n_off, unsigned long long* sat, unsigned long long* ufl) {
  if (M == 0) return cudaSuccess;
  if (C % 4 || Cpad % 4 || Cpad < kw * C || (!off && (T <= 0 || M % T)) || (off && n_off < 1)) return cudaErrorInvalidValue;
  const int pl = (kw - 1) / 2;                      // TF SAME at stride 1: total pad kw - 1, the smaller half on the left
  long long n = M * Cpad / 4; long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16;
  ++g_cgvc_launches;
  if (qmode) im2col_taps_kernel<1><<<(unsigned)nb, 256, 0, st>>>(x, M, T, C, kw, pl, dir, Cpad, hi, lo, off, n_off, sat, ufl);
  else im2col_taps_kernel<0><<<(unsigned)nb, 256, 0, st>>>(x, M, T, C, kw, pl, dir, Cpad, hi, lo, off, n_off, nullptr, nullptr);
  return cudaGetLastError();
}

// the inverse gather: y[m, c] = (bias ? bias[c] : 0) + sum_t z[m + dir*(t - pl), t*C + c] over the rows of the same sample; z row stride ldz.
// One thread per 4 output channels; the 15 partial sums are added in tap order (deterministic).
__global__ void __launch_bounds__(256)
col2im_taps_kernel(const float* __restrict__ z, int ldz, long long M, int T, int C, int kw, int pl, int dir, const float* __restrict__ bias, float* __restrict__ y,
                   const long long* __restrict__ off, int n_off) {
  const int cq = C / 4;
  const long long n = M * cq;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % cq) * 4; const long long m = i / cq;
    int len; const int w = tap_sample(m, T, off, n_off, len);
    float4 acc = bias ? *reinterpret_cast<const float4*>(bias + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = 0; t < kw; ++t) {
      const int ws = w + dir * (t - pl);
      if (ws < 0 || ws >= len) continue;
      const float4 q = *reinterpret_cast<const float4*>(z + (m + (long long)(ws - w)) * ldz + t * C + c);
      acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
    }
    *reinterpret_cast<float4*>(y + m * C + c) = acc;
  }
}

cudaError_t launch_col2im_taps(const float* z, int ldz, long long M, int T, int C, int kw, int dir, const float* bias, float* y, cudaStream_t st,
                               const long long* off, int n_off) {
  if (M == 0) return cudaSuccess;
  if (C % 4 || ldz % 4 || (!off && (T <= 0 || M % T)) || (off && n_off < 1)) return cudaErrorInvalidValue;
  const int pl = (kw - 1) / 2;
  long long n = M * (C / 4); long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 16) nb = CGVC_NUM_SMS * 16;
  ++g_cgvc_launches;
  col2im_taps_kernel<<<(unsigned)nb, 256, 0, st>>>(z, ldz, M, T, C, kw, pl, dir, bias, y, off, n_off);
  return cudaGetLastError();
}

// forward of the single-input-channel gated layer: P[m, n] = bias[n] + sum_t x[src(m,t)] * w[t][n], n over [a | g] columns.
// HBM-bound on the output write (N*4 bytes per position); one thread = one column quad, 4 positions per CTA sweep.
template <int NT, class... PKs>
__global__ void __launch_bounds__(256)
conv_c1_fwd_kernel(const __grid_constant__ GatherGeom g, const float* __restrict__ x, const float* __restrict__ wa, const float* __restrict__ wg,
                   const float* __restrict__ ba, const float* __restrict__ bg, int cout, float* __restrict__ P, int rows_per_block,
                   const PKs... pks) {
  __shared__ __align__(16) float xs[kC1Rows][kC1Pad];
  const int nq = (2 * cout) / 4;                       // column quads (host guarantees nq divides 256)
  const int cq = threadIdx.x % nq, rl = threadIdx.x / nq, rstep = 256 / nq;
  const int n = cq * 4;
  const float* w = n < cout ? wa + n : wg + (n - cout);
  float4 wq[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) wq[t] = t < g.ntaps ? *reinterpret_cast<const float4*>(w + (long long)g.widx[t] * cout) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 bq = *reinterpret_cast<const float4*>(n < cout ? ba + n : bg + (n - cout));
  const long long M = (long long)g.B * g.Hy * g.Wx;
  long long m0 = (long long)blockIdx.x * rows_per_block;
  long long m1 = m0 + rows_per_block < M ? m0 + rows_per_block : M;
  for (long long mb = m0; mb < m1; mb += kC1Rows) {
    __syncthreads();
    c1_stage_taps(g, x, mb, m1, xs, pks...);
    __syncthreads();
    const int cnt = (int)((m1 - mb) < kC1Rows ? (m1 - mb) : kC1Rows);
    for (int rr = rl; rr < cnt; rr += rstep) {
      float4 o = bq;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        if (t < g.ntaps) {
          float v = xs[rr][t];
          o.x = fmaf(v, wq[t].x, o.x); o.y = fmaf(v, wq[t].y, o.y); o.z = fmaf(v, wq[t].z, o.z); o.w = fmaf(v, wq[t].w, o.w);
        }
      }
      *reinterpret_cast<float4*>(P + (mb + rr) * (2 * cout) + n) = o;
    }
  }
}

cudaError_t launch_conv_c1_fwd(const GatherGeom& g, const float* x, const float* wa, const float* wg, const float* ba, const float* bg,
                               int cout, float* P, cudaStream_t st, const PackGeom* pk) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0) return cudaSuccess;
  int nq = (2 * cout) / 4;
  if (cout % 4 != 0 || nq > 256 || 256 % nq != 0 || (pk && (g.B != 1 || g.ntaps > 9))) return cudaErrorInvalidValue;
  int rpb = 4 * kC1Rows;
  ++g_cgvc_launches;
  if (pk) conv_c1_fwd_kernel<9, PackGeom2><<<(unsigned)((M + rpb - 1) / rpb), 256, 0, st>>>(g, x, wa, wg, ba, bg, cout, P, rpb, PackGeom2{*pk});
  else if (g.ntaps <= 9) conv_c1_fwd_kernel<9><<<(unsigned)((M + rpb - 1) / rpb), 256, 0, st>>>(g, x, wa, wg, ba, bg, cout, P, rpb);
  else conv_c1_fwd_kernel<CGVC_MAX_TAPS><<<(unsigned)((M + rpb - 1) / rpb), 256, 0, st>>>(g, x, wa, wg, ba, bg, cout, P, rpb);
  return cudaGetLastError();
}

// The same layer with its GLU (gate without instance norm, module.py:193-195) in the same pass: one thread computes the a-quad AND the
// g-quad of 4 channels, writes both to P (kept for the backward pass) and y = a * sigmoid(g) to the operand planes of the next layer
// (+ the fp32 copy when asked) -- P is not read back by a second kernel (B*24*64*256*4 bytes per application of the discriminator).
template <int NT, class... PKs>
__global__ void __launch_bounds__(256)
conv_c1_glu_fwd_kernel(const __grid_constant__ GatherGeom g, const float* __restrict__ x, const float* __restrict__ wa, const float* __restrict__ wg,
                       const float* __restrict__ ba, const float* __restrict__ bg, int cout, float* __restrict__ P,
                       float* __restrict__ y, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo, int qmode, long long plane_elems,
                       int rows_per_block, unsigned long long* __restrict__ sat, unsigned long long* __restrict__ ufl, const PKs... pks) {
  __shared__ __align__(16) float xs[kC1Rows][kC1Pad];
  const int nq = cout / 4;                             // channel quads (host guarantees nq divides 256)
  const int cq = threadIdx.x % nq, rl = threadIdx.x / nq, rstep = 256 / nq;
  const int n = cq * 4;
  float4 wqa[NT], wqg[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    wqa[t] = t < g.ntaps ? *reinterpret_cast<const float4*>(wa + n + (long long)g.widx[t] * cout) : make_float4(0.f, 0.f, 0.f, 0.f);
    wqg[t] = t < g.ntaps ? *reinterpret_cast<const float4*>(wg + n + (long long)g.widx[t] * cout) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float4 bqa = *reinterpret_cast<const float4*>(ba + n), bqg = *reinterpret_cast<const float4*>(bg + n);
  const long long M = (long long)g.B * g.Hy * g.Wx;
  long long m0 = (long long)blockIdx.x * rows_per_block;
  long long m1 = m0 + rows_per_block < M ? m0 + rows_per_block : M;
  for (long long mb = m0; mb < m1; mb += kC1Rows) {
    __syncthreads();
    c1_stage_taps(g, x, mb, m1, xs, pks...);
    __syncthreads();
    const int cnt = (int)((m1 - mb) < kC1Rows ? (m1 - mb) : kC1Rows);
    for (int rr = rl; rr < cnt; rr += rstep) {
      float4 a = bqa, gt = bqg;
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        if (t < g.ntaps) {
          const float v = xs[rr][t];
          a.x = fmaf(v, wqa[t].x, a.x); a.y = fmaf(v, wqa[t].y, a.y); a.z = fmaf(v, wqa[t].z, a.z); a.w = fmaf(v, wqa[t].w, a.w);
          gt.x = fmaf(v, wqg[t].x, gt.x); gt.y = fmaf(v, wqg[t].y, gt.y); gt.z = fmaf(v, wqg[t].z, gt.z); gt.w = fmaf(v, wqg[t].w, gt.w);
        }
      }
      const long long m = mb + rr;
      *reinterpret_cast<float4*>(P + m * (2 * cout) + n) = a;
      *reinterpret_cast<float4*>(P + m * (2 * cout) + cout + n) = gt;
      F4 o;
      o.v[0] = a.x * sigmoidf_(gt.x); o.v[1] = a.y * sigmoidf_(gt.y); o.v[2] = a.z * sigmoidf_(gt.z); o.v[3] = a.w * sigmoidf_(gt.w);
      const long long e = m * cout + n;
      if (y) st4(y + e, o);
      if (y_hi) {
        if (qmode) st4_quant(y_hi, y_lo, e, plane_elems, o, sat, ufl);
        else st4_split(y_hi + e, y_lo + e, o);
      }
    }
  }
}

cudaError_t launch_conv_c1_glu_fwd(const GatherGeom& g, const float* x, const float* wa, const float* wg, const float* ba, const float* bg,
                                   int cout, float* P, float* y, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo, int qmode, cudaStream_t st,
                                   unsigned long long* sat, unsigned long long* ufl, const PackGeom* pk) {
  long long M = (long long)g.B * g.Hy * g.Wx;
  if (M == 0) return cudaSuccess;
  int nq = cout / 4;
  if (cout % 4 != 0 || nq > 256 || 256 % nq != 0 || g.ntaps > 9 || (pk && g.B != 1)) return cudaErrorInvalidValue;
  int rpb = 4 * kC1Rows;
  ++g_cgvc_launches;
  if (pk) conv_c1_glu_fwd_kernel<9, PackGeom2><<<(unsigned)((M + rpb - 1) / rpb), 256, 0, st>>>(g, x, wa, wg, ba, bg, cout, P, y, y_hi, y_lo, qmode,
                                                                                                M * cout, rpb, sat, ufl, PackGeom2{*pk});
  else conv_c1_glu_fwd_kernel<9><<<(unsigned)((M + rpb - 1) / rpb), 256, 0, st>>>(g, x, wa, wg, ba, bg, cout, P, y, y_hi, y_lo, qmode, M * cout, rpb, sat, ufl);
  return cudaGetLastError();
}

// device scalars of a step, written by an eagerly launched kernel so that the captured CUDA graph of the step never
// contains a host-memory copy: s[off + i] = v[i]
struct Scalars6 { float v[6]; };
__global__ void set_scalars_kernel(float* s, Scalars6 x, int off, int n) {
  if (threadIdx.x < n) s[off + threadIdx.x] = x.v[threadIdx.x];
}
cudaError_t launch_set_scalars(float* s, int off, int n, const float* v6_host, cudaStream_t st) {
  Scalars6 x; for (int i = 0; i < 6; ++i) x.v[i] = i < n ? v6_host[i] : 0.f;
  ++g_cgvc_launches;
  set_scalars_kernel<<<1, 32, 0, st>>>(s, x, off, n);
  return cudaGetLastError();
}


// ------------------------------------------------------------------------------------------------------------------
// Device-resident training data (train.py:90-107 + preprocess.py:207-238 of the reference): the normalised MCEP corpus of both
// speakers lives in HBM; an epoch's pairing and crops are drawn on the device from a counter-based generator, so a training step
// needs no host -> device copy.  Contract (the host twin is preprocess.counter_sample_plan, compared index for index in the tests):
//   key(side, i)   = mix(mix(seed ^ (epoch << 20) ^ (side << 60)) + i)            side 0 = A, 1 = B
//   utterances of each side are taken in ascending key order (ties by index): two independent uniform shuffles, truncated to the
//   shorter list (num_pairs = min(n_A, n_B));  pair k = (order_A[k], order_B[k])
//   start(side, u) = mix(mix(seed ^ (epoch << 20) ^ ((side + 2) << 60)) + u) mod (frames(u) - crop + 1): one uniform crop per utterance
// ------------------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ unsigned long long cgvc_mix64(unsigned long long x) {     // splitmix64 finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ __forceinline__ unsigned long long cgvc_sample_key(unsigned long long seed, long long epoch, int stream, int i) {
  return cgvc_mix64(cgvc_mix64(seed ^ ((unsigned long long)epoch << 20) ^ ((unsigned long long)stream << 60)) + (unsigned long long)i);
}

// plan[0..3][num_pairs] = utt_A, start_A, utt_B, start_B.  One thread per (side, utterance): its rank among the keys of its side.
__global__ void sample_plan_kernel(const long long* __restrict__ off_A, int n_A, const long long* __restrict__ off_B, int n_B,
                                   unsigned long long seed, long long epoch, int crop, int num_pairs, int* __restrict__ plan, int* __restrict__ err) {
  const int side = blockIdx.y;
  const int n = side ? n_B : n_A;
  const long long* off = side ? off_B : off_A;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long ki = cgvc_sample_key(seed, epoch, side, i);
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const unsigned long long kj = cgvc_sample_key(seed, epoch, side, j);
      rank += (kj < ki || (kj == ki && j < i)) ? 1 : 0;
    }
    if (rank < num_pairs) {
      const long long len = off[i + 1] - off[i];
      if (len < crop) { atomicExch(err, i + 1 + (side ? (1 << 30) : 0)); continue; }      // preprocess.py:217,224: every utterance must hold a crop
      plan[(2 * side) * num_pairs + rank] = i;
      plan[(2 * side + 1) * num_pairs + rank] = (int)(cgvc_sample_key(seed, epoch, side + 2, i) % (unsigned long long)(len - crop + 1));
    }
  }
}

// out_X[b, f, t] = corpus_X[utt][f][start + t]; corpus_X holds utterance u as [F][len_u] at element F * off[u]
__global__ void gather_minibatch_kernel(const float* __restrict__ cA, const long long* __restrict__ off_A,
                                        const float* __restrict__ cB, const long long* __restrict__ off_B,
                                        const int* __restrict__ plan, int num_pairs, int first_pair, int F, int crop,
                                        float* __restrict__ out_A, float* __restrict__ out_B) {
  const int b = blockIdx.x, side = blockIdx.y;
  const int k = first_pair + b;
  const int utt = plan[(2 * side) * num_pairs + k], start = plan[(2 * side + 1) * num_pairs + k];
  const long long* off = side ? off_B : off_A;
  const float* src = (side ? cB : cA) + (long long)F * off[utt];
  const long long len = off[utt + 1] - off[utt];
  float* dst = (side ? out_B : out_A) + (long long)b * F * crop;
  for (int e = threadIdx.x; e < F * crop; e += blockDim.x) {
    const int f = e / crop, t = e - f * crop;
    dst[e] = src[(long long)f * len + start + t];
  }
}

cudaError_t launch_sample_plan(const long long* off_A, int n_A, const long long* off_B, int n_B, unsigned long long seed, long long epoch,
                               int crop, int* plan, int* err, cudaStream_t st) {
  const int num_pairs = n_A < n_B ? n_A : n_B;
  if (num_pairs <= 0) return cudaSuccess;
  const int n = n_A > n_B ? n_A : n_B;
  ++g_cgvc_launches;
  sample_plan_kernel<<<dim3((n + 127) / 128, 2), 128, 0, st>>>(off_A, n_A, off_B, n_B, seed, epoch, crop, num_pairs, plan, err);
  return cudaGetLastError();
}
cudaError_t launch_gather_minibatch(const float* cA, const long long* off_A, const float* cB, const long long* off_B, const int* plan,
                                    int num_pairs, int first_pair, int batch, int F, int crop, float* out_A, float* out_B, cudaStream_t st) {
  if (batch <= 0) return cudaSuccess;
  ++g_cgvc_launches;
  gather_minibatch_kernel<<<dim3(batch, 2), 256, 0, st>>>(cA, off_A, cB, off_B, plan, num_pairs, first_pair, F, crop, out_A, out_B);
  return cudaGetLastError();
}


// x *= a  (un-scaling the gradient arena after a loss-scaled backward pass whose result is handed out instead of going into Adam), or
// with div x *= a / *div; MUL: x *= a * *div (a tape backward's upstream gradient times the scaler's current loss scale)
template <bool MUL>
__global__ void __launch_bounds__(256) scale_kernel(float* __restrict__ x, long long n, float a, const float* __restrict__ div) {
  if (MUL) a = a * *div;
  else if (div) a = a / *div;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) x[i] *= a;
}
cudaError_t launch_scale(float* x, long long n, float a, cudaStream_t st, const float* div_dev) {
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 8) nb = CGVC_NUM_SMS * 8;
  ++g_cgvc_launches; scale_kernel<false><<<(unsigned)nb, 256, 0, st>>>(x, n, a, div_dev);
  return cudaGetLastError();
}
cudaError_t launch_scale_by(float* x, long long n, float a, const float* mul_dev, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  long long nb = (n + 255) / 256; if (nb > CGVC_NUM_SMS * 8) nb = CGVC_NUM_SMS * 8;
  ++g_cgvc_launches; scale_kernel<true><<<(unsigned)nb, 256, 0, st>>>(x, n, a, mul_dev);
  return cudaGetLastError();
}
