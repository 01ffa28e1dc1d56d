// Depthwise 5x5 convolution (groups == Cin == Cout = C, C % 8 == 0; stride 1 or 2, padding 2, dilation 1) on NHWC
// bf16 activations with fp32 accumulation: forward (+ per-channel BN statistics of the bf16 output), data gradient and
// weight gradient.  The 5x5 depthwise layers of MobileNetV3 (6 in -Large, 8 in -Small).  Same contracts as the 3x3
// kernels of depthwise.cu, same thread mapping (depthwise.cuh); only where the filter taps live differs:
//
// - forward / data gradient: 25 taps x 8 channels = 200 fp32 weights per thread would not fit the register file next to
//   the accumulators, so the block stages its slab's [25][8 * gpc] weights in shared memory (6.4 KB at most) once and
//   each tap reads its 8 weights as two 16-byte broadcasts (threads of a warp with the same channel group read the same
//   address).  What stays in registers is 8 accumulators (+ 16 statistics), so 3 blocks of 256 threads fit an SM.
// - weight gradient: 200 accumulators per thread would spill, so the grid's z dimension splits the filter rows: a block
//   owns one row r and accumulates its 5 taps x 8 channels = 40 products per thread (under 80 registers: 3 blocks per
//   SM), skipping the pixels whose row r falls in the padding.  The 5 row-blocks of a pixel range read the same dy
//   slab (L2-resident) and neighbouring x rows.
//
//   forward   y[n,p,q,c]  = sum_{r,s} x[n, p*st-2+r, q*st-2+s, c] * w[c][r][s]
//   dgrad     dx[n,h,w,c] = sum of dy[n,p,q,c] * w[c][r][s] over the taps with h = p*st-2+r, w = q*st-2+s (gather)
//   wgrad     gw[c][r][s] += sum_{n,p,q} dy[n,p,q,c] * x[n, p*st-2+r, q*st-2+s, c]
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"
#include "depthwise.cuh"

namespace ddl {

namespace {

using namespace dw;

constexpr int kTaps = 25;

// the block's weights [C][25] bf16, channels [slab0, slab0 + 8 << lg), as fp32 ws[tap][channel - slab0]
DDL_DEVICE void dw5_stage_weights(const __nv_bfloat16* w, int lg, float (*ws)[64]) {
  const int nch = 8 << lg;
  const __nv_bfloat16* src = w + (static_cast<size_t>(blockIdx.y) << (lg + 3)) * kTaps;     // contiguous nch * 25
  for (int e = threadIdx.x; e < nch * kTaps; e += kDwThreads) {
    const int c = e / kTaps, t = e - c * kTaps;
    ws[t][c] = __bfloat162float(src[e]);
  }
  __syncthreads();
}

// acc[i] += v[i] * ws[tap][cl + i]
DDL_DEVICE void dw5_fma_tap(float (&acc)[8], const float (&v)[8], const float* wrow) {
  const float4 a = reinterpret_cast<const float4*>(wrow)[0], b = reinterpret_cast<const float4*>(wrow)[1];
  acc[0] = fmaf(v[0], a.x, acc[0]); acc[1] = fmaf(v[1], a.y, acc[1]);
  acc[2] = fmaf(v[2], a.z, acc[2]); acc[3] = fmaf(v[3], a.w, acc[3]);
  acc[4] = fmaf(v[4], b.x, acc[4]); acc[5] = fmaf(v[5], b.y, acc[5]);
  acc[6] = fmaf(v[6], b.z, acc[6]); acc[7] = fmaf(v[7], b.w, acc[7]);
}

DDL_DEVICE uint4 dw5_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

// ---- forward ---------------------------------------------------------------------------------------------------
template <int STRIDE, bool STATS>
__global__ void __launch_bounds__(kDwThreads, 3) dwconv5_fwd_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  __shared__ __align__(16) float ws[kTaps][64];
  pdl_wait();
  dw5_stage_weights(a.w, a.lg_gpc, ws);
  const int cl = (threadIdx.x & ((1 << a.lg_gpc) - 1)) << 3;
  float st[16];                                   // [0, 8): sum y, [8, 16): sum y^2 of the bf16-rounded y
#pragma unroll
  for (int i = 0; i < 16; ++i) st[i] = 0.f;
  const int total = a.N * a.P * a.Q;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int q = o % a.Q;
    const int t = o / a.Q;
    const int p = t % a.P;
    const int n = t / a.P;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const int h = p * STRIDE - 2 + r;
      if (h < 0 || h >= a.H) continue;
      const __nv_bfloat16* row = a.x + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 5; ++s) {
        const int w = q * STRIDE - 2 + s;
        if (w < 0 || w >= a.W) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(w) * a.C, v);
        dw5_fma_tap(acc, v, &ws[r * 5 + s][cl]);
      }
    }
    const uint4 out = dw5_pack8(acc);
    *reinterpret_cast<uint4*>(a.y + static_cast<size_t>(o) * a.C + m.c0) = out;
    if (STATS) {
      float yb[8];
      dw_unpack8(out, yb);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        st[i] += yb[i];
        st[8 + i] = fmaf(yb[i], yb[i], st[8 + i]);
      }
    }
  }
  if (STATS) {
    __shared__ float red[kDwWarps * 8 * 16];
    dw_block_reduce<16>(st, a.lg_gpc, red, [&](int c, int which, float v) { atomicAdd((which ? a.sumsq : a.sum) + c, v); });
  }
}

// ---- data gradient (gather form) ---------------------------------------------------------------------------------
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads, 3) dwconv5_dgrad_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  __shared__ __align__(16) float ws[kTaps][64];
  pdl_wait();
  dw5_stage_weights(a.w, a.lg_gpc, ws);
  const int cl = (threadIdx.x & ((1 << a.lg_gpc) - 1)) << 3;
  const int total = a.N * a.H * a.W;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int w = o % a.W;
    const int t = o / a.W;
    const int h = t % a.H;
    const int n = t / a.H;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const int ph = h + 2 - r;                   // = p * STRIDE
      if (ph < 0 || (STRIDE == 2 && (ph & 1))) continue;
      const int p = ph / STRIDE;
      if (p >= a.P) continue;
      const __nv_bfloat16* row = a.dy + (static_cast<size_t>(n) * a.P + p) * a.Q * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 5; ++s) {
        const int qw = w + 2 - s;
        if (qw < 0 || (STRIDE == 2 && (qw & 1))) continue;
        const int q = qw / STRIDE;
        if (q >= a.Q) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(q) * a.C, v);
        dw5_fma_tap(acc, v, &ws[r * 5 + s][cl]);
      }
    }
    *reinterpret_cast<uint4*>(a.y + static_cast<size_t>(o) * a.C + m.c0) = dw5_pack8(acc);
  }
}

// ---- weight gradient -------------------------------------------------------------------------------------------
// Filter row r = blockIdx.z.  Each thread sums its pixels' 40 products (5 taps x 8 channels) in registers, the block
// folds them over its pixel lanes and adds one total per (channel, tap of row r) into the fp32 gradient with
// red.global.add.  Accumulates, never overwrites (see the 3x3 weight gradient).
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads, 3) dwconv5_wgrad_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  const int r = blockIdx.z;
  pdl_wait();
  float acc[40];                                  // acc[tap s * 8 + channel]
#pragma unroll
  for (int k = 0; k < 40; ++k) acc[k] = 0.f;
  const int total = a.N * a.P * a.Q;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int q = o % a.Q;
    const int t = o / a.Q;
    const int p = t % a.P;
    const int n = t / a.P;
    const int h = p * STRIDE - 2 + r;
    if (h < 0 || h >= a.H) continue;
    float d[8];
    dw_load8(a.dy + static_cast<size_t>(o) * a.C + m.c0, d);
    const __nv_bfloat16* row = a.x + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const int w = q * STRIDE - 2 + s;
      if (w < 0 || w >= a.W) continue;
      float v[8];
      dw_load8(row + static_cast<size_t>(w) * a.C, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[s * 8 + i] = fmaf(d[i], v[i], acc[s * 8 + i]);
    }
  }
  __shared__ float red[kDwWarps * 8 * 40];
  dw_block_reduce<40>(acc, a.lg_gpc, red, [&](int c, int s, float v) { atomicAdd(a.gw + c * kTaps + r * 5 + s, v); });
}

bool dw5_args_ok(const DwConvArgs& a) {
  if (a.C <= 0 || a.C % 8 != 0 || a.N <= 0 || a.H <= 0 || a.W <= 0) return false;
  if (a.stride != 1 && a.stride != 2) return false;
  return a.P == (a.H - 1) / a.stride + 1 && a.Q == (a.W - 1) / a.stride + 1;    // 5x5, padding 2
}

}  // namespace

cudaError_t launch_dwconv5_fwd(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw5_args_ok(a) || (a.sum == nullptr) != (a.sumsq == nullptr)) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  const dim3 grid = dw_grid(a.N * a.P * a.Q, a.C, a.lg_gpc, sms, 8);
  const bool stats = a.sum != nullptr;
  if (a.stride == 1)
    return stats ? launch_pdl(dwconv5_fwd_kernel<1, true>, grid, dim3(kDwThreads), 0, stream, 1, a)
                 : launch_pdl(dwconv5_fwd_kernel<1, false>, grid, dim3(kDwThreads), 0, stream, 1, a);
  return stats ? launch_pdl(dwconv5_fwd_kernel<2, true>, grid, dim3(kDwThreads), 0, stream, 1, a)
               : launch_pdl(dwconv5_fwd_kernel<2, false>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

cudaError_t launch_dwconv5_dgrad(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw5_args_ok(a)) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  const dim3 grid = dw_grid(a.N * a.H * a.W, a.C, a.lg_gpc, sms, 8);
  return a.stride == 1 ? launch_pdl(dwconv5_dgrad_kernel<1>, grid, dim3(kDwThreads), 0, stream, 1, a)
                       : launch_pdl(dwconv5_dgrad_kernel<2>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

cudaError_t launch_dwconv5_wgrad(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw5_args_ok(a) || a.gw == nullptr) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  // Atomic bound: every block issues 5 atomics (the taps of its filter row) per channel of its slab, and the (x, y)
  // grid holds at most 1 block per SM rounded up to whole slabs, gx <= ceil(SMs / slabs), times the 5 filter rows in z.
  // So a launch issues 25 * C * gx <= 25 * 64 * (SMs + slabs) atomics (about 0.24 M on 132 SMs for any layer) and each
  // gradient element receives gx of them, against 25 * N*P*Q*C multiply-adds.
  dim3 grid = dw_grid(a.N * a.P * a.Q, a.C, a.lg_gpc, sms, 1);
  grid.z = 5;
  return a.stride == 1 ? launch_pdl(dwconv5_wgrad_kernel<1>, grid, dim3(kDwThreads), 0, stream, 1, a)
                       : launch_pdl(dwconv5_wgrad_kernel<2>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

}  // namespace ddl
