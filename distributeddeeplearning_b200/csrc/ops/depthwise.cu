// Depthwise 3x3 convolution (groups == Cin == Cout = C, C % 8 == 0; stride 1 or 2, padding 1, dilation 1) on NHWC
// bf16 activations with fp32 accumulation: forward (+ per-channel BN statistics of the bf16 output), data gradient and
// weight gradient.  MobileNetV2's 17 depthwise layers.
//
// A depthwise 3x3 is 9 multiply-adds per output element: a stencil bound by HBM bandwidth, not a GEMM (the block-
// diagonal mode of the conv kernels would do 64x the useful MMA work at one channel per group).
//
// Thread mapping (all three kernels; depthwise.cuh): a thread owns 8 consecutive channels of a fixed channel slab and
// walks output (dgrad: input) pixels with a grid stride, so its 72 filter taps stay in registers.  The 3x3 windows of
// the neighbouring pixels of a warp overlap and the rows above and below were read moments earlier, so the taps are
// plain L1-cached 16-byte loads: HBM sees each input about once.
//
//   forward   y[n,p,q,c]  = sum_{r,s} x[n, p*st-1+r, q*st-1+s, c] * w[c][r][s]
//   dgrad     dx[n,h,w,c] = sum of dy[n,p,q,c] * w[c][r][s] over the taps with h = p*st-1+r, w = q*st-1+s (gather:
//             for stride 2 only the taps whose parity matches; every dx element is written once, no atomics)
//   wgrad     gw[c][r][s] += sum_{n,p,q} dy[n,p,q,c] * x[n, p*st-1+r, q*st-1+s, c]
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"
#include "depthwise.cuh"

namespace ddl {

namespace {

using namespace dw;

// the 9 taps of channels [c0, c0 + 8) of the bf16 [C][9] weights (72 contiguous elements) as wt[tap][channel]
DDL_DEVICE void dw_load_weights(const __nv_bfloat16* w, int c0, float (&wt)[9][8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
#pragma unroll
    for (int t = 0; t < 9; ++t) wt[t][i] = __bfloat162float(w[(c0 + i) * 9 + t]);
  }
}

// ---- forward ---------------------------------------------------------------------------------------------------
template <int STRIDE, bool STATS>
__global__ void __launch_bounds__(kDwThreads, 2) dwconv_fwd_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  pdl_wait();
  float wt[9][8];
  dw_load_weights(a.w, m.c0, wt);
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
    for (int r = 0; r < 3; ++r) {
      const int h = p * STRIDE - 1 + r;
      if (h < 0 || h >= a.H) continue;
      const __nv_bfloat16* row = a.x + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int w = q * STRIDE - 1 + s;
        if (w < 0 || w >= a.W) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(w) * a.C, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(v[i], wt[r * 3 + s][i], acc[i]);
      }
    }
    const uint4 out = make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                                 pack_bf16x2(acc[6], acc[7]));
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
__global__ void __launch_bounds__(kDwThreads, 2) dwconv_dgrad_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  pdl_wait();
  float wt[9][8];
  dw_load_weights(a.w, m.c0, wt);
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
    for (int r = 0; r < 3; ++r) {
      const int ph = h + 1 - r;                   // = p * STRIDE
      if (ph < 0 || (STRIDE == 2 && (ph & 1))) continue;
      const int p = ph / STRIDE;
      if (p >= a.P) continue;
      const __nv_bfloat16* row = a.dy + (static_cast<size_t>(n) * a.P + p) * a.Q * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int qw = w + 1 - s;
        if (qw < 0 || (STRIDE == 2 && (qw & 1))) continue;
        const int q = qw / STRIDE;
        if (q >= a.Q) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(q) * a.C, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(v[i], wt[r * 3 + s][i], acc[i]);
      }
    }
    *reinterpret_cast<uint4*>(a.y + static_cast<size_t>(o) * a.C + m.c0) =
        make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                   pack_bf16x2(acc[6], acc[7]));
  }
}

// ---- weight gradient -------------------------------------------------------------------------------------------
// Each thread sums its pixels' 72 products in registers, the block folds them over its pixel lanes (shuffles, then
// shared memory) and adds one total per (channel, tap) into the fp32 gradient with red.global.add.  Accumulates, never
// overwrites: the slot is the parameter's gradient (the fused engine's bucket arena), which may hold earlier passes.
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads, 2) dwconv_wgrad_kernel(DwConvArgs a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  pdl_wait();
  float acc[72];                                  // acc[tap * 8 + channel]
#pragma unroll
  for (int k = 0; k < 72; ++k) acc[k] = 0.f;
  const int total = a.N * a.P * a.Q;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int q = o % a.Q;
    const int t = o / a.Q;
    const int p = t % a.P;
    const int n = t / a.P;
    float d[8];
    dw_load8(a.dy + static_cast<size_t>(o) * a.C + m.c0, d);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = p * STRIDE - 1 + r;
      if (h < 0 || h >= a.H) continue;
      const __nv_bfloat16* row = a.x + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int w = q * STRIDE - 1 + s;
        if (w < 0 || w >= a.W) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(w) * a.C, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[(r * 3 + s) * 8 + i] = fmaf(d[i], v[i], acc[(r * 3 + s) * 8 + i]);
      }
    }
  }
  __shared__ float red[kDwWarps * 8 * 72];
  dw_block_reduce<72>(acc, a.lg_gpc, red, [&](int c, int tap, float v) { atomicAdd(a.gw + c * 9 + tap, v); });
}

bool dw_args_ok(const DwConvArgs& a) {
  if (a.C <= 0 || a.C % 8 != 0 || a.N <= 0 || a.H <= 0 || a.W <= 0) return false;
  if (a.stride != 1 && a.stride != 2) return false;
  return a.P == (a.H - 1) / a.stride + 1 && a.Q == (a.W - 1) / a.stride + 1;    // 3x3, padding 1
}

}  // namespace

cudaError_t launch_dwconv_fwd(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw_args_ok(a) || (a.sum == nullptr) != (a.sumsq == nullptr)) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  const dim3 grid = dw_grid(a.N * a.P * a.Q, a.C, a.lg_gpc, sms, 8);
  const bool stats = a.sum != nullptr;
  if (a.stride == 1)
    return stats ? launch_pdl(dwconv_fwd_kernel<1, true>, grid, dim3(kDwThreads), 0, stream, 1, a)
                 : launch_pdl(dwconv_fwd_kernel<1, false>, grid, dim3(kDwThreads), 0, stream, 1, a);
  return stats ? launch_pdl(dwconv_fwd_kernel<2, true>, grid, dim3(kDwThreads), 0, stream, 1, a)
               : launch_pdl(dwconv_fwd_kernel<2, false>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

cudaError_t launch_dwconv_dgrad(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw_args_ok(a)) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  const dim3 grid = dw_grid(a.N * a.H * a.W, a.C, a.lg_gpc, sms, 8);
  return a.stride == 1 ? launch_pdl(dwconv_dgrad_kernel<1>, grid, dim3(kDwThreads), 0, stream, 1, a)
                       : launch_pdl(dwconv_dgrad_kernel<2>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

cudaError_t launch_dwconv_wgrad(const DwConvArgs& a_in, int sms, cudaStream_t stream) {
  DwConvArgs a = a_in;
  if (!dw_args_ok(a) || a.gw == nullptr) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  // Atomic bound: every block issues 9 atomics per channel of its slab (8 << lg_gpc channels), and the grid holds at
  // most 2 blocks per SM rounded up to whole slabs, i.e. gx <= ceil(2 * SMs / slabs).  So a launch issues
  // 9 * C * gx <= 9 * 64 * (2 * SMs + slabs) atomics (about 0.16 M on 132 SMs for any layer) and each gradient
  // element receives gx of them, against 9 * N*P*Q*C multiply-adds.
  const dim3 grid = dw_grid(a.N * a.P * a.Q, a.C, a.lg_gpc, sms, 2);
  return a.stride == 1 ? launch_pdl(dwconv_wgrad_kernel<1>, grid, dim3(kDwThreads), 0, stream, 1, a)
                       : launch_pdl(dwconv_wgrad_kernel<2>, grid, dim3(kDwThreads), 0, stream, 1, a);
}

}  // namespace ddl
