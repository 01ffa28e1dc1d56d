// Depthwise 7x7 convolution with a bias (groups == Cin == Cout = C, C % 8 == 0; stride 1, padding 3, dilation 1) on NHWC
// bf16 activations with fp32 accumulation: forward (+ bias), data gradient (+ an optional same-shape addend) and weight
// gradient (+ the bias gradient).  The depthwise layer of every ConvNeXt block.  Same operand contracts as the 3x3 / 5x5
// kernels (depthwise.cu, depthwise5.cu): bf16 weights [C][49] (KRSC of [C, 1, 7, 7]) and an fp32 [C][49] gradient slot
// that the weight gradient accumulates into.
//
// - forward / data gradient: a 7x7 window reads every input pixel up to 49 times, so the block stages a halo tile in
//   shared memory: the (TH + 6) x (TW + 6) input pixels of its TH x TW output tile, for its 8 * gpc channels (gpc = 1, 2
//   or 4 groups of 8), and its [49][8 * gpc] weights as fp32.  Each thread then owns one output pixel x 8 channels and
//   reads its 49 taps from shared memory (one 16-byte load per tap, plus two 16-byte weight broadcasts).  With padding 3
//   and stride 1 the data gradient is the forward with the filter rotated by 180 degrees, so both share one kernel.
//   The launchers take `l1`: the 5x5 kernels' mapping instead (grid-stride pixels, taps read through L1), kept so that
//   tools/depthwise_bench.py can time the two against each other; the model path uses the halo tile.
// - weight gradient: 49 taps x 8 channels of accumulators would spill, so the grid's z dimension splits the filter rows
//   as in the 5x5 kernel: a block owns row r and accumulates 7 taps x 8 channels.  The centre row (r = 3) never falls
//   in the padding, so its blocks also sum dy for the bias gradient.
//
//   forward   y[n,p,q,c]  = b[c] + sum_{r,s} x[n, p-3+r, q-3+s, c] * w[c][r][s]
//   dgrad     dx[n,h,w,c] = add[n,h,w,c] + sum_{r,s} dy[n, h+3-r, w+3-s, c] * w[c][r][s]
//   wgrad     gw[c][r][s] += sum_{n,p,q} dy[n,p,q,c] * x[n, p-3+r, q-3+s, c];   gb[c] += sum_{n,p,q} dy[n,p,q,c]
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"
#include "depthwise.cuh"

namespace ddl {

namespace {

using namespace dw;

constexpr int kTaps7 = 49;
constexpr int kHaloMax = 14 * 14 * 4;      // (TH + 6) * (TW + 6) * gpc uint4 at most: 8x8 tile, 4 groups (8x16 x 2: 616,
                                           //   16x16 x 1: 484)

// output tile of a block: 256 threads = (pixels) x (gpc channel groups)
DDL_DEVICE int dw7_tile_w(int lg) { return lg == 2 ? 8 : 16; }
DDL_DEVICE int dw7_tile_h(int lg) { return lg == 0 ? 16 : 8; }

// the bf16 weights [C][49] of channels [slab0, slab0 + nch) as fp32 ws[tap][channel - slab0]; the data gradient takes
// tap 48 - tap (the filter rotated by 180 degrees).  Consecutive threads take consecutive channels of one tap, so the
// shared-memory stores of a warp fall in distinct banks.
template <bool DGRAD, int LD>
DDL_DEVICE void dw7_stage_weights(const __nv_bfloat16* w, int slab0, int nch, float (*ws)[LD]) {
  for (int e = threadIdx.x; e < nch * kTaps7; e += kDwThreads) {
    const int tap = e / nch, c = e - tap * nch;
    ws[DGRAD ? kTaps7 - 1 - tap : tap][c] = __bfloat162float(w[static_cast<size_t>(slab0 + c) * kTaps7 + tap]);
  }
}

// acc[i] += v[i] * wrow[i] (wrow: 8 fp32 weights in shared memory, 16-byte aligned)
DDL_DEVICE void dw7_fma_tap(float (&acc)[8], const float (&v)[8], const float* wrow) {
  const float4 w0 = reinterpret_cast<const float4*>(wrow)[0], w1 = reinterpret_cast<const float4*>(wrow)[1];
  acc[0] = fmaf(v[0], w0.x, acc[0]); acc[1] = fmaf(v[1], w0.y, acc[1]);
  acc[2] = fmaf(v[2], w0.z, acc[2]); acc[3] = fmaf(v[3], w0.w, acc[3]);
  acc[4] = fmaf(v[4], w1.x, acc[4]); acc[5] = fmaf(v[5], w1.y, acc[5]);
  acc[6] = fmaf(v[6], w1.z, acc[6]); acc[7] = fmaf(v[7], w1.w, acc[7]);
}

DDL_DEVICE uint4 dw7_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

template <bool DGRAD>
__global__ void __launch_bounds__(kDwThreads, 4) dwconv7_tile_kernel(Dw7Args a) {
  pdl_trigger();
  const int lg = a.lg_gpc;
  const int G = 1 << lg, nch = 8 << lg;
  const int TW = dw7_tile_w(lg), TH = dw7_tile_h(lg);
  const int HW_ = TW + 6, HH_ = TH + 6;
  const int tiles_w = (a.W + TW - 1) / TW, tiles_h = (a.H + TH - 1) / TH;
  int t = blockIdx.x;
  const int tw = t % tiles_w;
  t /= tiles_w;
  const int th = t % tiles_h;
  const int n = t / tiles_h;
  const int oh0 = th * TH, ow0 = tw * TW;
  const int slab0 = static_cast<int>(blockIdx.y) * nch;
  __shared__ __align__(16) uint4 halo[kHaloMax];
  __shared__ __align__(16) float ws[kTaps7][32];
  pdl_wait();
  const __nv_bfloat16* src = DGRAD ? a.dy : a.x;
  for (int e = threadIdx.x; e < HH_ * HW_ * G; e += kDwThreads) {
    const int g = e & (G - 1), pix = e >> lg;
    const int hy = pix / HW_, hx = pix - hy * HW_;
    const int h = oh0 - 3 + hy, w = ow0 - 3 + hx;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (h >= 0 && h < a.H && w >= 0 && w < a.W)
      v = __ldg(reinterpret_cast<const uint4*>(src + ((static_cast<size_t>(n) * a.H + h) * a.W + w) * a.C + slab0 + g * 8));
    halo[e] = v;
  }
  dw7_stage_weights<DGRAD>(a.w, slab0, nch, ws);
  __syncthreads();
  const int g = threadIdx.x & (G - 1), pix = threadIdx.x >> lg;
  const int ty = pix / TW, tx = pix - ty * TW;
  const int oh = oh0 + ty, ow = ow0 + tx;
  if (oh >= a.H || ow >= a.W) return;
  const int c0 = slab0 + g * 8;
  const size_t o = ((static_cast<size_t>(n) * a.H + oh) * a.W + ow) * a.C + c0;
  float acc[8];
  if (!DGRAD) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = __ldg(a.bias + c0 + i);      // fp32 parameter: no 16-byte alignment promised
  } else if (a.add != nullptr) {
    dw_load8(a.add + o, acc);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  }
#pragma unroll 1
  for (int r = 0; r < 7; ++r) {
    const uint4* hrow = halo + ((ty + r) * HW_ + tx) * G + g;
#pragma unroll
    for (int s = 0; s < 7; ++s) {
      float v[8];
      dw_unpack8(hrow[s * G], v);
      dw7_fma_tap(acc, v, &ws[r * 7 + s][g * 8]);
    }
  }
  *reinterpret_cast<uint4*>(a.y + o) = dw7_pack8(acc);
}

// ---- forward / data gradient, L1 mapping (the 5x5 kernels' mapping, for comparison with the halo tile) -------------
// A thread owns 8 channels of a fixed slab (up to 64 channels per block) and walks output pixels with a grid stride,
// reading its 49 taps from global memory through L1; only the weights are staged in shared memory.
template <bool DGRAD>
__global__ void __launch_bounds__(kDwThreads, 3) dwconv7_l1_kernel(Dw7Args a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  const int nch = 8 << a.lg_gpc, slab0 = static_cast<int>(blockIdx.y) * nch;
  __shared__ __align__(16) float ws[kTaps7][64];
  pdl_wait();
  dw7_stage_weights<DGRAD>(a.w, slab0, nch, ws);
  __syncthreads();
  const int cl = (threadIdx.x & ((1 << a.lg_gpc) - 1)) << 3;
  const __nv_bfloat16* src = DGRAD ? a.dy : a.x;
  const int total = a.N * a.H * a.W;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int q = o % a.W;
    const int t = o / a.W;
    const int p = t % a.H;
    const int n = t / a.H;
    const size_t off = static_cast<size_t>(o) * a.C + m.c0;
    float acc[8];
    if (!DGRAD) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = __ldg(a.bias + m.c0 + i);
    } else if (a.add != nullptr) {
      dw_load8(a.add + off, acc);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    }
#pragma unroll
    for (int r = 0; r < 7; ++r) {
      const int h = p - 3 + r;
      if (h < 0 || h >= a.H) continue;
      const __nv_bfloat16* row = src + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
      for (int s = 0; s < 7; ++s) {
        const int w = q - 3 + s;
        if (w < 0 || w >= a.W) continue;
        float v[8];
        dw_load8(row + static_cast<size_t>(w) * a.C, v);
        dw7_fma_tap(acc, v, &ws[r * 7 + s][cl]);
      }
    }
    *reinterpret_cast<uint4*>(a.y + off) = dw7_pack8(acc);
  }
}

// ---- weight gradient (+ bias gradient) ---------------------------------------------------------------------------
// Filter row r = blockIdx.z.  acc[s * 8 + i] for the 7 taps of row r, acc[56 + i] the bias sums (centre row only).
__global__ void __launch_bounds__(kDwThreads, 2) dwconv7_wgrad_kernel(Dw7Args a) {
  pdl_trigger();
  const DwMap m = dw_map(a.lg_gpc);
  const int r = blockIdx.z;
  pdl_wait();
  float acc[64];
#pragma unroll
  for (int k = 0; k < 64; ++k) acc[k] = 0.f;
  const int total = a.N * a.H * a.W;
  for (int o = m.lane; o < total; o += m.lanes) {
    const int q = o % a.W;
    const int t = o / a.W;
    const int p = t % a.H;
    const int n = t / a.H;
    const int h = p - 3 + r;
    if (h < 0 || h >= a.H) continue;
    float d[8];
    dw_load8(a.dy + static_cast<size_t>(o) * a.C + m.c0, d);
    if (r == 3) {
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[56 + i] += d[i];
    }
    const __nv_bfloat16* row = a.x + (static_cast<size_t>(n) * a.H + h) * a.W * a.C + m.c0;
#pragma unroll
    for (int s = 0; s < 7; ++s) {
      const int w = q - 3 + s;
      if (w < 0 || w >= a.W) continue;
      float v[8];
      dw_load8(row + static_cast<size_t>(w) * a.C, v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[s * 8 + i] = fmaf(d[i], v[i], acc[s * 8 + i]);
    }
  }
  __shared__ float red[kDwWarps * 8 * 64];
  dw_block_reduce<64>(acc, a.lg_gpc, red, [&](int c, int s, float v) {
    if (s < 7) atomicAdd(a.gw + c * kTaps7 + r * 7 + s, v);
    else if (r == 3 && a.gb != nullptr) atomicAdd(a.gb + c, v);
  });
}

bool dw7_args_ok(const Dw7Args& a) {
  return a.C > 0 && a.C % 8 == 0 && a.N > 0 && a.H > 0 && a.W > 0;
}

dim3 dw7_tile_grid(const Dw7Args& a) {
  const int TW = a.lg_gpc == 2 ? 8 : 16, TH = a.lg_gpc == 0 ? 16 : 8;
  const long long tiles = static_cast<long long>(a.N) * ((a.H + TH - 1) / TH) * ((a.W + TW - 1) / TW);
  return dim3(static_cast<unsigned>(tiles), static_cast<unsigned>((a.C / 8) >> a.lg_gpc));
}

template <bool DGRAD>
cudaError_t launch_dwconv7_window(Dw7Args a, int sms, bool l1, cudaStream_t stream) {
  if (l1) {
    a.lg_gpc = dw_lg_gpc(a.C);
    return launch_pdl(dwconv7_l1_kernel<DGRAD>, dw_grid(a.N * a.H * a.W, a.C, a.lg_gpc, sms, 8), dim3(kDwThreads), 0,
                      stream, 1, a);
  }
  a.lg_gpc = dw_lg_gpc(a.C) < 2 ? dw_lg_gpc(a.C) : 2;
  return launch_pdl(dwconv7_tile_kernel<DGRAD>, dw7_tile_grid(a), dim3(kDwThreads), 0, stream, 1, a);
}

}  // namespace

cudaError_t launch_dwconv7_fwd(const Dw7Args& a, int sms, bool l1, cudaStream_t stream) {
  if (!dw7_args_ok(a) || a.bias == nullptr) return cudaErrorInvalidValue;
  return launch_dwconv7_window<false>(a, sms, l1, stream);
}

cudaError_t launch_dwconv7_dgrad(const Dw7Args& a, int sms, bool l1, cudaStream_t stream) {
  if (!dw7_args_ok(a)) return cudaErrorInvalidValue;
  return launch_dwconv7_window<true>(a, sms, l1, stream);
}

cudaError_t launch_dwconv7_wgrad(const Dw7Args& a_in, int sms, cudaStream_t stream) {
  Dw7Args a = a_in;
  if (!dw7_args_ok(a) || a.gw == nullptr) return cudaErrorInvalidValue;
  a.lg_gpc = dw_lg_gpc(a.C);
  // as in the 5x5 weight gradient: at most ~1 block per SM in (x, y), times the 7 filter rows in z; each block issues
  // 7 atomics per channel of its slab (the centre row 8)
  dim3 grid = dw_grid(a.N * a.H * a.W, a.C, a.lg_gpc, sms, 1);
  grid.z = 7;
  return launch_pdl(dwconv7_wgrad_kernel, grid, dim3(kDwThreads), 0, stream, 1, a);
}

}  // namespace ddl
