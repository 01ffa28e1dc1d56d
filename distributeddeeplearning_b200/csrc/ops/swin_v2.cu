// Swin Transformer V2 per-block kernels: the continuous position bias (CPB) MLP and the 2x2 gather of PatchMergingV2.
//
// CPB: T[k][h] = 16 sigmoid(sum_m W2[h][m] relu(W1[m] . c_k + b1[m])) for the 225 relative coordinates c_k [225][2] (the
// stored relative_coords_table), hidden width 512, fp32 throughout.  The forward is one launch per block: CTA k < 225
// builds row k (the 512 hidden units in shared memory, then one warp per head sums its 512 products lane-strided and
// reduces them over the warp in a fixed order); CTA 225 writes the block's effective qkv bias [b_q, 0, b_v]
// (torchvision clones qkv.bias and zeroes its k-slice in every forward).  The backward is two launches: CTA (b, c) forms
// dZ = dT o T (1 - T / 16) of the 15 coordinates of row c of the 15 x 15 grid in shared memory, then its thread m (a
// hidden unit of block b) walks those k in order, recomputing relu(W1[m] . c_k + b1[m]) and accumulating dW2[.][m]
// (heads registers), dW1[m] and db1[m] into partials [15][heads * 512 + 1536]; a second kernel adds the 15 partials of
// every element in order.  Every gradient element is a fixed-order sum: no atomics, bit-identical run to run.
//
// Merge gather: y [N * H/2 * W/2][4C] = (x0, x1, x2, x3) = x[2i, 2j], x[2i+1, 2j], x[2i, 2j+1], x[2i+1, 2j+1] of the NHWC
// x [N][H][W][C] (H, W even, C % 8 == 0) in 16-byte vectors; the backward is the inverse permutation (dx from dy).
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kTab = 225;
constexpr int kHidden = 512;
constexpr int kMaxHeads = 32;
constexpr int kThreads = 128;
constexpr int kBwdThreads = 64;
constexpr int kSide = 15;                           // the 15 x 15 grid: 225 = kSide chunks of kSide coordinates

__global__ void __launch_bounds__(kThreads) cpb_fwd_kernel(const float* __restrict__ coords,
                                                           const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ w2, float* __restrict__ table,
                                                           const float* __restrict__ qkv_b, float* __restrict__ qkv_b_eff,
                                                           int heads, int C) {
  __shared__ float hid[kHidden];
  pdl_trigger();
  pdl_wait();
  const int k = blockIdx.x, tid = threadIdx.x;
  if (k == kTab) {
    if (qkv_b_eff == nullptr) return;
    for (int c = tid; c < 3 * C; c += kThreads) qkv_b_eff[c] = (c >= C && c < 2 * C) ? 0.f : qkv_b[c];
    return;
  }
  const float cy = coords[2 * k], cx = coords[2 * k + 1];
  for (int m = tid; m < kHidden; m += kThreads) hid[m] = fmaxf(fmaf(w1[2 * m], cy, fmaf(w1[2 * m + 1], cx, b1[m])), 0.f);
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  for (int h = warp; h < heads; h += kThreads / 32) {
    const float* w = w2 + static_cast<size_t>(h) * kHidden;
    float s = 0.f;
#pragma unroll 4
    for (int m = lane; m < kHidden; m += 32) s = fmaf(w[m], hid[m], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) table[k * heads + h] = 16.f / (1.f + expf(-s));
  }
}

__global__ void __launch_bounds__(kBwdThreads) cpb_bwd_kernel(const float* __restrict__ coords,
                                                              const float* __restrict__ w1, const float* __restrict__ b1,
                                                              const float* __restrict__ w2,
                                                              const float* __restrict__ table,
                                                              const float* __restrict__ dtable,
                                                              float* __restrict__ part, int heads) {
  __shared__ float dz[kSide * kMaxHeads];
  __shared__ float cs[2 * kSide];
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x, m = blockIdx.x * kBwdThreads + tid, k0 = blockIdx.y * kSide;
  for (int e = tid; e < kSide * heads; e += kBwdThreads) {
    const float t = table[k0 * heads + e];
    dz[e] = dtable[k0 * heads + e] * t * (1.f - t * (1.f / 16.f));
  }
  for (int e = tid; e < 2 * kSide; e += kBwdThreads) cs[e] = coords[2 * k0 + e];
  __syncthreads();
  const float wy = w1[2 * m], wx = w1[2 * m + 1], bm = b1[m];
  float w[kMaxHeads], acc[kMaxHeads];
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h) {
    w[h] = h < heads ? w2[static_cast<size_t>(h) * kHidden + m] : 0.f;
    acc[h] = 0.f;
  }
  float gy = 0.f, gx = 0.f, gb = 0.f;
  for (int k = 0; k < kSide; ++k) {
    const float cy = cs[2 * k], cx = cs[2 * k + 1];
    const float pre = fmaf(wy, cy, fmaf(wx, cx, bm));
    const float a = fmaxf(pre, 0.f);
    const float* d = dz + k * heads;
    float dh = 0.f;
#pragma unroll
    for (int h = 0; h < kMaxHeads; ++h) {
      if (h < heads) {
        acc[h] = fmaf(d[h], a, acc[h]);
        dh = fmaf(d[h], w[h], dh);
      }
    }
    if (pre > 0.f) {
      gy = fmaf(dh, cy, gy);
      gx = fmaf(dh, cx, gx);
      gb += dh;
    }
  }
  float* p = part + static_cast<size_t>(blockIdx.y) * (heads * kHidden + 3 * kHidden);
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h)
    if (h < heads) p[h * kHidden + m] = acc[h];
  p += heads * kHidden;
  p[2 * m] = gy;
  p[2 * m + 1] = gx;
  p[2 * kHidden + m] = gb;
}

// dW2 [heads][512], dW1 [512][2], db1 [512] += the kSide partials of each element, in order (each output optional)
__global__ void __launch_bounds__(kThreads) cpb_bwd_reduce_kernel(const float* __restrict__ part, float* dw1,
                                                                  float* db1, float* dw2, int heads) {
  pdl_trigger();
  pdl_wait();
  const int per = heads * kHidden + 3 * kHidden;
  const int e = blockIdx.x * kThreads + threadIdx.x;
  if (e >= per) return;
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < kSide; ++c) s += part[static_cast<size_t>(c) * per + e];
  const int w2n = heads * kHidden;
  if (e < w2n) {
    if (dw2 != nullptr) dw2[e] += s;
  } else if (e < w2n + 2 * kHidden) {
    if (dw1 != nullptr) dw1[e - w2n] += s;
  } else if (db1 != nullptr) {
    db1[e - w2n - 2 * kHidden] += s;
  }
}

// forward: y row (n, i, j) vector v of 4C/8 <- x[n][2i + (q & 1)][2j + (q >> 1)][c], q = v / (C/8); backward: the inverse
template <bool kFwd>
__global__ void __launch_bounds__(256) merge_gather_kernel(const __nv_bfloat16* __restrict__ src,
                                                            __nv_bfloat16* __restrict__ dst, int N, int H, int W,
                                                            int C) {
  pdl_trigger();
  pdl_wait();
  const int cv = C / 8, Ho = H / 2, Wo = W / 2;
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo * 4 * cv;
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < total;
       e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(e % (4 * cv));
    const int64_t row = e / (4 * cv);
    const int j = static_cast<int>(row % Wo), i = static_cast<int>((row / Wo) % Ho);
    const int64_t n = row / (static_cast<int64_t>(Wo) * Ho);
    const int q = v / cv, c = v - q * cv;
    const int64_t xi = ((n * H + 2 * i + (q & 1)) * W + 2 * j + (q >> 1)) * cv + c;
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    if (kFwd) d[e] = s[xi];
    else d[xi] = s[e];
  }
}

}  // namespace

cudaError_t launch_cpb_fwd(const float* coords, const float* w1, const float* b1, const float* w2, float* table,
                           const float* qkv_b, float* qkv_b_eff, int heads, int C, cudaStream_t stream) {
  if (heads <= 0 || heads > kMaxHeads || (qkv_b_eff != nullptr && (qkv_b == nullptr || C <= 0)))
    return cudaErrorInvalidValue;
  return launch_pdl(cpb_fwd_kernel, dim3(kTab + 1), dim3(kThreads), 0, stream, 1, coords, w1, b1, w2, table, qkv_b,
                    qkv_b_eff, heads, C);
}

size_t cpb_bwd_scratch_floats(int heads) { return static_cast<size_t>(kSide) * (heads * kHidden + 3 * kHidden); }

cudaError_t launch_cpb_bwd(const float* coords, const float* w1, const float* b1, const float* w2, const float* table,
                           const float* dtable, float* dw1, float* db1, float* dw2, float* scratch, int heads,
                           cudaStream_t stream) {
  if (heads <= 0 || heads > kMaxHeads) return cudaErrorInvalidValue;
  cudaError_t e = launch_pdl(cpb_bwd_kernel, dim3(kHidden / kBwdThreads, kSide), dim3(kBwdThreads), 0, stream, 1,
                             coords, w1, b1, w2, table, dtable, scratch, heads);
  if (e != cudaSuccess) return e;
  const int per = heads * kHidden + 3 * kHidden;
  return launch_pdl(cpb_bwd_reduce_kernel, dim3((per + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(scratch), dw1, db1, dw2, heads);
}

cudaError_t launch_merge_gather(const __nv_bfloat16* src, __nv_bfloat16* dst, int N, int H, int W, int C, bool forward,
                                int sms, cudaStream_t stream) {
  if (N <= 0 || H <= 0 || W <= 0 || H % 2 != 0 || W % 2 != 0 || C <= 0 || C % 8 != 0) return cudaErrorInvalidValue;
  const int64_t total = static_cast<int64_t>(N) * (H / 2) * (W / 2) * (C / 2);
  const int64_t want = (total + 255) / 256;
  const int blocks = static_cast<int>(want < 8LL * sms ? (want > 0 ? want : 1) : 8LL * sms);
  if (forward) return launch_pdl(merge_gather_kernel<true>, dim3(blocks), dim3(256), 0, stream, 1, src, dst, N, H, W, C);
  return launch_pdl(merge_gather_kernel<false>, dim3(blocks), dim3(256), 0, stream, 1, src, dst, N, H, W, C);
}

}  // namespace ddl
