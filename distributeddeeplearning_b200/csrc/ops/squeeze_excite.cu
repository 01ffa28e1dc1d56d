// Squeeze-excitation (MobileNetV3): y = x * hardsigmoid(s[n, c]) with s = fc2(relu(fc1(mean_hw(x)))) — the scale pass of
// the forward and the two passes of the backward.  The pooling and the two FCs run on global_avgpool_fwd and the GEMM
// kernels; s is their bf16 output [N][lds] (lds: the GEMM's padded width).  NHWC bf16 activations, x [N][HW][C],
// C % 8 == 0; a thread handles one 16-byte vector of 8 channels.
//
//   scale    y[n,p,c]  = x[n,p,c] * hsig(s[n,c])                         hsig(v) = clamp(v + 3, 0, 6) / 6
//   reduce   ds[n,c]   = hsig'(s[n,c]) * sum_p dy[n,p,c] * x[n,p,c]      hsig'(v) = 1/6 for -3 < v < 3, else 0
//   apply    dx[n,p,c] = dy[n,p,c] * hsig(s[n,c]) + dpooled[n,c] / HW   (the scale path's and the pooling path's
//                                                                          gradients of x, in one pass)
// The reduce is deterministic: one block per (sample, 64-channel chunk) sums its HW pixels in a fixed order (no atomics).
#include "../common.cuh"
#include "ops.h"

namespace ddl {

namespace {

constexpr int kSeThreads = 256;

DDL_DEVICE void se_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 se_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
DDL_DEVICE float hardsigmoid(float v) { return fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f); }

// the 8 gates hsig(s[n, c0 .. c0 + 8))
DDL_DEVICE void se_gates(const __nv_bfloat16* s, int lds, int n, int c0, float (&g)[8]) {
  se_unpack8(__ldg(reinterpret_cast<const uint4*>(s + static_cast<size_t>(n) * lds + c0)), g);
#pragma unroll
  for (int i = 0; i < 8; ++i) g[i] = hardsigmoid(g[i]);
}

__global__ void __launch_bounds__(kSeThreads) se_scale_kernel(const __nv_bfloat16* __restrict__ x,
                                                              const __nv_bfloat16* __restrict__ s, int lds,
                                                              __nv_bfloat16* __restrict__ y, int HW, int C, int64_t total) {
  const int groups = C / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const int n = static_cast<int>(i / groups / HW);
    float gate[8], v[8];
    se_gates(s, lds, n, g * 8, gate);
    se_unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] *= gate[k];
    reinterpret_cast<uint4*>(y)[i] = se_pack8(v);
  }
}

// block = (64-channel chunk blockIdx.x, sample blockIdx.y); thread = 8 channels (threadIdx.x & 7) x pixel lane
// (threadIdx.x >> 3, 32 lanes).  Channels [C, ldd) of the last chunk are written as zeros (the GEMM operand's padding).
__global__ void __launch_bounds__(kSeThreads) se_reduce_kernel(const __nv_bfloat16* __restrict__ dy,
                                                               const __nv_bfloat16* __restrict__ x,
                                                               const __nv_bfloat16* __restrict__ s, int lds,
                                                               __nv_bfloat16* __restrict__ ds, int ldd, int HW, int C) {
  const int cgl = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int n = blockIdx.y;
  const int c0 = blockIdx.x * 64 + cgl * 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (c0 < C) {
    const size_t base = static_cast<size_t>(n) * HW * C + c0;
    for (int p = rl; p < HW; p += 32) {
      float d[8], v[8];
      se_unpack8(__ldg(reinterpret_cast<const uint4*>(dy + base + static_cast<size_t>(p) * C)), d);
      se_unpack8(__ldg(reinterpret_cast<const uint4*>(x + base + static_cast<size_t>(p) * C)), v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(d[i], v[i], acc[i]);
    }
  }
  // lanes of a warp sharing a channel group: lane = (rl % 4) * 8 + cgl -> xor 8, 16
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
  }
  __shared__ float red[kSeThreads / 32][8][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) red[warp][lane][i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    const int c = blockIdx.x * 64 + g * 8 + i;
    float out = 0.f;
    if (c < C) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kSeThreads / 32; ++w) t += red[w][g][i];
      const float sv = __bfloat162float(s[static_cast<size_t>(n) * lds + c]);
      out = (sv > -3.f && sv < 3.f) ? t * (1.f / 6.f) : 0.f;
    }
    if (c < ldd) ds[static_cast<size_t>(n) * ldd + c] = __float2bfloat16_rn(out);
  }
}

__global__ void __launch_bounds__(kSeThreads) se_apply_kernel(const __nv_bfloat16* __restrict__ dy,
                                                              const __nv_bfloat16* __restrict__ s, int lds,
                                                              const __nv_bfloat16* __restrict__ dpooled,
                                                              __nv_bfloat16* __restrict__ dx, int HW, int C,
                                                              int64_t total) {
  const int groups = C / 8;
  const float inv_hw = 1.f / static_cast<float>(HW);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const int n = static_cast<int>(i / groups / HW);
    float gate[8], d[8], dp[8];
    se_gates(s, lds, n, g * 8, gate);
    se_unpack8(__ldg(reinterpret_cast<const uint4*>(dpooled + static_cast<size_t>(n) * C + g * 8)), dp);
    se_unpack8(reinterpret_cast<const uint4*>(dy)[i], d);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = fmaf(d[k], gate[k], dp[k] * inv_hw);
    reinterpret_cast<uint4*>(dx)[i] = se_pack8(d);
  }
}

// 16 blocks of 256 threads per SM at most (grid-stride beyond that)
inline int se_grid(int64_t vecs, int sms) {
  int64_t b = (vecs + kSeThreads - 1) / kSeThreads;
  const int64_t cap = static_cast<int64_t>(sms) * 16;
  if (b > cap) b = cap;
  return static_cast<int>(b < 1 ? 1 : b);
}

bool se_args_ok(int N, int HW, int C, int lds) {
  return N > 0 && HW > 0 && C > 0 && C % 8 == 0 && lds >= C && lds % 8 == 0;
}

}  // namespace

cudaError_t launch_se_scale(const __nv_bfloat16* x, const __nv_bfloat16* s, int lds, __nv_bfloat16* y, int N, int HW,
                            int C, int sms, cudaStream_t stream) {
  if (!se_args_ok(N, HW, C, lds)) return cudaErrorInvalidValue;
  const int64_t vecs = static_cast<int64_t>(N) * HW * (C / 8);
  se_scale_kernel<<<se_grid(vecs, sms), kSeThreads, 0, stream>>>(x, s, lds, y, HW, C, vecs);
  return cudaGetLastError();
}

cudaError_t launch_se_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* s, int lds,
                             __nv_bfloat16* ds, int ldd, int N, int HW, int C, cudaStream_t stream) {
  const int chunks = (C + 63) / 64;
  if (!se_args_ok(N, HW, C, lds) || ldd < C || ldd > chunks * 64) return cudaErrorInvalidValue;
  se_reduce_kernel<<<dim3(chunks, N), kSeThreads, 0, stream>>>(dy, x, s, lds, ds, ldd, HW, C);
  return cudaGetLastError();
}

cudaError_t launch_se_apply(const __nv_bfloat16* dy, const __nv_bfloat16* s, int lds, const __nv_bfloat16* dpooled,
                            __nv_bfloat16* dx, int N, int HW, int C, int sms, cudaStream_t stream) {
  if (!se_args_ok(N, HW, C, lds)) return cudaErrorInvalidValue;
  const int64_t vecs = static_cast<int64_t>(N) * HW * (C / 8);
  se_apply_kernel<<<se_grid(vecs, sms), kSeThreads, 0, stream>>>(dy, s, lds, dpooled, dx, HW, C, vecs);
  return cudaGetLastError();
}

}  // namespace ddl
