// Squeeze-excitation with a sigmoid gate (EfficientNet): y = x * sigmoid(s[n, c]) with s = fc2(silu(fc1(mean_hw(x)))).
// The same three passes as squeeze_excite.cu (MobileNetV3's hardsigmoid gate), kept in their own kernels so that those
// keep their code: NHWC bf16 activations, x [N][HW][C], C % 8 == 0; s the bf16 gate logits [N][lds].
//
//   scale    y[n,p,c]  = x[n,p,c] * g[n,c]                                   g = sigmoid(s)
//   reduce   ds[n,c]   = g (1 - g) * sum_p dy[n,p,c] * x[n,p,c]              (deterministic: one block per
//                                                                             (64-channel chunk, sample), no atomics)
//   apply    dx[n,p,c] = dy[n,p,c] * g[n,c] + dpooled[n,c] / HW
//
// EfficientNet's squeeze widths C' = C_in / 4 (4, 6, 10, 12, 14, ...) are not multiples of 8, so fc2's K = C' cannot be
// a TMA operand (row pitch not a multiple of 16 bytes).  The squeeze dimension is padded to C'8 = C' rounded up to 8 with
// zero columns: pad_cols builds the padded bf16 fc2 weight [C][C'8] each forward (graph capture records it), and
// fold_cols adds the padded fp32 weight gradient [C][C'8] into the compact slot [C][C'].
// Both take a batch of up to kPadMax matrices per launch, each padded in rows and columns: ShuffleNetV2's units pad
// every operand of a unit whose widths are not multiples of 8 (bf16 weights, fp32 BN parameters and running
// statistics) in one launch, and fold the padded gradients (or copy the running statistics) back in one more.
#include "../common.cuh"
#include "ops.h"

#include <algorithm>

namespace ddl {

namespace {

constexpr int kSgThreads = 256;

DDL_DEVICE void sg_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 sg_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
DDL_DEVICE float gate_sigmoid(float v) { return 1.f / (1.f + __expf(-v)); }

// the 8 gates sigmoid(s[n, c0 .. c0 + 8))
DDL_DEVICE void sg_gates(const __nv_bfloat16* s, int lds, int n, int c0, float (&g)[8]) {
  sg_unpack8(__ldg(reinterpret_cast<const uint4*>(s + static_cast<size_t>(n) * lds + c0)), g);
#pragma unroll
  for (int i = 0; i < 8; ++i) g[i] = gate_sigmoid(g[i]);
}

__global__ void __launch_bounds__(kSgThreads) sesig_scale_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 const __nv_bfloat16* __restrict__ s, int lds,
                                                                 __nv_bfloat16* __restrict__ y, int HW, int C,
                                                                 int64_t total) {
  const int groups = C / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % groups);
    const int n = static_cast<int>(i / groups / HW);
    float gate[8], v[8];
    sg_gates(s, lds, n, g * 8, gate);
    sg_unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] *= gate[k];
    reinterpret_cast<uint4*>(y)[i] = sg_pack8(v);
  }
}

// block = (64-channel chunk blockIdx.x, sample blockIdx.y); thread = 8 channels (threadIdx.x & 7) x pixel lane
// (threadIdx.x >> 3, 32 lanes).  Channels [C, ldd) of the last chunk are written as zeros (the GEMM operand's padding).
__global__ void __launch_bounds__(kSgThreads) sesig_reduce_kernel(const __nv_bfloat16* __restrict__ dy,
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
      sg_unpack8(__ldg(reinterpret_cast<const uint4*>(dy + base + static_cast<size_t>(p) * C)), d);
      sg_unpack8(__ldg(reinterpret_cast<const uint4*>(x + base + static_cast<size_t>(p) * C)), v);
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
  __shared__ float red[kSgThreads / 32][8][8];
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
      for (int w = 0; w < kSgThreads / 32; ++w) t += red[w][g][i];
      const float gv = gate_sigmoid(__bfloat162float(s[static_cast<size_t>(n) * lds + c]));
      out = t * gv * (1.f - gv);
    }
    if (c < ldd) ds[static_cast<size_t>(n) * ldd + c] = __float2bfloat16_rn(out);
  }
}

__global__ void __launch_bounds__(kSgThreads) sesig_apply_kernel(const __nv_bfloat16* __restrict__ dy,
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
    sg_gates(s, lds, n, g * 8, gate);
    sg_unpack8(__ldg(reinterpret_cast<const uint4*>(dpooled + static_cast<size_t>(n) * C + g * 8)), dp);
    sg_unpack8(reinterpret_cast<const uint4*>(dy)[i], d);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = fmaf(d[k], gate[k], dp[k] * inv_hw);
    reinterpret_cast<uint4*>(dx)[i] = sg_pack8(d);
  }
}

// blockIdx.y = matrix: dst [prows][kp] = src [rows][k] in its top-left corner, zeros elsewhere (2- or 4-byte elements)
__global__ void __launch_bounds__(kSgThreads) pad_cols_kernel(PadBatch b) {
  const PadMatrix& m = b.m[blockIdx.y];
  const int64_t total = static_cast<int64_t>(m.prows) * m.kp;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / m.kp), c = static_cast<int>(i % m.kp);
    const bool in = r < m.rows && c < m.k;
    const int64_t s = static_cast<int64_t>(r) * m.k + c;
    if (m.esize == 4)
      static_cast<uint32_t*>(m.dst)[i] = in ? static_cast<const uint32_t*>(m.src)[s] : 0u;
    else
      static_cast<uint16_t*>(m.dst)[i] = in ? static_cast<const uint16_t*>(m.src)[s] : static_cast<uint16_t>(0);
  }
}

// blockIdx.y = matrix: fp32 dst [rows][k] (+)= src [>= rows][kp] columns [0, k)
__global__ void __launch_bounds__(kSgThreads) fold_cols_kernel(FoldBatch b) {
  const FoldMatrix& m = b.m[blockIdx.y];
  const int64_t total = static_cast<int64_t>(m.rows) * m.k;
  const float* src = static_cast<const float*>(m.src);
  float* dst = static_cast<float*>(m.dst);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float v = src[(i / m.k) * m.kp + i % m.k];
    dst[i] = m.add ? dst[i] + v : v;
  }
}

// 16 blocks of 256 threads per SM at most (grid-stride beyond that)
inline int sg_grid(int64_t work, int sms) {
  int64_t b = (work + kSgThreads - 1) / kSgThreads;
  const int64_t cap = static_cast<int64_t>(sms) * 16;
  if (b > cap) b = cap;
  return static_cast<int>(b < 1 ? 1 : b);
}

bool sg_args_ok(int N, int HW, int C, int lds) {
  return N > 0 && HW > 0 && C > 0 && C % 8 == 0 && lds >= C && lds % 8 == 0;
}

}  // namespace

cudaError_t launch_se_sig_scale(const __nv_bfloat16* x, const __nv_bfloat16* s, int lds, __nv_bfloat16* y, int N, int HW,
                                int C, int sms, cudaStream_t stream) {
  if (!sg_args_ok(N, HW, C, lds)) return cudaErrorInvalidValue;
  const int64_t vecs = static_cast<int64_t>(N) * HW * (C / 8);
  sesig_scale_kernel<<<sg_grid(vecs, sms), kSgThreads, 0, stream>>>(x, s, lds, y, HW, C, vecs);
  return cudaGetLastError();
}

cudaError_t launch_se_sig_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* s, int lds,
                                 __nv_bfloat16* ds, int ldd, int N, int HW, int C, cudaStream_t stream) {
  const int chunks = (C + 63) / 64;
  if (!sg_args_ok(N, HW, C, lds) || ldd < C || ldd > chunks * 64) return cudaErrorInvalidValue;
  sesig_reduce_kernel<<<dim3(chunks, N), kSgThreads, 0, stream>>>(dy, x, s, lds, ds, ldd, HW, C);
  return cudaGetLastError();
}

cudaError_t launch_se_sig_apply(const __nv_bfloat16* dy, const __nv_bfloat16* s, int lds, const __nv_bfloat16* dpooled,
                                __nv_bfloat16* dx, int N, int HW, int C, int sms, cudaStream_t stream) {
  if (!sg_args_ok(N, HW, C, lds)) return cudaErrorInvalidValue;
  const int64_t vecs = static_cast<int64_t>(N) * HW * (C / 8);
  sesig_apply_kernel<<<sg_grid(vecs, sms), kSgThreads, 0, stream>>>(dy, s, lds, dpooled, dx, HW, C, vecs);
  return cudaGetLastError();
}

cudaError_t launch_pad_cols(const PadBatch& b, cudaStream_t stream) {
  if (b.n <= 0 || b.n > kPadMax) return cudaErrorInvalidValue;
  int64_t most = 0;
  for (int i = 0; i < b.n; ++i) {
    const PadMatrix& m = b.m[i];
    if (m.rows <= 0 || m.k <= 0 || m.prows < m.rows || m.kp < m.k || (m.esize != 2 && m.esize != 4)) return cudaErrorInvalidValue;
    most = std::max(most, static_cast<int64_t>(m.prows) * m.kp);
  }
  pad_cols_kernel<<<dim3(sg_grid(most, 132), b.n), kSgThreads, 0, stream>>>(b);
  return cudaGetLastError();
}

cudaError_t launch_fold_cols(const FoldBatch& b, cudaStream_t stream) {
  if (b.n <= 0 || b.n > kPadMax) return cudaErrorInvalidValue;
  int64_t most = 0;
  for (int i = 0; i < b.n; ++i) {
    const FoldMatrix& m = b.m[i];
    if (m.rows <= 0 || m.k <= 0 || m.kp < m.k) return cudaErrorInvalidValue;
    most = std::max(most, static_cast<int64_t>(m.rows) * m.k);
  }
  fold_cols_kernel<<<dim3(sg_grid(most, 132), b.n), kSgThreads, 0, stream>>>(b);
  return cudaGetLastError();
}

}  // namespace ddl
