// Patch merging of the Swin Transformer (V1): the 2x2 gather and the LayerNorm over 4C in one pass, and its backward.
//
// Forward: x is the NHWC activation [N][H][W][C] (H, W even); output row (n, i, j) of y [N * H/2 * W/2][4C] is
// LayerNorm(x[n, 2i, 2j] | x[n, 2i+1, 2j] | x[n, 2i, 2j+1] | x[n, 2i+1, 2j+1]), torchvision's concat order
// (x0, x1, x2, x3), with fp32 mean / rstd [rows] saved.  The reduction linear that follows is a 1x1 conv-GEMM.
// Backward: dx = LN_bwd(dy) scattered back to the four source pixels (a bijection: every element of dx is stored once,
// nothing accumulates); dgamma / dbeta are summed in a fixed order: per lane in registers over the rows of its warp, per
// block over its warps in warp order in shared memory, then over the blocks in block order by a second kernel.
//
// Mapping: one warp per output row; lane l holds the 16-byte vectors l, l + 32, ... (K = ceil(4C / 256) of them, the
// widths 384 .. 2048 of swin_t / _s / _b give K = 2 .. 8).  The forward takes a two-pass variance over registers; the
// backward makes two passes over (x, dy), the second one from L1.  Registers: 8K floats of data in the forward; 16K of
// dgamma / dbeta sums in the backward (128 at 4C = 2048, within the 255 of one 256-thread block per SM).
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

DDL_DEVICE void pm_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 pm_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

struct MergeArgs {
  const __nv_bfloat16* x;        // [N][H][W][C]
  const __nv_bfloat16* dy;       // backward: [M][4C]
  const float* gamma;
  const float* beta;
  __nv_bfloat16* y;              // forward: [M][4C]
  __nv_bfloat16* dx;             // backward: [N][H][W][C]
  float* mean;
  float* rstd;
  float* part;                   // backward: [blocks][2][4C]
  int M, H, W, C;                // M = N * H/2 * W/2
  float eps;
};

// offset in x of vector v (of 4C / 8) of output row `row`
DDL_DEVICE size_t src_off(const MergeArgs& a, int row, int v) {
  const int ho = a.H >> 1, wo = a.W >> 1, cv = a.C >> 3;
  const int n = row / (ho * wo), rem = row - n * ho * wo, i = rem / wo, j = rem - i * wo;
  const int q = v / cv, c = (v - q * cv) * 8;
  const int yy = 2 * i + (q & 1), xx = 2 * j + (q >> 1);
  return ((static_cast<size_t>(n) * a.H + yy) * a.W + xx) * a.C + c;
}

template <int K>
__global__ void __launch_bounds__(kThreads) patch_merge_fwd_kernel(MergeArgs a) {
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = gridDim.x * kWarps;
  const int vecs = a.C >> 1, C4 = 4 * a.C;
  const float inv_c = 1.f / static_cast<float>(C4);
  pdl_wait();
  for (int row = warp; row < a.M; row += nwarps) {
    float v[K][8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int vi = lane + 32 * k;
      if (vi < vecs) {
        pm_unpack8(__ldg(reinterpret_cast<const uint4*>(a.x + src_off(a, row, vi))), v[k]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[k][i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[k][i];
    }
    const float mu = warp_sum(s) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (lane + 32 * k >= vecs) continue;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[k][i] -= mu;
        q = fmaf(v[k][i], v[k][i], q);
      }
    }
    const float rs = rsqrtf(warp_sum(q) * inv_c + a.eps);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int vi = lane + 32 * k;
      if (vi >= vecs) continue;
      const int c = vi * 8;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(v[k][i] * rs, __ldg(a.gamma + c + i), __ldg(a.beta + c + i));
      *reinterpret_cast<uint4*>(a.y + static_cast<size_t>(row) * C4 + c) = pm_pack8(o);
    }
    if (lane == 0) {
      a.mean[row] = mu;
      a.rstd[row] = rs;
    }
  }
}

template <int K>
__global__ void __launch_bounds__(kThreads) patch_merge_bwd_kernel(MergeArgs a) {
  pdl_trigger();
  extern __shared__ float sh[];                   // [2][4C]: the block's dgamma, dbeta
  const int C4 = 4 * a.C, vecs = a.C >> 1;
  for (int c = threadIdx.x; c < 2 * C4; c += kThreads) sh[c] = 0.f;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int warp = blockIdx.x * kWarps + wib, nwarps = gridDim.x * kWarps;
  const float inv_c = 1.f / static_cast<float>(C4);
  float dg[K][8], db[K][8];
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dg[k][i] = db[k][i] = 0.f;
  }
  pdl_wait();
  for (int row = warp; row < a.M; row += nwarps) {
    const float mu = a.mean[row], rs = a.rstd[row];
    const size_t yoff = static_cast<size_t>(row) * C4;
    float s1 = 0.f, s2 = 0.f;                     // sum g dy, sum g dy xhat
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int vi = lane + 32 * k;
      if (vi >= vecs) continue;
      const int c = vi * 8;
      float x[8], d[8];
      pm_unpack8(__ldg(reinterpret_cast<const uint4*>(a.x + src_off(a, row, vi))), x);
      pm_unpack8(__ldg(reinterpret_cast<const uint4*>(a.dy + yoff + c)), d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float gd = d[i] * __ldg(a.gamma + c + i);
        s1 += gd;
        s2 = fmaf(gd, (x[i] - mu) * rs, s2);
      }
    }
    s1 = warp_sum(s1) * inv_c;
    s2 = warp_sum(s2) * inv_c;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int vi = lane + 32 * k;
      if (vi >= vecs) continue;
      const int c = vi * 8;
      const size_t xo = src_off(a, row, vi);
      float x[8], d[8], o[8];
      pm_unpack8(__ldg(reinterpret_cast<const uint4*>(a.x + xo)), x);
      pm_unpack8(__ldg(reinterpret_cast<const uint4*>(a.dy + yoff + c)), d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (x[i] - mu) * rs;
        o[i] = rs * (d[i] * __ldg(a.gamma + c + i) - s1 - xh * s2);
        dg[k][i] = fmaf(d[i], xh, dg[k][i]);
        db[k][i] += d[i];
      }
      *reinterpret_cast<uint4*>(a.dx + xo) = pm_pack8(o);
    }
  }
  __syncthreads();
  for (int w = 0; w < kWarps; ++w) {              // fold the warps in order
    if (wib == w) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int vi = lane + 32 * k;
        if (vi >= vecs) continue;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          sh[vi * 8 + i] += dg[k][i];
          sh[C4 + vi * 8 + i] += db[k][i];
        }
      }
    }
    __syncthreads();
  }
  float* part = a.part + static_cast<size_t>(blockIdx.x) * 2 * C4;
  for (int c = threadIdx.x; c < 2 * C4; c += kThreads) part[c] = sh[c];
}

// dgamma[c] += sum over the blocks in order, dbeta likewise (one thread per column of [2][4C])
__global__ void __launch_bounds__(kThreads) patch_merge_reduce_kernel(const float* __restrict__ part, float* dgamma,
                                                                      float* dbeta, int blocks, int C4) {
  pdl_trigger();
  pdl_wait();
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= 2 * C4) return;
  float s = 0.f;
#pragma unroll 8
  for (int b = 0; b < blocks; ++b) s += part[static_cast<size_t>(b) * 2 * C4 + c];
  float* dst = c < C4 ? dgamma : dbeta;
  if (dst) dst[c < C4 ? c : c - C4] += s;
}

bool merge_shape_ok(int N, int H, int W, int C) {
  return N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && C >= 8 && C <= 512 &&
         static_cast<int64_t>(N) * (H / 2) * (W / 2) < (static_cast<int64_t>(1) << 31);
}

#define DDL_PM_LAUNCH(KERNEL)                                                                                        \
  switch ((a.C / 2 + 31) / 32) {                                                                                     \
    case 1: return launch_pdl(KERNEL<1>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 2: return launch_pdl(KERNEL<2>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 3: return launch_pdl(KERNEL<3>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 4: return launch_pdl(KERNEL<4>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 5: return launch_pdl(KERNEL<5>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 6: return launch_pdl(KERNEL<6>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 7: return launch_pdl(KERNEL<7>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 8: return launch_pdl(KERNEL<8>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    default: return cudaErrorInvalidValue;                                                                           \
  }

}  // namespace

int patch_merge_bwd_blocks(int sms) { return sms > 0 ? sms : 1; }

cudaError_t launch_patch_merge_fwd(const __nv_bfloat16* x, const float* gamma, const float* beta, __nv_bfloat16* y,
                                   float* mean, float* rstd, int N, int H, int W, int C, float eps, int sms,
                                   cudaStream_t stream) {
  if (!merge_shape_ok(N, H, W, C)) return cudaErrorInvalidValue;
  MergeArgs a{};
  a.x = x; a.gamma = gamma; a.beta = beta; a.y = y; a.mean = mean; a.rstd = rstd;
  a.M = N * (H / 2) * (W / 2); a.H = H; a.W = W; a.C = C; a.eps = eps;
  int64_t blocks = (static_cast<int64_t>(a.M) + kWarps - 1) / kWarps;
  if (blocks > static_cast<int64_t>(sms) * 8) blocks = static_cast<int64_t>(sms) * 8;
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 0;
  DDL_PM_LAUNCH(patch_merge_fwd_kernel)
}

cudaError_t launch_patch_merge_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean, const float* rstd,
                                   const float* gamma, __nv_bfloat16* dx, float* dgamma, float* dbeta, float* scratch,
                                   int N, int H, int W, int C, int sms, cudaStream_t stream) {
  if (!merge_shape_ok(N, H, W, C)) return cudaErrorInvalidValue;
  MergeArgs a{};
  a.x = x; a.dy = dy; a.gamma = gamma; a.dx = dx; a.mean = const_cast<float*>(mean); a.rstd = const_cast<float*>(rstd);
  a.part = scratch; a.M = N * (H / 2) * (W / 2); a.H = H; a.W = W; a.C = C;
  const int blocks = patch_merge_bwd_blocks(sms);
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 8 * static_cast<size_t>(C) * sizeof(float);
  cudaError_t e = [&]() -> cudaError_t { DDL_PM_LAUNCH(patch_merge_bwd_kernel) }();
  if (e != cudaSuccess) return e;
  const int C4 = 4 * C;
  return launch_pdl(patch_merge_reduce_kernel, dim3((2 * C4 + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(scratch), dgamma, dbeta, blocks, C4);
}

}  // namespace ddl
