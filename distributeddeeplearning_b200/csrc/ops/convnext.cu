// Row kernels of the ConvNeXt block (NHWC bf16 activations viewed as [M][C] rows, fp32 math):
// - LayerNorm over the channels of each row, forward and backward;
// - exact (erf) GELU, forward and a backward that also reduces fc1's bias gradient;
// - layer scale + stochastic depth + residual add, forward and a backward that also reduces the layer-scale and fc2
//   bias gradients.
//
// LayerNorm thread mapping: T threads (a power of two <= 32) share a row, each holding V = C / (8 T) 16-byte vectors
// (V <= 6); T is the largest power of two <= 32 dividing C / 8, so every thread has the same work (C = 96: 4 threads x 3
// vectors, 8 rows per warp).  Row statistics are shuffles within the T lanes.  The forward keeps the row in registers and
// takes the variance as the mean of (x - mean)^2 (two passes over registers, no E[x^2] - E[x]^2 cancellation for rows
// whose mean is far larger than their spread).  The backward makes two passes over (x, dy), the second from L1, so that
// its registers hold the per-thread dgamma / dbeta partial sums rather than the row.
//
// The parameter-gradient reductions (LayerNorm dgamma / dbeta, GELU's bias, layer scale and fc2's bias) sum in
// registers, fold the block's partial sums in shared memory and add one value per channel and block to the fp32 slot.
// A bias gradient is the column sum of the bf16 gradient the kernel stores, the operand its GEMM's data and weight
// gradients consume (as bias_relu_bwd sums the bf16 dy it reads), not of the fp32 value before rounding.
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kThreads = 256;

DDL_DEVICE void cx_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 cx_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
DDL_DEVICE void cx_load8(const __nv_bfloat16* p, float (&v)[8]) { cx_unpack8(__ldg(reinterpret_cast<const uint4*>(p)), v); }

struct LnArgs {
  const __nv_bfloat16* x;
  const __nv_bfloat16* dy;
  const float* gamma;
  const float* beta;
  __nv_bfloat16* y;          // forward: y; backward: dx
  float* mean;
  float* rstd;
  float* dgamma;
  float* dbeta;
  int M, C, lg_t;
  float eps;
};

// sum over the T = 1 << lg_t lanes of this row (lanes of a warp with the same row differ in bits < lg_t)
DDL_DEVICE float row_sum(float v, int lg_t) {
  for (int off = 1; off < (1 << lg_t); off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <int V>
__global__ void __launch_bounds__(kThreads, V <= 5 ? 2 : 1) layer_norm_fwd_kernel(LnArgs a) {
  pdl_trigger();
  const int T = 1 << a.lg_t, rpw = 32 >> a.lg_t;
  const int lane = threadIdx.x & 31, sub = lane >> a.lg_t, j = lane & (T - 1);
  const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = gridDim.x * (kThreads / 32);
  const float inv_c = 1.f / static_cast<float>(a.C);
  pdl_wait();
  // the loop bound is uniform over the warp (every lane takes part in the shuffles); rows past M are masked
  for (int base = warp * rpw; base < a.M; base += nwarps * rpw) {
    const int row = base + sub;
    const bool valid = row < a.M;
    const __nv_bfloat16* xr = a.x + static_cast<size_t>(row) * a.C;
    float v[V][8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      if (valid) cx_load8(xr + (j + k * T) * 8, v[k]);
      else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[k][i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[k][i];
    }
    const float mu = row_sum(s, a.lg_t) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[k][i] -= mu;
        q = fmaf(v[k][i], v[k][i], q);
      }
    }
    const float rs = rsqrtf(row_sum(q, a.lg_t) * inv_c + a.eps);
    if (!valid) continue;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(v[k][i] * rs, __ldg(a.gamma + c + i), __ldg(a.beta + c + i));
      *reinterpret_cast<uint4*>(a.y + static_cast<size_t>(row) * a.C + c) = cx_pack8(o);
    }
    if (j == 0) {
      a.mean[row] = mu;
      a.rstd[row] = rs;
    }
  }
}

template <int V>
__global__ void __launch_bounds__(kThreads, V <= 3 ? 2 : 1) layer_norm_bwd_kernel(LnArgs a) {
  pdl_trigger();
  extern __shared__ float sh[];                   // [2][C]: the block's dgamma, dbeta
  for (int c = threadIdx.x; c < 2 * a.C; c += kThreads) sh[c] = 0.f;
  const int T = 1 << a.lg_t, rpw = 32 >> a.lg_t;
  const int lane = threadIdx.x & 31, sub = lane >> a.lg_t, j = lane & (T - 1);
  const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = gridDim.x * (kThreads / 32);
  const float inv_c = 1.f / static_cast<float>(a.C);
  float dg[V][8], db[V][8];
#pragma unroll
  for (int k = 0; k < V; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dg[k][i] = db[k][i] = 0.f;
  }
  pdl_wait();
  for (int base = warp * rpw; base < a.M; base += nwarps * rpw) {
    const int row = base + sub;
    const bool valid = row < a.M;
    const size_t off = static_cast<size_t>(valid ? row : 0) * a.C;
    const float mu = valid ? a.mean[row] : 0.f, rs = valid ? a.rstd[row] : 0.f;
    float s1 = 0.f, s2 = 0.f;                     // sum g dy, sum g dy xhat
    if (valid) {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const int c = (j + k * T) * 8;
        float x[8], d[8];
        cx_load8(a.x + off + c, x);
        cx_load8(a.dy + off + c, d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float gd = d[i] * __ldg(a.gamma + c + i);
          s1 += gd;
          s2 = fmaf(gd, (x[i] - mu) * rs, s2);
        }
      }
    }
    s1 = row_sum(s1, a.lg_t) * inv_c;
    s2 = row_sum(s2, a.lg_t) * inv_c;
    if (!valid) continue;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
      float x[8], d[8], o[8];
      cx_load8(a.x + off + c, x);
      cx_load8(a.dy + off + c, d);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (x[i] - mu) * rs;
        o[i] = rs * (d[i] * __ldg(a.gamma + c + i) - s1 - xh * s2);
        dg[k][i] = fmaf(d[i], xh, dg[k][i]);
        db[k][i] += d[i];
      }
      *reinterpret_cast<uint4*>(a.y + off + c) = cx_pack8(o);
    }
  }
  // fold the lanes of the warp that own the same channels (they differ in bits >= lg_t), then the warps in shared memory
#pragma unroll
  for (int k = 0; k < V; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      for (int o = T; o < 32; o <<= 1) {
        dg[k][i] += __shfl_xor_sync(0xffffffffu, dg[k][i], o);
        db[k][i] += __shfl_xor_sync(0xffffffffu, db[k][i], o);
      }
    }
  }
  __syncthreads();                                // sh zeroed by every thread before any adds
  if (sub == 0) {
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        atomicAdd(sh + c + i, dg[k][i]);
        atomicAdd(sh + a.C + c + i, db[k][i]);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < a.C; c += kThreads) {
    if (a.dgamma) atomicAdd(a.dgamma + c, sh[c]);
    if (a.dbeta) atomicAdd(a.dbeta + c, sh[a.C + c]);
  }
}

// ---- exact GELU ------------------------------------------------------------------------------------------------------
DDL_DEVICE float gelu_f(float h) { return 0.5f * h * (1.f + erff(h * 0.70710678118654752f)); }
DDL_DEVICE float gelu_grad(float h) {     // Phi(h) + h phi(h)
  return 0.5f * (1.f + erff(h * 0.70710678118654752f)) + h * 0.39894228040143268f * __expf(-0.5f * h * h);
}

__global__ void __launch_bounds__(kThreads) gelu_fwd_kernel(const __nv_bfloat16* __restrict__ h,
                                                            __nv_bfloat16* __restrict__ g, int64_t n8) {
  pdl_trigger();
  pdl_wait();
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    float v[8];
    cx_unpack8(__ldg(reinterpret_cast<const uint4*>(h) + i), v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = gelu_f(v[k]);
    reinterpret_cast<uint4*>(g)[i] = cx_pack8(v);
  }
}

// Column-reduction mapping shared by the two backward kernels below: thread `tid` owns the 8-channel group tid % (C/8)
// and walks the rows tid / (C/8), + stride; the launcher makes the thread count a multiple of C/8.
struct ColMap {
  int g, row0, stride;
};
DDL_DEVICE ColMap col_map(int C) {
  const int groups = C / 8;
  const int tid = blockIdx.x * kThreads + threadIdx.x;
  return ColMap{tid % groups, tid / groups, static_cast<int>(gridDim.x * kThreads) / groups};
}

// add `nsum` per-thread vectors of 8 channel sums into the block's shared [nsum][C] and then into the fp32 slots
template <int NS>
DDL_DEVICE void col_flush(float (&s)[NS][8], float* sh, int C, int g, float* const (&dst)[NS]) {
#pragma unroll
  for (int k = 0; k < NS; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) atomicAdd(sh + k * C + g * 8 + i, s[k][i]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kThreads) {
#pragma unroll
    for (int k = 0; k < NS; ++k)
      if (dst[k]) atomicAdd(dst[k] + c, sh[k * C + c]);
  }
}

__global__ void __launch_bounds__(kThreads) gelu_bwd_kernel(const __nv_bfloat16* __restrict__ dg,
                                                            const __nv_bfloat16* __restrict__ h,
                                                            __nv_bfloat16* __restrict__ dh, float* dbias, int M, int C) {
  pdl_trigger();
  extern __shared__ float sh[];
  for (int c = threadIdx.x; c < C; c += kThreads) sh[c] = 0.f;
  const ColMap m = col_map(C);
  float s[1][8] = {{0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}};
  pdl_wait();
  __syncthreads();
  for (int r = m.row0; r < M; r += m.stride) {
    const size_t off = static_cast<size_t>(r) * C + m.g * 8;
    float d[8], v[8];
    cx_load8(dg + off, d);
    cx_load8(h + off, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      d[i] = bf16_round(d[i] * gelu_grad(v[i]));      // the bias gradient sums the dh fc1's GEMMs consume
      s[0][i] += d[i];
    }
    *reinterpret_cast<uint4*>(dh + off) = cx_pack8(d);
  }
  float* const dst[1] = {dbias};
  col_flush<1>(s, sh, C, m.g, dst);
}

// ---- layer scale + stochastic depth + residual -------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) layer_scale_fwd_kernel(const __nv_bfloat16* __restrict__ y,
                                                                   const float* __restrict__ ls,
                                                                   const float* __restrict__ keep,
                                                                   const __nv_bfloat16* __restrict__ x,
                                                                   __nv_bfloat16* __restrict__ z, int64_t n8, int C,
                                                                   int hw) {
  pdl_trigger();
  pdl_wait();
  const int groups = C / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    const int64_t m = i / groups;
    const int c = static_cast<int>(i - m * groups) * 8;
    const float kp = keep ? __ldg(keep + m / hw) : 1.f;
    float u[8], v[8];
    cx_unpack8(__ldg(reinterpret_cast<const uint4*>(y) + i), u);
    cx_unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaf(__ldg(ls + c + k) * kp, u[k], v[k]);
    reinterpret_cast<uint4*>(z)[i] = cx_pack8(v);
  }
}

__global__ void __launch_bounds__(kThreads) layer_scale_bwd_kernel(const __nv_bfloat16* __restrict__ dz,
                                                                   const __nv_bfloat16* __restrict__ y,
                                                                   const float* __restrict__ ls,
                                                                   const float* __restrict__ keep,
                                                                   __nv_bfloat16* __restrict__ dy, float* dls,
                                                                   float* dbias, int M, int C, int hw) {
  pdl_trigger();
  extern __shared__ float sh[];                   // [2][C]: dls, dbias
  for (int c = threadIdx.x; c < 2 * C; c += kThreads) sh[c] = 0.f;
  const ColMap m = col_map(C);
  float s[2][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[0][i] = s[1][i] = 0.f;
  pdl_wait();
  float l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) l[i] = __ldg(ls + m.g * 8 + i);
  __syncthreads();
  for (int r = m.row0; r < M; r += m.stride) {
    const size_t off = static_cast<size_t>(r) * C + m.g * 8;
    const float kp = keep ? __ldg(keep + r / hw) : 1.f;
    float d[8], v[8];
    cx_load8(dz + off, d);
    cx_load8(y + off, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float dk = d[i] * kp;
      s[0][i] = fmaf(dk, v[i], s[0][i]);
      d[i] = dk * l[i];
      s[1][i] += bf16_round(d[i]);               // the bias gradient sums the dy fc2's GEMMs consume
    }
    *reinterpret_cast<uint4*>(dy + off) = cx_pack8(d);
  }
  float* const dst[2] = {dls, dbias};
  col_flush<2>(s, sh, C, m.g, dst);
}

// blocks of the column-reduction kernels: about 4 blocks per SM, thread count a multiple of C/8
int col_blocks(int M, int C, int sms) {
  const int64_t groups = C / 8;
  int64_t threads = static_cast<int64_t>(M) * groups;
  const int64_t cap = static_cast<int64_t>(sms) * 4 * kThreads;
  if (threads > cap) threads = cap;
  int64_t l = groups;
  while (l % kThreads != 0) l += groups;     // smallest multiple of groups that is a whole number of blocks
  const int64_t unit = l / kThreads;
  int64_t blocks = (threads + kThreads - 1) / kThreads;
  blocks = (blocks + unit - 1) / unit * unit;
  return static_cast<int>(blocks);
}

// blocks of the elementwise kernels: one vector per thread, at most 16 blocks per SM (grid-stride beyond)
inline int grid_for(int64_t work, int sms) {
  int64_t b = (work + kThreads - 1) / kThreads;
  if (b > static_cast<int64_t>(sms) * 16) b = static_cast<int64_t>(sms) * 16;
  return static_cast<int>(b < 1 ? 1 : b);
}

// T (as log2) and V of the LayerNorm mapping, or -1 when C is not covered
int ln_mapping(int C, int* v_out) {
  if (C <= 0 || C % 8 != 0) return -1;
  const int vecs = C / 8;
  int lg = 0;
  while (lg < 5 && vecs % (2 << lg) == 0) ++lg;
  const int v = vecs >> lg;
  if (v > 6) return -1;
  *v_out = v;
  return lg;
}

#define DDL_LN_LAUNCH(KERNEL)                                                                                        \
  switch (v) {                                                                                                       \
    case 1: return launch_pdl(KERNEL<1>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 2: return launch_pdl(KERNEL<2>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 3: return launch_pdl(KERNEL<3>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 4: return launch_pdl(KERNEL<4>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 5: return launch_pdl(KERNEL<5>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    case 6: return launch_pdl(KERNEL<6>, grid, dim3(kThreads), smem, stream, 1, a);                                  \
    default: return cudaErrorInvalidValue;                                                                           \
  }

}  // namespace

cudaError_t launch_layer_norm_fwd(const __nv_bfloat16* x, const float* gamma, const float* beta, __nv_bfloat16* y,
                                  float* mean, float* rstd, int M, int C, float eps, int sms, cudaStream_t stream) {
  int v = 0;
  const int lg = ln_mapping(C, &v);
  if (lg < 0 || M <= 0) return cudaErrorInvalidValue;
  LnArgs a{};
  a.x = x; a.gamma = gamma; a.beta = beta; a.y = y; a.mean = mean; a.rstd = rstd; a.M = M; a.C = C; a.lg_t = lg;
  a.eps = eps;
  const int rows_per_block = (kThreads / 32) * (32 >> lg);
  int64_t blocks = (static_cast<int64_t>(M) + rows_per_block - 1) / rows_per_block;
  if (blocks > static_cast<int64_t>(sms) * 8) blocks = static_cast<int64_t>(sms) * 8;
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 0;
  DDL_LN_LAUNCH(layer_norm_fwd_kernel)
}

cudaError_t launch_layer_norm_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean, const float* rstd,
                                  const float* gamma, __nv_bfloat16* dx, float* dgamma, float* dbeta, int M, int C, int sms,
                                  cudaStream_t stream) {
  int v = 0;
  const int lg = ln_mapping(C, &v);
  if (lg < 0 || M <= 0) return cudaErrorInvalidValue;
  LnArgs a{};
  a.x = x; a.dy = dy; a.gamma = gamma; a.y = dx; a.mean = const_cast<float*>(mean); a.rstd = const_cast<float*>(rstd);
  a.dgamma = dgamma; a.dbeta = dbeta; a.M = M; a.C = C; a.lg_t = lg;
  const int rows_per_block = (kThreads / 32) * (32 >> lg);
  int64_t blocks = (static_cast<int64_t>(M) + rows_per_block - 1) / rows_per_block;
  if (blocks > static_cast<int64_t>(sms) * 2) blocks = static_cast<int64_t>(sms) * 2;
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 2 * static_cast<size_t>(C) * sizeof(float);
  DDL_LN_LAUNCH(layer_norm_bwd_kernel)
}

cudaError_t launch_gelu_fwd(const __nv_bfloat16* h, __nv_bfloat16* g, int64_t n, int sms, cudaStream_t stream) {
  if (n <= 0 || n % 8 != 0) return cudaErrorInvalidValue;
  return launch_pdl(gelu_fwd_kernel, dim3(grid_for(n / 8, sms)), dim3(kThreads), 0, stream, 1, h, g, n / 8);
}

cudaError_t launch_gelu_bwd(const __nv_bfloat16* dg, const __nv_bfloat16* h, __nv_bfloat16* dh, float* dbias, int M, int C,
                            int sms, cudaStream_t stream) {
  if (M <= 0 || C <= 0 || C % 8 != 0 || C > 8192) return cudaErrorInvalidValue;
  return launch_pdl(gelu_bwd_kernel, dim3(col_blocks(M, C, sms)), dim3(kThreads), static_cast<size_t>(C) * sizeof(float),
                    stream, 1, dg, h, dh, dbias, M, C);
}

cudaError_t launch_layer_scale_fwd(const __nv_bfloat16* y, const float* ls, const float* keep, const __nv_bfloat16* x,
                                   __nv_bfloat16* z, int M, int C, int hw, int sms, cudaStream_t stream) {
  if (M <= 0 || C <= 0 || C % 8 != 0 || hw <= 0 || M % hw != 0) return cudaErrorInvalidValue;
  const int64_t n8 = static_cast<int64_t>(M) * (C / 8);
  return launch_pdl(layer_scale_fwd_kernel, dim3(grid_for(n8, sms)), dim3(kThreads), 0, stream, 1, y, ls, keep, x, z, n8, C,
                    hw);
}

cudaError_t launch_layer_scale_bwd(const __nv_bfloat16* dz, const __nv_bfloat16* y, const float* ls, const float* keep,
                                   __nv_bfloat16* dy, float* dls, float* dbias, int M, int C, int hw, int sms,
                                   cudaStream_t stream) {
  if (M <= 0 || C <= 0 || C % 8 != 0 || C > 4096 || hw <= 0 || M % hw != 0) return cudaErrorInvalidValue;
  return launch_pdl(layer_scale_bwd_kernel, dim3(col_blocks(M, C, sms)), dim3(kThreads),
                    2 * static_cast<size_t>(C) * sizeof(float), stream, 1, dz, y, ls, keep, dy, dls, dbias, M, C, hw);
}

}  // namespace ddl
