// Row kernels of the Vision Transformer (bf16 [rows][C] token matrices, fp32 math):
// - residual add + LayerNorm, forward: x1 = x + a, t = LN(x1), writing x1, t and fp32 mean / rstd in one pass;
// - LayerNorm backward with an addend: dx = LN_bwd(dt) + dres, also reducing dgamma / dbeta, so that each residual
//   gradient of the encoder block is one store;
// - patchify: an NHWC4 image [N][H][W][4] to the patch rows [N * (H/P) * (W/P)][P * P * 3] in (r, s, c) order (KRSC, the
//   pad channel dropped), which a channels_last conv_proj weight [C, 3, P, P] multiplies as it is;
// - token assembly: tokens[n, 0] = cls + pos[0], tokens[n, 1 + p] = patch[n, p] + pos[1 + p]; its backward copies the
//   patch rows of dtokens out and sums dtokens over the images per token (dpos, dcls) and over the patch tokens (the
//   conv_proj bias gradient), in a fixed order.
//
// The LayerNorm kernels use convnext.cu's row mapping: T threads (a power of two <= 32) share a row, each holding
// V = C / (8 T) 16-byte vectors; the forward takes a two-pass variance over registers, the backward makes two passes
// over (x, dy) and keeps per-thread dgamma / dbeta sums, folded per block in shared memory and added once per block.
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kThreads = 256;

DDL_DEVICE void vt_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 vt_pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
DDL_DEVICE void vt_load8(const __nv_bfloat16* p, float (&v)[8]) { vt_unpack8(__ldg(reinterpret_cast<const uint4*>(p)), v); }

DDL_DEVICE float lane_sum(float v, int lg_t) {
  for (int off = 1; off < (1 << lg_t); off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

struct AddLnArgs {
  const __nv_bfloat16* x;        // forward: x; backward: the saved LN input
  const __nv_bfloat16* a;        // forward: the addend a; backward: dres
  const __nv_bfloat16* dy;       // backward: dt
  const float* gamma;
  const float* beta;
  __nv_bfloat16* x1;             // forward: x + a
  __nv_bfloat16* y;              // forward: t; backward: dx
  float* mean;
  float* rstd;
  float* dgamma;
  float* dbeta;
  int M, C, lg_t;
  float eps;
};

template <int V>
__global__ void __launch_bounds__(kThreads, V <= 5 ? 2 : 1) add_layer_norm_fwd_kernel(AddLnArgs a) {
  pdl_trigger();
  const int T = 1 << a.lg_t, rpw = 32 >> a.lg_t;
  const int lane = threadIdx.x & 31, sub = lane >> a.lg_t, j = lane & (T - 1);
  const int warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = gridDim.x * (kThreads / 32);
  const float inv_c = 1.f / static_cast<float>(a.C);
  pdl_wait();
  for (int base = warp * rpw; base < a.M; base += nwarps * rpw) {
    const int row = base + sub;
    const bool valid = row < a.M;
    const size_t off = static_cast<size_t>(valid ? row : 0) * a.C;
    float v[V][8];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
      if (valid) {
        float u[8];
        vt_load8(a.x + off + c, v[k]);
        vt_load8(a.a + off + c, u);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[k][i] = bf16_round(v[k][i] + u[i]);     // the stored x1 is what LN normalises
        *reinterpret_cast<uint4*>(a.x1 + off + c) = vt_pack8(v[k]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[k][i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[k][i];
    }
    const float mu = lane_sum(s, a.lg_t) * inv_c;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < V; ++k) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[k][i] -= mu;
        q = fmaf(v[k][i], v[k][i], q);
      }
    }
    const float rs = rsqrtf(lane_sum(q, a.lg_t) * inv_c + a.eps);
    if (!valid) continue;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = fmaf(v[k][i] * rs, __ldg(a.gamma + c + i), __ldg(a.beta + c + i));
      *reinterpret_cast<uint4*>(a.y + off + c) = vt_pack8(o);
    }
    if (j == 0) {
      a.mean[row] = mu;
      a.rstd[row] = rs;
    }
  }
}

template <int V>
__global__ void __launch_bounds__(kThreads, V <= 3 ? 2 : 1) layer_norm_bwd_add_kernel(AddLnArgs a) {
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
        vt_load8(a.x + off + c, x);
        vt_load8(a.dy + off + c, d);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float gd = d[i] * __ldg(a.gamma + c + i);
          s1 += gd;
          s2 = fmaf(gd, (x[i] - mu) * rs, s2);
        }
      }
    }
    s1 = lane_sum(s1, a.lg_t) * inv_c;
    s2 = lane_sum(s2, a.lg_t) * inv_c;
    if (!valid) continue;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = (j + k * T) * 8;
      float x[8], d[8], r[8], o[8];
      vt_load8(a.x + off + c, x);
      vt_load8(a.dy + off + c, d);
      vt_load8(a.a + off + c, r);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float xh = (x[i] - mu) * rs;
        o[i] = rs * (d[i] * __ldg(a.gamma + c + i) - s1 - xh * s2) + r[i];
        dg[k][i] = fmaf(d[i], xh, dg[k][i]);
        db[k][i] += d[i];
      }
      *reinterpret_cast<uint4*>(a.y + off + c) = vt_pack8(o);
    }
  }
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
  __syncthreads();
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

// ---- patch embedding -----------------------------------------------------------------------------------------------
// one thread per (patch, r, s): reads the 4 channels of one pixel, writes its 3 real channels
__global__ void __launch_bounds__(kThreads) patchify_kernel(const __nv_bfloat16* __restrict__ img,
                                                            __nv_bfloat16* __restrict__ out, int H, int W, int P,
                                                            int64_t total) {
  pdl_trigger();
  pdl_wait();
  const int gw = W / P, pp = P * P, per_img = (H / P) * gw;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    const int64_t patch = i / pp;
    const int rs = static_cast<int>(i - patch * pp), r = rs / P, s = rs - r * P;
    const int n = static_cast<int>(patch / per_img), pidx = static_cast<int>(patch - static_cast<int64_t>(n) * per_img);
    const int py = pidx / gw, px = pidx - py * gw;
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(img + ((static_cast<size_t>(n) * H + py * P + r) * W + px * P + s) * 4));
    __nv_bfloat16* d = out + i * 3;
    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&v.x);
    const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&v.y);
    d[0] = lo.x;
    d[1] = lo.y;
    d[2] = hi.x;
  }
}

// ---- token assembly --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) tokens_fwd_kernel(const __nv_bfloat16* __restrict__ patch,
                                                              const float* __restrict__ cls,
                                                              const float* __restrict__ pos,
                                                              __nv_bfloat16* __restrict__ tok, int L, int C,
                                                              int64_t n8) {
  pdl_trigger();
  pdl_wait();
  const int groups = C / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    const int64_t row = i / groups;                // n * L + l
    const int c = static_cast<int>(i - row * groups) * 8;
    const int n = static_cast<int>(row / L), l = static_cast<int>(row - static_cast<int64_t>(n) * L);
    float v[8];
    if (l == 0) {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = __ldg(cls + c + k);
    } else {
      vt_load8(patch + (static_cast<size_t>(n) * (L - 1) + l - 1) * C + c, v);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] += __ldg(pos + static_cast<size_t>(l) * C + c + k);
    reinterpret_cast<uint4*>(tok)[i] = vt_pack8(v);
  }
}

// pass 1: thread (l, 8 columns) sums dtokens[n, l] over the images in order into colsum[l] and copies the patch rows
// out; pass 2 (one thread per column) adds colsum into dpos / dcls and the patch-token total into dbias
__global__ void __launch_bounds__(kThreads) tokens_bwd_kernel(const __nv_bfloat16* __restrict__ dtok,
                                                              __nv_bfloat16* __restrict__ dpatch,
                                                              float* __restrict__ colsum, int N, int L, int C) {
  pdl_trigger();
  pdl_wait();
  const int groups = C / 8;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  if (i >= static_cast<int64_t>(L) * groups) return;
  const int l = static_cast<int>(i / groups), c = static_cast<int>(i - static_cast<int64_t>(l) * groups) * 8;
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int n = 0; n < N; ++n) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(dtok + (static_cast<size_t>(n) * L + l) * C + c));
    float v[8];
    vt_unpack8(u, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] += v[k];
    if (l > 0 && dpatch) *reinterpret_cast<uint4*>(dpatch + (static_cast<size_t>(n) * (L - 1) + l - 1) * C + c) = u;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) colsum[static_cast<size_t>(l) * C + c + k] = s[k];
}

__global__ void __launch_bounds__(kThreads) tokens_bwd_reduce_kernel(const float* __restrict__ colsum, float* dpos,
                                                                     float* dcls, float* dbias, int L, int C) {
  pdl_trigger();
  pdl_wait();
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  float tot = 0.f;
  for (int l = 0; l < L; ++l) {
    const float v = colsum[static_cast<size_t>(l) * C + c];
    if (dpos) dpos[static_cast<size_t>(l) * C + c] += v;
    if (l > 0) tot += v;
  }
  if (dcls) dcls[c] += colsum[c];
  if (dbias) dbias[c] += tot;
}

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

inline int grid_for(int64_t work, int sms) {
  int64_t b = (work + kThreads - 1) / kThreads;
  if (b > static_cast<int64_t>(sms) * 16) b = static_cast<int64_t>(sms) * 16;
  return static_cast<int>(b < 1 ? 1 : b);
}

#define DDL_VIT_LN_LAUNCH(KERNEL)                                                                                    \
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

cudaError_t launch_add_layer_norm_fwd(const __nv_bfloat16* x, const __nv_bfloat16* add, const float* gamma,
                                      const float* beta, __nv_bfloat16* x1, __nv_bfloat16* y, float* mean, float* rstd,
                                      int M, int C, float eps, int sms, cudaStream_t stream) {
  int v = 0;
  const int lg = ln_mapping(C, &v);
  if (lg < 0 || M <= 0) return cudaErrorInvalidValue;
  AddLnArgs a{};
  a.x = x; a.a = add; a.gamma = gamma; a.beta = beta; a.x1 = x1; a.y = y; a.mean = mean; a.rstd = rstd;
  a.M = M; a.C = C; a.lg_t = lg; a.eps = eps;
  const int rows_per_block = (kThreads / 32) * (32 >> lg);
  int64_t blocks = (static_cast<int64_t>(M) + rows_per_block - 1) / rows_per_block;
  if (blocks > static_cast<int64_t>(sms) * 8) blocks = static_cast<int64_t>(sms) * 8;
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 0;
  DDL_VIT_LN_LAUNCH(add_layer_norm_fwd_kernel)
}

cudaError_t launch_layer_norm_bwd_add(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean,
                                      const float* rstd, const float* gamma, const __nv_bfloat16* dres, __nv_bfloat16* dx,
                                      float* dgamma, float* dbeta, int M, int C, int sms, cudaStream_t stream) {
  int v = 0;
  const int lg = ln_mapping(C, &v);
  if (lg < 0 || M <= 0) return cudaErrorInvalidValue;
  AddLnArgs a{};
  a.x = x; a.a = dres; a.dy = dy; a.gamma = gamma; a.y = dx; a.mean = const_cast<float*>(mean);
  a.rstd = const_cast<float*>(rstd); a.dgamma = dgamma; a.dbeta = dbeta; a.M = M; a.C = C; a.lg_t = lg;
  const int rows_per_block = (kThreads / 32) * (32 >> lg);
  int64_t blocks = (static_cast<int64_t>(M) + rows_per_block - 1) / rows_per_block;
  if (blocks > static_cast<int64_t>(sms) * 2) blocks = static_cast<int64_t>(sms) * 2;
  const dim3 grid(static_cast<unsigned>(blocks));
  const size_t smem = 2 * static_cast<size_t>(C) * sizeof(float);
  DDL_VIT_LN_LAUNCH(layer_norm_bwd_add_kernel)
}

cudaError_t launch_patchify(const __nv_bfloat16* img, __nv_bfloat16* out, int N, int H, int W, int P, int sms,
                            cudaStream_t stream) {
  if (N <= 0 || P <= 0 || H <= 0 || W <= 0 || H % P != 0 || W % P != 0) return cudaErrorInvalidValue;
  const int64_t total = static_cast<int64_t>(N) * H * W;
  return launch_pdl(patchify_kernel, dim3(grid_for(total, sms)), dim3(kThreads), 0, stream, 1, img, out, H, W, P, total);
}

cudaError_t launch_tokens_fwd(const __nv_bfloat16* patch, const float* cls, const float* pos, __nv_bfloat16* tok, int N,
                              int L, int C, int sms, cudaStream_t stream) {
  if (N <= 0 || L <= 1 || C <= 0 || C % 8 != 0) return cudaErrorInvalidValue;
  const int64_t n8 = static_cast<int64_t>(N) * L * (C / 8);
  return launch_pdl(tokens_fwd_kernel, dim3(grid_for(n8, sms)), dim3(kThreads), 0, stream, 1, patch, cls, pos, tok, L, C,
                    n8);
}

cudaError_t launch_tokens_bwd(const __nv_bfloat16* dtok, __nv_bfloat16* dpatch, float* colsum, float* dpos, float* dcls,
                              float* dbias, int N, int L, int C, cudaStream_t stream) {
  if (N <= 0 || L <= 1 || C <= 0 || C % 8 != 0) return cudaErrorInvalidValue;
  const int64_t work = static_cast<int64_t>(L) * (C / 8);
  cudaError_t e = launch_pdl(tokens_bwd_kernel, dim3(static_cast<unsigned>((work + kThreads - 1) / kThreads)),
                             dim3(kThreads), 0, stream, 1, dtok, dpatch, colsum, N, L, C);
  if (e != cudaSuccess) return e;
  return launch_pdl(tokens_bwd_reduce_kernel, dim3((C + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(colsum), dpos, dcls, dbias, L, C);
}

}  // namespace ddl
