// GoogLeNet's Inception module (ops/googlenet.py runs it as one autograd node on these kernels, the conv kernels and the
// max-pool kernels), and its auxiliary head.
//
// Segmented BatchNorm + ReLU: one launch applies up to kSegMax BatchNorms, each to a channel segment that is read from
// and written to strided row slices ([M][ld] tensors at a column offset), so the module's branch BNs write straight into
// their slices of the concatenated output and read their slices of the merged 1x1 GEMM's output: no concat or split copy.
//   forward   z = relu(x * scale + shift), per channel; train: scale / shift from the conv epilogue's (sum, sumsq), mean /
//             invstd saved, running statistics updated, with the same expressions as bn_act_fwd (bit-equal outputs)
//   backward  pass 1 (reduce): g = dz masked by relu'(x * gamma invstd + beta - mean gamma invstd) (the mask recomputed
//             from the saved pre-BN input, so the BN output is never saved), S1 = sum g, S2 = sum g x per block; the last
//             block of each 64-channel chunk sums the blocks' partials in a fixed order: dbeta = S1, dgamma = invstd
//             (S2 - mean S1), into this step's scratch and the .grad slots.  Deterministic; no atomics on activations.
//             pass 2 (apply): dx = gamma invstd (g - dbeta / M - xhat dgamma / M)
// Thread mapping (both directions): a block owns one 64-channel chunk of one segment (blockIdx.y) and 32 row lanes; a
// thread owns 8 consecutive channels, so every load and store is a 16-byte vector (pitches and offsets are multiples
// of 8).
//
// Adaptive average pooling (torch's windows [floor(i H / P), ceil((i + 1) H / P)), which overlap when P does not divide
// H) on NHWC activations; the backward is a gather over the windows that contain each input pixel.
//
// transpose_rows: out[n][b][a] = in[n][a][b].  The auxiliary head flattens its [N, 4, 4, 128] NHWC activation in
// torchvision's NCHW order (a = pixel, b = channel), and the backward is the same kernel with the roles swapped.
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kSegThreads = 256;

DDL_DEVICE void seg_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE void seg_store8(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                                            pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

// the segment of chunk blockIdx.y and the first channel (within the segment) of this thread's 8
DDL_DEVICE const BnSeg& seg_of_block(const BnSegArgs& a, int& c0, int& chunk) {
  int s = 0;
  while (s + 1 < a.n && static_cast<int>(blockIdx.y) >= a.chunk0[s + 1]) ++s;
  chunk = blockIdx.y - a.chunk0[s];
  c0 = chunk * 64 + (threadIdx.x & 7) * 8;
  return a.s[s];
}

template <bool TRAIN>
__global__ void __launch_bounds__(kSegThreads, 4) bn_seg_fwd_kernel(BnSegArgs a) {
  pdl_trigger();
  pdl_wait();
  int c0, chunk;
  const BnSeg& sg = seg_of_block(a, c0, chunk);
  if (c0 >= sg.C) return;
  const int row0 = blockIdx.x * 32 + (threadIdx.x >> 3);
  float scale[8], shift[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + i;
    if (TRAIN) {
      const float inv_n = 1.f / static_cast<float>(a.M);
      const float mean = sg.sum[c] * inv_n;
      const float var = fmaxf(sg.sumsq[c] * inv_n - mean * mean, 0.f);
      const float invstd = rsqrtf(var + sg.eps);
      scale[i] = sg.gamma[c] * invstd;
      shift[i] = sg.beta[c] - mean * scale[i];
      if (row0 == 0) {
        sg.mean[c] = mean;
        sg.invstd[c] = invstd;
        if (sg.running_mean) {
          const float unbiased = a.M > 1 ? var * static_cast<float>(a.M) / static_cast<float>(a.M - 1) : var;
          sg.running_mean[c] = (1.f - sg.momentum) * sg.running_mean[c] + sg.momentum * mean;
          sg.running_var[c] = (1.f - sg.momentum) * sg.running_var[c] + sg.momentum * unbiased;
        }
      }
    } else {
      scale[i] = sg.gamma[c] * rsqrtf(sg.running_var[c] + sg.eps);
      shift[i] = sg.beta[c] - sg.running_mean[c] * scale[i];
    }
  }
  const __nv_bfloat16* x = sg.x + sg.colx + c0;
  __nv_bfloat16* z = sg.z + sg.colz + c0;
  for (int r = row0; r < a.M; r += gridDim.x * 32) {
    float v[8];
    seg_unpack8(ld_stream_u4(x + static_cast<size_t>(r) * sg.ldx), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = fmaxf(fmaf(v[i], scale[i], shift[i]), 0.f);
    seg_store8(z + static_cast<size_t>(r) * sg.ldz, v);
  }
}

__global__ void __launch_bounds__(kSegThreads, 4) bn_seg_bwd_reduce_kernel(BnSegArgs a) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[kSegThreads / 32][8][16];
  __shared__ bool last;
  int c0, chunk;
  const BnSeg& sg = seg_of_block(a, c0, chunk);
  const bool live = c0 < sg.C;
  float s1[8], s2[8], msc[8], msh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    s1[i] = 0.f; s2[i] = 0.f; msc[i] = 0.f; msh[i] = 0.f;
    if (live) {
      msc[i] = sg.gamma[c0 + i] * sg.invstd[c0 + i];
      msh[i] = sg.beta[c0 + i] - sg.mean[c0 + i] * msc[i];
    }
  }
  const __nv_bfloat16* x = sg.x + sg.colx + c0;
  const __nv_bfloat16* dz = sg.dz + sg.coldz + c0;
  for (int r = live ? blockIdx.x * 32 + (threadIdx.x >> 3) : a.M; r < a.M; r += gridDim.x * 32) {
    float g[8], v[8];
    seg_unpack8(ld_stream_u4(dz + static_cast<size_t>(r) * sg.lddz), g);
    seg_unpack8(ld_stream_u4(x + static_cast<size_t>(r) * sg.ldx), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float gi = fmaf(v[i], msc[i], msh[i]) > 0.f ? g[i] : 0.f;
      s1[i] += gi;
      s2[i] = fmaf(gi, v[i], s2[i]);
    }
  }
  // lanes of a warp sharing a channel group: lane = (row lane % 4) * 8 + group -> xor 8, 16
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], off);
      s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], off);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { red[warp][lane][i] = s1[i]; red[warp][lane][8 + i] = s2[i]; }
  }
  __syncthreads();
  float* part = a.partial + (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * 128;
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int w = 0; w < kSegThreads / 32; ++w) { t1 += red[w][g][i]; t2 += red[w][g][8 + i]; }
    part[threadIdx.x] = t1;
    part[64 + threadIdx.x] = t2;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(a.done + blockIdx.y, 1u);
    last = prev == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  // the chunk's last block: sum the blocks' partials in block order (a fixed order: deterministic)
  if (threadIdx.x < 64) {
    const int ch = chunk * 64 + threadIdx.x;
    const float* base = a.partial + static_cast<size_t>(blockIdx.y) * gridDim.x * 128;
    float t1 = 0.f, t2 = 0.f;
    for (unsigned int b = 0; b < gridDim.x; ++b) {
      t1 += __ldcg(base + b * 128 + threadIdx.x);
      t2 += __ldcg(base + b * 128 + 64 + threadIdx.x);
    }
    if (ch < sg.C) {
      const float dg = sg.invstd[ch] * (t2 - sg.mean[ch] * t1);
      sg.dbeta[ch] = t1;
      sg.dgamma[ch] = dg;
      if (sg.gamma_grad) sg.gamma_grad[ch] += dg;
      if (sg.beta_grad) sg.beta_grad[ch] += t1;
    }
  }
  if (threadIdx.x == 0) a.done[blockIdx.y] = 0u;
}

__global__ void __launch_bounds__(kSegThreads, 4) bn_seg_bwd_apply_kernel(BnSegArgs a) {
  pdl_trigger();
  pdl_wait();
  int c0, chunk;
  const BnSeg& sg = seg_of_block(a, c0, chunk);
  if (c0 >= sg.C) return;
  const float inv_n = 1.f / static_cast<float>(a.M);
  float k1[8], cA[8], cB[8], msh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + i;
    const float invstd = sg.invstd[c], mean = sg.mean[c];
    k1[i] = sg.gamma[c] * invstd;
    cB[i] = -k1[i] * invstd * sg.dgamma[c] * inv_n;
    cA[i] = -k1[i] * sg.dbeta[c] * inv_n - mean * cB[i];
    msh[i] = sg.beta[c] - mean * k1[i];
  }
  const __nv_bfloat16* x = sg.x + sg.colx + c0;
  const __nv_bfloat16* dz = sg.dz + sg.coldz + c0;
  __nv_bfloat16* dx = sg.dx + sg.coldx + c0;
  for (int r = blockIdx.x * 32 + (threadIdx.x >> 3); r < a.M; r += gridDim.x * 32) {
    float g[8], v[8];
    seg_unpack8(ld_stream_u4(dz + static_cast<size_t>(r) * sg.lddz), g);
    seg_unpack8(ld_stream_u4(x + static_cast<size_t>(r) * sg.ldx), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float gi = fmaf(v[i], k1[i], msh[i]) > 0.f ? g[i] : 0.f;
      v[i] = fmaf(gi, k1[i], fmaf(v[i], cB[i], cA[i]));
    }
    seg_store8(dx + static_cast<size_t>(r) * sg.lddx, v);
  }
}

// ---- adaptive average pooling ------------------------------------------------------------------
// one thread per (n, p, q, 8-channel group)
__global__ void __launch_bounds__(256) adaptive_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                   __nv_bfloat16* __restrict__ y, int N, int H, int W,
                                                                   int C, int P, int Q) {
  pdl_trigger();
  pdl_wait();
  const int groups = C / 8;
  const int64_t total = static_cast<int64_t>(N) * P * Q * groups;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(t % groups);
    int64_t rest = t / groups;
    const int q = static_cast<int>(rest % Q);
    rest /= Q;
    const int p = static_cast<int>(rest % P);
    const int n = static_cast<int>(rest / P);
    const int h0 = p * H / P, h1 = ((p + 1) * H + P - 1) / P;
    const int w0 = q * W / Q, w1 = ((q + 1) * W + Q - 1) / Q;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int h = h0; h < h1; ++h) {
      for (int w = w0; w < w1; ++w) {
        float v[8];
        seg_unpack8(*reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + h) * W + w) * C + g * 8), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += v[i];
      }
    }
    const float inv = 1.f / static_cast<float>((h1 - h0) * (w1 - w0));
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= inv;
    seg_store8(y + ((static_cast<size_t>(n) * P + p) * Q + q) * C + g * 8, acc);
  }
}

// one thread per (n, h, w, 8-channel group): the windows containing row h are p in [floor(h P / H), ceil((h+1) P / H))
__global__ void __launch_bounds__(256) adaptive_avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                   __nv_bfloat16* __restrict__ dx, int N, int H, int W,
                                                                   int C, int P, int Q) {
  pdl_trigger();
  pdl_wait();
  const int groups = C / 8;
  const int64_t total = static_cast<int64_t>(N) * H * W * groups;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(t % groups);
    int64_t rest = t / groups;
    const int w = static_cast<int>(rest % W);
    rest /= W;
    const int h = static_cast<int>(rest % H);
    const int n = static_cast<int>(rest / H);
    const int p0 = h * P / H, p1 = ((h + 1) * P + H - 1) / H;
    const int q0 = w * Q / W, q1 = ((w + 1) * Q + W - 1) / W;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int p = p0; p < p1; ++p) {
      const int hc = ((p + 1) * H + P - 1) / P - p * H / P;
      for (int q = q0; q < q1; ++q) {
        const int wc = ((q + 1) * W + Q - 1) / Q - q * W / Q;
        const float inv = 1.f / static_cast<float>(hc * wc);
        float v[8];
        seg_unpack8(*reinterpret_cast<const uint4*>(dy + ((static_cast<size_t>(n) * P + p) * Q + q) * C + g * 8), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(v[i], inv, acc[i]);
      }
    }
    seg_store8(dx + ((static_cast<size_t>(n) * H + h) * W + w) * C + g * 8, acc);
  }
}

// ---- out[n][b][a] = in[n][a][b]: one thread per 8 consecutive a of one (n, b) ---------------------
__global__ void __launch_bounds__(256) transpose_rows_kernel(const __nv_bfloat16* __restrict__ in,
                                                             __nv_bfloat16* __restrict__ out, int N, int A, int B) {
  pdl_trigger();
  pdl_wait();
  const int ga = A / 8;
  const int64_t total = static_cast<int64_t>(N) * B * ga;
  const uint16_t* src = reinterpret_cast<const uint16_t*>(in);
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int a0 = static_cast<int>(t % ga) * 8;
    const int64_t nb = t / ga;
    const int b = static_cast<int>(nb % B);
    const int64_t n = nb / B;
    const uint16_t* s = src + (n * A + a0) * B + b;
    uint16_t h[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) h[k] = s[static_cast<int64_t>(k) * B];
    *reinterpret_cast<uint4*>(out + nb * A + a0) =
        make_uint4(h[0] | (static_cast<uint32_t>(h[1]) << 16), h[2] | (static_cast<uint32_t>(h[3]) << 16),
                   h[4] | (static_cast<uint32_t>(h[5]) << 16), h[6] | (static_cast<uint32_t>(h[7]) << 16));
  }
}

unsigned int seg_grid(int64_t work, int sms) {
  int64_t blocks = (work + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sms) * 8;
  if (blocks > cap) blocks = cap;
  return static_cast<unsigned int>(blocks < 1 ? 1 : blocks);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// validates the segments and fills chunk0; returns the number of 64-channel chunks (0: invalid)
int seg_prepare(BnSegArgs& a, bool fwd) {
  if (a.n <= 0 || a.n > kSegMax || a.M <= 0) return 0;
  int chunks = 0;
  for (int s = 0; s < a.n; ++s) {
    const BnSeg& g = a.s[s];
    if (g.C <= 0 || g.C % 8 != 0 || !g.x || !g.gamma || !g.beta || g.ldx % 8 || g.colx % 8 || g.colx + g.C > g.ldx ||
        !aligned16(g.x))
      return 0;
    if (fwd && (!g.z || g.ldz % 8 || g.colz % 8 || g.colz + g.C > g.ldz || !aligned16(g.z))) return 0;
    if (!fwd && (!g.dz || !g.dx || !g.mean || !g.invstd || !g.dgamma || !g.dbeta || g.lddz % 8 || g.coldz % 8 ||
                 g.coldz + g.C > g.lddz || g.lddx % 8 || g.coldx % 8 || g.coldx + g.C > g.lddx || !aligned16(g.dz) ||
                 !aligned16(g.dx)))
      return 0;
    a.chunk0[s] = chunks;
    chunks += (g.C + 63) / 64;
  }
  a.chunk0[a.n] = chunks;
  return chunks;
}

}  // namespace

int bn_seg_grid_x(int M, int chunks, int sms) {
  int gx = (M + 32 * 8 - 1) / (32 * 8);
  const int cap = (sms * 8 + chunks - 1) / chunks;
  if (gx > cap) gx = cap;
  return gx < 1 ? 1 : gx;
}

cudaError_t launch_bn_seg_fwd(BnSegArgs a, bool train, int sms, cudaStream_t stream) {
  const int chunks = seg_prepare(a, true);
  if (chunks == 0) return cudaErrorInvalidValue;
  for (int s = 0; s < a.n; ++s) {
    const BnSeg& g = a.s[s];
    if (train ? (!g.sum || !g.sumsq || !g.mean || !g.invstd) : (!g.running_mean || !g.running_var))
      return cudaErrorInvalidValue;
  }
  const dim3 grid(bn_seg_grid_x(a.M, chunks, sms), chunks);
  return train ? launch_pdl(bn_seg_fwd_kernel<true>, grid, dim3(kSegThreads), 0, stream, 1, a)
               : launch_pdl(bn_seg_fwd_kernel<false>, grid, dim3(kSegThreads), 0, stream, 1, a);
}

cudaError_t launch_bn_seg_bwd(BnSegArgs a, int grid_x, cudaStream_t stream) {
  const int chunks = seg_prepare(a, false);
  if (chunks == 0 || grid_x <= 0 || !a.partial || !a.done) return cudaErrorInvalidValue;
  const dim3 grid(grid_x, chunks);
  const cudaError_t e = launch_pdl(bn_seg_bwd_reduce_kernel, grid, dim3(kSegThreads), 0, stream, 1, a);
  if (e != cudaSuccess) return e;
  return launch_pdl(bn_seg_bwd_apply_kernel, grid, dim3(kSegThreads), 0, stream, 1, a);
}

cudaError_t launch_adaptive_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int N, int H, int W, int C, int P,
                                        int Q, int sms, cudaStream_t stream) {
  if (C % 8 != 0 || P <= 0 || Q <= 0 || P > H || Q > W || !aligned16(x) || !aligned16(y)) return cudaErrorInvalidValue;
  return launch_pdl(adaptive_avgpool_fwd_kernel, dim3(seg_grid(static_cast<int64_t>(N) * P * Q * (C / 8), sms)),
                    dim3(256), 0, stream, 1, x, y, N, H, W, C, P, Q);
}

cudaError_t launch_adaptive_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int N, int H, int W, int C, int P,
                                        int Q, int sms, cudaStream_t stream) {
  if (C % 8 != 0 || P <= 0 || Q <= 0 || P > H || Q > W || !aligned16(dy) || !aligned16(dx)) return cudaErrorInvalidValue;
  return launch_pdl(adaptive_avgpool_bwd_kernel, dim3(seg_grid(static_cast<int64_t>(N) * H * W * (C / 8), sms)),
                    dim3(256), 0, stream, 1, dy, dx, N, H, W, C, P, Q);
}

cudaError_t launch_transpose_rows(const __nv_bfloat16* in, __nv_bfloat16* out, int N, int A, int B, int sms,
                                  cudaStream_t stream) {
  if (N <= 0 || A <= 0 || B <= 0 || A % 8 != 0 || !aligned16(out)) return cudaErrorInvalidValue;
  return launch_pdl(transpose_rows_kernel, dim3(seg_grid(static_cast<int64_t>(N) * B * (A / 8), sms)), dim3(256), 0,
                    stream, 1, in, out, N, A, B);
}

}  // namespace ddl
