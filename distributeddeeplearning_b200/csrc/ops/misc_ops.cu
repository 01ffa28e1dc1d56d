// Memory-bound support kernels (NHWC bf16): pooling, fused softmax-cross-entropy(+top-k), Philox
// synthetic data, layout/dtype conversion, bias/ReLU backward, dropout.
// Reference op inventory: SURVEY.md K1 (synthetic batch), K8 (max-pool), K9 (avg-pool), K11
// (cross-entropy), K17 (accuracy), K20 (bias / dropout), K21 (normalise + layout convert).
#include "../common.cuh"
#include "ops.h"

namespace ddl {
namespace {

DDL_DEVICE void unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE uint4 pack8(const float (&v)[8]) {
  return make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

// ---------------------------------------------------------------------------------------------
// channel statistics (fallback when the producer did not fuse them)
// ---------------------------------------------------------------------------------------------
// block = one 64-channel chunk (blockIdx.y) x 32 row lanes; thread = 8 channels of one row lane (any C % 8 == 0)
__global__ void __launch_bounds__(256) channel_stats_kernel(const __nv_bfloat16* __restrict__ x, float* sum,
                                                            float* sumsq, int M, int C) {
  const int cgl = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + cgl * 8;
  const bool live = c0 < C;
  float s[8], ss[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; ss[i] = 0.f; }
  for (int r = live ? blockIdx.x * 32 + rl : M; r < M; r += gridDim.x * 32) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(x + static_cast<size_t>(r) * C + c0), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] += v[i]; ss[i] = fmaf(v[i], v[i], ss[i]); }
  }
  // lanes of a warp sharing a channel group: lane = (rl % 4) * 8 + cgl -> xor 8, 16
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i] += __shfl_xor_sync(0xffffffffu, s[i], off);
      ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], off);
    }
  }
  __shared__ float red[8][8][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { red[warp][lane][i] = s[i]; red[warp][lane][8 + i] = ss[i]; }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) { t1 += red[w][g][i]; t2 += red[w][g][8 + i]; }
    const int ch = blockIdx.y * 64 + g * 8 + i;
    if (ch < C) {
      atomicAdd(sum + ch, t1);
      atomicAdd(sumsq + ch, t2);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// pooling: one thread = one output (or input) pixel x 8 channels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* y,
                                                          uint8_t* argmax, PoolArgs p) {
  const int groups = p.C / 8;
  const int64_t total = static_cast<int64_t>(p.N) * p.P * p.Q * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t pix = idx / groups;
    const int q = pix % p.Q; pix /= p.Q;
    const int pp = pix % p.P;
    const int n = pix / p.P;
    float best[8];
    int bi[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; bi[i] = 0; }
    for (int r = 0; r < p.k; ++r) {
      const int h = pp * p.stride - p.pad + r;
      if (h < 0 || h >= p.H) continue;
      for (int s = 0; s < p.k; ++s) {
        const int w = q * p.stride - p.pad + s;
        if (w < 0 || w >= p.W) continue;
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * p.C + g * 8), v);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (v[i] > best[i]) { best[i] = v[i]; bi[i] = r * p.k + s; }
      }
    }
    const size_t o = ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * p.C + g * 8;
    *reinterpret_cast<uint4*>(y + o) = pack8(best);
    if (argmax) {
      uint2 a;
      a.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
      a.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
      *reinterpret_cast<uint2*>(argmax + o) = a;
    }
  }
}

// gather formulation: each INPUT pixel sums the dy of the windows whose arg-max it is (no atomics)
// 3x3 / stride 2 / pad 1 forward (the ResNet / DenseNet stem pool): all nine 16-byte window loads of a thread are issued
// before the first compare (the generic kernel's tap loop exposes one L2 round trip per tap on the ~565 MB this layer
// moves at batch 256).  Out-of-image taps load nothing and can never win.
__global__ void __launch_bounds__(256) maxpool_fwd_k3s2_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* y,
                                                               uint8_t* argmax, PoolArgs p) {
  const int groups = p.C / 8;
  const int64_t total = static_cast<int64_t>(p.N) * p.P * p.Q * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t pix = idx / groups;
    const int q = pix % p.Q; pix /= p.Q;
    const int pp = pix % p.P;
    const int n = pix / p.P;
    const int h0 = pp * 2 - 1, w0 = q * 2 - 1;
    const __nv_bfloat16* base = x + (static_cast<size_t>(n) * p.H * p.W) * p.C + g * 8;
    uint4 t[9];
    bool ok[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int h = h0 + r, w = w0 + s;
        ok[r * 3 + s] = h >= 0 && h < p.H && w >= 0 && w < p.W;
        t[r * 3 + s] = ok[r * 3 + s] ? __ldg(reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h) * p.W + w) * p.C))
                                     : make_uint4(0, 0, 0, 0);
      }
    float best[8];
    int bi[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; bi[i] = 0; }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (!ok[k]) continue;
      float v[8];
      unpack8(t[k], v);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (v[i] > best[i]) { best[i] = v[i]; bi[i] = k; }
    }
    const size_t o = ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * p.C + g * 8;
    *reinterpret_cast<uint4*>(y + o) = pack8(best);
    if (argmax) {
      uint2 a;
      a.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
      a.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
      *reinterpret_cast<uint2*>(argmax + o) = a;
    }
  }
}

__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                          const uint8_t* __restrict__ argmax, __nv_bfloat16* dx,
                                                          PoolArgs p) {
  const int groups = p.C / 8;
  const int64_t total = static_cast<int64_t>(p.N) * p.H * p.W * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t pix = idx / groups;
    const int w = pix % p.W; pix /= p.W;
    const int h = pix % p.H;
    const int n = pix / p.H;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    // windows (pp, q) covering (h, w): pp*stride - pad + r == h with 0 <= r < k  ->  at most ceil(k/stride) per axis
    const int pp_hi = (h + p.pad) / p.stride, q_hi = (w + p.pad) / p.stride;
    for (int pp = pp_hi; pp >= 0; --pp) {
      const int r = h + p.pad - pp * p.stride;
      if (r >= p.k) break;
      if (pp >= p.P) continue;
      for (int q = q_hi; q >= 0; --q) {
        const int s = w + p.pad - q * p.stride;
        if (s >= p.k) break;
        if (q >= p.Q) continue;
        const size_t o = ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * p.C + g * 8;
        const uint2 am = *reinterpret_cast<const uint2*>(argmax + o);
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + o), v);
        const int code = r * p.k + s;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int a = ((i < 4 ? am.x : am.y) >> (8 * (i & 3))) & 0xff;
          if (a == code) acc[i] += v[i];
        }
      }
    }
    *reinterpret_cast<uint4*>(dx + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * p.C + g * 8) = pack8(acc);
  }
}

// 3x3 / stride 2 / pad 1 specialisation (ResNet / DenseNet stem; H, W even): one thread = one 2x2 patch of input
// pixels x 8 channels.  The patch is covered by exactly the 4 windows (a..a+1, b..b+1), each loaded ONCE; which window
// tap lands on which of the 4 pixels is a compile-time table, so the generic kernel's index arithmetic and its
// 2.25 window visits per pixel (it was instruction-bound at ~22 % of the HBM roofline) collapse into 4 loads + 9 compares.
__global__ void __launch_bounds__(256) maxpool_bwd_k3s2_kernel(const __nv_bfloat16* __restrict__ dy,
                                                               const uint8_t* __restrict__ argmax, __nv_bfloat16* dx,
                                                               PoolArgs p) {
  const int groups = p.C / 8;
  const int H2 = p.H / 2, W2 = p.W / 2;
  const int64_t total = static_cast<int64_t>(p.N) * H2 * W2 * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t t = idx / groups;
    const int b = t % W2; t /= W2;
    const int a = t % H2;
    const int n = t / H2;
    float o00[8], o01[8], o10[8], o11[8];       // gradients of pixels (2a, 2b), (2a, 2b+1), (2a+1, 2b), (2a+1, 2b+1)
#pragma unroll
    for (int i = 0; i < 8; ++i) { o00[i] = 0.f; o01[i] = 0.f; o10[i] = 0.f; o11[i] = 0.f; }
    // the four windows that touch this 2x2 patch: all eight loads in flight before anything is consumed
    uint4 gv[4];
    uint2 av[4];
    bool live[4];
#pragma unroll
    for (int w4 = 0; w4 < 4; ++w4) {
      const int pp = a + (w4 >> 1), q = b + (w4 & 1);
      live[w4] = pp < p.P && q < p.Q;
      const size_t o = ((static_cast<size_t>(n) * p.P + (live[w4] ? pp : 0)) * p.Q + (live[w4] ? q : 0)) * p.C + g * 8;
      gv[w4] = live[w4] ? ld_stream_u4(dy + o) : make_uint4(0, 0, 0, 0);
      av[w4] = live[w4] ? ld_stream_u2(argmax + o) : make_uint2(0xffffffffu, 0xffffffffu);
    }
#pragma unroll
    for (int dp = 0; dp < 2; ++dp) {
#pragma unroll
      for (int dq = 0; dq < 2; ++dq) {
        if (!live[dp * 2 + dq]) continue;
        const uint2 am = av[dp * 2 + dq];
        float v[8];
        unpack8(gv[dp * 2 + dq], v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int code = ((i < 4 ? am.x : am.y) >> (8 * (i & 3))) & 0xff;      // r * 3 + s of the arg-max tap
          // window (a + dp, b + dq) touches patch pixel (y, x) with tap r = 2*(y - dp) + 1 - ... (table below)
          if (dp == 0 && dq == 0) {
            if (code == 4) o00[i] += v[i]; else if (code == 5) o01[i] += v[i];
            else if (code == 7) o10[i] += v[i]; else if (code == 8) o11[i] += v[i];
          } else if (dp == 0 && dq == 1) {
            if (code == 3) o01[i] += v[i]; else if (code == 6) o11[i] += v[i];
          } else if (dp == 1 && dq == 0) {
            if (code == 1) o10[i] += v[i]; else if (code == 2) o11[i] += v[i];
          } else {
            if (code == 0) o11[i] += v[i];
          }
        }
      }
    }
    const size_t base = ((static_cast<size_t>(n) * p.H + 2 * a) * p.W + 2 * b) * p.C + g * 8;
    *reinterpret_cast<uint4*>(dx + base) = pack8(o00);
    *reinterpret_cast<uint4*>(dx + base + p.C) = pack8(o01);
    *reinterpret_cast<uint4*>(dx + base + static_cast<size_t>(p.W) * p.C) = pack8(o10);
    *reinterpret_cast<uint4*>(dx + base + static_cast<size_t>(p.W + 1) * p.C) = pack8(o11);
  }
}

__global__ void __launch_bounds__(256) avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* y,
                                                          PoolArgs p, int count_include_pad) {
  const int groups = p.C / 8;
  const int64_t total = static_cast<int64_t>(p.N) * p.P * p.Q * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t pix = idx / groups;
    const int q = pix % p.Q; pix /= p.Q;
    const int pp = pix % p.P;
    const int n = pix / p.P;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    int cnt = 0;
    for (int r = 0; r < p.k; ++r) {
      const int h = pp * p.stride - p.pad + r;
      if (h < 0 || h >= p.H) continue;
      for (int s = 0; s < p.k; ++s) {
        const int w = q * p.stride - p.pad + s;
        if (w < 0 || w >= p.W) continue;
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * p.C + g * 8), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] += v[i];
        ++cnt;
      }
    }
    const float inv = 1.f / static_cast<float>(count_include_pad ? p.k * p.k : max(cnt, 1));
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= inv;
    *reinterpret_cast<uint4*>(y + ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * p.C + g * 8) = pack8(acc);
  }
}

__global__ void __launch_bounds__(256) avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* dx,
                                                          PoolArgs p, int count_include_pad) {
  const int groups = p.C / 8;
  const int64_t total = static_cast<int64_t>(p.N) * p.H * p.W * groups;
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    int64_t pix = idx / groups;
    const int w = pix % p.W; pix /= p.W;
    const int h = pix % p.H;
    const int n = pix / p.H;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int r = 0; r < p.k; ++r) {
      const int th = h + p.pad - r;
      if (th < 0 || th % p.stride != 0) continue;
      const int pp = th / p.stride;
      if (pp >= p.P) continue;
      for (int s = 0; s < p.k; ++s) {
        const int tw = w + p.pad - s;
        if (tw < 0 || tw % p.stride != 0) continue;
        const int q = tw / p.stride;
        if (q >= p.Q) continue;
        float inv;
        if (count_include_pad) {
          inv = 1.f / static_cast<float>(p.k * p.k);
        } else {
          const int h0 = max(pp * p.stride - p.pad, 0), h1 = min(pp * p.stride - p.pad + p.k, p.H);
          const int w0 = max(q * p.stride - p.pad, 0), w1 = min(q * p.stride - p.pad + p.k, p.W);
          inv = 1.f / static_cast<float>(max((h1 - h0) * (w1 - w0), 1));
        }
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(dy + ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * p.C + g * 8), v);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(v[i], inv, acc[i]);
      }
    }
    *reinterpret_cast<uint4*>(dx + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * p.C + g * 8) = pack8(acc);
  }
}

__global__ void __launch_bounds__(256) global_avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                 __nv_bfloat16* y, int N, int HW, int C) {
  const int groups = C / 8;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * groups) return;
  const int g = idx % groups, n = idx / groups;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const __nv_bfloat16* base = x + static_cast<size_t>(n) * HW * C + g * 8;
  for (int t = 0; t < HW; ++t) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(base + static_cast<size_t>(t) * C), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] += v[i];
  }
  const float inv = 1.f / static_cast<float>(HW);
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] *= inv;
  *reinterpret_cast<uint4*>(y + static_cast<size_t>(n) * C + g * 8) = pack8(acc);
}

__global__ void __launch_bounds__(256) global_avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                 __nv_bfloat16* dx, int N, int HW, int C) {
  const int groups = C / 8;
  const int64_t total = static_cast<int64_t>(N) * HW * groups;
  const float inv = 1.f / static_cast<float>(HW);
  for (int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = idx % groups;
    const int64_t pix = idx / groups;
    const int n = pix / HW;
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(dy + static_cast<size_t>(n) * C + g * 8), v);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] *= inv;
    *reinterpret_cast<uint4*>(dx + static_cast<size_t>(pix) * C + g * 8) = pack8(v);
  }
}

// ---------------------------------------------------------------------------------------------
// fused softmax cross-entropy forward + backward + top-1/top-5: one warp per sample
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) softmax_xent_kernel(XentArgs a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.B) return;
  const __nv_bfloat16* row = a.logits + static_cast<size_t>(warp) * a.ld;
  const int label = static_cast<int>(a.labels[warp]);
  float mx = -INFINITY;
  for (int c = lane; c < a.classes; c += 32) mx = fmaxf(mx, __bfloat162float(row[c]));
  mx = warp_max(mx);
  float se = 0.f;
  for (int c = lane; c < a.classes; c += 32) se += __expf(__bfloat162float(row[c]) - mx);
  se = warp_sum(se);
  const float xl = __bfloat162float(row[label]);
  const float lse = mx + __logf(se);
  const float loss = lse - xl;
  if (a.correct) {
    // rank of the label logit: number of classes with a strictly larger logit (ties: lower index wins)
    int larger = 0;
    for (int c = lane; c < a.classes; c += 32) {
      const float v = __bfloat162float(row[c]);
      larger += (v > xl) || (v == xl && c < label);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) larger += __shfl_xor_sync(0xffffffffu, larger, o);
    if (lane == 0) {
      if (larger < 1) atomicAdd(a.correct, 1);
      if (larger < 5) atomicAdd(a.correct + 1, 1);
    }
  }
  if (lane == 0) {
    if (a.per_sample) a.per_sample[warp] = loss;
    if (a.loss_sum) atomicAdd(a.loss_sum, loss * a.loss_scale);
  }
  if (a.dlogits) {
    __nv_bfloat16* drow = a.dlogits + static_cast<size_t>(warp) * a.ld;
    const float inv = 1.f / se;
    for (int c = lane; c < a.ld; c += 32) {
      float g = 0.f;
      if (c < a.classes) {
        g = __expf(__bfloat162float(row[c]) - mx) * inv;
        if (c == label) g -= 1.f;
        g *= a.grad_scale;
      }
      drow[c] = __float2bfloat16_rn(g);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Philox synthetic data (K1): normal(0,1) NHWC images, uniform labels
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) philox_normal_nhwc_kernel(__nv_bfloat16* out, int64_t pixels, int c_valid,
                                                                 int cpad, uint64_t seed, uint64_t offset) {
  // one Philox block (4 normals) per pixel; channels beyond c_valid are zero (cpad <= 4)
  const uint2 key = make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < pixels;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint64_t ctr = offset + static_cast<uint64_t>(i);
    const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x4e48u, 0), key);
    const float2 n0 = box_muller(r.x, r.y), n1 = box_muller(r.z, r.w);
    float v[4] = {n0.x, n0.y, n1.x, n1.y};
    for (int c = 0; c < cpad; ++c) out[i * cpad + c] = __float2bfloat16_rn(c < c_valid ? v[c] : 0.f);
  }
}

__global__ void __launch_bounds__(256) philox_labels_kernel(int64_t* out, int64_t n, int classes, uint64_t seed,
                                                            uint64_t offset) {
  const uint2 key = make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t ctr = offset + static_cast<uint64_t>(i);
  const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x4c42u, 0), key);
  out[i] = static_cast<int64_t>(r.x % static_cast<uint32_t>(classes));
}

// ---------------------------------------------------------------------------------------------
// layout / dtype
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nchw_to_nhwc_norm_kernel(const float* __restrict__ in, __nv_bfloat16* out,
                                                                int N, int C, int H, int W, int cpad,
                                                                const float* mean, const float* stdv) {
  const int64_t total = static_cast<int64_t>(N) * H * W;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t hw = i % (static_cast<int64_t>(H) * W);
    const int64_t n = i / (static_cast<int64_t>(H) * W);
    for (int c = 0; c < cpad; ++c) {
      float v = 0.f;
      if (c < C) {
        v = in[(n * C + c) * static_cast<int64_t>(H) * W + hw];
        if (mean) v = (v - mean[c]) / stdv[c];
      }
      out[i * cpad + c] = __float2bfloat16_rn(v);
    }
  }
}

// uint8 NHWC3 (decoded image bytes) -> bf16 NHWC4, (x/255 - mean) / std, 4 pixels per thread
__global__ void __launch_bounds__(256) nhwc_u8_to_nhwc4_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* out,
                                                               int64_t pixels, const float* mean, const float* stdv) {
  float m[3] = {0.f, 0.f, 0.f}, is[3] = {1.f / 255.f, 1.f / 255.f, 1.f / 255.f};
  if (mean) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { m[c] = mean[c]; is[c] = 1.f / (255.f * stdv[c]); }
  }
  const int64_t quads = pixels / 4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < quads;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    // 4 pixels = 12 bytes in, 32 bytes out
    const uint32_t* src = reinterpret_cast<const uint32_t*>(in + i * 12);
    const uint32_t w0 = src[0], w1 = src[1], w2 = src[2];
    const uint8_t b[12] = {uint8_t(w0), uint8_t(w0 >> 8), uint8_t(w0 >> 16), uint8_t(w0 >> 24),
                           uint8_t(w1), uint8_t(w1 >> 8), uint8_t(w1 >> 16), uint8_t(w1 >> 24),
                           uint8_t(w2), uint8_t(w2 >> 8), uint8_t(w2 >> 16), uint8_t(w2 >> 24)};
    uint32_t o[8];
#pragma unroll
    for (int px = 0; px < 4; ++px) {
      const float r = b[3 * px] * is[0] - m[0] * is[0] * 255.f;
      const float g = b[3 * px + 1] * is[1] - m[1] * is[1] * 255.f;
      const float bl = b[3 * px + 2] * is[2] - m[2] * is[2] * 255.f;
      o[2 * px] = pack_bf16x2(r, g);
      o[2 * px + 1] = pack_bf16x2(bl, 0.f);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + i * 16);
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
  // tail (pixels % 4)
  if (blockIdx.x == 0 && threadIdx.x < (pixels & 3)) {
    const int64_t px = quads * 4 + threadIdx.x;
    for (int c = 0; c < 4; ++c) {
      float v = 0.f;
      if (c < 3) v = in[px * 3 + c] * is[c] - m[c] * is[c] * 255.f;
      out[px * 4 + c] = __float2bfloat16_rn(v);
    }
  }
}

__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* out,
                                                            int64_t n) {
  const int64_t n4 = n / 4;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    reinterpret_cast<uint2*>(out)[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) out[n4 * 4 + threadIdx.x] = __float2bfloat16_rn(in[n4 * 4 + threadIdx.x]);
}

// w: fp32 KRSC [Cout][R][S][Cin] ; packed: bf16 [Cout][RP][SP][4], zero padded (RP >= R, SP >= S)
__global__ void pack_stem_weight_kernel(const float* __restrict__ w, __nv_bfloat16* packed, int Cout, int R, int S,
                                        int Cin, int RP, int SP) {
  const int total = Cout * RP * SP * 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    // packed index = ((co * KB + j) * SP + s) * RPK*4 + g*4 + c  with filter row r = j*RPK + g: inside a k-block the
    // order is (tap, row-in-block, channel) — the order in which the row-interleaved stem image (pad_nhwc4) lays out
    // the 128 bytes one output pixel needs, so a single contiguous TMA box yields the operand row
    const int RPK = 16 / SP;
    const int c = i & 3;
    int t = i >> 2;
    const int g = t % RPK; t /= RPK;
    const int s = t % SP; t /= SP;
    const int j = t % (RP / RPK);
    const int co = t / (RP / RPK);
    const int r = j * RPK + g;
    float v = 0.f;
    if (c < Cin && s < S && r < R) v = w[((co * R + r) * S + s) * Cin + c];
    packed[i] = __float2bfloat16_rn(v);
  }
}
__global__ void unpack_stem_grad_kernel(const float* __restrict__ packed, float* gw, int Cout, int R, int S, int Cin,
                                        int RP, int SP) {
  const int total = Cout * R * S * Cin;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i % Cin;
    int t = i / Cin;
    const int s = t % S; t /= S;
    const int r = t % R;
    const int co = t / R;
    const int RPK = 16 / SP, j = r / RPK, g = r - j * RPK;
    gw[i] += packed[(((co * (RP / RPK) + j) * SP + s) * RPK + g) * 4 + c];
  }
}

// ---------------------------------------------------------------------------------------------
// bias / relu backward, dropout, add
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bias_relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                            const __nv_bfloat16* __restrict__ z, __nv_bfloat16* dx,
                                                            float* dbias, int M, int C, int c_valid, int relu) {
  const int groups = C / 8;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int g = tid % groups, row0 = tid / groups;
  const int row_stride = (gridDim.x * blockDim.x) / groups;
  float s[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) s[i] = 0.f;
  for (int r = row0; r < M; r += row_stride) {
    const size_t off = static_cast<size_t>(r) * C + g * 8;
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(dy + off), v);
    if (relu) {
      float zz[8];
      unpack8(*reinterpret_cast<const uint4*>(z + off), zz);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = zz[i] > 0.f ? v[i] : 0.f;
      *reinterpret_cast<uint4*>(dx + off) = pack8(v);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i] += v[i];
  }
  if (dbias) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (g * 8 + i < c_valid) atomicAdd(dbias + g * 8 + i, s[i]);
  }
}

__global__ void __launch_bounds__(256) dropout_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* y,
                                                      int64_t n8, float p, uint64_t seed, uint64_t offset,
                                                      const int64_t* __restrict__ step) {
  // mask is a pure function of (seed, step, offset, element index): backward recomputes it (no mask tensor).
  // `step` is an optional device-resident counter advanced once per training step: it keeps the masks fresh when the
  // whole step — launch arguments included — is replayed from a CUDA graph.
  const uint64_t sd = seed + (step ? static_cast<uint64_t>(*step) * 0x9E3779B97F4A7C15ull : 0ull);
  const uint2 key = make_uint2(static_cast<uint32_t>(sd), static_cast<uint32_t>(sd >> 32));
  const float scale = 1.f / (1.f - p);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint64_t ctr = offset + static_cast<uint64_t>(i);
    const uint4 r0 = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x4450u, 0), key);
    const uint4 r1 = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x4450u, 1), key);
    const uint32_t rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
    float v[8];
    unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = (u32_to_unit(rr[k]) > p) ? v[k] * scale : 0.f;
    reinterpret_cast<uint4*>(y)[i] = pack8(v);
  }
}

__global__ void __launch_bounds__(256) add_bf16_kernel(const __nv_bfloat16* __restrict__ a,
                                                       const __nv_bfloat16* __restrict__ b, __nv_bfloat16* y,
                                                       int64_t n8) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float u[8], v[8];
    unpack8(reinterpret_cast<const uint4*>(a)[i], u);
    unpack8(reinterpret_cast<const uint4*>(b)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) u[k] += v[k];
    reinterpret_cast<uint4*>(y)[i] = pack8(u);
  }
}

// hardswish on a [B][F] activation (MobileNetV3's classifier): y = x * clamp(x + 3, 0, 6) / 6, and its backward from the
// saved pre-activation x: dx = dy * (0 for x <= -3, x / 3 + 1/2 for -3 < x < 3, 1 for x >= 3)
__global__ void __launch_bounds__(256) hardswish_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* y,
                                                            int64_t n8) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float v[8];
    unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = v[k] * fminf(fmaxf(v[k] + 3.f, 0.f), 6.f) * (1.f / 6.f);
    reinterpret_cast<uint4*>(y)[i] = pack8(v);
  }
}

__global__ void __launch_bounds__(256) hardswish_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                            const __nv_bfloat16* __restrict__ x, __nv_bfloat16* dx,
                                                            int64_t n8) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float d[8], v[8];
    unpack8(reinterpret_cast<const uint4*>(dy)[i], d);
    unpack8(reinterpret_cast<const uint4*>(x)[i], v);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = v[k] <= -3.f ? 0.f : (v[k] >= 3.f ? d[k] : d[k] * fmaf(v[k], 1.f / 3.f, 0.5f));
    reinterpret_cast<uint4*>(dx)[i] = pack8(d);
  }
}

// SiLU on the rows of a small bf16 matrix (EfficientNet's squeeze-excitation fc1 output [N][ldx]): y = x * sigmoid(x) into
// [N][ldy] (ldy <= ldx: the next GEMM's K), and its backward from the saved x into a zero-padded GEMM operand
// [N][ldx]: dx = dy * s * (1 + x * (1 - s)) for columns < c_valid, 0 beyond.  One thread per 8-column vector.
__global__ void __launch_bounds__(256) silu_rows_fwd_kernel(const __nv_bfloat16* __restrict__ x, int ldx,
                                                            __nv_bfloat16* __restrict__ y, int ldy, int64_t total) {
  const int g8 = ldy / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = i / g8;
    const int c = static_cast<int>(i % g8) * 8;
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(x + n * ldx + c), v);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = v[k] / (1.f + __expf(-v[k]));
    *reinterpret_cast<uint4*>(y + n * ldy + c) = pack8(v);
  }
}

__global__ void __launch_bounds__(256) silu_rows_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int ldy,
                                                            const __nv_bfloat16* __restrict__ x, int ldx,
                                                            __nv_bfloat16* __restrict__ dx, int c_valid, int64_t total) {
  const int g8 = ldx / 8;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t n = i / g8;
    const int c = static_cast<int>(i % g8) * 8;
    float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < c_valid) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(x + n * ldx + c), v);
      unpack8(*reinterpret_cast<const uint4*>(dy + n * ldy + c), d);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float sg = 1.f / (1.f + __expf(-v[k]));
        d[k] = c + k < c_valid ? d[k] * sg * fmaf(v[k], 1.f - sg, 1.f) : 0.f;
      }
    }
    *reinterpret_cast<uint4*>(dx + n * ldx + c) = pack8(d);
  }
}

// stochastic depth ("row" mode): one keep scale per sample, 0 or 1 / (1 - p), from the dropout Philox stream (same key
// and device step counter as dropout_kernel, its own counter word) so that CUDA-graph replays draw fresh vectors
__global__ void __launch_bounds__(256) stochastic_depth_keep_kernel(float* __restrict__ keep, int n, float p,
                                                                    uint64_t seed, uint64_t offset,
                                                                    const int64_t* __restrict__ step) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t sd = seed + (step ? static_cast<uint64_t>(*step) * 0x9E3779B97F4A7C15ull : 0ull);
  const uint2 key = make_uint2(static_cast<uint32_t>(sd), static_cast<uint32_t>(sd >> 32));
  const uint64_t ctr = offset + static_cast<uint64_t>(i);
  const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x5344u, 0), key);
  keep[i] = u32_to_unit(r.x) > p ? 1.f / (1.f - p) : 0.f;
}

inline int grid_for(int64_t work, int per_block = 256, int cap = 132 * 16) {     // 16 blocks per SM of an H100 SXM
  int64_t b = (work + per_block - 1) / per_block;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

// out[n][h][w][g][0..3] = in[n][h - pt + g][w - pl][0..3] (zero outside the source image), g < G
__global__ void __launch_bounds__(256) pad_nhwc4_kernel(const uint2* __restrict__ in, uint2* __restrict__ out, int N,
                                                        int H, int W, int Hp, int Wp, int pt, int pl, int G) {
  const int64_t total = static_cast<int64_t>(N) * Hp * Wp * G;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(i % G);
    int64_t t = i / G;
    const int w = static_cast<int>(t % Wp); t /= Wp;
    const int h = static_cast<int>(t % Hp);
    const int64_t n = t / Hp;
    const int sh = h - pt + g, sw = w - pl;
    uint2 v = make_uint2(0u, 0u);
    if (sh >= 0 && sh < H && sw >= 0 && sw < W) v = in[(n * H + sh) * W + sw];
    out[i] = v;
  }
}

// one thread = one 16-byte vector of the concatenated row; the part is found by walking the (<= 8) channel counts
template <bool SCATTER>
__global__ void __launch_bounds__(256) concat_channels_kernel(CatArgs a) {
  const int groups = a.ctot / 8;
  const int64_t total = static_cast<int64_t>(a.M) * groups;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t row = i / groups;
    int ch = static_cast<int>(i - row * groups) * 8;
    int p = 0;
#pragma unroll
    for (int k = 0; k < kCatMax - 1; ++k)
      if (p < a.n - 1 && ch >= a.c[p]) { ch -= a.c[p]; ++p; }
    uint4* w = reinterpret_cast<uint4*>(a.whole) + i;
    uint4* q = reinterpret_cast<uint4*>(a.part[p] + row * a.c[p] + ch);
    if (SCATTER) *q = *w;
    else *w = *q;
  }
}

}  // namespace

cudaError_t launch_channel_stats(const __nv_bfloat16* x, float* sum, float* sumsq, int M, int C, int sms,
                                 cudaStream_t stream) {
  if (C % 8 != 0 || C <= 0) return cudaErrorInvalidValue;
  const int chunks = (C + 63) / 64;
  int gx = (M + 32 * 8 - 1) / (32 * 8);
  const int cap = (sms * 8 + chunks - 1) / chunks;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  channel_stats_kernel<<<dim3(gx, chunks), 256, 0, stream>>>(x, sum, sumsq, M, C);
  return cudaGetLastError();
}

cudaError_t launch_maxpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* argmax, const PoolArgs& p,
                               cudaStream_t stream) {
  if (p.C % 8 != 0) return cudaErrorInvalidValue;
  if (p.k == 3 && p.stride == 2 && p.pad == 1)
    maxpool_fwd_k3s2_kernel<<<grid_for(static_cast<int64_t>(p.N) * p.P * p.Q * (p.C / 8)), 256, 0, stream>>>(x, y, argmax, p);
  else
    maxpool_fwd_kernel<<<grid_for(static_cast<int64_t>(p.N) * p.P * p.Q * (p.C / 8)), 256, 0, stream>>>(x, y, argmax, p);
  return cudaGetLastError();
}
cudaError_t launch_maxpool_bwd(const __nv_bfloat16* dy, const uint8_t* argmax, __nv_bfloat16* dx, const PoolArgs& p,
                               cudaStream_t stream) {
  if (p.C % 8 != 0) return cudaErrorInvalidValue;
  if (p.k == 3 && p.stride == 2 && p.pad == 1 && p.H % 2 == 0 && p.W % 2 == 0 && p.P == p.H / 2 && p.Q == p.W / 2) {
    maxpool_bwd_k3s2_kernel<<<grid_for(static_cast<int64_t>(p.N) * (p.H / 2) * (p.W / 2) * (p.C / 8)), 256, 0, stream>>>(
        dy, argmax, dx, p);
    return cudaGetLastError();
  }
  maxpool_bwd_kernel<<<grid_for(static_cast<int64_t>(p.N) * p.H * p.W * (p.C / 8)), 256, 0, stream>>>(dy, argmax, dx, p);
  return cudaGetLastError();
}
cudaError_t launch_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, const PoolArgs& p, int count_include_pad,
                               cudaStream_t stream) {
  if (p.C % 8 != 0) return cudaErrorInvalidValue;
  avgpool_fwd_kernel<<<grid_for(static_cast<int64_t>(p.N) * p.P * p.Q * (p.C / 8)), 256, 0, stream>>>(x, y, p, count_include_pad);
  return cudaGetLastError();
}
cudaError_t launch_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, const PoolArgs& p, int count_include_pad,
                               cudaStream_t stream) {
  if (p.C % 8 != 0) return cudaErrorInvalidValue;
  avgpool_bwd_kernel<<<grid_for(static_cast<int64_t>(p.N) * p.H * p.W * (p.C / 8)), 256, 0, stream>>>(dy, dx, p, count_include_pad);
  return cudaGetLastError();
}
cudaError_t launch_global_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int N, int HW, int C,
                                      cudaStream_t stream) {
  if (C % 8 != 0) return cudaErrorInvalidValue;
  const int total = N * (C / 8);
  global_avgpool_fwd_kernel<<<(total + 255) / 256, 256, 0, stream>>>(x, y, N, HW, C);
  return cudaGetLastError();
}
cudaError_t launch_global_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int N, int HW, int C,
                                      cudaStream_t stream) {
  if (C % 8 != 0) return cudaErrorInvalidValue;
  global_avgpool_bwd_kernel<<<grid_for(static_cast<int64_t>(N) * HW * (C / 8)), 256, 0, stream>>>(dy, dx, N, HW, C);
  return cudaGetLastError();
}

cudaError_t launch_softmax_xent(const XentArgs& a, cudaStream_t stream) {
  const int warps_per_block = 8;
  softmax_xent_kernel<<<(a.B + warps_per_block - 1) / warps_per_block, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_philox_normal_nhwc(__nv_bfloat16* out, int64_t pixels, int c_valid, int cpad, uint64_t seed,
                                      uint64_t offset, cudaStream_t stream) {
  if (cpad > 4 || c_valid > cpad) return cudaErrorInvalidValue;
  philox_normal_nhwc_kernel<<<grid_for(pixels), 256, 0, stream>>>(out, pixels, c_valid, cpad, seed, offset);
  return cudaGetLastError();
}
cudaError_t launch_philox_labels(int64_t* out, int64_t n, int classes, uint64_t seed, uint64_t offset,
                                 cudaStream_t stream) {
  philox_labels_kernel<<<static_cast<int>((n + 255) / 256), 256, 0, stream>>>(out, n, classes, seed, offset);
  return cudaGetLastError();
}

cudaError_t launch_nchw_to_nhwc_norm(const float* in, __nv_bfloat16* out, int N, int C, int H, int W, int cpad,
                                     const float* mean, const float* stdv, cudaStream_t stream) {
  nchw_to_nhwc_norm_kernel<<<grid_for(static_cast<int64_t>(N) * H * W), 256, 0, stream>>>(in, out, N, C, H, W, cpad, mean, stdv);
  return cudaGetLastError();
}
cudaError_t launch_nhwc_u8_to_nhwc4(const uint8_t* in, __nv_bfloat16* out, int64_t pixels, const float* mean,
                                    const float* stdv, cudaStream_t stream) {
  nhwc_u8_to_nhwc4_kernel<<<grid_for(pixels / 4 + 1), 256, 0, stream>>>(in, out, pixels, mean, stdv);
  return cudaGetLastError();
}
cudaError_t launch_cast_f32_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t stream) {
  cast_f32_bf16_kernel<<<grid_for(n / 4 + 1), 256, 0, stream>>>(in, out, n);
  return cudaGetLastError();
}
cudaError_t launch_pack_stem_weight(const float* w, __nv_bfloat16* packed, int Cout, int R, int S, int Cin, int RP,
                                    int SP, cudaStream_t stream) {
  pack_stem_weight_kernel<<<grid_for(static_cast<int64_t>(Cout) * RP * SP * 4), 256, 0, stream>>>(w, packed, Cout, R, S, Cin, RP, SP);
  return cudaGetLastError();
}
cudaError_t launch_unpack_stem_grad(const float* packed, float* gw, int Cout, int R, int S, int Cin, int RP, int SP,
                                    cudaStream_t stream) {
  unpack_stem_grad_kernel<<<grid_for(static_cast<int64_t>(Cout) * R * S * Cin), 256, 0, stream>>>(packed, gw, Cout, R, S, Cin, RP, SP);
  return cudaGetLastError();
}

cudaError_t launch_bias_relu_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* z, __nv_bfloat16* dx, float* dbias,
                                 int M, int C, int c_valid, int relu, int sms, cudaStream_t stream) {
  const int groups = C / 8;
  if (C % 8 != 0) return cudaErrorInvalidValue;
  // total threads must be a multiple of `groups`
  int64_t threads = static_cast<int64_t>(M) * groups;
  int64_t cap = static_cast<int64_t>(sms) * 4 * 256;
  if (threads > cap) threads = cap;
  int64_t unit = 256;                       // lcm(256, groups) / 256 blocks granularity
  int64_t l = groups;
  while (l % 256 != 0) l += groups;         // smallest multiple of groups divisible by 256
  unit = l / 256;
  int64_t blocks = (threads + 255) / 256;
  blocks = (blocks + unit - 1) / unit * unit;
  bias_relu_bwd_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(dy, z, dx, dbias, M, C, c_valid, relu);
  return cudaGetLastError();
}
cudaError_t launch_dropout(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, float p, uint64_t seed,
                           uint64_t offset, const int64_t* step, cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  dropout_kernel<<<grid_for(n / 8), 256, 0, stream>>>(x, y, n / 8, p, seed, offset, step);
  return cudaGetLastError();
}
cudaError_t launch_hardswish_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  hardswish_fwd_kernel<<<grid_for(n / 8), 256, 0, stream>>>(x, y, n / 8);
  return cudaGetLastError();
}
cudaError_t launch_hardswish_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, __nv_bfloat16* dx, int64_t n,
                                 cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  hardswish_bwd_kernel<<<grid_for(n / 8), 256, 0, stream>>>(dy, x, dx, n / 8);
  return cudaGetLastError();
}
cudaError_t launch_silu_rows_fwd(const __nv_bfloat16* x, int ldx, __nv_bfloat16* y, int ldy, int N, cudaStream_t stream) {
  if (N <= 0 || ldy <= 0 || ldy % 8 != 0 || ldx % 8 != 0 || ldy > ldx) return cudaErrorInvalidValue;
  const int64_t total = static_cast<int64_t>(N) * (ldy / 8);
  silu_rows_fwd_kernel<<<grid_for(total), 256, 0, stream>>>(x, ldx, y, ldy, total);
  return cudaGetLastError();
}
cudaError_t launch_silu_rows_bwd(const __nv_bfloat16* dy, int ldy, const __nv_bfloat16* x, int ldx, __nv_bfloat16* dx,
                                 int c_valid, int N, cudaStream_t stream) {
  if (N <= 0 || ldy % 8 != 0 || ldx % 8 != 0 || c_valid <= 0 || c_valid > ldy || ldy > ldx) return cudaErrorInvalidValue;
  const int64_t total = static_cast<int64_t>(N) * (ldx / 8);
  silu_rows_bwd_kernel<<<grid_for(total), 256, 0, stream>>>(dy, ldy, x, ldx, dx, c_valid, total);
  return cudaGetLastError();
}
cudaError_t launch_stochastic_depth_keep(float* keep, int n, float p, uint64_t seed, uint64_t offset, const int64_t* step,
                                         cudaStream_t stream) {
  if (n <= 0 || !(p > 0.f && p < 1.f)) return cudaErrorInvalidValue;
  stochastic_depth_keep_kernel<<<(n + 255) / 256, 256, 0, stream>>>(keep, n, p, seed, offset, step);
  return cudaGetLastError();
}
cudaError_t launch_pad_nhwc4(const __nv_bfloat16* in, __nv_bfloat16* out, int N, int H, int W, int Hp, int Wp, int pt,
                             int pl, int G, cudaStream_t stream) {
  if (Hp < H + pt || Wp < W + pl || pt < 0 || pl < 0 || G < 1 || G > 4) return cudaErrorInvalidValue;
  pad_nhwc4_kernel<<<grid_for(static_cast<int64_t>(N) * Hp * Wp * G), 256, 0, stream>>>(
      reinterpret_cast<const uint2*>(in), reinterpret_cast<uint2*>(out), N, H, W, Hp, Wp, pt, pl, G);
  return cudaGetLastError();
}
cudaError_t launch_concat_channels(const CatArgs& a, bool scatter, cudaStream_t stream) {
  if (a.n < 1 || a.n > kCatMax || a.ctot % 8 != 0) return cudaErrorInvalidValue;
  int tot = 0;
  for (int i = 0; i < a.n; ++i) {
    if (a.c[i] % 8 != 0 || a.c[i] <= 0) return cudaErrorInvalidValue;
    tot += a.c[i];
  }
  if (tot != a.ctot) return cudaErrorInvalidValue;
  const int64_t vecs = static_cast<int64_t>(a.M) * (a.ctot / 8);
  if (scatter) concat_channels_kernel<true><<<grid_for(vecs), 256, 0, stream>>>(a);
  else concat_channels_kernel<false><<<grid_for(vecs), 256, 0, stream>>>(a);
  return cudaGetLastError();
}
cudaError_t launch_add_bf16(const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* y, int64_t n,
                            cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  add_bf16_kernel<<<grid_for(n / 8), 256, 0, stream>>>(a, b, y, n / 8);
  return cudaGetLastError();
}

}  // namespace ddl
