// Fused BatchNorm(train) + ReLU (+ residual add) forward / backward on NHWC bf16 activations.
//
// Replaces cuDNN BN fwd/bwd + ATen ReLU + ATen add of the reference step (SURVEY.md K5, K6, K7).
// The batch statistics (sum, sum of squares per channel) arrive from the conv epilogue
// (conv_gemm.cu, STATS) — the activation tensor is never re-read just to reduce it.
//
//   forward   z = relu( (x - mean) * invstd * gamma + beta  (+ residual) )          1 read (+1), 1 write
//   backward  pass 1: dbeta = sum dy, dgamma = sum dy * xhat   with dy = dz * mask
//             pass 2: dx = gamma*invstd * (dy - dbeta/M - xhat*dgamma/M),  dres = dy
//   mask: none (no ReLU) | z > 0 (residual layers; z is read) | x*scale + shift > 0 (no residual: the
//   mask is recomputed from x, so z is never read: 2 reads in pass 1, 2 reads + 1 write in pass 2)
//   ReLU6 (relu == 2, MobileNetV2): z = min(max(v, 0), 6) and the gradient passes where 0 < v < 6 (PyTorch's hardtanh
//   backward), v being z or the recomputed pre-activation.  Its own template instantiations, so that the ReLU
//   kernels of the ResNet path keep their code and registers; not combined with the residual bit mask.
//   Hardswish (relu == 3, MobileNetV3): z = v * clamp(v + 3, 0, 6) / 6; the gradient is dz * (0 for v <= -3,
//   v / 3 + 1/2 for -3 < v < 3, 1 for v >= 3), v recomputed from x (mask-from-x mode only).  Its own forward kernel
//   (bn_hswish_fwd_kernel, sharing the body) and backward mask value; no residual, bit mask or fp8 twin.
//   SiLU (relu == 4, EfficientNet): z = v * sigmoid(v); the gradient is dz * s * (1 + v * (1 - s)) with s = sigmoid(v),
//   v recomputed from x.  Own forward kernel (bn_silu_fwd_kernel) and mask value; the same refusals as hardswish.
//   GELU (relu == 5, MaxViT): z = v * Phi(v), exact (erf); the gradient is dz * (Phi(v) + v * phi(v)), v recomputed from
//   x.  Own forward kernel (bn_gelu_fwd_kernel) and mask value (9); the same refusals as hardswish.
//   Stochastic depth (sample_scale, EfficientNet's residual blocks): z = BN(x) * keep[n] + residual with one scale per
//   sample (row / hw), no activation.  The statistics cover every sample, dropped ones included; backward feeds
//   dz * keep[n] to the BN and returns dres = dz.  Own forward kernel (bn_sd_fwd_kernel, train only) and mask value.
//
// Thread mapping: a thread owns 8 consecutive channels (one 16-byte vector) of a FIXED channel
// group and walks rows with a grid stride, so per-channel constants live in registers.  The loops
// work on raw x (sum dy*x, then a closed-form fix-up) to keep the live register set under 64 so that
// 4 CTAs x 256 threads stay resident per SM (these kernels are pure HBM streams).
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kBnThreads = 256;
enum { kMaskNone = 0, kMaskZ = 1, kMaskX = 2, kMaskBits = 3, kMaskZ6 = 4, kMaskX6 = 5, kMaskXH = 6, kMaskXS = 7,
       kMaskSD = 8, kMaskXG = 9 };
constexpr bool mask_from_z(int m) { return m == kMaskZ || m == kMaskZ6; }
constexpr bool mask_from_x(int m) { return m == kMaskX || m == kMaskX6 || m == kMaskXH || m == kMaskXS || m == kMaskXG; }
// sigmoid on the MUFU exp and reciprocal (__fdividef, no IEEE division: with `1.f / (...)` the SiLU backward's chunked
// apply pass spilled at 64 registers).  Relative accuracy holds in the negative tail, where sigmoid(v) is tiny; for
// v < -87 the denominator overflows to inf and the result is 0.
DDL_DEVICE float sigmoid(float v) { return __fdividef(1.f, 1.f + __expf(-v)); }
// Phi(v) and e = exp(-v^2 / 2) from one MUFU exponential: erf by Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7), with
// 0.5 erfc(|v| / sqrt 2) formed directly so that the negative tail keeps its relative accuracy.  The GELU backward's
// apply pass spilled at 64 registers with erff; the forward keeps erff.
DDL_DEVICE float gelu_cdf(float v, float& e) {
  const float t = __fdividef(1.f, fmaf(0.3275911f * 0.70710678118654752f, fabsf(v), 1.f));
  e = __expf(-0.5f * v * v);
  const float tail = 0.5f * e * t *
      fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  return v >= 0.f ? 1.f - tail : tail;
}
// whether the gradient passes the activation at pre-activation (or output) value v
template <int MASK>
DDL_DEVICE bool act_passes(float v) {
  return (MASK == kMaskZ6 || MASK == kMaskX6) ? (v > 0.f && v < 6.f) : v > 0.f;
}
// the gradient dz of the activation's output as a gradient of its input, at pre-activation value v
template <int MASK>
DDL_DEVICE float act_bwd(float v, float dz) {
  if (MASK == kMaskXH) return v <= -3.f ? 0.f : (v >= 3.f ? dz : dz * fmaf(v, 1.f / 3.f, 0.5f));
  if (MASK == kMaskXS) {
    const float sg = sigmoid(v);
    return dz * sg * fmaf(v, 1.f - sg, 1.f);
  }
  if (MASK == kMaskXG) {     // Phi(v) + v phi(v), phi(v) = exp(-v^2 / 2) / sqrt(2 pi)
    float e;
    const float cdf = gelu_cdf(v, e);
    return dz * fmaf(v * 0.39894228040143268f, e, cdf);
  }
  return act_passes<MASK>(v) ? dz : 0.f;
}
// forward activations of bn_act_fwd_body
enum { kActRelu = 0, kActRelu6 = 1, kActHswish = 2, kActSilu = 3, kActSD = 4, kActGelu = 5 };
DDL_DEVICE float hardswish(float v) { return v * fminf(fmaxf(v + 3.f, 0.f), 6.f) * (1.f / 6.f); }

struct Vec8 {
  float v[8];
};
DDL_DEVICE void unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE void store8_bf16(__nv_bfloat16* p, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]),
                                            pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}
DDL_DEVICE Vec8 load8_f32(const float* p) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  Vec8 r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}

// ---- forward --------------------------------------------------------------------------------
// TRAIN: scale/shift derived from (sum, sumsq); also emits mean/invstd (saved for backward) and
// updates running stats.  EVAL: scale/shift from running stats.
// Thread -> (channel group, row lane).  FLAT: threads are spread over the C/8 channel groups of consecutive rows
// (needs C/8 to divide, or be a multiple of, the block size: the power-of-two widths of ResNet/VGG).  CHUNKED: a
// block owns the 64-channel chunk blockIdx.y and 32 row lanes — any C that is a multiple of 8 (Inception's 48, 80,
// 96, 160, 192, 288, 320, 384, 448, 768, 1280; DenseNet's growth steps), channel groups beyond C idle.
template <bool CHUNKED>
DDL_DEVICE bool bn_thread_map(int C, int& c0, int& row0, int& row_stride) {
  if (CHUNKED) {
    c0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
    row0 = blockIdx.x * 32 + (threadIdx.x >> 3);
    row_stride = gridDim.x * 32;
    return c0 < C;
  }
  const int groups = C / 8;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  c0 = (tid % groups) * 8;
  row0 = tid / groups;
  row_stride = (gridDim.x * blockDim.x) / groups;
  return true;
}

// FP8: also emit the e4m3 twin of z (z * slot scale) and fold max|z| into the slot — the quantisation pass of the fp8
// training mode rides in this kernel's streaming pass (+1 byte written per element) instead of re-reading z.
// BLOCK_WIDE: every thread of the block reaches this point (flat thread mapping): fold through shared memory and issue ONE
// atomic per block instead of ~9.5k same-address atomics per launch (one per warp), which serialise on one address.
template <bool BLOCK_WIDE>
DDL_DEVICE void fp8_fold_amax(Fp8Slot* slot, float amax) {
  amax = warp_max(amax);
  if (BLOCK_WIDE) {
    __shared__ float s_amax[kBnThreads / 32];
    if ((threadIdx.x & 31) == 0) s_amax[threadIdx.x >> 5] = amax;
    __syncthreads();
    if (threadIdx.x < 32) {
      float v = threadIdx.x < kBnThreads / 32 ? s_amax[threadIdx.x] : 0.f;
      v = warp_max(v);
      if (threadIdx.x == 0 && v > 0.f) atomicMax(reinterpret_cast<unsigned int*>(&slot->amax), __float_as_uint(v));
    }
  } else if ((threadIdx.x & 31) == 0 && amax > 0.f) {
    atomicMax(reinterpret_cast<unsigned int*>(&slot->amax), __float_as_uint(amax));    // chunked mapping: idle threads left early
  }
}

// ACT: kActRelu (ReLU when a.relu, else none), kActRelu6 (when a.relu), kActHswish / kActSilu / kActGelu (always) or kActSD (no
// activation; the BN output scaled by the row's sample scale before the residual add)
template <bool TRAIN, bool CHUNKED, bool FP8, int ACT>
DDL_DEVICE void bn_act_fwd_body(const BnFwdArgs& a) {
  pdl_trigger();
  pdl_wait();      // nothing to prepare here: the gain is the launch latency and the block ramp-up
  int c0, row0, row_stride;
  if (!bn_thread_map<CHUNKED>(a.C, c0, row0, row_stride)) return;
  const float qscale = FP8 ? a.zq_slot->scale : 1.f;
  float amax = 0.f;
  float scale[8], shift[8];
  {
    Vec8 gam = load8_f32(a.gamma + c0), bet = load8_f32(a.beta + c0);
    if (TRAIN) {
      Vec8 s = load8_f32(a.sum + c0), ss = load8_f32(a.sumsq + c0);
      const float inv_n = 1.f / static_cast<float>(a.M);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float mean = s.v[i] * inv_n;
        const float var = fmaxf(ss.v[i] * inv_n - mean * mean, 0.f);
        const float invstd = rsqrtf(var + a.eps);
        scale[i] = gam.v[i] * invstd;
        shift[i] = bet.v[i] - mean * scale[i];
        if (row0 == 0) {
          a.mean[c0 + i] = mean;
          a.invstd[c0 + i] = invstd;
          if (a.running_mean) {
            const float unbiased = a.M > 1 ? var * static_cast<float>(a.M) / static_cast<float>(a.M - 1) : var;
            a.running_mean[c0 + i] = (1.f - a.momentum) * a.running_mean[c0 + i] + a.momentum * mean;
            a.running_var[c0 + i] = (1.f - a.momentum) * a.running_var[c0 + i] + a.momentum * unbiased;
          }
        }
      }
    } else {
      Vec8 rm = load8_f32(a.running_mean + c0), rv = load8_f32(a.running_var + c0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        scale[i] = gam.v[i] * rsqrtf(rv.v[i] + a.eps);
        shift[i] = bet.v[i] - rm.v[i] * scale[i];
      }
    }
  }
  // two rows per iteration: both rows' 16-byte loads are in flight before either is consumed (one load per thread
  // leaves only ~16 KB per SM outstanding, short of the ~30 KB an HBM3e stream needs at this latency)
  auto finish = [&](const uint4& ux, const uint4& ur, size_t off) {
    float x[8], z[8];
    unpack8(ux, x);
    if (ACT == kActSD) {
      float res[8];
      unpack8(ur, res);
      const float ks = a.sample_scale[off / (static_cast<size_t>(a.hw) * a.C)];
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaf(fmaf(x[i], scale[i], shift[i]), ks, res[i]);
    } else if (a.residual) {
      float res[8];
      unpack8(ur, res);
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaf(x[i], scale[i], shift[i]) + res[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaf(x[i], scale[i], shift[i]);
    }
    if (ACT == kActHswish) {
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = hardswish(z[i]);
    } else if (ACT == kActSilu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] *= sigmoid(z[i]);
    } else if (ACT == kActGelu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] *= fmaf(0.5f, erff(z[i] * 0.70710678118654752f), 0.5f);
    } else if (ACT != kActSD && a.relu) {
      if (a.mask) {
        uint32_t bits = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) bits |= (z[i] > 0.f ? 1u : 0u) << i;
        a.mask[off >> 3] = static_cast<uint8_t>(bits);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = ACT == kActRelu6 ? fminf(fmaxf(z[i], 0.f), 6.f) : fmaxf(z[i], 0.f);
    }
    store8_bf16(a.z + off, z);
    if (FP8) {
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(z[i]));
      *reinterpret_cast<uint2*>(a.zq + off) =
          make_uint2(fp8_cvt4<false>(z[0] * qscale, z[1] * qscale, z[2] * qscale, z[3] * qscale),
                     fp8_cvt4<false>(z[4] * qscale, z[5] * qscale, z[6] * qscale, z[7] * qscale));
    }
  };
  // logical row r -> physical row: mirrored when the tensor's tail is what the producer left in L2 (BnFwdArgs::reverse)
  const int last = a.M - 1;
  auto phys = [&](int rr) { return a.reverse ? last - rr : rr; };
  int r = row0;
  for (; r + row_stride < a.M; r += 2 * row_stride) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const size_t off1 = static_cast<size_t>(phys(r + row_stride)) * a.C + c0;
    const uint4 x0 = ld_stream_u4(a.x + off0), x1 = ld_stream_u4(a.x + off1);
    uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;
    if (a.residual) { r0 = ld_stream_u4(a.residual + off0); r1 = ld_stream_u4(a.residual + off1); }
    finish(x0, r0, off0);
    finish(x1, r1, off1);
  }
  if (r < a.M) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const uint4 x0 = ld_stream_u4(a.x + off0);
    uint4 r0 = make_uint4(0, 0, 0, 0);
    if (a.residual) r0 = ld_stream_u4(a.residual + off0);
    finish(x0, r0, off0);
  }
  if (FP8) fp8_fold_amax<!CHUNKED>(a.zq_slot, amax);
}

template <bool TRAIN, bool CHUNKED, bool FP8, bool RELU6>
__global__ void __launch_bounds__(kBnThreads, 4) bn_act_fwd_kernel(BnFwdArgs a) {
  bn_act_fwd_body<TRAIN, CHUNKED, FP8, RELU6 ? kActRelu6 : kActRelu>(a);
}

template <bool TRAIN, bool CHUNKED>
__global__ void __launch_bounds__(kBnThreads, 4) bn_hswish_fwd_kernel(BnFwdArgs a) {
  bn_act_fwd_body<TRAIN, CHUNKED, false, kActHswish>(a);
}

template <bool TRAIN, bool CHUNKED>
__global__ void __launch_bounds__(kBnThreads, 4) bn_silu_fwd_kernel(BnFwdArgs a) {
  bn_act_fwd_body<TRAIN, CHUNKED, false, kActSilu>(a);
}

template <bool TRAIN, bool CHUNKED>
__global__ void __launch_bounds__(kBnThreads, 4) bn_gelu_fwd_kernel(BnFwdArgs a) {
  bn_act_fwd_body<TRAIN, CHUNKED, false, kActGelu>(a);
}

// stochastic depth is drawn in training only: eval takes the plain residual kernels
template <bool CHUNKED>
__global__ void __launch_bounds__(kBnThreads, 4) bn_sd_fwd_kernel(BnFwdArgs a) {
  bn_act_fwd_body<true, CHUNKED, false, kActSD>(a);
}

// ---- backward pass 1: per-channel reductions ----------------------------------------------------
// accumulates S1 = sum dy and S2 = sum dy * x (raw x); dbeta = S1, dgamma = invstd * (S2 - mean * S1).
// Mapping: a block owns ONE 64-channel chunk (blockIdx.y) and 32 row lanes (thread = 8 channels x 1 row lane),
// so a block ends with 64 x 2 partial sums -> 128 atomics per block and only gridDim.x contributions per address.
// (A block spanning all channels would issue C x 2 atomics per block: ~5 M contended atomics for C = 2048, enough to
// dominate the small layers.)
template <int MASK>
__global__ void __launch_bounds__(kBnThreads, 4) bn_act_bwd_reduce_kernel(BnBwdArgs a) {
  pdl_trigger();
  pdl_wait();      // nothing to prepare here: the gain is the launch latency and the block ramp-up
  const int cgl = threadIdx.x & 7;                 // channel group within the 64-channel chunk
  const int rl = threadIdx.x >> 3;                 // row lane 0..31
  const int c0 = blockIdx.y * 64 + cgl * 8;
  const bool live = c0 < a.C;                      // last chunk of a width that is not a multiple of 64
  float s1[8], s2[8], msc[8], msh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s1[i] = 0.f; s2[i] = 0.f; msc[i] = 0.f; msh[i] = 0.f; }
  if (mask_from_x(MASK) && live) {
    Vec8 mean = load8_f32(a.mean + c0), invstd = load8_f32(a.invstd + c0);
    Vec8 gam = load8_f32(a.gamma + c0), bet = load8_f32(a.beta + c0);
#pragma unroll
    for (int i = 0; i < 8; ++i) { msc[i] = gam.v[i] * invstd.v[i]; msh[i] = bet.v[i] - mean.v[i] * msc[i]; }
  }
  auto accumulate = [&](const uint4& udz, const uint4& ux, const uint4& uz) {
    float dz[8], x[8];
    unpack8(udz, dz);
    unpack8(ux, x);
    if (mask_from_z(MASK)) {
      float z[8];
      unpack8(uz, z);
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = act_passes<MASK>(z[i]) ? dz[i] : 0.f;
    } else if (MASK == kMaskBits) {        // uz.x carries the 8 mask bits of this (row, channel group)
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = ((uz.x >> i) & 1u) ? dz[i] : 0.f;
    } else if (mask_from_x(MASK)) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = act_bwd<MASK>(fmaf(x[i], msc[i], msh[i]), dz[i]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1[i] += dz[i];
      s2[i] = fmaf(dz[i], x[i], s2[i]);
    }
  };
  // two rows per iteration so that 4 (6 with the z mask) 16-byte loads are outstanding per thread
  const int rstep = gridDim.x * 32;
  const int last = a.M - 1;
  auto phys = [&](int rr) { return a.reverse ? last - rr : rr; };      // see BnBwdArgs::reverse
  int r = live ? blockIdx.x * 32 + rl : a.M;
  if constexpr (MASK == kMaskXH || MASK == kMaskXS || MASK == kMaskXG) {
    // one row per iteration: the hardswish / SiLU / GELU gradient keeps more values live than a mask, and two rows would spill
    for (; r < a.M; r += rstep) {
      const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
      accumulate(ld_stream_u4(a.dz + off0), ld_stream_u4(a.x + off0), make_uint4(0, 0, 0, 0));
    }
  }
  if constexpr (MASK == kMaskSD) {        // the BN sees dz * keep[sample]
    for (; r < a.M; r += rstep) {
      const int pr = phys(r);
      const size_t off0 = static_cast<size_t>(pr) * a.C + c0;
      const float ks = a.sample_scale[pr / a.hw];
      float dz[8], x[8];
      unpack8(ld_stream_u4(a.dz + off0), dz);
      unpack8(ld_stream_u4(a.x + off0), x);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s1[i] = fmaf(dz[i], ks, s1[i]);
        s2[i] = fmaf(dz[i] * ks, x[i], s2[i]);
      }
    }
  }
  for (; MASK != kMaskXH && MASK != kMaskXS && MASK != kMaskXG && MASK != kMaskSD && r + rstep < a.M; r += 2 * rstep) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const size_t off1 = static_cast<size_t>(phys(r + rstep)) * a.C + c0;
    const uint4 d0 = ld_stream_u4(a.dz + off0), d1 = ld_stream_u4(a.dz + off1);
    const uint4 x0 = ld_stream_u4(a.x + off0), x1 = ld_stream_u4(a.x + off1);
    uint4 z0 = make_uint4(0, 0, 0, 0), z1 = z0;
    if (mask_from_z(MASK)) { z0 = ld_stream_u4(a.z + off0); z1 = ld_stream_u4(a.z + off1); }
    if (MASK == kMaskBits) { z0.x = a.zmask[off0 >> 3]; z1.x = a.zmask[off1 >> 3]; }
    accumulate(d0, x0, z0);
    accumulate(d1, x1, z1);
  }
  if (r < a.M) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const uint4 d0 = ld_stream_u4(a.dz + off0);
    const uint4 x0 = ld_stream_u4(a.x + off0);
    uint4 z0 = make_uint4(0, 0, 0, 0);
    if (mask_from_z(MASK)) z0 = ld_stream_u4(a.z + off0);
    if (MASK == kMaskBits) z0.x = a.zmask[off0 >> 3];
    accumulate(d0, x0, z0);
  }
  // lanes of a warp sharing a channel group: lane = (rl % 4) * 8 + cgl -> xor 8, 16
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], off);
      s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], off);
    }
  }
  __shared__ float red[kBnThreads / 32][8][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { red[warp][lane][i] = s1[i]; red[warp][lane][8 + i] = s2[i]; }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int w = 0; w < kBnThreads / 32; ++w) { t1 += red[w][g][i]; t2 += red[w][g][8 + i]; }
    const int ch = blockIdx.y * 64 + g * 8 + i;
    if (ch < a.C) {
      atomicAdd(a.dbeta + ch, t1);
      atomicAdd(a.dgamma + ch, a.invstd[ch] * (t2 - a.mean[ch] * t1));
    }
  }
}

// ---- backward pass 2: elementwise ----------------------------------------------------------------
// dx = k1*dy + x*B + A   with k1 = gamma*invstd, B = -k1*invstd*dgamma/M, A = -k1*dbeta/M - mean*B
template <int MASK, bool CHUNKED, bool FP8>
__global__ void __launch_bounds__(kBnThreads, 4) bn_act_bwd_apply_kernel(BnBwdArgs a) {
  pdl_trigger();
  pdl_wait();      // nothing to prepare here: the gain is the launch latency and the block ramp-up
  int c0, row0, row_stride;
  if (!bn_thread_map<CHUNKED>(a.C, c0, row0, row_stride)) return;
  const float qscale = FP8 ? a.dxq_slot->scale : 1.f;
  float amax = 0.f;
  float k1[8], cA[8], cB[8], msh[8];
  {
    Vec8 mean = load8_f32(a.mean + c0), invstd = load8_f32(a.invstd + c0), gam = load8_f32(a.gamma + c0);
    Vec8 db = load8_f32(a.dbeta + c0), dg = load8_f32(a.dgamma + c0);
    const float inv_n = 1.f / static_cast<float>(a.M);
    if (row0 == 0) {   // exactly one thread per channel group: accumulate parameter grads (each one only if it trains)
      if (a.gamma_grad) {
#pragma unroll
        for (int i = 0; i < 8; ++i) a.gamma_grad[c0 + i] += dg.v[i];
      }
      if (a.beta_grad) {
#pragma unroll
        for (int i = 0; i < 8; ++i) a.beta_grad[c0 + i] += db.v[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      k1[i] = gam.v[i] * invstd.v[i];
      cB[i] = -k1[i] * invstd.v[i] * dg.v[i] * inv_n;
      cA[i] = -k1[i] * db.v[i] * inv_n - mean.v[i] * cB[i];
      msh[i] = 0.f;
    }
    if (mask_from_x(MASK)) {
      Vec8 bet = load8_f32(a.beta + c0);
#pragma unroll
      for (int i = 0; i < 8; ++i) msh[i] = bet.v[i] - mean.v[i] * k1[i];
    }
  }
  for (int r = row0; r < a.M; r += row_stride) {
    const size_t off = static_cast<size_t>(r) * a.C + c0;
    float dz[8], x[8];
    unpack8(ld_stream_u4(a.dz + off), dz);
    unpack8(ld_stream_u4(a.x + off), x);
    if (mask_from_z(MASK)) {
      float z[8];
      unpack8(ld_stream_u4(a.z + off), z);
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = act_passes<MASK>(z[i]) ? dz[i] : 0.f;
    } else if (MASK == kMaskBits) {
      const uint32_t bits = a.zmask[off >> 3];
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = ((bits >> i) & 1u) ? dz[i] : 0.f;
    } else if (mask_from_x(MASK)) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = act_bwd<MASK>(fmaf(x[i], k1[i], msh[i]), dz[i]);
    }
    if (a.dres) store8_bf16(a.dres + off, dz);
    if constexpr (MASK == kMaskSD) {
      const float ks = a.sample_scale[r / a.hw];
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] *= ks;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = fmaf(dz[i], k1[i], fmaf(x[i], cB[i], cA[i]));
    store8_bf16(a.dx + off, x);
    if (FP8) {       // e5m2 twin of the gradient for the data-gradient convolution (same rounding source: fp32 x[])
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(x[i]));
      *reinterpret_cast<uint2*>(a.dxq + off) =
          make_uint2(fp8_cvt4<true>(x[0] * qscale, x[1] * qscale, x[2] * qscale, x[3] * qscale),
                     fp8_cvt4<true>(x[4] * qscale, x[5] * qscale, x[6] * qscale, x[7] * qscale));
    }
  }
  if (FP8) fp8_fold_amax<!CHUNKED>(a.dxq_slot, amax);
}

// ---------------------------------------------------------------------------------------------
// stem fusion: conv -> BN -> ReLU -> max-pool (ResNet / DenseNet first layers)
// ---------------------------------------------------------------------------------------------
// forward: the BN+ReLU output (the largest activation of the network, 112 x 112 x 64 per image) is never written —
// each pooled pixel applies scale/shift to its window of the raw conv output and keeps max + arg-max code.
// backward: BN's input gradient dz is rebuilt on the fly from the pooled gradient and the arg-max codes (the
// gather of maxpool_bwd_kernel), so neither max-pool backward's 112 x 112 output nor its two re-reads exist.
template <bool CHUNKED_UNUSED = false>
DDL_DEVICE void bn_scale_shift(const BnFwdArgs& a, int c0, bool writer, float (&scale)[8], float (&shift)[8]) {
  Vec8 gam = load8_f32(a.gamma + c0), bet = load8_f32(a.beta + c0);
  Vec8 s = load8_f32(a.sum + c0), ss = load8_f32(a.sumsq + c0);
  const float inv_n = 1.f / static_cast<float>(a.M);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float mean = s.v[i] * inv_n;
    const float var = fmaxf(ss.v[i] * inv_n - mean * mean, 0.f);
    const float invstd = rsqrtf(var + a.eps);
    scale[i] = gam.v[i] * invstd;
    shift[i] = bet.v[i] - mean * scale[i];
    if (writer) {
      a.mean[c0 + i] = mean;
      a.invstd[c0 + i] = invstd;
      if (a.running_mean) {
        const float unbiased = a.M > 1 ? var * static_cast<float>(a.M) / static_cast<float>(a.M - 1) : var;
        a.running_mean[c0 + i] = (1.f - a.momentum) * a.running_mean[c0 + i] + a.momentum * mean;
        a.running_var[c0 + i] = (1.f - a.momentum) * a.running_var[c0 + i] + a.momentum * unbiased;
      }
    }
  }
}

// block = one 64-channel chunk x 32 pooled-pixel lanes (same mapping as the reduce kernel: any C % 8 == 0)
__global__ void __launch_bounds__(kBnThreads, 4)
bn_relu_maxpool_fwd_kernel(BnFwdArgs a, PoolArgs p, __nv_bfloat16* pooled, uint8_t* argmax) {
  const int c0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
  if (c0 >= a.C) return;
  const int lane = blockIdx.x * 32 + (threadIdx.x >> 3);
  float scale[8], shift[8];
  bn_scale_shift(a, c0, lane == 0, scale, shift);
  const int total = p.N * p.P * p.Q;
  for (int o = lane; o < total; o += gridDim.x * 32) {
    const int q = o % p.Q;
    const int t = o / p.Q;
    const int pp = t % p.P;
    const int n = t / p.P;
    float best[8];
    uint32_t code[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = -INFINITY; code[i] = 0; }
    for (int r = 0; r < p.k; ++r) {
      const int h = pp * p.stride - p.pad + r;
      if (h < 0 || h >= p.H) continue;
      for (int sx = 0; sx < p.k; ++sx) {
        const int w = q * p.stride - p.pad + sx;
        if (w < 0 || w >= p.W) continue;
        float v[8];
        unpack8(ld_stream_u4(a.x + ((static_cast<size_t>(n) * p.H + h) * p.W + w) * a.C + c0), v);
        const uint32_t cd = r * p.k + sx;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float z = bf16_round(fmaf(v[i], scale[i], shift[i]));     // the value the unfused path would store
          if (z > best[i]) { best[i] = z; code[i] = cd; }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) best[i] = fmaxf(best[i], 0.f);           // ReLU commutes with max
    const size_t off = static_cast<size_t>(o) * a.C + c0;
    store8_bf16(pooled + off, best);
    uint2 am;
    am.x = code[0] | (code[1] << 8) | (code[2] << 16) | (code[3] << 24);
    am.y = code[4] | (code[5] << 8) | (code[6] << 16) | (code[7] << 24);
    *reinterpret_cast<uint2*>(argmax + off) = am;
  }
}

// gradient of the max-pool input pixel (n, h, w), channels [c0, c0+8): sum of the pooled gradients of the windows
// whose arg-max is this pixel
DDL_DEVICE void pool_gather(const __nv_bfloat16* __restrict__ dyp, const uint8_t* __restrict__ argmax, const PoolArgs& p,
                            int C, int n, int h, int w, int c0, float (&acc)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const int pp_hi = (h + p.pad) / p.stride, q_hi = (w + p.pad) / p.stride;
  for (int pp = pp_hi; pp >= 0; --pp) {
    const int r = h + p.pad - pp * p.stride;
    if (r >= p.k) break;
    if (pp >= p.P) continue;
    for (int q = q_hi; q >= 0; --q) {
      const int sx = w + p.pad - q * p.stride;
      if (sx >= p.k) break;
      if (q >= p.Q) continue;
      const size_t o = ((static_cast<size_t>(n) * p.P + pp) * p.Q + q) * C + c0;
      const uint2 am = *reinterpret_cast<const uint2*>(argmax + o);
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(dyp + o), v);
      const uint32_t code = r * p.k + sx;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t ai = ((i < 4 ? am.x : am.y) >> (8 * (i & 3))) & 0xffu;
        if (ai == code) acc[i] += v[i];
      }
    }
  }
}

// pass 1 of the fused stem backward: S1 = sum dm, S2 = sum dm * x with dm = pool_gather(...) * [x*scale + shift > 0]
__global__ void __launch_bounds__(kBnThreads, 4)
bn_pool_bwd_reduce_kernel(BnBwdArgs a, PoolArgs p, const __nv_bfloat16* __restrict__ dyp,
                          const uint8_t* __restrict__ argmax) {
  const int cgl = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + cgl * 8;
  const bool live = c0 < a.C;
  float s1[8], s2[8], msc[8], msh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s1[i] = 0.f; s2[i] = 0.f; msc[i] = 0.f; msh[i] = 0.f; }
  if (live) {
    Vec8 mean = load8_f32(a.mean + c0), invstd = load8_f32(a.invstd + c0);
    Vec8 gam = load8_f32(a.gamma + c0), bet = load8_f32(a.beta + c0);
#pragma unroll
    for (int i = 0; i < 8; ++i) { msc[i] = gam.v[i] * invstd.v[i]; msh[i] = bet.v[i] - mean.v[i] * msc[i]; }
  }
  for (int r = live ? blockIdx.x * 32 + rl : a.M; r < a.M; r += gridDim.x * 32) {
    const int w = r % p.W;
    const int t = r / p.W;
    const int h = t % p.H;
    const int n = t / p.H;
    float dz[8], x[8];
    unpack8(ld_stream_u4(a.x + static_cast<size_t>(r) * a.C + c0), x);
    pool_gather(dyp, argmax, p, a.C, n, h, w, c0, dz);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float dm = fmaf(x[i], msc[i], msh[i]) > 0.f ? dz[i] : 0.f;
      s1[i] += dm;
      s2[i] = fmaf(dm, x[i], s2[i]);
    }
  }
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], off);
      s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], off);
    }
  }
  __shared__ float red[kBnThreads / 32][8][16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { red[warp][lane][i] = s1[i]; red[warp][lane][8 + i] = s2[i]; }
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int wv = 0; wv < kBnThreads / 32; ++wv) { t1 += red[wv][g][i]; t2 += red[wv][g][8 + i]; }
    const int ch = blockIdx.y * 64 + g * 8 + i;
    if (ch < a.C) {
      atomicAdd(a.dbeta + ch, t1);
      atomicAdd(a.dgamma + ch, a.invstd[ch] * (t2 - a.mean[ch] * t1));
    }
  }
}

// pass 2: dx = k1*dm + x*B + A (see bn_act_bwd_apply_kernel) with dm rebuilt from the pooled gradient
__global__ void __launch_bounds__(kBnThreads, 4)
bn_pool_bwd_apply_kernel(BnBwdArgs a, PoolArgs p, const __nv_bfloat16* __restrict__ dyp,
                         const uint8_t* __restrict__ argmax) {
  const int c0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
  if (c0 >= a.C) return;
  const int row0 = blockIdx.x * 32 + (threadIdx.x >> 3);
  float k1[8], cA[8], cB[8], msh[8];
  {
    Vec8 mean = load8_f32(a.mean + c0), invstd = load8_f32(a.invstd + c0), gam = load8_f32(a.gamma + c0);
    Vec8 db = load8_f32(a.dbeta + c0), dg = load8_f32(a.dgamma + c0), bet = load8_f32(a.beta + c0);
    const float inv_n = 1.f / static_cast<float>(a.M);
    if (row0 == 0) {
      if (a.gamma_grad) {
#pragma unroll
        for (int i = 0; i < 8; ++i) a.gamma_grad[c0 + i] += dg.v[i];
      }
      if (a.beta_grad) {
#pragma unroll
        for (int i = 0; i < 8; ++i) a.beta_grad[c0 + i] += db.v[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      k1[i] = gam.v[i] * invstd.v[i];
      cB[i] = -k1[i] * invstd.v[i] * dg.v[i] * inv_n;
      cA[i] = -k1[i] * db.v[i] * inv_n - mean.v[i] * cB[i];
      msh[i] = bet.v[i] - mean.v[i] * k1[i];
    }
  }
  for (int r = row0; r < a.M; r += gridDim.x * 32) {
    const int w = r % p.W;
    const int t = r / p.W;
    const int h = t % p.H;
    const int n = t / p.H;
    const size_t off = static_cast<size_t>(r) * a.C + c0;
    float dz[8], x[8];
    unpack8(ld_stream_u4(a.x + off), x);
    pool_gather(dyp, argmax, p, a.C, n, h, w, c0, dz);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float dm = fmaf(x[i], k1[i], msh[i]) > 0.f ? dz[i] : 0.f;
      x[i] = fmaf(dm, k1[i], fmaf(x[i], cB[i], cA[i]));
    }
    store8_bf16(a.dx + off, x);
  }
}

// grid: every block must hold a whole number of channel groups AND total threads % groups == 0
inline int bn_grid(int M, int C, int sms) {
  const int groups = C / 8;
  const long long total_vec = static_cast<long long>(M) * groups;
  long long blocks = (total_vec + kBnThreads - 1) / kBnThreads;
  const long long cap = static_cast<long long>(sms) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (groups > kBnThreads) {
    const int need = groups / kBnThreads;
    blocks = (blocks + need - 1) / need * need;
  }
  return static_cast<int>(blocks);
}

}  // namespace

// chunked mapping: blocks = (row blocks, 64-channel chunks); >= 8 rows per thread, <= 8 resident waves of blocks
inline dim3 bn_chunk_grid(int M, int C, int sms) {
  const int chunks = (C + 63) / 64;
  int gx = (M + 32 * 8 - 1) / (32 * 8);
  const int cap = (sms * 8 + chunks - 1) / chunks;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3(gx, chunks);
}

inline bool bn_flat_ok(int C) {
  const int groups = C / 8;
  return (kBnThreads % groups == 0) || (groups % kBnThreads == 0);
}

int g_bn_reverse = 1;        // tuning hook (set_bn_reverse / DDL_BN_REVERSE): BN forward and the backward reduce pass walk rows from the end
void set_bn_reverse(int on) { g_bn_reverse = on; }

void pdl_early_bn(int trig) { cudaMemcpyToSymbol(c_pdl_trigger, &trig, sizeof(int)); }

namespace {

// ReLU6 layers get no fp8 twin (not instantiated: no MobileNetV2 convolution meets the fp8 shape rules)
template <bool CHUNKED, bool RELU6>
cudaError_t launch_bn_fwd_variant(const BnFwdArgs& a, bool train, bool f8, dim3 grid, cudaStream_t stream) {
  if (f8) {
    if constexpr (RELU6) return cudaErrorInvalidValue;
    else return launch_pdl(bn_act_fwd_kernel<true, CHUNKED, true, false>, grid, dim3(kBnThreads), 0, stream, 1, a);
  }
  if (train) return launch_pdl(bn_act_fwd_kernel<true, CHUNKED, false, RELU6>, grid, dim3(kBnThreads), 0, stream, 1, a);
  return launch_pdl(bn_act_fwd_kernel<false, CHUNKED, false, RELU6>, grid, dim3(kBnThreads), 0, stream, 1, a);
}

template <int MASK>
cudaError_t launch_bn_bwd_mask(const BnBwdArgs& a, int sms, cudaStream_t stream, bool skip_reduce) {
  const dim3 rgrid = bn_chunk_grid(a.M, a.C, sms);
  if (!skip_reduce) {
    const cudaError_t e = launch_pdl(bn_act_bwd_reduce_kernel<MASK>, rgrid, dim3(kBnThreads), 0, stream, 1, a);
    if (e != cudaSuccess) return e;
  }
  const bool f8 = a.dxq != nullptr && a.dxq_slot != nullptr;
  const bool flat = bn_flat_ok(a.C);
  const dim3 grid = flat ? dim3(bn_grid(a.M, a.C, sms)) : rgrid;
  if constexpr (MASK == kMaskZ6 || MASK == kMaskX6 || MASK == kMaskXH || MASK == kMaskXS || MASK == kMaskXG ||
                MASK == kMaskSD) {
    if (f8) return cudaErrorInvalidValue;
  } else if (f8) {
    return flat ? launch_pdl(bn_act_bwd_apply_kernel<MASK, false, true>, grid, dim3(kBnThreads), 0, stream, 1, a)
                : launch_pdl(bn_act_bwd_apply_kernel<MASK, true, true>, grid, dim3(kBnThreads), 0, stream, 1, a);
  }
  return flat ? launch_pdl(bn_act_bwd_apply_kernel<MASK, false, false>, grid, dim3(kBnThreads), 0, stream, 1, a)
              : launch_pdl(bn_act_bwd_apply_kernel<MASK, true, false>, grid, dim3(kBnThreads), 0, stream, 1, a);
}

}  // namespace

cudaError_t launch_bn_act_fwd(const BnFwdArgs& a_in, bool train, int sms, cudaStream_t stream) {
  BnFwdArgs a = a_in;
  a.reverse = g_bn_reverse;
  if (a.C % 8 != 0 || a.C <= 0) return cudaErrorInvalidValue;
  const bool flat = bn_flat_ok(a.C);
  const dim3 grid = flat ? dim3(bn_grid(a.M, a.C, sms)) : bn_chunk_grid(a.M, a.C, sms);
  if (a.sample_scale != nullptr) {     // stochastic depth: train only, a residual, no activation, bit mask or fp8 twin
    if (!train || a.relu != 0 || a.residual == nullptr || a.mask != nullptr || (a.zq != nullptr && a.zq_slot != nullptr) ||
        a.hw <= 0 || a.M % a.hw != 0)
      return cudaErrorInvalidValue;
    return flat ? launch_pdl(bn_sd_fwd_kernel<false>, grid, dim3(kBnThreads), 0, stream, 1, a)
                : launch_pdl(bn_sd_fwd_kernel<true>, grid, dim3(kBnThreads), 0, stream, 1, a);
  }
  if (a.relu == 3 || a.relu == 4 || a.relu == 5) {    // hardswish / SiLU / GELU: no residual, bit mask or fp8 twin
    if (a.residual != nullptr || a.mask != nullptr || (a.zq != nullptr && a.zq_slot != nullptr)) return cudaErrorInvalidValue;
    if (a.relu == 5) {
      if (flat)
        return train ? launch_pdl(bn_gelu_fwd_kernel<true, false>, grid, dim3(kBnThreads), 0, stream, 1, a)
                     : launch_pdl(bn_gelu_fwd_kernel<false, false>, grid, dim3(kBnThreads), 0, stream, 1, a);
      return train ? launch_pdl(bn_gelu_fwd_kernel<true, true>, grid, dim3(kBnThreads), 0, stream, 1, a)
                   : launch_pdl(bn_gelu_fwd_kernel<false, true>, grid, dim3(kBnThreads), 0, stream, 1, a);
    }
    if (a.relu == 4) {
      if (flat)
        return train ? launch_pdl(bn_silu_fwd_kernel<true, false>, grid, dim3(kBnThreads), 0, stream, 1, a)
                     : launch_pdl(bn_silu_fwd_kernel<false, false>, grid, dim3(kBnThreads), 0, stream, 1, a);
      return train ? launch_pdl(bn_silu_fwd_kernel<true, true>, grid, dim3(kBnThreads), 0, stream, 1, a)
                   : launch_pdl(bn_silu_fwd_kernel<false, true>, grid, dim3(kBnThreads), 0, stream, 1, a);
    }
    if (flat)
      return train ? launch_pdl(bn_hswish_fwd_kernel<true, false>, grid, dim3(kBnThreads), 0, stream, 1, a)
                   : launch_pdl(bn_hswish_fwd_kernel<false, false>, grid, dim3(kBnThreads), 0, stream, 1, a);
    return train ? launch_pdl(bn_hswish_fwd_kernel<true, true>, grid, dim3(kBnThreads), 0, stream, 1, a)
                 : launch_pdl(bn_hswish_fwd_kernel<false, true>, grid, dim3(kBnThreads), 0, stream, 1, a);
  }
  if (a.relu < 0 || a.relu > 2 || (a.relu == 2 && a.mask != nullptr)) return cudaErrorInvalidValue;   // no ReLU6 bit mask
  const bool f8 = a.zq != nullptr && a.zq_slot != nullptr && train;
  const bool r6 = a.relu == 2;
  if (flat) {
    return r6 ? launch_bn_fwd_variant<false, true>(a, train, f8, grid, stream)
              : launch_bn_fwd_variant<false, false>(a, train, f8, grid, stream);
  }
  return r6 ? launch_bn_fwd_variant<true, true>(a, train, f8, grid, stream)
            : launch_bn_fwd_variant<true, false>(a, train, f8, grid, stream);
}

cudaError_t launch_bn_act_bwd(const BnBwdArgs& a_in, int sms, cudaStream_t stream, bool skip_reduce) {
  BnBwdArgs a = a_in;
  a.reverse = g_bn_reverse;
  if (a.C % 8 != 0 || a.C <= 0) return cudaErrorInvalidValue;
  if (a.sample_scale != nullptr) {     // stochastic depth: no activation, no fp8 twin, sums not pre-reduced
    if (a.relu != 0 || a.zmask != nullptr || skip_reduce || (a.dxq != nullptr && a.dxq_slot != nullptr) || a.hw <= 0 ||
        a.M % a.hw != 0)
      return cudaErrorInvalidValue;
    return launch_bn_bwd_mask<kMaskSD>(a, sms, stream, false);
  }
  if (a.relu == 3 || a.relu == 4 || a.relu == 5) {    // hardswish / SiLU / GELU: pre-activation recomputed from x only,
    if (!a.mask_from_x || a.zmask != nullptr || a.dres != nullptr) return cudaErrorInvalidValue;   // no dres
    if (a.relu == 5) return launch_bn_bwd_mask<kMaskXG>(a, sms, stream, skip_reduce);
    return a.relu == 3 ? launch_bn_bwd_mask<kMaskXH>(a, sms, stream, skip_reduce)
                       : launch_bn_bwd_mask<kMaskXS>(a, sms, stream, skip_reduce);
  }
  if (a.relu < 0 || a.relu > 2 || (a.relu == 2 && a.zmask != nullptr)) return cudaErrorInvalidValue;   // no ReLU6 bit mask
  switch (!a.relu ? kMaskNone
                  : a.relu == 2 ? (a.mask_from_x ? kMaskX6 : kMaskZ6)
                                : (a.mask_from_x ? kMaskX : (a.zmask ? kMaskBits : kMaskZ))) {
    case kMaskNone: return launch_bn_bwd_mask<kMaskNone>(a, sms, stream, skip_reduce);
    case kMaskZ: return launch_bn_bwd_mask<kMaskZ>(a, sms, stream, skip_reduce);
    case kMaskBits: return launch_bn_bwd_mask<kMaskBits>(a, sms, stream, skip_reduce);
    case kMaskX: return launch_bn_bwd_mask<kMaskX>(a, sms, stream, skip_reduce);
    case kMaskZ6: return launch_bn_bwd_mask<kMaskZ6>(a, sms, stream, skip_reduce);
    default: return launch_bn_bwd_mask<kMaskX6>(a, sms, stream, skip_reduce);
  }
}


cudaError_t launch_bn_relu_maxpool_fwd(const BnFwdArgs& a, const PoolArgs& p, __nv_bfloat16* pooled, uint8_t* argmax,
                                       int sms, cudaStream_t stream) {
  if (a.C % 8 != 0 || a.C <= 0 || a.M != p.N * p.H * p.W || a.C != p.C || p.k * p.k > 255) return cudaErrorInvalidValue;
  const dim3 grid = bn_chunk_grid(p.N * p.P * p.Q, a.C, sms);
  bn_relu_maxpool_fwd_kernel<<<grid, kBnThreads, 0, stream>>>(a, p, pooled, argmax);
  return cudaGetLastError();
}

cudaError_t launch_bn_pool_bwd(const BnBwdArgs& a, const PoolArgs& p, const __nv_bfloat16* dy_pooled, const uint8_t* argmax,
                               int sms, cudaStream_t stream) {
  if (a.C % 8 != 0 || a.C <= 0 || a.M != p.N * p.H * p.W || a.C != p.C) return cudaErrorInvalidValue;
  const dim3 grid = bn_chunk_grid(a.M, a.C, sms);
  bn_pool_bwd_reduce_kernel<<<grid, kBnThreads, 0, stream>>>(a, p, dy_pooled, argmax);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  bn_pool_bwd_apply_kernel<<<grid, kBnThreads, 0, stream>>>(a, p, dy_pooled, argmax);
  return cudaGetLastError();
}

}  // namespace ddl
