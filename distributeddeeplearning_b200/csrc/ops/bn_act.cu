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
enum { kMaskNone = 0, kMaskZ = 1, kMaskX = 2, kMaskBits = 3 };

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

template <bool TRAIN, bool CHUNKED, bool FP8>
__global__ void __launch_bounds__(kBnThreads, 4) bn_act_fwd_kernel(BnFwdArgs a) {
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
    if (a.residual) {
      float res[8];
      unpack8(ur, res);
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaf(x[i], scale[i], shift[i]) + res[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaf(x[i], scale[i], shift[i]);
    }
    if (a.relu) {
      if (a.mask) {
        uint32_t bits = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) bits |= (z[i] > 0.f ? 1u : 0u) << i;
        a.mask[off >> 3] = static_cast<uint8_t>(bits);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) z[i] = fmaxf(z[i], 0.f);
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
  if (MASK == kMaskX && live) {
    Vec8 mean = load8_f32(a.mean + c0), invstd = load8_f32(a.invstd + c0);
    Vec8 gam = load8_f32(a.gamma + c0), bet = load8_f32(a.beta + c0);
#pragma unroll
    for (int i = 0; i < 8; ++i) { msc[i] = gam.v[i] * invstd.v[i]; msh[i] = bet.v[i] - mean.v[i] * msc[i]; }
  }
  auto accumulate = [&](const uint4& udz, const uint4& ux, const uint4& uz) {
    float dz[8], x[8];
    unpack8(udz, dz);
    unpack8(ux, x);
    if (MASK == kMaskZ) {
      float z[8];
      unpack8(uz, z);
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = z[i] > 0.f ? dz[i] : 0.f;
    } else if (MASK == kMaskBits) {        // uz.x carries the 8 mask bits of this (row, channel group)
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = ((uz.x >> i) & 1u) ? dz[i] : 0.f;
    } else if (MASK == kMaskX) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = fmaf(x[i], msc[i], msh[i]) > 0.f ? dz[i] : 0.f;
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
  for (; r + rstep < a.M; r += 2 * rstep) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const size_t off1 = static_cast<size_t>(phys(r + rstep)) * a.C + c0;
    const uint4 d0 = ld_stream_u4(a.dz + off0), d1 = ld_stream_u4(a.dz + off1);
    const uint4 x0 = ld_stream_u4(a.x + off0), x1 = ld_stream_u4(a.x + off1);
    uint4 z0 = make_uint4(0, 0, 0, 0), z1 = z0;
    if (MASK == kMaskZ) { z0 = ld_stream_u4(a.z + off0); z1 = ld_stream_u4(a.z + off1); }
    if (MASK == kMaskBits) { z0.x = a.zmask[off0 >> 3]; z1.x = a.zmask[off1 >> 3]; }
    accumulate(d0, x0, z0);
    accumulate(d1, x1, z1);
  }
  if (r < a.M) {
    const size_t off0 = static_cast<size_t>(phys(r)) * a.C + c0;
    const uint4 d0 = ld_stream_u4(a.dz + off0);
    const uint4 x0 = ld_stream_u4(a.x + off0);
    uint4 z0 = make_uint4(0, 0, 0, 0);
    if (MASK == kMaskZ) z0 = ld_stream_u4(a.z + off0);
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
    if (row0 == 0 && a.gamma_grad) {   // exactly one thread per channel group: accumulate parameter grads
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        a.gamma_grad[c0 + i] += dg.v[i];
        a.beta_grad[c0 + i] += db.v[i];
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      k1[i] = gam.v[i] * invstd.v[i];
      cB[i] = -k1[i] * invstd.v[i] * dg.v[i] * inv_n;
      cA[i] = -k1[i] * db.v[i] * inv_n - mean.v[i] * cB[i];
      msh[i] = 0.f;
    }
    if (MASK == kMaskX) {
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
    if (MASK == kMaskZ) {
      float z[8];
      unpack8(ld_stream_u4(a.z + off), z);
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = z[i] > 0.f ? dz[i] : 0.f;
    } else if (MASK == kMaskBits) {
      const uint32_t bits = a.zmask[off >> 3];
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = ((bits >> i) & 1u) ? dz[i] : 0.f;
    } else if (MASK == kMaskX) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dz[i] = fmaf(x[i], k1[i], msh[i]) > 0.f ? dz[i] : 0.f;
    }
    if (a.dres) store8_bf16(a.dres + off, dz);
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
    if (row0 == 0 && a.gamma_grad) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        a.gamma_grad[c0 + i] += dg.v[i];
        a.beta_grad[c0 + i] += db.v[i];
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

cudaError_t launch_bn_act_fwd(const BnFwdArgs& a_in, bool train, int sms, cudaStream_t stream) {
  BnFwdArgs a = a_in;
  a.reverse = g_bn_reverse;
  if (a.C % 8 != 0 || a.C <= 0) return cudaErrorInvalidValue;
  const bool f8 = a.zq != nullptr && a.zq_slot != nullptr && train;
  cudaError_t e = cudaSuccess;
  if (bn_flat_ok(a.C)) {
    const int grid = bn_grid(a.M, a.C, sms);
    if (f8) e = launch_pdl(bn_act_fwd_kernel<true, false, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
    else if (train) e = launch_pdl(bn_act_fwd_kernel<true, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
    else e = launch_pdl(bn_act_fwd_kernel<false, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
  } else {
    const dim3 grid = bn_chunk_grid(a.M, a.C, sms);
    if (f8) e = launch_pdl(bn_act_fwd_kernel<true, true, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
    else if (train) e = launch_pdl(bn_act_fwd_kernel<true, true, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
    else e = launch_pdl(bn_act_fwd_kernel<false, true, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a);
  }
  return e;
}

cudaError_t launch_bn_act_bwd(const BnBwdArgs& a_in, int sms, cudaStream_t stream, bool skip_reduce) {
  BnBwdArgs a = a_in;
  a.reverse = g_bn_reverse;
  if (a.C % 8 != 0 || a.C <= 0) return cudaErrorInvalidValue;
  const int mask = !a.relu ? kMaskNone : (a.mask_from_x ? kMaskX : (a.zmask ? kMaskBits : kMaskZ));
  const dim3 rgrid = bn_chunk_grid(a.M, a.C, sms);
  cudaError_t e = cudaSuccess;
  if (!skip_reduce) switch (mask) {
    case kMaskNone: e = launch_pdl(bn_act_bwd_reduce_kernel<kMaskNone>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
    case kMaskZ: e = launch_pdl(bn_act_bwd_reduce_kernel<kMaskZ>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
    case kMaskBits: e = launch_pdl(bn_act_bwd_reduce_kernel<kMaskBits>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
    default: e = launch_pdl(bn_act_bwd_reduce_kernel<kMaskX>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
  }
  if (e != cudaSuccess) return e;
  const bool f8 = a.dxq != nullptr && a.dxq_slot != nullptr;
  if (bn_flat_ok(a.C)) {
    const int grid = bn_grid(a.M, a.C, sms);
    switch (mask) {
      case kMaskNone: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskNone, false, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskNone, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); break;
      case kMaskZ: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskZ, false, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskZ, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); break;
      case kMaskBits: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskBits, false, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskBits, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); break;
      default: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskX, false, true>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskX, false, false>, dim3(grid), dim3(kBnThreads), 0, stream, 1, a); break;
    }
  } else {
    switch (mask) {
      case kMaskNone: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskNone, true, true>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskNone, true, false>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
      case kMaskZ: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskZ, true, true>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskZ, true, false>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
      case kMaskBits: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskBits, true, true>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskBits, true, false>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
      default: if (f8) e = launch_pdl(bn_act_bwd_apply_kernel<kMaskX, true, true>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); else e = launch_pdl(bn_act_bwd_apply_kernel<kMaskX, true, false>, dim3(rgrid), dim3(kBnThreads), 0, stream, 1, a); break;
    }
  }
  return e;
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
