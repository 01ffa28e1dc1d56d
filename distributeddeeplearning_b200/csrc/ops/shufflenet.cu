// ShuffleNetV2's channel split, concat and shuffle, fused into the BatchNorm of the branch's last convolution
// (ops/shufflenet.py runs a whole unit as one autograd node on these kernels and the conv / depthwise / BN kernels).
//
// A unit's output interleaves two halves of `half` channels each:  s[2i] = a[i],  s[2i+1] = relu(BN_b(b[i])).
//   stride 1: a is the unit's pass-through input (copied bit for bit), b the branch's last 1x1 conv output;
//   stride 2: a is relu(BN_a(a[i])) of branch1's last conv output, applied in the same pass.
// s is stored whole ([M][ld_s]) or as its two channel halves lo = s[:, :half] and hi = s[:, half:] ([M][ld_ab] each),
// which the next stride-1 unit reads as its pass-through and its branch input: no split copy.  Every stored tensor
// holds its real channels first, then zeros up to its pitch (a multiple of 8).
//
//   forward   one pass: read a and b once, write s (16-byte stores); train: the BN statistics come from the conv
//             epilogue (sum, sum of squares); mean / invstd saved, running statistics updated for the real channels
//   backward  pass 1 (reduce): de-interleave ds on the fly, S1 = sum g, S2 = sum g * y of the BN-ReLU half (halves),
//             g the output gradient masked by relu'(BN(y)); stride 1 also writes the pass-through gradient (bit copy)
//             pass 2 (apply): read ds again, dy = gamma invstd (g - dbeta / M - xhat dgamma / M); no de-interleaved copy
//             of the branch gradient is ever stored
//
// Thread mapping (both directions): a block owns a 64-wide chunk of channels (blockIdx.y) and 32 row lanes; a thread
// owns 8 consecutive channels of the tensor it stores, so that its stores are 16-byte vectors.  In forward those are 8
// output channels of s / lo / hi (their sources are 4 + 4 scattered a / b channels, read as 2-byte values); in backward
// 8 consecutive channel pairs (a[i], b[i]), each one 4-byte word of ds (half is even, so a pair never straddles lo / hi).
#include "../common.cuh"
#include "ops.h"

namespace ddl {

namespace {

constexpr int kShThreads = 256;

DDL_DEVICE float bf16_bits_to_float(uint16_t h) { return __uint_as_float(static_cast<uint32_t>(h) << 16); }
DDL_DEVICE uint16_t float_to_bf16_bits(float v) {
  __nv_bfloat16 b = __float2bfloat16_rn(v);
  return *reinterpret_cast<uint16_t*>(&b);
}

// scale / shift of one BN channel; TRAIN and `writer`: also the saved mean / invstd and the running statistics
template <bool TRAIN>
DDL_DEVICE void sh_bn_channel(const ShuffleBn& bn, int c, int M, bool writer, float& scale, float& shift) {
  if (TRAIN) {
    const float inv_n = 1.f / static_cast<float>(M);
    const float mean = bn.sum[c] * inv_n;
    const float var = fmaxf(bn.sumsq[c] * inv_n - mean * mean, 0.f);
    const float invstd = rsqrtf(var + bn.eps);
    scale = bn.gamma[c] * invstd;
    shift = bn.beta[c] - mean * scale;
    if (writer) {
      bn.mean[c] = mean;
      bn.invstd[c] = invstd;
      if (bn.running_mean) {
        const float unbiased = M > 1 ? var * static_cast<float>(M) / static_cast<float>(M - 1) : var;
        bn.running_mean[c] = (1.f - bn.momentum) * bn.running_mean[c] + bn.momentum * mean;
        bn.running_var[c] = (1.f - bn.momentum) * bn.running_var[c] + bn.momentum * unbiased;
      }
    }
  } else {
    scale = bn.gamma[c] * rsqrtf(bn.running_var[c] + bn.eps);
    shift = bn.beta[c] - bn.running_mean[c] * scale;
  }
}

template <bool TRAIN, bool ABN>
__global__ void __launch_bounds__(kShThreads) shuffle_fwd_kernel(ShuffleArgs p) {
  const int width = p.split ? 2 * p.ld_s : p.ld_s;       // stored channels: lo then hi, or s
  const int v0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
  if (v0 >= width) return;
  const int dest = p.split ? v0 / p.ld_s : 0;
  const int j0 = v0 - dest * p.ld_s;
  const int real = p.split ? p.half : 2 * p.half;        // real channels of the destination
  const int row0 = blockIdx.x * 32 + (threadIdx.x >> 3);
  const bool writer = TRAIN && row0 == 0;                // exactly one thread per output channel group
  __nv_bfloat16* out = dest ? p.s1 : p.s0;
  int col[8];          // source channel, -1 in the pad
  bool fromb[8];
  float scale[8], shift[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int j = j0 + k;
    scale[k] = 1.f;
    shift[k] = 0.f;
    fromb[k] = false;
    col[k] = -1;
    if (j < real) {
      const int o = dest * p.half + j;
      col[k] = o >> 1;
      fromb[k] = o & 1;
      if (fromb[k]) sh_bn_channel<TRAIN>(p.bn_b, col[k], p.M, writer, scale[k], shift[k]);
      else if (ABN) sh_bn_channel<TRAIN>(p.bn_a, col[k], p.M, writer, scale[k], shift[k]);
    }
  }
  const uint16_t* a = reinterpret_cast<const uint16_t*>(p.a);
  const uint16_t* b = reinterpret_cast<const uint16_t*>(p.b);
  for (int r = row0; r < p.M; r += gridDim.x * 32) {
    const size_t rb = static_cast<size_t>(r) * p.ld_ab;
    uint16_t h[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (col[k] < 0) {
        h[k] = 0;
      } else if (fromb[k] || ABN) {
        const uint16_t raw = __ldg((fromb[k] ? b : a) + rb + col[k]);
        h[k] = float_to_bf16_bits(fmaxf(fmaf(bf16_bits_to_float(raw), scale[k], shift[k]), 0.f));
      } else {
        h[k] = __ldg(a + rb + col[k]);                  // the pass-through half: a bit copy
      }
    }
    const uint4 v = make_uint4(h[0] | (static_cast<uint32_t>(h[1]) << 16), h[2] | (static_cast<uint32_t>(h[3]) << 16),
                               h[4] | (static_cast<uint32_t>(h[5]) << 16), h[6] | (static_cast<uint32_t>(h[7]) << 16));
    *reinterpret_cast<uint4*>(out + static_cast<size_t>(r) * p.ld_s + j0) = v;
  }
}

// element offset of pair i's 4-byte word within a row of ds (whole) or of dlo / dhi (split), -1 beyond `half`
DDL_DEVICE int sh_pair_offset(const ShuffleArgs& p, int i, int& sel) {
  sel = 0;
  if (i >= p.half) return -1;
  const int o = 2 * i;
  if (!p.split) return o;
  sel = o >= p.half;
  return o - sel * p.half;
}

DDL_DEVICE void sh_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}

// the BN-ReLU mask constants of 8 channels starting at i0 (zeros beyond `half`)
DDL_DEVICE void sh_mask_consts(const ShuffleBn& bn, int i0, int half, float (&msc)[8], float (&msh)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = i0 + k;
    msc[k] = c < half ? bn.gamma[c] * bn.invstd[c] : 0.f;
    msh[k] = c < half ? bn.beta[c] - bn.mean[c] * msc[k] : 0.f;
  }
}

// block-wide sum of s1 / s2 over the 32 row lanes of each channel group, then one atomic per channel and sum
DDL_DEVICE void sh_reduce_store(const ShuffleBn& bn, int half, float (&s1)[8], float (&s2)[8], float (*red)[8][16]) {
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {       // lanes sharing a channel group: lane = (row lane % 4) * 8 + group
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
  if (threadIdx.x < 64) {
    const int g = threadIdx.x >> 3, i = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int w = 0; w < kShThreads / 32; ++w) { t1 += red[w][g][i]; t2 += red[w][g][8 + i]; }
    const int ch = blockIdx.y * 64 + g * 8 + i;
    if (ch < half) {
      atomicAdd(bn.dbeta + ch, t1);
      atomicAdd(bn.dgamma + ch, bn.invstd[ch] * (t2 - bn.mean[ch] * t1));
    }
  }
}

template <bool ABN>
__global__ void __launch_bounds__(kShThreads) shuffle_bwd_reduce_kernel(ShuffleArgs p) {
  __shared__ float red_b[kShThreads / 32][8][16];
  __shared__ float red_a[ABN ? kShThreads / 32 : 1][8][16];
  const int i0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
  const bool live = i0 < p.ld_ab;
  int off[8], sel[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) off[k] = sh_pair_offset(p, i0 + k, sel[k]);
  float s1b[8], s2b[8], mscb[8], mshb[8], s1a[8], s2a[8], msca[8], msha[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s1b[k] = 0.f; s2b[k] = 0.f; s1a[k] = 0.f; s2a[k] = 0.f; }
  sh_mask_consts(p.bn_b, i0, p.half, mscb, mshb);      // zeros for the channels beyond `half` (and idle threads)
  if (ABN) sh_mask_consts(p.bn_a, i0, p.half, msca, msha);
  const uint32_t* d0 = reinterpret_cast<const uint32_t*>(p.ds0);
  const uint32_t* d1 = reinterpret_cast<const uint32_t*>(p.ds1);
  for (int r = live ? blockIdx.x * 32 + (threadIdx.x >> 3) : p.M; r < p.M; r += gridDim.x * 32) {
    const size_t rb = static_cast<size_t>(r) * p.ld_ab + i0;
    const size_t rs = static_cast<size_t>(r) * (p.ld_s / 2);          // row pitch of ds / dlo / dhi in words
    float yb[8], ya[8];
    sh_unpack8(ld_stream_u4(p.b + rb), yb);
    if (ABN) sh_unpack8(ld_stream_u4(p.a + rb), ya);
    uint16_t pass[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t w = off[k] < 0 ? 0u : __ldg((sel[k] ? d1 : d0) + rs + off[k] / 2);
      pass[k] = static_cast<uint16_t>(w & 0xffffu);
      const float gb = fmaf(yb[k], mscb[k], mshb[k]) > 0.f ? bf16_bits_to_float(static_cast<uint16_t>(w >> 16)) : 0.f;
      s1b[k] += gb;
      s2b[k] = fmaf(gb, yb[k], s2b[k]);
      if (ABN) {
        const float ga = fmaf(ya[k], msca[k], msha[k]) > 0.f ? bf16_bits_to_float(pass[k]) : 0.f;
        s1a[k] += ga;
        s2a[k] = fmaf(ga, ya[k], s2a[k]);
      }
    }
    if (!ABN) {
      *reinterpret_cast<uint4*>(p.da + rb) =
          make_uint4(pass[0] | (static_cast<uint32_t>(pass[1]) << 16), pass[2] | (static_cast<uint32_t>(pass[3]) << 16),
                     pass[4] | (static_cast<uint32_t>(pass[5]) << 16), pass[6] | (static_cast<uint32_t>(pass[7]) << 16));
    }
  }
  sh_reduce_store(p.bn_b, p.half, s1b, s2b, red_b);
  if (ABN) sh_reduce_store(p.bn_a, p.half, s1a, s2a, red_a);
}

// dx = k1 g + y cB + cA with k1 = gamma invstd, cB = -k1 invstd dgamma / M, cA = -k1 dbeta / M - mean cB
DDL_DEVICE void sh_apply_consts(const ShuffleBn& bn, int i0, int half, int M, bool writer, float (&k1)[8],
                                float (&cA)[8], float (&cB)[8], float (&msh)[8]) {
  const float inv_n = 1.f / static_cast<float>(M);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = i0 + k;
    k1[k] = 0.f; cA[k] = 0.f; cB[k] = 0.f; msh[k] = 0.f;
    if (c < half) {
      const float invstd = bn.invstd[c], mean = bn.mean[c], dg = bn.dgamma[c], db = bn.dbeta[c];
      k1[k] = bn.gamma[c] * invstd;
      cB[k] = -k1[k] * invstd * dg * inv_n;
      cA[k] = -k1[k] * db * inv_n - mean * cB[k];
      msh[k] = bn.beta[c] - mean * k1[k];
      if (writer) {
        if (bn.gamma_grad) bn.gamma_grad[c] += dg;
        if (bn.beta_grad) bn.beta_grad[c] += db;
      }
    }
  }
}

template <bool ABN>
__global__ void __launch_bounds__(kShThreads) shuffle_bwd_apply_kernel(ShuffleArgs p) {
  const int i0 = blockIdx.y * 64 + (threadIdx.x & 7) * 8;
  if (i0 >= p.ld_ab) return;
  const int row0 = blockIdx.x * 32 + (threadIdx.x >> 3);
  int off[8], sel[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) off[k] = sh_pair_offset(p, i0 + k, sel[k]);
  float k1b[8], cAb[8], cBb[8], mshb[8], k1a[8], cAa[8], cBa[8], msha[8];
  sh_apply_consts(p.bn_b, i0, p.half, p.M, row0 == 0, k1b, cAb, cBb, mshb);
  if (ABN) sh_apply_consts(p.bn_a, i0, p.half, p.M, row0 == 0, k1a, cAa, cBa, msha);
  const uint32_t* d0 = reinterpret_cast<const uint32_t*>(p.ds0);
  const uint32_t* d1 = reinterpret_cast<const uint32_t*>(p.ds1);
  for (int r = row0; r < p.M; r += gridDim.x * 32) {
    const size_t rb = static_cast<size_t>(r) * p.ld_ab + i0;
    const size_t rs = static_cast<size_t>(r) * (p.ld_s / 2);
    float yb[8], ya[8], ob[8], oa[8];
    sh_unpack8(ld_stream_u4(p.b + rb), yb);
    if (ABN) sh_unpack8(ld_stream_u4(p.a + rb), ya);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t w = off[k] < 0 ? 0u : __ldg((sel[k] ? d1 : d0) + rs + off[k] / 2);
      const float gb = fmaf(yb[k], k1b[k], mshb[k]) > 0.f ? bf16_bits_to_float(static_cast<uint16_t>(w >> 16)) : 0.f;
      ob[k] = fmaf(gb, k1b[k], fmaf(yb[k], cBb[k], cAb[k]));
      if (ABN) {
        const float ga = fmaf(ya[k], k1a[k], msha[k]) > 0.f ? bf16_bits_to_float(static_cast<uint16_t>(w & 0xffffu)) : 0.f;
        oa[k] = fmaf(ga, k1a[k], fmaf(ya[k], cBa[k], cAa[k]));
      }
    }
    *reinterpret_cast<uint4*>(p.db + rb) = make_uint4(pack_bf16x2(ob[0], ob[1]), pack_bf16x2(ob[2], ob[3]),
                                                      pack_bf16x2(ob[4], ob[5]), pack_bf16x2(ob[6], ob[7]));
    if (ABN)
      *reinterpret_cast<uint4*>(p.da + rb) = make_uint4(pack_bf16x2(oa[0], oa[1]), pack_bf16x2(oa[2], oa[3]),
                                                        pack_bf16x2(oa[4], oa[5]), pack_bf16x2(oa[6], oa[7]));
  }
}

inline dim3 sh_grid(int M, int width, int sms) {
  const int chunks = (width + 63) / 64;
  int gx = (M + 32 * 8 - 1) / (32 * 8);
  const int cap = (sms * 8 + chunks - 1) / chunks;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3(gx, chunks);
}

bool sh_args_ok(const ShuffleArgs& p) {
  if (p.M <= 0 || p.half <= 0 || p.half % 2 != 0 || p.ld_ab % 8 != 0 || p.ld_ab < p.half) return false;
  return p.split ? p.ld_s == p.ld_ab : (p.ld_s % 8 == 0 && p.ld_s >= 2 * p.half);
}

}  // namespace

cudaError_t launch_shuffle_fwd(const ShuffleArgs& p, int sms, cudaStream_t stream) {
  if (!sh_args_ok(p) || p.a == nullptr || p.b == nullptr || p.s0 == nullptr || (p.split && p.s1 == nullptr))
    return cudaErrorInvalidValue;
  const dim3 grid = sh_grid(p.M, p.split ? 2 * p.ld_s : p.ld_s, sms);
  if (p.train) {
    if (p.a_bn) shuffle_fwd_kernel<true, true><<<grid, kShThreads, 0, stream>>>(p);
    else shuffle_fwd_kernel<true, false><<<grid, kShThreads, 0, stream>>>(p);
  } else {
    if (p.a_bn) shuffle_fwd_kernel<false, true><<<grid, kShThreads, 0, stream>>>(p);
    else shuffle_fwd_kernel<false, false><<<grid, kShThreads, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

cudaError_t launch_shuffle_bwd(const ShuffleArgs& p, int sms, cudaStream_t stream) {
  if (!sh_args_ok(p) || p.b == nullptr || p.ds0 == nullptr || (p.split && p.ds1 == nullptr) || p.da == nullptr ||
      p.db == nullptr || (p.a_bn && p.a == nullptr))
    return cudaErrorInvalidValue;
  const dim3 grid = sh_grid(p.M, p.ld_ab, sms);
  if (p.a_bn) {
    shuffle_bwd_reduce_kernel<true><<<grid, kShThreads, 0, stream>>>(p);
    shuffle_bwd_apply_kernel<true><<<grid, kShThreads, 0, stream>>>(p);
  } else {
    shuffle_bwd_reduce_kernel<false><<<grid, kShThreads, 0, stream>>>(p);
    shuffle_bwd_apply_kernel<false><<<grid, kShThreads, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

}  // namespace ddl
