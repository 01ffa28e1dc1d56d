// Helpers shared by the depthwise convolution kernels: depthwise.cu (3x3) and depthwise5.cu (5x5).
//
// Thread mapping (every depthwise kernel): a thread owns 8 consecutive channels (one 16-byte vector) of a fixed channel
// slab and walks output (dgrad: input) pixels with a grid stride.  A block of 256 threads covers `gpc` channel groups x
// 256/gpc pixel lanes, gpc being the largest power of two <= 8 that divides C/8: every thread is live for any
// C % 8 == 0, and a pixel's slab is gpc*16 contiguous bytes.  blockIdx.y picks the slab.
#pragma once

#include "../common.cuh"

namespace ddl {
namespace dw {

constexpr int kDwThreads = 256;
constexpr int kDwWarps = kDwThreads / 32;

DDL_DEVICE void dw_unpack8(const uint4& u, float (&v)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
DDL_DEVICE void dw_load8(const __nv_bfloat16* p, float (&v)[8]) {
  dw_unpack8(__ldg(reinterpret_cast<const uint4*>(p)), v);
}

// this thread's channel slab and pixel lane
struct DwMap {
  int c0, lane, lanes;
};
DDL_DEVICE DwMap dw_map(int lg) {
  DwMap m;
  m.c0 = (static_cast<int>(blockIdx.y) << (lg + 3)) + ((threadIdx.x & ((1 << lg) - 1)) << 3);
  m.lane = blockIdx.x * (kDwThreads >> lg) + (threadIdx.x >> lg);
  m.lanes = gridDim.x * (kDwThreads >> lg);
  return m;
}

// Sum v[K] over the pixel lanes of the block that share this thread's channel group (v[k] belongs to channel k % 8),
// then hand each of the block's gpc*K totals to `emit(channel, k / 8, total)` on one thread: the caller's one atomic per
// channel and statistic (or tap) per block.  Lanes of a warp with the same channel group differ in lane bits >= lg.
template <int K, typename Emit>
DDL_DEVICE void dw_block_reduce(float (&v)[K], int lg, float* red /* [kDwWarps][8][K] */, Emit emit) {
  for (int off = 1 << lg; off < 32; off <<= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], off);
  }
  const int warp = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l < (1 << lg)) {
#pragma unroll
    for (int k = 0; k < K; ++k) red[(warp * 8 + l) * K + k] = v[k];
  }
  __syncthreads();
  const int slab0 = static_cast<int>(blockIdx.y) << (lg + 3);
  for (int e = threadIdx.x; e < (K << lg); e += kDwThreads) {
    const int g = e / K, k = e - g * K;
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kDwWarps; ++w) t += red[(w * 8 + g) * K + k];
    emit(slab0 + g * 8 + (k & 7), k >> 3, t);
  }
}

// largest power of two <= 8 dividing C/8, as its log2
inline int dw_lg_gpc(int C) {
  const int groups = C / 8;
  int lg = 0;
  while (lg < 3 && groups % (2 << lg) == 0) ++lg;
  return lg;
}

// (pixel blocks, channel slabs): at least 4 pixels per thread (amortises the weight loads), at most
// `blocks_per_sm` * SMs blocks in all
inline dim3 dw_grid(int pixels, int C, int lg, int sms, int blocks_per_sm) {
  const int slabs = (C / 8) >> lg;
  const int lanes = kDwThreads >> lg;
  long long gx = (static_cast<long long>(pixels) + 4LL * lanes - 1) / (4LL * lanes);
  const long long cap = (static_cast<long long>(sms) * blocks_per_sm + slabs - 1) / slabs;
  if (gx > cap) gx = cap;
  if (gx < 1) gx = 1;
  return dim3(static_cast<unsigned>(gx), static_cast<unsigned>(slabs));
}

}  // namespace dw
}  // namespace ddl
