// Warp-level bf16 tensor-core tile code of the attention kernels (attention.cu, window_attention.cu,
// window_attention_v2.cu): mma.sync.m16n8k16 with fp32 accumulators, ldmatrix operand loads from shared tiles of any
// row stride, the 16-row warp tile products, the per-relative-index dS sums of the bias gradients and the first level
// of their deterministic reduction.
//
// Fragment layout (PTX ISA, mma.m16n8k16): lane l holds rows l/4 and l/4 + 8, columns 8j + 2(l%4) + {0, 1} of every
// 8-column n-tile j of a 16-row accumulator tile; the accumulator pair of n-tiles 2k, 2k+1 rounded to bf16 is the A
// fragment of k-slice k, so a score tile is the A operand of the next product without leaving registers.
#pragma once

#include <cuda_bf16.h>
#include <stdint.h>

#include "../common.cuh"

namespace ddl {
namespace mma_tile {

DDL_DEVICE void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
DDL_DEVICE void ldsm4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
DDL_DEVICE void ldsm4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// lane addresses of ldmatrix on a tile of row stride LD (lane l feeds row l % 8 of matrix l / 8):
// A fragment of rows m0.., columns k0.. (row-major A), and B of a [k][n]-stored operand (trans)
template <int LD>
DDL_DEVICE uint32_t addr_a(uint32_t tile, int r0, int c0, int lane) {
  const int i = lane >> 3, r = lane & 7;
  return tile + static_cast<uint32_t>(((r0 + (i & 1) * 8 + r) * LD + c0 + (i >> 1) * 8) * 2);
}
// B of an [n][k]-stored operand (non-trans): matrices (n0, k0), (n0, k0+8), (n0+8, k0), (n0+8, k0+8)
template <int LD>
DDL_DEVICE uint32_t addr_bn(uint32_t tile, int n0, int k0, int lane) {
  const int i = lane >> 3, r = lane & 7;
  return tile + static_cast<uint32_t>(((n0 + (i >> 1) * 8 + r) * LD + k0 + (i & 1) * 8) * 2);
}
// A fragment of the transpose of a row-major [k][m] tile (trans): A rows m0.., columns k0..
template <int LD>
DDL_DEVICE uint32_t addr_at(uint32_t tile, int m0, int k0, int lane) {
  const int i = lane >> 3, r = lane & 7;
  return tile + static_cast<uint32_t>(((k0 + (i >> 1) * 8 + r) * LD + m0 + (i & 1) * 8) * 2);
}

// S[16 x 64] = A[16 x 16 KSLICES] B^T with B a [64 = n][16 KSLICES = k] tile of stride LDB (K in S = Q K^T, ...)
template <int LDB, int KSLICES>
DDL_DEVICE void mm_abt(float (&s)[8][4], const uint32_t (&a)[KSLICES][4], uint32_t tile, int lane) {
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < KSLICES; ++kk) {
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t b[4];
      ldsm4(addr_bn<LDB>(tile, 16 * jp, 16 * kk, lane), b);
      mma_bf16(s[2 * jp], a[kk], b[0], b[1]);
      mma_bf16(s[2 * jp + 1], a[kk], b[2], b[3]);
    }
  }
}
// acc[16 x 8 NTILES] += P[16 x 64] B with B a [64 = k][8 NTILES = n] tile of stride LDB (V in O += P V, ...);
// P given as the accumulator-layout fp32 tile, rounded to bf16 here
template <int LDB, int NTILES>
DDL_DEVICE void mm_pb(float (&acc)[NTILES][4], const float (&p)[8][4], uint32_t tile, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(p[2 * kk][0], p[2 * kk][1]), pack_bf16x2(p[2 * kk][2], p[2 * kk][3]),
                           pack_bf16x2(p[2 * kk + 1][0], p[2 * kk + 1][1]),
                           pack_bf16x2(p[2 * kk + 1][2], p[2 * kk + 1][3])};
#pragma unroll
    for (int jp = 0; jp < NTILES / 2; ++jp) {
      uint32_t b[4];
      ldsm4_t(addr_a<LDB>(tile, 16 * kk, 16 * jp, lane), b);
      mma_bf16(acc[2 * jp], a, b[0], b[1]);
      mma_bf16(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}
// acc[16 x 32] += A^T[16 x 64] B with A^T the transpose of the rows m0.. of a [64 = k][64 = m] tile of stride LDA and
// B a [64 = k][32 = n] tile of stride LDB  (dV = P^T dO, dK = dS^T Q)
template <int LDA, int LDB>
DDL_DEVICE void mm_atb(float (&acc)[4][4], uint32_t at, int m0, uint32_t tile, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    ldsm4_t(addr_at<LDA>(at, m0, 16 * kk, lane), a);
#pragma unroll
    for (int jp = 0; jp < 2; ++jp) {
      uint32_t b[4];
      ldsm4_t(addr_a<LDB>(tile, 16 * kk, 16 * jp, lane), b);
      mma_bf16(acc[2 * jp], a, b[0], b[1]);
      mma_bf16(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}

// sum of dS over the pairs (i, j) of a WIN x WIN window with relative index
// k = (iy - jy + WIN - 1) (2 WIN - 1) + (ix - jx + WIN - 1), in row-major order of i; dS of (i, j) at dsf[i * LDF + j]
template <int WIN, int LDF>
DDL_DEVICE float rel_sum(const float* dsf, int k) {
  constexpr int kW = 2 * WIN - 1;
  const int dy = k / kW - (WIN - 1), dx = k - (k / kW) * kW - (WIN - 1);
  float s = 0.f;
  for (int iy = dy > 0 ? dy : 0; iy < (dy < 0 ? WIN + dy : WIN); ++iy)
    for (int ix = dx > 0 ? dx : 0; ix < (dx < 0 ? WIN + dx : WIN); ++ix)
      s += dsf[(iy * WIN + ix) * LDF + (iy - dy) * WIN + ix - dx];
  return s;
}

// Kernels here are templates in an unnamed namespace: each translation unit that launches one gets its own instance
// and host stub, and one that does not compiles none.
namespace {

// first level of a parameter-gradient reduction that is bit-identical run to run: chunk c of the P partial rows of
// `per` floats, summed in order -> chunk [CHUNKS][per]
template <int THREADS, int CHUNKS>
__global__ void __launch_bounds__(THREADS) grad_chunk_kernel(const float* __restrict__ part, float* __restrict__ chunk,
                                                             int P, int per) {
  pdl_trigger();
  pdl_wait();
  const int e = blockIdx.x * THREADS + threadIdx.x, c = blockIdx.y;
  if (e >= per) return;
  const int p0 = static_cast<int>(static_cast<int64_t>(P) * c / CHUNKS);
  const int p1 = static_cast<int>(static_cast<int64_t>(P) * (c + 1) / CHUNKS);
  float s = 0.f;
#pragma unroll 8
  for (int p = p0; p < p1; ++p) s += part[static_cast<size_t>(p) * per + e];
  chunk[static_cast<size_t>(c) * per + e] = s;
}

}  // namespace

}  // namespace mma_tile
}  // namespace ddl
