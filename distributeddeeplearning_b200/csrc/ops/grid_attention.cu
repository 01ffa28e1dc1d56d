// Partition attention of MaxViT (torchvision's PartitionAttentionLayer): 49-token sequences, head dim 32, a learned
// relative-position bias and no mask, on the image-order qkv rows of the layer.  Two token maps, one per layer type:
//
//   grid   (WindowPartition(p = H/7) + SwapAxes): sequence (i, j), i, j in [0, p), token t = 7a + b at pixel (a p + i,
//          b p + j): the 49 tokens are spaced p pixels apart along both axes.
//   window (WindowPartition(7)): sequence (i, j), i, j in [0, H/7), token t = 7a + b at pixel (7i + a, 7j + b).
//
// Both maps cut a square H = W = 7p map into p x p sequences, so the CTA layout is the same and only the token -> row
// map differs (a compile-time flag).  The map is square because torchvision's grid partition takes one p for both axes.
//
// Logits: S = q . k * scale + table[(a - a' + 6) * 13 + (b - b' + 6)][h], with the fp32 table [169][heads] read
// directly and scale a runtime value: torchvision's RelativePositionalMultiHeadAttention scales k by feat_dim^-1/2, the
// layer's channel count C, not the head dim (1/sqrt(32) only for one head).  This is why MaxViT's window layer does not
// run on window_attention.cu, whose scale is 1/sqrt(32).
//
// Layout: qkv is the bf16 [N*H*W][3C] output of the qkv GEMM on the NHWC rows in image order; head h's Q, K and V are
// the 32 columns at 32h, C + 32h and 2C + 32h.  O of token t goes back to the same row of o [N*H*W][C]; lse
// [N*H*W][heads] fp32 is the natural-log log-sum-exp of the logits of every (token, head).  There is no partition, swap
// or reverse copy.
//
// Mapping and tiles are those of window_attention.cu: one CTA of 4 warps per (sequence, head, image) in the forward,
// mma.sync.m16n8k16 bf16 with fp32 accumulators, 64-row tiles (rows 49..63 zero, keys 49..63 at -inf), single-pass fp32
// softmax in base 2.  Backward: one CTA per (sequence row i, head, image) walks the sequences j = 0, 1, ... in order;
// dS in fp32 feeds the bias gradient, summed per relative index in a fixed order, then over (n, i) in fixed chunks and
// over the chunks in order by two small kernels.  No atomics: dqkv and dtable are bit-identical run to run.
#include <math.h>

#include "../common.cuh"
#include "ops.h"
#include "tc_utils.cuh"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kP = 7;
constexpr int kL = kP * kP;       // 49 tokens per sequence
constexpr int kD = 32;            // head dim
constexpr int kRows = 64;         // tile rows
constexpr int kThreads = 128;     // 4 warps x 16 rows
constexpr int kLd = 40;           // shared row stride (bf16) of the Q / K / V / dO tiles
constexpr int kLdP = 72;          // shared row stride (bf16) of the P / dS tiles
constexpr int kTab = 169;         // (2 * 7 - 1)^2 relative positions
constexpr int kChunks = 64;       // first-level chunks of the bias-gradient reduction
constexpr float kLog2e = 1.4426950408889634f;

struct GridArgs {
  const __nv_bfloat16* qkv;      // [N*H*W][3C]
  const __nv_bfloat16* o;        // [N*H*W][C]
  const __nv_bfloat16* dout;     // [N*H*W][C]   (backward)
  const float* table;            // [169][heads]
  __nv_bfloat16* out;            // forward: O; backward: dqkv
  float* lse;                    // [N*H*W][heads]
  float* part;                   // backward: [N * ns][heads][169]
  int H, C, heads, ns;           // ns = H / 7 sequences per side
  float scale;
};

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
// B of an [n][k]-stored operand (non-trans)
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

// S[16 x 64] = A[16 x 32] B^T with B a [64 = n][32 = k] tile of stride kLd
DDL_DEVICE void mm_abt(float (&s)[8][4], const uint32_t (&a)[2][4], uint32_t tile, int lane) {
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      uint32_t b[4];
      ldsm4(addr_bn<kLd>(tile, 16 * jp, 16 * kk, lane), b);
      mma_bf16(s[2 * jp], a[kk], b[0], b[1]);
      mma_bf16(s[2 * jp + 1], a[kk], b[2], b[3]);
    }
  }
}
// acc[16 x 32] += P[16 x 64] B with B a [64 = k][32 = n] tile of stride kLd; P in the accumulator layout (fp32)
DDL_DEVICE void mm_pb(float (&acc)[4][4], const float (&p)[8][4], uint32_t tile, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(p[2 * kk][0], p[2 * kk][1]), pack_bf16x2(p[2 * kk][2], p[2 * kk][3]),
                           pack_bf16x2(p[2 * kk + 1][0], p[2 * kk + 1][1]),
                           pack_bf16x2(p[2 * kk + 1][2], p[2 * kk + 1][3])};
#pragma unroll
    for (int jp = 0; jp < 2; ++jp) {
      uint32_t b[4];
      ldsm4_t(addr_a<kLd>(tile, 16 * kk, 16 * jp, lane), b);
      mma_bf16(acc[2 * jp], a, b[0], b[1]);
      mma_bf16(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}
// acc[16 x 32] += A^T[16 x 64] B with A^T the transpose of the rows m0.. of a [64 = k][64 = m] tile of stride kLdP and
// B a [64 = k][32 = n] tile of stride kLd  (dV = P^T dO, dK = dS^T Q)
DDL_DEVICE void mm_atb(float (&acc)[4][4], uint32_t at, int m0, uint32_t tile, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    ldsm4_t(addr_at<kLdP>(at, m0, 16 * kk, lane), a);
#pragma unroll
    for (int jp = 0; jp < 2; ++jp) {
      uint32_t b[4];
      ldsm4_t(addr_a<kLd>(tile, 16 * kk, 16 * jp, lane), b);
      mma_bf16(acc[2 * jp], a, b[0], b[1]);
      mma_bf16(acc[2 * jp + 1], a, b[2], b[3]);
    }
  }
}

// image-order row of token t = 7a + b of sequence (i, j) of image n
template <bool GRID>
DDL_DEVICE size_t token_row(const GridArgs& g, int n, int i, int j, int t) {
  const int ta = t / kP, tb = t - ta * kP;
  const int y = GRID ? ta * g.ns + i : kP * i + ta;
  const int x = GRID ? tb * g.ns + j : kP * j + tb;
  return (static_cast<size_t>(n) * g.H + y) * g.H + x;
}
DDL_DEVICE int rel_key(int t) { const int ta = t / kP; return ta * 13 + (t - ta * kP); }

// 64 rows x 32 bf16 of head columns `col` of the sequence's tokens (rows >= 49 zero-filled) into a tile of stride kLd
template <bool GRID>
DDL_DEVICE void load_seq(uint32_t tile, const GridArgs& g, const __nv_bfloat16* base, int ld, int col, int n, int i,
                         int j, int tid) {
#pragma unroll
  for (int it = 0; it < (kRows * 4) / kThreads; ++it) {
    const int c = tid + it * kThreads, r = c >> 2, ch = c & 3;
    const bool ok = r < kL;
    const __nv_bfloat16* src = base + (ok ? token_row<GRID>(g, n, i, j, r) : 0) * ld + col + ch * 8;
    tc::cp_async_16(tile + static_cast<uint32_t>((r * kLd + ch * 8) * 2), src, ok);
  }
}

// the base-2 logits of a warp's 16 x 64 score tile: s * scale + bias, keys >= 49 at -inf
DDL_DEVICE void logits(float (&s)[8][4], const GridArgs& g, int h, int row0, int lane) {
  const int gr = lane >> 2, t = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = row0 + gr + 8 * r;
    const int ri = rel_key(i < kL ? i : 0) + 84;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jj = 8 * j + 2 * t + e;
        float& x = s[j][2 * r + e];
        x = jj < kL ? fmaf(x, g.scale, __ldg(g.table + (ri - rel_key(jj)) * g.heads + h)) * kLog2e : -INFINITY;
      }
    }
  }
}

// sum of dS over the pairs (t, u) of relative index k = (ta - ua + 6) * 13 + (tb - ub + 6), in row-major order of t
DDL_DEVICE float rel_sum(const float* sSf, int k) {
  const int dy = k / 13 - 6, dx = k - (k / 13) * 13 - 6;
  float s = 0.f;
  for (int iy = dy > 0 ? dy : 0; iy < (dy < 0 ? kP + dy : kP); ++iy)
    for (int ix = dx > 0 ? dx : 0; ix < (dx < 0 ? kP + dx : kP); ++ix)
      s += sSf[(iy * kP + ix) * kL + (iy - dy) * kP + ix - dx];
  return s;
}

template <bool GRID>
__global__ void __launch_bounds__(kThreads) part_attn_fwd_kernel(GridArgs g) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[kRows * kLd];
  pdl_trigger();
  const int seq = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int si = seq / g.ns, sj = seq - si * g.ns;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gr = lane >> 2, t = lane & 3;
  const int ld = 3 * g.C;
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV);
  pdl_wait();
  load_seq<GRID>(q_s, g, g.qkv, ld, h * kD, n, si, sj, tid);
  load_seq<GRID>(k_s, g, g.qkv, ld, g.C + h * kD, n, si, sj, tid);
  load_seq<GRID>(v_s, g, g.qkv, ld, 2 * g.C + h * kD, n, si, sj, tid);
  tc::cp_async_commit();
  tc::cp_async_wait<0>();
  __syncthreads();
  uint32_t qf[2][4];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) ldsm4(addr_a<kLd>(q_s, 16 * warp, 16 * kk, lane), qf[kk]);
  float s[8][4];
  mm_abt(s, qf, k_s, lane);
  logits(s, g, h, 16 * warp, lane);
  float m[2], l[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(s[j][2 * r], s[j][2 * r + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    float ls = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& x = s[j][2 * r + e];
        x = exp2f(x - mx);
        ls += x;
      }
    }
    ls += __shfl_xor_sync(0xffffffffu, ls, 1);
    ls += __shfl_xor_sync(0xffffffffu, ls, 2);
    m[r] = mx;
    l[r] = ls;
  }
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  mm_pb(acc, s, v_s, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = 16 * warp + gr + 8 * r;
    if (i >= kL) continue;
    const size_t row = token_row<GRID>(g, n, si, sj, i);
    const float inv = 1.f / l[r];
    __nv_bfloat16* dst = g.out + row * g.C + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) g.lse[row * g.heads + h] = (m[r] + log2f(l[r])) * (1.f / kLog2e);
  }
}

template <bool GRID>
__global__ void __launch_bounds__(kThreads) part_attn_bwd_kernel(GridArgs g) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sO[kRows * kLd];        // dO
  __shared__ __align__(128) __nv_bfloat16 sP[kRows * kLdP];
  __shared__ __align__(128) __nv_bfloat16 sS[kRows * kLdP];       // dS
  __shared__ float sSf[kL * kL];                                  // dS (fp32) of the real pairs
  __shared__ float sD[kRows];
  pdl_trigger();
  const int si = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gr = lane >> 2, t = lane & 3;
  const int C = g.C, ld = 3 * C;
  const float scale = g.scale;
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV), o_s = tc::smem_u32(sO);
  const uint32_t p_s = tc::smem_u32(sP), s_s = tc::smem_u32(sS);
  float dt_sum = 0.f, dt_sum2 = 0.f;         // bias-gradient sums of relative index tid (and tid + 128 < 169)
  pdl_wait();
  for (int sj = 0; sj < g.ns; ++sj) {
    load_seq<GRID>(q_s, g, g.qkv, ld, h * kD, n, si, sj, tid);
    load_seq<GRID>(k_s, g, g.qkv, ld, C + h * kD, n, si, sj, tid);
    load_seq<GRID>(v_s, g, g.qkv, ld, 2 * C + h * kD, n, si, sj, tid);
    load_seq<GRID>(o_s, g, g.dout, C, h * kD, n, si, sj, tid);
    tc::cp_async_commit();
    {   // D = rowsum(dO o O): two threads per row, 16 columns each
      const int r = tid >> 1, c0 = h * kD + (tid & 1) * 16;
      float d = 0.f;
      if (r < kL) {
        const size_t off = token_row<GRID>(g, n, si, sj, r) * C + c0;
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const uint4 x = __ldg(reinterpret_cast<const uint4*>(g.dout + off) + v);
          const uint4 y = __ldg(reinterpret_cast<const uint4*>(g.o + off) + v);
          const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 u = unpack_bf16x2(xs[k]), w = unpack_bf16x2(ys[k]);
            d = fmaf(u.x, w.x, fmaf(u.y, w.y, d));
          }
        }
      }
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      if ((tid & 1) == 0) sD[r] = d;
    }
    tc::cp_async_wait<0>();
    __syncthreads();
    {
      uint32_t qf[2][4], df[2][4];
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {
        ldsm4(addr_a<kLd>(q_s, 16 * warp, 16 * kk, lane), qf[kk]);
        ldsm4(addr_a<kLd>(o_s, 16 * warp, 16 * kk, lane), df[kk]);
      }
      float p[8][4], dp[8][4];
      mm_abt(p, qf, k_s, lane);
      logits(p, g, h, 16 * warp, lane);
      mm_abt(dp, df, v_s, lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = 16 * warp + gr + 8 * r;
        const bool ok = i < kL;
        const float lse2 = ok ? g.lse[token_row<GRID>(g, n, si, sj, i) * g.heads + h] * kLog2e : 0.f;
        const float dr = sD[i];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int q = 2 * r + e, jj = 8 * j + 2 * t + e;
            const float pv = ok ? exp2f(p[j][q] - lse2) : 0.f;          // keys >= 49: exp2(-inf) = 0
            const float ds = pv * (dp[j][q] - dr);
            p[j][q] = pv;
            dp[j][q] = ds;
            if (ok && jj < kL) sSf[i * kL + jj] = ds;
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int off = (16 * warp + gr + 8 * r) * kLdP + 8 * j + 2 * t;
          *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16x2(p[j][2 * r], p[j][2 * r + 1]);
          *reinterpret_cast<uint32_t*>(sS + off) = pack_bf16x2(dp[j][2 * r], dp[j][2 * r + 1]);
        }
      }
      float dq[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;
      mm_pb(dq, dp, k_s, lane);                                      // dQ = dS K
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = 16 * warp + gr + 8 * r;
        if (i >= kL) continue;
        __nv_bfloat16* dst = g.out + token_row<GRID>(g, n, si, sj, i) * ld + h * kD + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(dq[j][2 * r] * scale, dq[j][2 * r + 1] * scale);
      }
    }
    __syncthreads();
    {
      float dk[4][4], dv[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
      mm_atb(dv, p_s, 16 * warp, o_s, lane);                         // dV = P^T dO
      mm_atb(dk, s_s, 16 * warp, q_s, lane);                         // dK = dS^T Q
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int k = 16 * warp + gr + 8 * r;
        if (k >= kL) continue;
        __nv_bfloat16* dst = g.out + token_row<GRID>(g, n, si, sj, k) * ld + h * kD + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          *reinterpret_cast<uint32_t*>(dst + C + 8 * j) = pack_bf16x2(dk[j][2 * r] * scale, dk[j][2 * r + 1] * scale);
          *reinterpret_cast<uint32_t*>(dst + 2 * C + 8 * j) = pack_bf16x2(dv[j][2 * r], dv[j][2 * r + 1]);
        }
      }
    }
    // bias gradient: the pairs (t, u) with ta - ua = dy and tb - ub = dx, in row-major order of t
    if (tid < kTab) dt_sum += rel_sum(sSf, tid);
    if (tid + kThreads < kTab) dt_sum2 += rel_sum(sSf, tid + kThreads);
    __syncthreads();                              // the tiles and sSf are refilled by the next sequence
  }
  float* part = g.part + ((static_cast<size_t>(n) * g.ns + si) * g.heads + h) * kTab;
  if (tid < kTab) part[tid] = dt_sum;
  if (tid + kThreads < kTab) part[tid + kThreads] = dt_sum2;
}

// first level: chunk c of the P = N * ns partials, summed in order, for every (head, k) -> chunk [kChunks][heads*169]
__global__ void __launch_bounds__(kThreads) part_bias_grad_chunk_kernel(const float* __restrict__ part,
                                                                        float* __restrict__ chunk, int P, int per) {
  pdl_trigger();
  pdl_wait();
  const int e = blockIdx.x * kThreads + threadIdx.x, c = blockIdx.y;
  if (e >= per) return;
  const int p0 = static_cast<int>(static_cast<int64_t>(P) * c / kChunks);
  const int p1 = static_cast<int>(static_cast<int64_t>(P) * (c + 1) / kChunks);
  float s = 0.f;
#pragma unroll 8
  for (int p = p0; p < p1; ++p) s += part[static_cast<size_t>(p) * per + e];
  chunk[static_cast<size_t>(c) * per + e] = s;
}

// second level: dtable[k][h] += sum over the chunks in order
__global__ void __launch_bounds__(kThreads) part_bias_grad_final_kernel(const float* __restrict__ chunk,
                                                                        float* __restrict__ dtable, int heads) {
  pdl_trigger();
  pdl_wait();
  const int e = blockIdx.x * kThreads + threadIdx.x, per = heads * kTab;
  if (e >= per || dtable == nullptr) return;
  float s = 0.f;
#pragma unroll 8
  for (int c = 0; c < kChunks; ++c) s += chunk[static_cast<size_t>(c) * per + e];
  const int h = e / kTab, k = e - h * kTab;
  dtable[k * heads + h] += s;
}

bool grid_shape_ok(int N, int H, int W, int heads, int C) {
  return N > 0 && N <= 65535 && heads > 0 && heads <= 65535 && C == kD * heads && H > 0 && H == W && H % kP == 0 &&
         (H / kP) * (H / kP) <= 65535;
}

GridArgs grid_args(const __nv_bfloat16* qkv, int H, int heads, int C, float scale) {
  GridArgs g{};
  g.qkv = qkv; g.H = H; g.C = C; g.heads = heads; g.ns = H / kP; g.scale = scale;
  return g;
}

}  // namespace

size_t grid_attention_bwd_scratch_floats(int N, int H, int heads) {
  return (static_cast<size_t>(N) * (H / kP) + kChunks) * heads * kTab;
}

cudaError_t launch_grid_attention_fwd(const __nv_bfloat16* qkv, const float* table, __nv_bfloat16* o, float* lse,
                                      int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream) {
  if (!grid_shape_ok(N, H, W, heads, C)) return cudaErrorInvalidValue;
  GridArgs g = grid_args(qkv, H, heads, C, scale);
  g.table = table; g.out = o; g.lse = lse;
  const dim3 blocks(g.ns * g.ns, heads, N);
  return grid ? launch_pdl(part_attn_fwd_kernel<true>, blocks, dim3(kThreads), 0, stream, 1, g)
              : launch_pdl(part_attn_fwd_kernel<false>, blocks, dim3(kThreads), 0, stream, 1, g);
}

cudaError_t launch_grid_attention_bwd(const __nv_bfloat16* qkv, const float* table, const __nv_bfloat16* o,
                                      const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv, float* dtable,
                                      float* scratch, int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream) {
  if (!grid_shape_ok(N, H, W, heads, C)) return cudaErrorInvalidValue;
  GridArgs g = grid_args(qkv, H, heads, C, scale);
  g.table = table; g.o = o; g.dout = dout; g.lse = const_cast<float*>(lse); g.out = dqkv; g.part = scratch;
  const dim3 blocks(g.ns, heads, N);
  cudaError_t e = grid ? launch_pdl(part_attn_bwd_kernel<true>, blocks, dim3(kThreads), 0, stream, 1, g)
                       : launch_pdl(part_attn_bwd_kernel<false>, blocks, dim3(kThreads), 0, stream, 1, g);
  if (e != cudaSuccess) return e;
  const int P = N * g.ns, per = heads * kTab;
  float* chunk = scratch + static_cast<size_t>(P) * per;
  e = launch_pdl(part_bias_grad_chunk_kernel, dim3((per + kThreads - 1) / kThreads, kChunks), dim3(kThreads), 0,
                 stream, 1, static_cast<const float*>(scratch), chunk, P, per);
  if (e != cudaSuccess) return e;
  return launch_pdl(part_bias_grad_final_kernel, dim3((per + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(chunk), dtable, heads);
}

}  // namespace ddl
