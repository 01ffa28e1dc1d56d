// Fused multi-head self-attention, head dim 64, on the packed in-projection output of a transformer encoder block.
//
// Layout (no transposes anywhere): qkv is the bf16 [N*L][3C] output of the in-projection GEMM; head h's Q, K and V are
// the 64 columns at 64h, C + 64h and 2C + 64h of the rows n*L .. n*L + L - 1 of image n.  The forward writes
// O = softmax(Q K^T / 8) V into [N*L][C] (head h at columns 64h, out_proj's GEMM input as it is) and the fp32 natural-log
// log-sum-exp of every (image, head, query) into [N][H][L].  The backward writes dQ, dK and dV into one bf16 [N*L][3C]
// buffer in qkv's layout, the operand of the in-projection's data, weight and bias gradients.
//
// Mapping: one CTA of 4 warps per (64-row tile, head, image); each warp owns 16 rows and runs the warp-level
// mma.sync.m16n8k16 bf16 tensor-core instruction with fp32 accumulators.  The streamed operand (K/V in the forward and
// the dQ kernel, Q/dO in the dK/dV kernel) comes in 64-row blocks through a two-stage cp.async pipeline into shared rows
// of 72 bf16 (144 B: ldmatrix rows stay 16-byte aligned and the 8 rows of each 8x8 matrix fall in distinct banks).  The
// score tile S of a warp (16 x 64, in the accumulator layout) is, after the softmax, exactly the register A operand of
// the next product: the accumulator pair of n-tiles 2k, 2k+1 is the A fragment of k-slice k, so P never leaves registers.
//
// Masking: rows past L are loaded as zeros (cp.async zero-fill) and never stored.  Key columns past L are set to -inf
// before the softmax (forward, dQ) and query columns past L get P = 0 (dK/dV): a zero-filled key would score 0, not -inf.
//
// Softmax: online over the key blocks, in fp32, in the base-2 domain with the scale folded in (x = s * log2(e) / 8,
// p = exp2(x - m)).  The saved LSE is natural-log: lse = (m + log2(l)) / log2(e).
//
// Backward (deterministic: no atomics, no fp32 scratch beyond D):
//   dQ kernel,   per query tile: D = rowsum(dO o O) -> [N][H][L]; over key blocks: S = Q K^T, P = exp2(S' - lse'),
//                dP = dO V^T, dS = P o (dP - D), dQ += dS K; dQ *= 1/8.
//   dK/dV kernel, per key block: over query tiles: S^T = K Q^T, P^T = exp2(S^T' - lse'), dV += P^T dO,
//                dP^T = V dO^T, dS^T = P^T o (dP^T - D), dK += dS^T Q; dK *= 1/8.
// P, dS (and their transposes) are rounded to bf16 as A operands; D uses the stored bf16 O.
#include <math.h>

#include "../common.cuh"
#include "ops.h"
#include "mma_tile.cuh"
#include "tc_utils.cuh"
#include "../launch.h"

namespace ddl {

namespace {

using namespace mma_tile;

constexpr int kD = 64;           // head dim
constexpr int kTile = 64;        // rows per CTA and per streamed block
constexpr int kThreads = 128;    // 4 warps x 16 rows
constexpr int kLd = 72;          // shared row stride in bf16
constexpr float kLog2e = 1.4426950408889634f;
constexpr uint32_t kStage = kTile * kLd * 2;     // bytes of one tile

struct AttnArgs {
  const __nv_bfloat16* qkv;      // [N*L][3C]
  const __nv_bfloat16* o;        // [N*L][C]   (backward)
  const __nv_bfloat16* dout;     // [N*L][C]   (backward)
  __nv_bfloat16* out;            // forward: O [N*L][C]; backward: dqkv [N*L][3C]
  float* lse;                    // [N][H][L]
  float* delta;                  // [N][H][L]  (backward: D, written by the dQ kernel, read by the dK/dV kernel)
  int L, H, C;
};

// 64 rows x 64 bf16 of a row-major matrix (row stride ld) from row r0 (rows >= rows_valid are zero-filled) into a tile
DDL_DEVICE void load_tile(uint32_t tile, const __nv_bfloat16* base, int ld, int r0, int col, int rows_valid, int tid) {
#pragma unroll
  for (int it = 0; it < (kTile * 8) / kThreads; ++it) {
    const int c = tid + it * kThreads, r = c >> 3, ch = c & 7;
    const bool ok = r0 + r < rows_valid;
    const __nv_bfloat16* src = base + static_cast<size_t>(ok ? r0 + r : 0) * ld + col + ch * 8;
    tc::cp_async_16(tile + static_cast<uint32_t>((r * kLd + ch * 8) * 2), src, ok);
  }
}

// A fragments (16 rows x 64) of a warp straight from global memory (rows >= rows_valid are zero)
DDL_DEVICE void load_a_global(uint32_t (&f)[4][4], const __nv_bfloat16* base, int ld, int r0, int col, int rows_valid,
                              int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + g + 8 * h;
    const bool ok = r < rows_valid;
    const __nv_bfloat16* p = base + static_cast<size_t>(ok ? r : 0) * ld + col + 2 * t;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      f[kk][h] = ok ? __ldg(reinterpret_cast<const unsigned int*>(p + 16 * kk)) : 0u;
      f[kk][2 + h] = ok ? __ldg(reinterpret_cast<const unsigned int*>(p + 16 * kk + 8)) : 0u;
    }
  }
}

__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(AttnArgs a) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kTile * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[2][kTile * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[2][kTile * kLd];
  pdl_trigger();
  const int q0 = blockIdx.x * kTile, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, ld = 3 * a.C, nkb = (L + kTile - 1) / kTile;
  const float sl2 = kLog2e * 0.125f;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(n) * L * ld;
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK[0]), v_s = tc::smem_u32(sV[0]);
  pdl_wait();
  load_tile(q_s, base, ld, q0, h * kD, L, tid);
  load_tile(k_s, base, ld, 0, a.C + h * kD, L, tid);
  load_tile(v_s, base, ld, 0, 2 * a.C + h * kD, L, tid);
  tc::cp_async_commit();

  uint32_t qf[4][4];
  float acc[8][4], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    const int cur = kb & 1;
    if (kb + 1 < nkb) {
      load_tile(k_s + (cur ^ 1) * kStage, base, ld, (kb + 1) * kTile, a.C + h * kD, L, tid);
      load_tile(v_s + (cur ^ 1) * kStage, base, ld, (kb + 1) * kTile, 2 * a.C + h * kD, L, tid);
      tc::cp_async_commit();
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();
    if (kb == 0) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) ldsm4(addr_a<kLd>(q_s, 16 * warp, 16 * kk, lane), qf[kk]);
    }
    float s[8][4];
    mm_abt<kLd>(s, qf, k_s + cur * kStage, lane);
    const int key0 = kb * kTile + 2 * t;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = s[j][2 * r + e];
          x = key0 + 8 * j + e < L ? x * sl2 : -INFINITY;
          mx = fmaxf(mx, x);
        }
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[r], mx);        // finite: every key block holds at least one key < L
      const float corr = exp2f(m[r] - mn);
      m[r] = mn;
      float ls = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& x = s[j][2 * r + e];
          x = exp2f(x - mn);
          ls += x;
        }
        acc[j][2 * r] *= corr;
        acc[j][2 * r + 1] *= corr;
      }
      l[r] = l[r] * corr + ls;
    }
    mm_pb<kLd>(acc, s, v_s + cur * kStage, lane);
    __syncthreads();                           // everyone is done with stage cur before it is refilled
  }
  const size_t head = (static_cast<size_t>(n) * a.H + h) * L;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float lt = l[r];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const int q = q0 + 16 * warp + g + 8 * r;
    if (q >= L) continue;
    const float inv = 1.f / lt;
    __nv_bfloat16* dst = a.out + (static_cast<size_t>(n) * L + q) * a.C + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) a.lse[head + q] = (m[r] + log2f(lt)) * (1.f / kLog2e);
  }
}

__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(AttnArgs a) {
  __shared__ __align__(128) __nv_bfloat16 sK[2][kTile * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[2][kTile * kLd];
  __shared__ float sD[kTile];
  pdl_trigger();
  const int q0 = blockIdx.x * kTile, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, C = a.C, ld = 3 * C, nkb = (L + kTile - 1) / kTile;
  const float sl2 = kLog2e * 0.125f;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(n) * L * ld;
  const size_t head = (static_cast<size_t>(n) * a.H + h) * L;
  const uint32_t k_s = tc::smem_u32(sK[0]), v_s = tc::smem_u32(sV[0]);
  pdl_wait();
  load_tile(k_s, base, ld, 0, C + h * kD, L, tid);
  load_tile(v_s, base, ld, 0, 2 * C + h * kD, L, tid);
  tc::cp_async_commit();
  {   // D = rowsum(dO o O): two threads per row, 32 columns each
    const int r = tid >> 1, q = q0 + r, c0 = h * kD + (tid & 1) * 32;
    float d = 0.f;
    if (q < L) {
      const size_t off = (static_cast<size_t>(n) * L + q) * C + c0;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const uint4 x = __ldg(reinterpret_cast<const uint4*>(a.dout + off) + v);
        const uint4 y = __ldg(reinterpret_cast<const uint4*>(a.o + off) + v);
        const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 u = unpack_bf16x2(xs[k]), w = unpack_bf16x2(ys[k]);
          d = fmaf(u.x, w.x, fmaf(u.y, w.y, d));
        }
      }
    }
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    if ((tid & 1) == 0) {
      sD[r] = d;
      if (q < L) a.delta[head + q] = d;
    }
  }
  uint32_t qf[4][4], df[4][4];
  load_a_global(qf, base, ld, q0 + 16 * warp, h * kD, L, lane);
  load_a_global(df, a.dout + static_cast<size_t>(n) * L * C, C, q0 + 16 * warp, h * kD, L, lane);
  float lse2[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + 16 * warp + g + 8 * r;
    lse2[r] = q < L ? a.lse[head + q] * kLog2e : 0.f;
  }
  float dq[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    const int cur = kb & 1;
    if (kb + 1 < nkb) {
      load_tile(k_s + (cur ^ 1) * kStage, base, ld, (kb + 1) * kTile, C + h * kD, L, tid);
      load_tile(v_s + (cur ^ 1) * kStage, base, ld, (kb + 1) * kTile, 2 * C + h * kD, L, tid);
      tc::cp_async_commit();
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();                           // (also publishes sD on the first pass)
    float p[8][4], dp[8][4];
    mm_abt<kLd>(p, qf, k_s + cur * kStage, lane);
    mm_abt<kLd>(dp, df, v_s + cur * kStage, lane);
    const int key0 = kb * kTile + 2 * t;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float dr = sD[16 * warp + g + 8 * r];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 2 * r + e;
          const float pv = key0 + 8 * j + e < L ? exp2f(fmaf(p[j][i], sl2, -lse2[r])) : 0.f;
          p[j][i] = pv * (dp[j][i] - dr);      // dS
        }
      }
    }
    mm_pb<kLd>(dq, p, k_s + cur * kStage, lane);
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + 16 * warp + g + 8 * r;
    if (q >= L) continue;
    __nv_bfloat16* dst = a.out + (static_cast<size_t>(n) * L + q) * ld + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(dq[j][2 * r] * 0.125f, dq[j][2 * r + 1] * 0.125f);
  }
}

__global__ void __launch_bounds__(kThreads) attn_bwd_dkv_kernel(AttnArgs a) {
  __shared__ __align__(128) __nv_bfloat16 sQ[2][kTile * kLd];
  __shared__ __align__(128) __nv_bfloat16 sO[2][kTile * kLd];      // dO
  __shared__ float sL[2][kTile], sD[2][kTile];                     // lse * log2(e), D of the query tile
  pdl_trigger();
  const int k0 = blockIdx.x * kTile, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int L = a.L, C = a.C, ld = 3 * C, nqb = (L + kTile - 1) / kTile;
  const float sl2 = kLog2e * 0.125f;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(n) * L * ld;
  const __nv_bfloat16* dob = a.dout + static_cast<size_t>(n) * L * C;
  const size_t head = (static_cast<size_t>(n) * a.H + h) * L;
  const uint32_t q_s = tc::smem_u32(sQ[0]), o_s = tc::smem_u32(sO[0]);
  pdl_wait();
  auto stage = [&](int qb, int buf) {
    load_tile(q_s + buf * kStage, base, ld, qb * kTile, h * kD, L, tid);
    load_tile(o_s + buf * kStage, dob, C, qb * kTile, h * kD, L, tid);
    tc::cp_async_commit();
    if (tid < kTile) {
      const int q = qb * kTile + tid;
      sL[buf][tid] = q < L ? a.lse[head + q] * kLog2e : 0.f;
      sD[buf][tid] = q < L ? a.delta[head + q] : 0.f;
    }
  };
  stage(0, 0);
  uint32_t kf[4][4], vf[4][4];
  load_a_global(kf, base, ld, k0 + 16 * warp, C + h * kD, L, lane);
  load_a_global(vf, base, ld, k0 + 16 * warp, 2 * C + h * kD, L, lane);
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
  for (int qb = 0; qb < nqb; ++qb) {
    const int cur = qb & 1;
    if (qb + 1 < nqb) {
      stage(qb + 1, cur ^ 1);
      tc::cp_async_wait<1>();
    } else {
      tc::cp_async_wait<0>();
    }
    __syncthreads();
    float p[8][4];
    mm_abt<kLd>(p, kf, q_s + cur * kStage, lane);        // S^T = K Q^T
    const int qc0 = qb * kTile + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 8 * j + 2 * t + (i & 1);
        p[j][i] = qc0 + 8 * j + (i & 1) < L ? exp2f(fmaf(p[j][i], sl2, -sL[cur][c])) : 0.f;
      }
    }
    mm_pb<kLd>(dv, p, o_s + cur * kStage, lane);         // dV += P^T dO
    float dp[8][4];
    mm_abt<kLd>(dp, vf, o_s + cur * kStage, lane);       // dP^T = V dO^T
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int i = 0; i < 4; ++i) p[j][i] *= dp[j][i] - sD[cur][8 * j + 2 * t + (i & 1)];
    }
    mm_pb<kLd>(dk, p, q_s + cur * kStage, lane);         // dK += dS^T Q
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int k = k0 + 16 * warp + g + 8 * r;
    if (k >= L) continue;
    __nv_bfloat16* dst = a.out + (static_cast<size_t>(n) * L + k) * ld + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(dst + C + 8 * j) = pack_bf16x2(dk[j][2 * r] * 0.125f, dk[j][2 * r + 1] * 0.125f);
      *reinterpret_cast<uint32_t*>(dst + 2 * C + 8 * j) = pack_bf16x2(dv[j][2 * r], dv[j][2 * r + 1]);
    }
  }
}

bool attn_shape_ok(int N, int L, int H, int C) {
  return N > 0 && L > 0 && H > 0 && H <= 65535 && N <= 65535 && C == kD * H;
}

}  // namespace

cudaError_t launch_attention_fwd(const __nv_bfloat16* qkv, __nv_bfloat16* o, float* lse, int N, int L, int H, int C,
                                 cudaStream_t stream) {
  if (!attn_shape_ok(N, L, H, C)) return cudaErrorInvalidValue;
  AttnArgs a{};
  a.qkv = qkv; a.out = o; a.lse = lse; a.L = L; a.H = H; a.C = C;
  const dim3 grid((L + kTile - 1) / kTile, H, N);
  return launch_pdl(attn_fwd_kernel, grid, dim3(kThreads), 0, stream, 1, a);
}

cudaError_t launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* o, const __nv_bfloat16* dout,
                                 const float* lse, float* delta, __nv_bfloat16* dqkv, int N, int L, int H, int C,
                                 cudaStream_t stream) {
  if (!attn_shape_ok(N, L, H, C)) return cudaErrorInvalidValue;
  AttnArgs a{};
  a.qkv = qkv; a.o = o; a.dout = dout; a.out = dqkv; a.lse = const_cast<float*>(lse); a.delta = delta;
  a.L = L; a.H = H; a.C = C;
  const dim3 grid((L + kTile - 1) / kTile, H, N);
  cudaError_t e = launch_pdl(attn_bwd_dq_kernel, grid, dim3(kThreads), 0, stream, 1, a);
  if (e != cudaSuccess) return e;
  return launch_pdl(attn_bwd_dkv_kernel, grid, dim3(kThreads), 0, stream, 1, a);
}

}  // namespace ddl
